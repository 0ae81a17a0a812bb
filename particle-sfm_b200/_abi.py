"""ctypes mirror of include/psfm_b200.h (structs + enums).  Shared by the product
binding (`_lib.py`) and by the oracle loader (oracle/__init__.py) so that both sides of a
parity test receive byte-identical inputs."""
import ctypes as C

import numpy as np

PSFM_OK = 0
PSFM_ZERO_RESIDUALS = 1
PSFM_ERR_INVALID = -1
PSFM_ERR_NO_DEVICE = -2
PSFM_ERR_CUDA = -3
PSFM_ERR_UNSUPPORTED = -4
PSFM_ERR_NCCL = -5

LOSS_TRIVIAL, LOSS_SOFT_L1, LOSS_CAUCHY = 0, 1, 2
SOLVER_AUTO, SOLVER_EXACT_SCHUR, SOLVER_ITERATIVE_SCHUR = 0, 1, 2

TERMINATION_NAMES = {
    0: "CONVERGENCE (gradient tolerance)",
    1: "CONVERGENCE (parameter tolerance)",
    2: "CONVERGENCE (function tolerance)",
    3: "NO_CONVERGENCE (max iterations)",
    4: "FAILURE",
    5: "CONVERGENCE (min trust region radius)",
}

NCCL_UNIQUE_ID_BYTES = 128


class TrajOptions(C.Structure):
    _fields_ = [
        ("max_num_iterations", C.c_int32),
        ("function_tolerance", C.c_double),
        ("gradient_tolerance", C.c_double),
        ("parameter_tolerance", C.c_double),
        ("initial_trust_region_radius", C.c_double),
        ("max_trust_region_radius", C.c_double),
        ("min_trust_region_radius", C.c_double),
        ("min_relative_decrease", C.c_double),
        ("max_num_consecutive_invalid_steps", C.c_int32),
        ("jacobi_scaling", C.c_int32),
    ]


class TrajSummary(C.Structure):
    _fields_ = [
        ("num_iterations", C.c_int32),
        ("num_successful_steps", C.c_int32),
        ("num_unsuccessful_steps", C.c_int32),
        ("termination", C.c_int32),
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("solve_ms", C.c_double),
        ("total_ms", C.c_double),
    ]


class BAOptions(C.Structure):
    _fields_ = [
        ("loss_function_type", C.c_int32),
        ("loss_function_scale", C.c_double),
        ("refine_focal_length", C.c_int32),
        ("refine_principal_point", C.c_int32),
        ("refine_extra_params", C.c_int32),
        ("refine_extrinsics", C.c_int32),
        ("refine_rotation", C.c_int32),
        ("print_summary", C.c_int32),
        ("minimizer_progress_to_stdout", C.c_int32),
        ("function_tolerance", C.c_double),
        ("gradient_tolerance", C.c_double),
        ("parameter_tolerance", C.c_double),
        ("max_num_iterations", C.c_int32),
        ("max_linear_solver_iterations", C.c_int32),
        ("max_num_consecutive_invalid_steps", C.c_int32),
        ("linear_solver", C.c_int32),
        ("eta", C.c_double),
        ("exact_r_tolerance", C.c_double),
        ("exact_max_iterations", C.c_int32),
        ("initial_trust_region_radius", C.c_double),
        ("max_trust_region_radius", C.c_double),
        ("min_trust_region_radius", C.c_double),
        ("min_relative_decrease", C.c_double),
        ("min_lm_diagonal", C.c_double),
        ("max_lm_diagonal", C.c_double),
        ("jacobi_scaling", C.c_int32),
        ("pcg_check_period", C.c_int32),
    ]

    def copy(self):
        o = BAOptions()
        C.memmove(C.byref(o), C.byref(self), C.sizeof(BAOptions))
        return o


class BAProblemStruct(C.Structure):
    _fields_ = [
        ("num_images", C.c_int32),
        ("num_points", C.c_int32),
        ("num_observations", C.c_int32),
        ("num_cameras", C.c_int32),
        ("qvec", C.POINTER(C.c_double)),
        ("tvec", C.POINTER(C.c_double)),
        ("xyz", C.POINTER(C.c_double)),
        ("cam_params", C.POINTER(C.c_double)),
        ("obs_image", C.POINTER(C.c_int32)),
        ("obs_point", C.POINTER(C.c_int32)),
        ("obs_xy", C.POINTER(C.c_double)),
        ("image_camera", C.POINTER(C.c_int32)),
        ("pose_constant", C.POINTER(C.c_uint8)),
        ("tvec_constant_mask", C.POINTER(C.c_uint8)),
        ("camera_constant", C.POINTER(C.c_uint8)),
    ]


class BASummary(C.Structure):
    _fields_ = [
        ("num_residuals_reduced", C.c_int32),
        ("num_effective_parameters_reduced", C.c_int32),
        ("num_successful_steps", C.c_int32),
        ("num_unsuccessful_steps", C.c_int32),
        ("num_iterations", C.c_int32),
        ("num_linear_iterations", C.c_int32),
        ("termination", C.c_int32),
        ("initial_cost", C.c_double),
        ("final_cost", C.c_double),
        ("total_time_in_seconds", C.c_double),
        ("device_ms", C.c_double),
        ("linearize_ms", C.c_double),
        ("schur_product_ms", C.c_double),
        ("num_linearize", C.c_int32),
        ("num_schur_products", C.c_int32),
        ("linear_solver_used", C.c_int32),
        ("world_size", C.c_int32),
        ("num_explicit_solves", C.c_int32),
        ("schur_w_ms", C.c_double),
        ("schur_pairs_ms", C.c_double),
        ("cholesky_ms", C.c_double),
        ("num_pair_entries", C.c_int64),
        ("num_pair_tasks", C.c_int32),
        ("explicit_fused", C.c_int32),
        ("explicit_dense_tiles", C.c_int32),
    ]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


MAX_REFINEMENTS = 8   # PSFM_BA_MAX_REFINEMENTS


class BARefineOptions(C.Structure):
    _fields_ = [
        ("max_refinements", C.c_int32),
        ("max_refinement_change", C.c_double),
        ("filter_max_reproj_error", C.c_double),
        ("filter_min_tri_angle", C.c_double),
        ("normalize_extent", C.c_double),
        ("normalize_p0", C.c_double),
        ("normalize_p1", C.c_double),
    ]


class BARefineReport(C.Structure):
    _fields_ = [
        ("num_rounds", C.c_int32),
        ("ba_iterations", C.c_int32 * MAX_REFINEMENTS),
        ("ba_termination", C.c_int32 * MAX_REFINEMENTS),
        ("num_observations", C.c_int64 * MAX_REFINEMENTS),
        ("num_negative_depth", C.c_int64 * MAX_REFINEMENTS),
        ("num_changed", C.c_int64 * MAX_REFINEMENTS),
        ("changed", C.c_double * MAX_REFINEMENTS),
        ("ba_final_cost", C.c_double * MAX_REFINEMENTS),
        ("final_num_observations", C.c_int64),
        ("total_time_in_seconds", C.c_double),
    ]

    def rounds(self):
        return [dict(num_observations=self.num_observations[i], num_negative_depth=self.num_negative_depth[i],
                     changed_observations=self.num_changed[i], changed=self.changed[i],
                     ba_iterations=self.ba_iterations[i], final_cost=self.ba_final_cost[i],
                     termination=self.ba_termination[i]) for i in range(self.num_rounds)]


def _ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype)) if a is not None else None


class BAProblem:
    """Flattened bundle-adjustment problem (host numpy arrays) = what
    BundleAdjuster::SetUp builds from (Reconstruction, BundleAdjustmentConfig)
    (reference sfm/gmapper/src/optim/bundle_adjustment.cc:326-447).  Owns contiguous
    arrays and hands out the C struct view; qvec/tvec/xyz/cam_params are updated in place
    by a solve, like the reference mutates the Reconstruction."""

    def __init__(self, qvec, tvec, xyz, cam_params, obs_image, obs_point, obs_xy, image_camera,
                 pose_constant=None, tvec_constant_mask=None, camera_constant=None):
        self.qvec = np.ascontiguousarray(qvec, dtype=np.float64).reshape(-1, 4)
        self.tvec = np.ascontiguousarray(tvec, dtype=np.float64).reshape(-1, 3)
        self.xyz = np.ascontiguousarray(xyz, dtype=np.float64).reshape(-1, 3)
        self.cam_params = np.ascontiguousarray(cam_params, dtype=np.float64).reshape(-1, 3)
        self.obs_image = np.ascontiguousarray(obs_image, dtype=np.int32).reshape(-1)
        self.obs_point = np.ascontiguousarray(obs_point, dtype=np.int32).reshape(-1)
        self.obs_xy = np.ascontiguousarray(obs_xy, dtype=np.float64).reshape(-1, 2)
        self.image_camera = np.ascontiguousarray(image_camera, dtype=np.int32).reshape(-1)
        F, Cn = self.qvec.shape[0], self.cam_params.shape[0]
        self.pose_constant = (np.zeros(F, np.uint8) if pose_constant is None
                              else np.ascontiguousarray(pose_constant, dtype=np.uint8))
        self.tvec_constant_mask = (np.zeros(F, np.uint8) if tvec_constant_mask is None
                                   else np.ascontiguousarray(tvec_constant_mask, dtype=np.uint8))
        self.camera_constant = (np.zeros(Cn, np.uint8) if camera_constant is None
                                else np.ascontiguousarray(camera_constant, dtype=np.uint8))
        assert self.tvec.shape[0] == F and self.image_camera.shape[0] == F
        assert self.obs_point.shape[0] == self.obs_image.shape[0] == self.obs_xy.shape[0]

    num_images = property(lambda s: s.qvec.shape[0])
    num_points = property(lambda s: s.xyz.shape[0])
    num_observations = property(lambda s: s.obs_image.shape[0])
    num_cameras = property(lambda s: s.cam_params.shape[0])

    def copy(self):
        return BAProblem(self.qvec.copy(), self.tvec.copy(), self.xyz.copy(), self.cam_params.copy(),
                         self.obs_image, self.obs_point, self.obs_xy, self.image_camera,
                         self.pose_constant, self.tvec_constant_mask, self.camera_constant)

    def shard(self, rank, world):
        """Point-sharded view for rank `rank` of `world` (SURVEY.md §8e): contiguous point
        ranges balanced by observation count; cameras/images replicated.  Point arrays keep
        their global size (only the shard's points receive observations)."""
        if world == 1:
            return self
        counts = np.bincount(self.obs_point, minlength=self.num_points)
        cum = np.cumsum(counts)
        total = int(cum[-1]) if len(cum) else 0
        lo_obs, hi_obs = total * rank // world, total * (rank + 1) // world
        p_lo = int(np.searchsorted(cum, lo_obs, side="right")) if rank > 0 else 0
        p_hi = int(np.searchsorted(cum, hi_obs, side="right")) if rank + 1 < world else self.num_points
        sel = (self.obs_point >= p_lo) & (self.obs_point < p_hi)
        return BAProblem(self.qvec, self.tvec, self.xyz, self.cam_params, self.obs_image[sel],
                         self.obs_point[sel], self.obs_xy[sel], self.image_camera,
                         self.pose_constant, self.tvec_constant_mask, self.camera_constant)

    def struct(self):
        s = BAProblemStruct()
        s.num_images, s.num_points = self.num_images, self.num_points
        s.num_observations, s.num_cameras = self.num_observations, self.num_cameras
        s.qvec, s.tvec = _ptr(self.qvec, C.c_double), _ptr(self.tvec, C.c_double)
        s.xyz, s.cam_params = _ptr(self.xyz, C.c_double), _ptr(self.cam_params, C.c_double)
        s.obs_image, s.obs_point = _ptr(self.obs_image, C.c_int32), _ptr(self.obs_point, C.c_int32)
        s.obs_xy, s.image_camera = _ptr(self.obs_xy, C.c_double), _ptr(self.image_camera, C.c_int32)
        s.pose_constant = _ptr(self.pose_constant, C.c_uint8)
        s.tvec_constant_mask = _ptr(self.tvec_constant_mask, C.c_uint8)
        s.camera_constant = _ptr(self.camera_constant, C.c_uint8)
        return s


ROTATION_MAX_L1_ROUNDS = 16   # PSFM_ROTATION_MAX_L1_ROUNDS
NO_ROTATIONS = 2              # PSFM_NO_ROTATIONS


class RotationOptions(C.Structure):
    _fields_ = [
        ("max_num_l1_iterations", C.c_int32),
        ("l1_step_convergence_threshold", C.c_double),
        ("max_num_irls_iterations", C.c_int32),
        ("irls_step_convergence_threshold", C.c_double),
        ("irls_loss_parameter_sigma", C.c_double),
        ("rotation_filter_max_degrees", C.c_double),
    ]


class RotationSummary(C.Structure):
    _fields_ = [
        ("num_l1_rounds", C.c_int32),
        ("admm_iterations", C.c_int32 * ROTATION_MAX_L1_ROUNDS),
        ("num_irls_iterations", C.c_int32),
        ("l1_final_step", C.c_double),
        ("irls_final_step", C.c_double),
        ("gauge_image", C.c_int32),
        ("num_images_connected", C.c_int32),
        ("num_pairs_connected", C.c_int32),
        ("num_images_kept", C.c_int32),
        ("num_pairs_kept", C.c_int32),
        ("num_launches", C.c_int64),
        ("host_ms", C.c_double),
        ("device_ms", C.c_double),
    ]
