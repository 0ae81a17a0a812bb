"""Host-side mirror of the reference's bundle-adjustment interface (HP2).

Mirrors, name for name, what `gcolmap` uses around `BundleAdjuster::Solve`
(reference sfm/gmapper/src/optim/bundle_adjustment.{h,cc}):

  BundleAdjustmentOptions   bundle_adjustment.h:48-102
  BundleAdjustmentConfig    bundle_adjustment.h:105-158, .cc:78-251
  BundleAdjuster            bundle_adjustment.h:161-198, .cc:253-320
  global_bundle_adjustment_options()   GlobalMapperOptions::GlobalBundleAdjustment,
                                       controllers/global_mapper.cc:41-71
  adjust_global_bundle()    GlobalMapper::AdjustGlobalBundle, sfm/global_mapper.cc:402-448
                            (gauge fixing + Normalize) and the option policy of
                            controllers/global_mapper.cc:215-243

The numerical work is done by the CUDA library through the C ABI (`_lib.py`); this
module only flattens a Reconstruction-like container into `psfm_ba_problem` and scatters
the result back in place, as the reference mutates its Reconstruction in place.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

from . import _abi, _lib
from ._abi import BAProblem, BAOptions, BASummary  # noqa: F401

SIMPLE_PINHOLE = 0  # colmap camera model id (sfm/colmap_utils/read_write_model.py:56)


# ----------------------------------------------------------------------------- options

class LossFunctionType:
    TRIVIAL, SOFT_L1, CAUCHY = 0, 1, 2


@dataclass
class SolverOptions:
    """The ceres::Solver::Options fields the reference touches (bundle_adjustment.h:80-95)."""
    function_tolerance: float = 0.0
    gradient_tolerance: float = 0.0
    parameter_tolerance: float = 0.0
    minimizer_progress_to_stdout: bool = False
    max_num_iterations: int = 100
    max_linear_solver_iterations: int = 200
    max_num_consecutive_invalid_steps: int = 10
    max_consecutive_nonmonotonic_steps: int = 10   # inert: use_nonmonotonic_steps stays false
    num_threads: int = -1                          # meaningless on the GPU; kept for the surface
    # extensions (not in the reference): which reduced-system solve to use
    linear_solver: int = _abi.SOLVER_AUTO
    eta: float = 0.1


@dataclass
class BundleAdjustmentOptions:
    loss_function_type: int = LossFunctionType.TRIVIAL
    loss_function_scale: float = 1.0
    refine_focal_length: bool = True
    refine_principal_point: bool = False
    refine_extra_params: bool = True
    refine_extrinsics: bool = True
    refine_rotation: bool = True
    print_summary: bool = True
    min_num_residuals_for_multi_threading: int = 50000   # CPU-thread policy, unused here
    solver_options: SolverOptions = field(default_factory=SolverOptions)

    def Check(self):
        if not self.loss_function_scale >= 0:
            raise ValueError("loss_function_scale must be >= 0")   # CHECK_OPTION_GE, .cc:72
        return True

    def to_struct(self):
        o = _abi.BAOptions()
        _lib.lib().psfm_ba_default_options(C.byref(o))
        so = self.solver_options
        o.loss_function_type = int(self.loss_function_type)
        o.loss_function_scale = float(self.loss_function_scale)
        o.refine_focal_length = int(self.refine_focal_length)
        o.refine_principal_point = int(self.refine_principal_point)
        o.refine_extra_params = int(self.refine_extra_params)
        o.refine_extrinsics = int(self.refine_extrinsics)
        o.refine_rotation = int(self.refine_rotation)
        o.print_summary = int(self.print_summary)
        o.minimizer_progress_to_stdout = int(so.minimizer_progress_to_stdout)
        o.function_tolerance = so.function_tolerance
        o.gradient_tolerance = so.gradient_tolerance
        o.parameter_tolerance = so.parameter_tolerance
        o.max_num_iterations = so.max_num_iterations
        o.max_linear_solver_iterations = so.max_linear_solver_iterations
        o.max_num_consecutive_invalid_steps = so.max_num_consecutive_invalid_steps
        o.linear_solver = so.linear_solver
        o.eta = so.eta
        return o


def global_bundle_adjustment_options(ba_global_max_num_iterations=50, num_threads=-1):
    """GlobalMapperOptions::GlobalBundleAdjustment (controllers/global_mapper.cc:41-71)."""
    o = BundleAdjustmentOptions()
    so = o.solver_options
    so.function_tolerance = 1e-6
    so.gradient_tolerance = 1.0
    so.parameter_tolerance = 1e-8
    so.max_num_iterations = ba_global_max_num_iterations
    so.max_linear_solver_iterations = 100
    so.minimizer_progress_to_stdout = True
    so.num_threads = num_threads
    o.print_summary = True
    o.refine_rotation = False
    o.refine_focal_length = False
    o.refine_principal_point = False
    o.refine_extra_params = False
    o.loss_function_type = LossFunctionType.SOFT_L1
    return o


# ----------------------------------------------------------------------------- config

class BundleAdjustmentConfig:
    """Which images / cameras / poses take part and which are constant
    (bundle_adjustment.cc:78-251).  Variable/constant *points* are not supported by the
    CUDA path (the global BA never adds any: sfm/global_mapper.cc:416-435)."""

    def __init__(self):
        self._images, self._const_cams, self._const_poses, self._const_tvecs = set(), set(), set(), {}

    def NumImages(self): return len(self._images)
    def NumConstantCameras(self): return len(self._const_cams)
    def NumConstantPoses(self): return len(self._const_poses)
    def NumConstantTvecs(self): return len(self._const_tvecs)
    def NumPoints(self): return 0
    def NumVariablePoints(self): return 0
    def NumConstantPoints(self): return 0

    def NumResiduals(self, reconstruction):
        return 2 * sum(int(np.count_nonzero(reconstruction.images[i].point3D_ids >= 0)) for i in self._images)

    def AddImage(self, image_id): self._images.add(image_id)
    def HasImage(self, image_id): return image_id in self._images
    def RemoveImage(self, image_id): self._images.discard(image_id)
    def SetConstantCamera(self, camera_id): self._const_cams.add(camera_id)
    def SetVariableCamera(self, camera_id): self._const_cams.discard(camera_id)
    def IsConstantCamera(self, camera_id): return camera_id in self._const_cams

    def SetConstantPose(self, image_id):
        if not self.HasImage(image_id) or self.HasConstantTvec(image_id):
            raise RuntimeError("SetConstantPose: image not added or has a constant tvec")   # CHECKs .cc:170-171
        self._const_poses.add(image_id)

    def SetVariablePose(self, image_id): self._const_poses.discard(image_id)
    def HasConstantPose(self, image_id): return image_id in self._const_poses

    def SetConstantTvec(self, image_id, idxs):
        idxs = list(idxs)
        if not (0 < len(idxs) <= 3) or not self.HasImage(image_id) or self.HasConstantPose(image_id) \
                or len(set(idxs)) != len(idxs):
            raise RuntimeError("SetConstantTvec: invalid arguments")   # CHECKs .cc:185-191
        self._const_tvecs[image_id] = idxs

    def RemoveConstantTvec(self, image_id): self._const_tvecs.pop(image_id, None)
    def HasConstantTvec(self, image_id): return image_id in self._const_tvecs
    def Images(self): return self._images
    def ConstantTvec(self, image_id): return self._const_tvecs[image_id]
    def VariablePoints(self): return set()
    def ConstantPoints(self): return set()


# ----------------------------------------------------------------------------- model container

@dataclass
class Camera:
    camera_id: int
    model_id: int
    width: int
    height: int
    params: np.ndarray          # SIMPLE_PINHOLE: f, cx, cy


@dataclass
class Image:
    image_id: int
    qvec: np.ndarray            # w, x, y, z
    tvec: np.ndarray
    camera_id: int
    name: str = ""
    xys: np.ndarray = None      # [n, 2] Point2D::XY()
    point3D_ids: np.ndarray = None   # [n] int64, -1 = no 3D point


@dataclass
class Point3D:
    point3D_id: int
    xyz: np.ndarray
    rgb: np.ndarray = None
    error: float = 0.0
    image_ids: np.ndarray = None
    point2D_idxs: np.ndarray = None


class Reconstruction:
    """The slice of colmap::Reconstruction the BA touches: cameras, registered images
    with their 2D observations, 3D points (base/reconstruction.h).  Same field names as
    sfm/colmap_utils/read_write_model.py so that models read from disk plug in."""

    def __init__(self, cameras=None, images=None, points3D=None, reg_image_ids=None):
        self.cameras, self.images, self.points3D = cameras or {}, images or {}, points3D or {}
        # reg_image_ids_ is REGISTRATION order in the reference (base/reconstruction.h); a model read
        # from disk registers its images in file order (ReadImagesBinary, reconstruction.cc:1733-1790).
        # The gauge of the global BA fixes reg[0] and reg[1] (sfm/global_mapper.cc:431-435), so the
        # order is part of the result.  Default: insertion order of `images`.
        self.reg_image_ids = list(reg_image_ids) if reg_image_ids is not None else None

    def RegImageIds(self):
        if self.reg_image_ids is not None:
            return [i for i in self.reg_image_ids if i in self.images]
        return list(self.images.keys())

    def NumRegImages(self):
        return len(self.RegImageIds())

    def ComputeNumObservations(self):
        """base/reconstruction.cc:756-762."""
        return int(sum(np.count_nonzero(self.images[i].point3D_ids >= 0) for i in self.RegImageIds()
                       if self.images[i].point3D_ids is not None))

    def DeletePoint3D(self, point3D_id):
        """base/reconstruction.cc:279-298: reset every Point2D of the track, erase the point."""
        p = self.points3D.pop(point3D_id, None)
        if p is None:
            return
        if p.image_ids is not None and len(p.image_ids):
            for iid, j in zip(p.image_ids, p.point2D_idxs):
                im = self.images.get(int(iid))
                if im is not None and im.point3D_ids is not None and im.point3D_ids[int(j)] == point3D_id:
                    im.point3D_ids[int(j)] = -1
        else:                                   # container built without tracks: search
            for im in self.images.values():
                if im.point3D_ids is not None:
                    im.point3D_ids[im.point3D_ids == point3D_id] = -1

    def DeleteObservation(self, image_id, point2D_idx):
        """base/reconstruction.cc:300-320: the whole point goes once its track length is <= 2;
        otherwise the track element is removed and the Point2D reset."""
        im = self.images[image_id]
        pid = int(im.point3D_ids[point2D_idx])
        p = self.points3D[pid]
        length = len(p.image_ids) if p.image_ids is not None else self._track_length(pid)
        if length <= 2:
            self.DeletePoint3D(pid)
            return
        if p.image_ids is not None:
            keep = ~((p.image_ids == image_id) & (p.point2D_idxs == point2D_idx))
            p.image_ids, p.point2D_idxs = p.image_ids[keep], p.point2D_idxs[keep]
        im.point3D_ids[point2D_idx] = -1

    def _track_length(self, point3D_id):
        return int(sum(np.count_nonzero(im.point3D_ids == point3D_id) for im in self.images.values()
                       if im.point3D_ids is not None))

    def FilterObservationsWithNegativeDepth(self):
        """base/reconstruction.cc:711-729: DeleteObservation for every Point2D whose point is not in
        front of its camera (HasPointPositiveDepth: P.row(2) . [X; 1] >= eps), images in registration
        order.  Returns the number of DeleteObservation calls, like the reference."""
        from .synthetic import qvec_to_rotmat
        eps = np.finfo(np.float64).eps
        n = 0
        for i in self.RegImageIds():
            im = self.images[i]
            if im.point3D_ids is None:
                continue
            R = qvec_to_rotmat(im.qvec / np.linalg.norm(im.qvec))
            for j in np.nonzero(im.point3D_ids >= 0)[0]:
                pid = int(im.point3D_ids[j])
                if pid < 0 or pid not in self.points3D:
                    continue                       # its point was deleted by an earlier call
                if R[2] @ self.points3D[pid].xyz + im.tvec[2] >= eps:
                    continue
                self.DeleteObservation(i, int(j))
                n += 1
        return n

    def Normalize(self, extent=10.0, p0=0.1, p1=0.9, use_images=True):
        """base/reconstruction.cc:373-468: per-axis sorted float32 camera-centre
        coordinates, P0 = floor(p0 (n-1)), P1 = floor(p1 (n-1)) (0 and n-1 when n <= 3); the
        box is [coords[P0], coords[P1]] per axis, the translation the mean of the sorted
        coordinates in P0..P1; scale = extent / |box diagonal|."""
        from .synthetic import camera_centres, qvec_to_rotmat
        ids = self.RegImageIds()
        if (use_images and len(ids) < 2) or (not use_images and len(self.points3D) < 2):
            return
        q = np.stack([self.images[i].qvec for i in ids])
        q = q / np.linalg.norm(q, axis=1, keepdims=True)
        t = np.stack([self.images[i].tvec for i in ids])
        cen = camera_centres(q, t)
        coords = cen if use_images else np.stack([p.xyz for p in self.points3D.values()])
        cs = np.sort(coords.astype(np.float32), axis=0)
        n = cs.shape[0]
        P0 = int(p0 * (n - 1)) if n > 3 else 0
        P1 = int(p1 * (n - 1)) if n > 3 else n - 1
        lo, hi = cs[P0].astype(np.float64), cs[P1].astype(np.float64)
        mean = np.zeros(3)
        for k in range(P0, P1 + 1):                 # accumulated sequentially, as the reference does
            mean += cs[k].astype(np.float64)
        mean /= (P1 - P0 + 1)
        old_extent = np.linalg.norm(hi - lo)
        scale = 1.0 if old_extent < np.finfo(np.float64).eps else extent / old_extent
        R = qvec_to_rotmat(q)
        for k, i in enumerate(ids):
            self.images[i].tvec = R[k] @ (-(cen[k] - mean) * scale)
        for p in self.points3D.values():
            p.xyz = (p.xyz - mean) * scale
        return mean, scale


def flatten(reconstruction, config):
    """BundleAdjuster::SetUp (bundle_adjustment.cc:326-447) as arrays: one observation per
    Point2D with a Point3D in an image of the config.  Returns (BAProblem, index maps)."""
    reg = reconstruction.RegImageIds()
    image_ids = [i for i in reg if config.HasImage(i)] + sorted(i for i in config.Images() if i not in set(reg))
    cam_ids = sorted({reconstruction.images[i].camera_id for i in image_ids})
    cam_index = {c: k for k, c in enumerate(cam_ids)}
    for c in cam_ids:
        if reconstruction.cameras[c].model_id != SIMPLE_PINHOLE:
            raise _lib.PsfmError("only SIMPLE_PINHOLE cameras are supported (the pipeline imports "
                                 "features with --ImageReader.camera_model SIMPLE_PINHOLE)")
    pt_ids = sorted(reconstruction.points3D.keys())
    pt_index = {p: k for k, p in enumerate(pt_ids)}
    obs_image, obs_point, obs_xy, obs_p2d = [], [], [], []
    for k, i in enumerate(image_ids):
        im = reconstruction.images[i]
        if im.point3D_ids is None:
            continue
        sel = np.nonzero(im.point3D_ids >= 0)[0]
        obs_p2d.append(sel.astype(np.int64))
        obs_image.append(np.full(sel.shape[0], k, np.int32))
        obs_point.append(np.array([pt_index[int(p)] for p in im.point3D_ids[sel]], np.int32))
        obs_xy.append(np.asarray(im.xys, np.float64)[sel])
    cat = (lambda l, shape, dt: np.concatenate(l) if l else np.zeros(shape, dt))
    # ParameterizePoints (bundle_adjustment.cc:546-552) holds constant every point whose track is longer
    # than its residuals in the problem (it is also seen by images outside the config).  The flattened
    # problem has no constant points (the global BA adds every registered image): refuse instead of
    # silently moving points the reference would hold fixed.
    if obs_point:
        in_cfg = np.bincount(np.concatenate(obs_point), minlength=len(pt_ids))
        for k, pid in enumerate(pt_ids):
            p3 = reconstruction.points3D[pid]
            if p3.image_ids is not None and in_cfg[k] and len(p3.image_ids) > in_cfg[k]:
                raise _lib.PsfmError(f"point {pid} is observed by images outside the BundleAdjustmentConfig: constant points "
                                     "(bundle_adjustment.cc:546-552) are not supported by the flattened problem")
    F = len(image_ids)
    pose_constant = np.array([config.HasConstantPose(i) for i in image_ids], np.uint8)
    tmask = np.zeros(F, np.uint8)
    for k, i in enumerate(image_ids):
        if config.HasConstantTvec(i):
            for j in config.ConstantTvec(i):
                tmask[k] |= (1 << j)
    prob = BAProblem(
        np.stack([reconstruction.images[i].qvec for i in image_ids]) if F else np.zeros((0, 4)),
        np.stack([reconstruction.images[i].tvec for i in image_ids]) if F else np.zeros((0, 3)),
        np.stack([reconstruction.points3D[p].xyz for p in pt_ids]) if pt_ids else np.zeros((0, 3)),
        np.stack([reconstruction.cameras[c].params[:3] for c in cam_ids]),
        cat(obs_image, (0,), np.int32), cat(obs_point, (0,), np.int32), cat(obs_xy, (0, 2), np.float64),
        np.array([cam_index[reconstruction.images[i].camera_id] for i in image_ids], np.int32),
        pose_constant, tmask, np.array([config.IsConstantCamera(c) for c in cam_ids], np.uint8))
    return prob, dict(image_ids=image_ids, cam_ids=cam_ids, pt_ids=pt_ids,
                      obs_point2D_idx=cat(obs_p2d, (0,), np.int64))


def apply_observation_mask(problem, maps, reconstruction, alive, point_errors=None):
    """Make the container agree with the solver's ALIVE mask (what the reference's filters did to
    its Tracks / Point2Ds): dead observations lose their point, points without observations are
    deleted, tracks are rebuilt from the survivors; Point3D::Error from the last point filter."""
    image_ids, pt_ids = maps["image_ids"], maps["pt_ids"]
    dead = np.nonzero(~alive)[0]
    for m in dead:
        im = reconstruction.images[image_ids[problem.obs_image[m]]]
        im.point3D_ids[maps["obs_point2D_idx"][m]] = -1
    tracks = {}
    for m in np.nonzero(alive)[0]:
        tracks.setdefault(int(problem.obs_point[m]), []).append((image_ids[problem.obs_image[m]], int(maps["obs_point2D_idx"][m])))
    for k, pid in enumerate(pt_ids):
        if k not in tracks:
            reconstruction.points3D.pop(pid, None)
            continue
        p = reconstruction.points3D[pid]
        p.image_ids = np.array([t[0] for t in tracks[k]], np.int32)
        p.point2D_idxs = np.array([t[1] for t in tracks[k]], np.int32)
        if point_errors is not None and not np.isnan(point_errors[k]):
            p.error = float(point_errors[k])


def scatter(problem, maps, reconstruction):
    for k, i in enumerate(maps["image_ids"]):
        reconstruction.images[i].qvec = problem.qvec[k].copy()
        reconstruction.images[i].tvec = problem.tvec[k].copy()
    for k, c in enumerate(maps["cam_ids"]):
        reconstruction.cameras[c].params[:3] = problem.cam_params[k]
    for k, p in enumerate(maps["pt_ids"]):
        reconstruction.points3D[p].xyz = problem.xyz[k].copy()


# ----------------------------------------------------------------------------- solver entry points

def solve_problem(problem, options_struct):
    """psfm_ba_solve on a flattened BAProblem (host buffers; in-place update)."""
    s = BASummary()
    st = problem.struct()
    _lib.check(_lib.lib().psfm_ba_solve(C.byref(st), C.byref(options_struct), C.byref(s)), "psfm_ba_solve")
    return s


class ResidentSolver:
    """Observations and structure uploaded once; state re-set / re-solved many times
    (the refinement loop of controllers/global_mapper.cc:253-268)."""

    def __init__(self, problem):
        self.problem = problem
        self._h = C.c_void_p()
        st = problem.struct()
        _lib.check(_lib.lib().psfm_ba_create(C.byref(st), C.byref(self._h)), "psfm_ba_create")

    def set_state(self, qvec=None, tvec=None, xyz=None, cam_params=None):
        a = [None if v is None else np.ascontiguousarray(v, np.float64) for v in (qvec, tvec, xyz, cam_params)]
        _lib.check(_lib.lib().psfm_ba_set_state(self._h, *[_lib.dptr(v) for v in a]), "psfm_ba_set_state")

    def run(self, options_struct):
        s = BASummary()
        _lib.check(_lib.lib().psfm_ba_run(self._h, C.byref(options_struct), C.byref(s)), "psfm_ba_run")
        return s

    def get_state(self):
        p = self.problem
        _lib.check(_lib.lib().psfm_ba_get_state(self._h, _lib.dptr(p.qvec), _lib.dptr(p.tvec), _lib.dptr(p.xyz),
                                                _lib.dptr(p.cam_params)), "psfm_ba_get_state")
        return p

    def evaluate(self, options_struct):
        p = self.problem
        cost = C.c_double()
        r = np.zeros((p.num_observations, 2))
        gc = np.zeros(6 * p.num_images + 3 * p.num_cameras)
        gp = np.zeros((p.num_points, 3))
        _lib.check(_lib.lib().psfm_ba_evaluate(self._h, C.byref(options_struct), C.byref(cost), _lib.dptr(r),
                                               _lib.dptr(gc), _lib.dptr(gp)), "psfm_ba_evaluate")
        return cost.value, r, gc, gp

    def linear_step(self, options_struct, radius):
        p = self.problem
        sc = np.zeros(6 * p.num_images + 3 * p.num_cameras)
        sp = np.zeros((p.num_points, 3))
        it = C.c_int32()
        _lib.check(_lib.lib().psfm_ba_linear_step(self._h, C.byref(options_struct), radius, _lib.dptr(sc),
                                                  _lib.dptr(sp), C.byref(it)), "psfm_ba_linear_step")
        return sc, sp, it.value

    # ---- the refinement loop around the BA, on the resident problem (csrc/ba_refine.cuh) ----
    def filter_negative_depth(self):
        """Reconstruction::FilterObservationsWithNegativeDepth; returns num_filtered."""
        n = C.c_int64()
        _lib.check(_lib.lib().psfm_ba_filter_negative_depth(self._h, C.byref(n)), "psfm_ba_filter_negative_depth")
        return n.value

    def filter_points(self, max_reproj_error=4.0, min_tri_angle=1.5):
        """Reconstruction::FilterAllPoints3D; returns num_filtered."""
        n = C.c_int64()
        _lib.check(_lib.lib().psfm_ba_filter_points(self._h, max_reproj_error, min_tri_angle, C.byref(n)),
                   "psfm_ba_filter_points")
        return n.value

    def normalize(self, extent=10.0, p0=0.1, p1=0.9):
        """Reconstruction::Normalize on the solver's state; returns (translation, scale)."""
        t, s = np.zeros(3), C.c_double()
        _lib.check(_lib.lib().psfm_ba_normalize(self._h, extent, p0, p1, _lib.dptr(t), C.byref(s)), "psfm_ba_normalize")
        return t, s.value

    def num_observations(self):
        n = C.c_int64()
        _lib.check(_lib.lib().psfm_ba_num_observations(self._h, C.byref(n)), "psfm_ba_num_observations")
        return n.value

    def observation_mask(self):
        m = np.zeros(self.problem.num_observations, np.uint8)
        _lib.check(_lib.lib().psfm_ba_get_observation_mask(self._h, m.ctypes.data_as(C.POINTER(C.c_uint8))),
                   "psfm_ba_get_observation_mask")
        return m.astype(bool)

    def point_errors(self):
        e = np.zeros(self.problem.num_points)
        _lib.check(_lib.lib().psfm_ba_get_point_errors(self._h, _lib.dptr(e)), "psfm_ba_get_point_errors")
        return e

    def iterative_refinement(self, options_struct, refine_options=None):
        """One IterativeGlobalRefinement pass (controllers/global_mapper.cc:245-271); returns the report."""
        rep = _abi.BARefineReport()
        ro = C.byref(refine_options) if refine_options is not None else None
        _lib.check(_lib.lib().psfm_ba_iterative_refinement(self._h, C.byref(options_struct), ro, C.byref(rep)),
                   "psfm_ba_iterative_refinement")
        return rep

    def close(self):
        if self._h:
            _lib.lib().psfm_ba_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class BundleAdjuster:
    """BundleAdjuster(options, config).Solve(reconstruction) — bundle_adjustment.cc:253-320."""

    def __init__(self, options, config):
        options.Check()
        self.options_, self.config_ = options, config
        self.summary_ = None
        self._used = False

    def Solve(self, reconstruction):
        if self._used:
            raise RuntimeError("Cannot use the same BundleAdjuster multiple times")   # CHECK .cc:261
        self._used = True
        problem, maps = flatten(reconstruction, self.config_)
        self.summary_ = solve_problem(problem, self.options_.to_struct())
        if problem.num_observations == 0:
            return False                                                              # .cc:268-271
        scatter(problem, maps, reconstruction)
        return True

    def Summary(self):
        return self.summary_


def adjust_global_bundle(reconstruction, force_update_rotation, ba_refine_focal_length=True,
                         ba_refine_principal_point=False, ba_refine_extra_params=False,
                         ba_fix_prior_rotation=False, ba_global_max_num_iterations=50, quiet=True,
                         linear_solver=_abi.SOLVER_AUTO):
    """AdjustGlobalBundle (controllers/global_mapper.cc:215-243) followed by
    GlobalMapper::AdjustGlobalBundle (sfm/global_mapper.cc:402-448)."""
    o = global_bundle_adjustment_options(ba_global_max_num_iterations)
    if force_update_rotation:
        o.refine_rotation = not ba_fix_prior_rotation
        o.refine_focal_length = ba_refine_focal_length
        o.refine_principal_point = ba_refine_principal_point
        o.refine_extra_params = ba_refine_extra_params
    reg = reconstruction.RegImageIds()
    if len(reg) < 10:                      # kMinNumRegImagesForFastBA (:226-235)
        so = o.solver_options
        so.function_tolerance /= 10
        so.gradient_tolerance /= 10
        so.parameter_tolerance /= 10
        so.max_num_iterations *= 2
        so.max_linear_solver_iterations = 200
    if quiet:
        o.print_summary = False
        o.solver_options.minimizer_progress_to_stdout = False
    o.solver_options.linear_solver = linear_solver
    if len(reg) < 2:
        raise RuntimeError("At least two images must be registered for global bundle-adjustment")
    reconstruction.FilterObservationsWithNegativeDepth()
    cfg = BundleAdjustmentConfig()
    for i in reg:
        cfg.AddImage(i)
    cfg.SetConstantPose(reg[0])            # fix 7 DoF (sfm/global_mapper.cc:431-435)
    cfg.SetConstantTvec(reg[1], [0])
    ba = BundleAdjuster(o, cfg)
    if not ba.Solve(reconstruction):
        return False, ba.Summary()
    reconstruction.Normalize()
    return True, ba.Summary()


def _global_ba_options(force_update_rotation, ba_refine_focal_length, ba_refine_principal_point, ba_refine_extra_params,
                       ba_fix_prior_rotation, ba_global_max_num_iterations, quiet, linear_solver):
    o = global_bundle_adjustment_options(ba_global_max_num_iterations)
    if force_update_rotation:
        o.refine_rotation = not ba_fix_prior_rotation
        o.refine_focal_length = ba_refine_focal_length
        o.refine_principal_point = ba_refine_principal_point
        o.refine_extra_params = ba_refine_extra_params
    if quiet:
        o.print_summary = False
        o.solver_options.minimizer_progress_to_stdout = False
    o.solver_options.linear_solver = linear_solver
    return o


def iterative_global_refinement(reconstruction, force_update_rotation, ba_refine_focal_length=True,
                                ba_refine_principal_point=False, ba_refine_extra_params=False,
                                ba_fix_prior_rotation=False, ba_global_max_num_iterations=50,
                                ba_global_max_refinements=5, ba_global_max_refinement_change=0.0005,
                                filter_max_reproj_error=4.0, filter_min_tri_angle=1.5, quiet=True,
                                linear_solver=_abi.SOLVER_AUTO):
    """IterativeGlobalRefinement (controllers/global_mapper.cc:245-271) on a Reconstruction: the whole
    loop — negative-depth filter, BA, Normalize, FilterAllPoints3D, <= 5 rounds — runs on the resident
    device problem (psfm_ba_iterative_refinement); the container is updated once at the end.  The
    IncrementalTriangulator steps of the reference (CompleteAndMergeTracks, Retriangulate) and
    FilterImages are not part of this library.  Returns the BARefineReport."""
    reg = reconstruction.RegImageIds()
    if len(reg) < 2:
        raise RuntimeError("At least two images must be registered for global bundle-adjustment")
    o = _global_ba_options(force_update_rotation, ba_refine_focal_length, ba_refine_principal_point,
                           ba_refine_extra_params, ba_fix_prior_rotation, ba_global_max_num_iterations, quiet,
                           linear_solver)
    cfg = BundleAdjustmentConfig()
    for i in reg:
        cfg.AddImage(i)
    cfg.SetConstantPose(reg[0])            # fix 7 DoF (sfm/global_mapper.cc:431-435)
    cfg.SetConstantTvec(reg[1], [0])
    problem, maps = flatten(reconstruction, cfg)
    ro = _abi.BARefineOptions()
    _lib.lib().psfm_ba_default_refine_options(C.byref(ro))
    ro.max_refinements = ba_global_max_refinements
    ro.max_refinement_change = ba_global_max_refinement_change
    ro.filter_max_reproj_error = filter_max_reproj_error
    ro.filter_min_tri_angle = filter_min_tri_angle
    S = ResidentSolver(problem)
    try:
        rep = S.iterative_refinement(o.to_struct(), ro)
        S.get_state()
        alive = S.observation_mask()
        err = S.point_errors()
    finally:
        S.close()
    scatter(problem, maps, reconstruction)
    apply_observation_mask(problem, maps, reconstruction, alive, err)
    return rep


# ----------------------------------------------------------------------------- triangulation -> BA -> model on the device

class TriangulationModel:
    """What psfm_ba_get_model returns, in the triangulation's layout (image / camera index, point row = point id - 1):
    qvec [F][4], tvec [F][3], cam_params [C][3], xyz [P][3], track_ptr [P + 1] (length 0: a deleted point),
    track_image / track_point2D [E], point3D_of_keypoint [K] (row, -1), error [P] (Point3D::Error, 0 where no point
    filter set it)."""

    def __init__(self, **arrays):
        self.__dict__.update(arrays)


class TriangulationSolver:
    """The resident problem of an init_geometry.ResidentTriangulation (psfm_ba_create_from_triangulation): the problem
    `flatten` builds from Triangulation.to_reconstruction with every registered image in the config, built on the
    device.  qvec [F][4], tvec [F][3] and cam_params [C][3] are indexed like the triangulation's inputs; the masks too
    (None: nothing constant).  The refinement loop and its filters act on it as on a ResidentSolver; get_model()
    compacts the surviving observations into tracks on the device.  num_images / num_cameras / num_observations are the
    problem's sizes as created; num_alive() counts the observations still in the problem."""

    def __init__(self, triangulation, qvec, tvec, cam_params, pose_constant=None, tvec_constant_mask=None,
                 camera_constant=None):
        self._h = C.c_void_p()
        self._q = np.ascontiguousarray(qvec, np.float64).reshape(-1, 4)
        self._t = np.ascontiguousarray(tvec, np.float64).reshape(-1, 3)
        self._k = np.ascontiguousarray(cam_params, np.float64).reshape(-1, 3)
        u8 = C.POINTER(C.c_uint8)
        masks = [None if m is None else np.ascontiguousarray(m, np.uint8) for m in (pose_constant, tvec_constant_mask, camera_constant)]
        for m, n in zip(masks, (len(self._q), len(self._q), len(self._k))):
            if m is not None and m.shape != (n,):
                raise ValueError("pose_constant / tvec_constant_mask need one entry per image, camera_constant per camera")
        if len(self._t) != len(self._q):
            raise ValueError("qvec and tvec must describe the same images")
        F, Cn, M = C.c_int32(), C.c_int32(), C.c_int64()
        _lib.check(_lib.lib().psfm_ba_create_from_triangulation(
            triangulation.handle, _lib.dptr(self._q), _lib.dptr(self._t), _lib.dptr(self._k),
            *(m.ctypes.data_as(u8) if m is not None else None for m in masks), C.byref(self._h), C.byref(F), C.byref(Cn),
            C.byref(M)), "psfm_ba_create_from_triangulation")
        self.num_images, self.num_cameras, self.num_observations = F.value, Cn.value, M.value
        self.num_points = triangulation.num_points3D

    # the entry points that only need the handle are ResidentSolver's
    filter_negative_depth = ResidentSolver.filter_negative_depth
    filter_points = ResidentSolver.filter_points
    normalize = ResidentSolver.normalize
    iterative_refinement = ResidentSolver.iterative_refinement
    num_alive = ResidentSolver.num_observations
    close = ResidentSolver.close
    __del__ = ResidentSolver.__del__

    def observation_mask(self):
        """alive [num_observations] bool over the observations the problem was created with."""
        m = np.zeros(self.num_observations, np.uint8)
        _lib.check(_lib.lib().psfm_ba_get_observation_mask(self._h, m.ctypes.data_as(C.POINTER(C.c_uint8))),
                   "psfm_ba_get_observation_mask")
        return m.astype(bool)

    def observations(self):
        """The observations the problem was built with: obs_image [M] (problem image = rank among the registered
        images), obs_point [M] (point row), obs_xy [M][2], point2D_idx [M]."""
        M = self.num_observations
        img, pt, p2d, xy = np.zeros(M, np.int32), np.zeros(M, np.int32), np.zeros(M, np.int32), np.zeros((M, 2))
        ip = C.POINTER(C.c_int32)
        _lib.check(_lib.lib().psfm_ba_get_observations(self._h, img.ctypes.data_as(ip), pt.ctypes.data_as(ip), _lib.dptr(xy),
                                                       p2d.ctypes.data_as(ip)), "psfm_ba_get_observations")
        return img, pt, xy, p2d

    def point_errors(self):
        e = np.zeros(self.num_points)
        _lib.check(_lib.lib().psfm_ba_get_point_errors(self._h, _lib.dptr(e)), "psfm_ba_get_point_errors")
        return e

    def get_model(self, num_keypoints):
        """TriangulationModel of the solver's current state; num_keypoints: the triangulation's K."""
        P, M = self.num_points, self.num_observations
        q, t, k = self._q.copy(), self._t.copy(), self._k.copy()
        xyz, track_ptr = np.zeros((P, 3)), np.zeros(P + 1, np.int64)
        ti, tp = np.zeros(M, np.int32), np.zeros(M, np.int32)
        p3 = np.zeros(int(num_keypoints), np.int64)
        ip, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
        _lib.check(_lib.lib().psfm_ba_get_model(self._h, _lib.dptr(q), _lib.dptr(t), _lib.dptr(k), _lib.dptr(xyz),
                                                track_ptr.ctypes.data_as(i64), ti.ctypes.data_as(ip), tp.ctypes.data_as(ip),
                                                p3.ctypes.data_as(i64)), "psfm_ba_get_model")
        E = int(track_ptr[-1])
        err = self.point_errors()
        return TriangulationModel(qvec=q, tvec=t, cam_params=k, xyz=xyz, track_ptr=track_ptr, track_image=ti[:E].copy(),
                                  track_point2D=tp[:E].copy(), point3D_of_keypoint=p3,
                                  error=np.where(np.isnan(err), 0.0, err))
