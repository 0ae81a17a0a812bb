"""Host mirror of the two batched initialisation ops of SURVEY.md 8(f) row f-4 (csrc/init_geometry.cu).

Names and argument meaning follow the reference:
* `optimize_relative_position_with_known_rotation(points1, points2, rotation1, rotation2)` —
  OptimizeRelativePositionWithKnownRotation, sfm/gmapper/src/global/known_rotation_util.cc:107-196
  (normalised image points, quaternions (w, x, y, z); returns the unit relative position);
* `batch_optimize_relative_position_with_known_rotation(pairs)` — BatchOptimize..., :198-229, every pair in
  one launch instead of one ThreadPool task per pair;
* `triangulate_multi_view_points(tracks)` — the multi-view DLT behind IncrementalTriangulator::Create
  (sfm/incremental_triangulator.cc:463-548), every track in one launch;
* `estimate_relative_poses(...)` — TwoViewGeometry::EstimateRelativePose (estimators/two_view_geometry.cc:172-239)
  of every verified pair in one call, instead of the ThreadPool loop of DatabaseCache::Load
  (base/database_cache.cc:206-228); its inputs are what `handoff.read_two_view_geometries` reads from a database;
* `estimate_global_rotations(...)` — EstimateGlobalRotations (global/robust_rotation_estimator.cc:310-331), the
  first step of the global mapper: pair relative rotations in, one orientation per image out, which
  `batch_optimize_relative_position_with_known_rotation` takes as its rotations.
There is no CPU fallback: the library raises without a CUDA device."""
import ctypes as C

import numpy as np

from . import _abi, _lib


def _ptr(sizes):
    p = np.zeros(len(sizes) + 1, np.int32)
    np.cumsum(sizes, out=p[1:])
    return p


def batch_optimize_relative_position_with_known_rotation(pairs, return_iterations=False):
    """pairs: sequence of (points1 [n][2], points2 [n][2], rotation1 [4], rotation2 [4]); returns [len(pairs)][3]."""
    pairs = list(pairs)
    n = len(pairs)
    tvec = np.zeros((n, 3))
    its = np.zeros(n, np.int32)
    if n == 0:
        return (tvec, its) if return_iterations else tvec
    for a, b, _, _ in pairs:
        if np.shape(a) != np.shape(b):
            raise ValueError("points1 and points2 must have the same shape")       # CHECK_EQ, known_rotation_util.cc:115
    ptr = _ptr([len(a) for a, _, _, _ in pairs])
    p1 = np.ascontiguousarray(np.concatenate([np.asarray(a, np.float64).reshape(-1, 2) for a, _, _, _ in pairs]))
    p2 = np.ascontiguousarray(np.concatenate([np.asarray(b, np.float64).reshape(-1, 2) for _, b, _, _ in pairs]))
    q1 = np.ascontiguousarray(np.array([np.asarray(q, np.float64) for _, _, q, _ in pairs]).reshape(n, 4))
    q2 = np.ascontiguousarray(np.array([np.asarray(q, np.float64) for _, _, _, q in pairs]).reshape(n, 4))
    ip = C.POINTER(C.c_int32)
    _lib.check(_lib.lib().psfm_known_rotation_translations(_lib.dptr(p1), _lib.dptr(p2), ptr.ctypes.data_as(ip), _lib.dptr(q1),
                                                           _lib.dptr(q2), n, _lib.dptr(tvec), its.ctypes.data_as(ip)),
               "psfm_known_rotation_translations")
    return (tvec, its) if return_iterations else tvec


def optimize_relative_position_with_known_rotation(points1, points2, rotation1, rotation2):
    return batch_optimize_relative_position_with_known_rotation([(points1, points2, rotation1, rotation2)])[0]


def triangulate_multi_view_points(tracks):
    """tracks: sequence of (proj_matrices [v][3][4], points [v][2] normalised); returns [len(tracks)][3]."""
    tracks = list(tracks)
    n = len(tracks)
    xyz = np.zeros((n, 3))
    if n == 0:
        return xyz
    ptr = _ptr([len(p) for p, _ in tracks])
    P = np.ascontiguousarray(np.concatenate([np.asarray(p, np.float64).reshape(-1, 12) for p, _ in tracks]))
    x = np.ascontiguousarray(np.concatenate([np.asarray(q, np.float64).reshape(-1, 2) for _, q in tracks]))
    if len(P) != len(x):
        raise ValueError("one image point per projection matrix")
    _lib.check(_lib.lib().psfm_triangulate_tracks(_lib.dptr(P), _lib.dptr(x), ptr.ctypes.data_as(C.POINTER(C.c_int32)), n, _lib.dptr(xyz)),
               "psfm_triangulate_tracks")
    return xyz


class RelativePoses:
    """Per pair: qvec [R][4] (w, x, y, z), tvec [R][3], tri_angle [R] (radians), config [R] (PLANAR_OR_PANORAMIC
    resolved), num_points3D [R] int64, estimated [R] bool (False: config not estimable, everything else zero)."""

    def __init__(self, qvec, tvec, tri_angle, config, num_points3D, estimated):
        self.qvec, self.tvec, self.tri_angle = qvec, tvec, tri_angle
        self.config, self.num_points3D, self.estimated = config, num_points3D, estimated


def estimate_relative_poses(keypoint_ptr, keypoints, image_camera, cameras, pair_images, config, E, F, H, inlier_ptr,
                            inlier_matches):
    """keypoint_ptr [F + 1] (image f owns keypoints keypoint_ptr[f] .. keypoint_ptr[f + 1]), keypoints [K][2] (as
    stored in the database), image_camera [F], cameras [C][3] SIMPLE_PINHOLE (f, cx, cy), pair_images [R][2] image
    indices, config [R], E / F / H [R][3][3], inlier_ptr [R + 1], inlier_matches [N][2] (keypoint in image 1,
    keypoint in image 2).  Returns RelativePoses (psfm_two_view_relative_poses, csrc/two_view.cu)."""
    kp_ptr = np.ascontiguousarray(keypoint_ptr, np.int64)
    kps = np.ascontiguousarray(keypoints, np.float32).reshape(-1, 2)
    cam_of = np.ascontiguousarray(image_camera, np.int32)
    cams = np.ascontiguousarray(cameras, np.float64).reshape(-1, 3)
    pairs = np.ascontiguousarray(pair_images, np.int32).reshape(-1, 2)
    cfg = np.ascontiguousarray(config, np.int32)
    R = cfg.shape[0]
    E, F, H = (np.ascontiguousarray(m, np.float64).reshape(R, 9) for m in (E, F, H))
    iptr = np.ascontiguousarray(inlier_ptr, np.int64)
    m = np.ascontiguousarray(inlier_matches, np.uint32).reshape(-1, 2)
    num_images = kp_ptr.shape[0] - 1
    if pairs.shape[0] != R or iptr.shape[0] != R + 1 or cam_of.shape[0] != num_images:
        raise ValueError("pair_images, config, E, F, H and inlier_ptr must describe the same pairs, image_camera the same images")
    if iptr[-1] != m.shape[0] or kp_ptr[-1] != kps.shape[0]:
        raise ValueError("inlier_ptr / keypoint_ptr must end at the number of matches / keypoints")
    out = RelativePoses(np.zeros((R, 4)), np.zeros((R, 3)), np.zeros(R), np.zeros(R, np.int32), np.zeros(R, np.int64),
                        np.zeros(R, np.uint8))
    i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    _lib.check(_lib.lib().psfm_two_view_relative_poses(
        num_images, kp_ptr.ctypes.data_as(i64), kps.ctypes.data_as(C.POINTER(C.c_float)), cam_of.ctypes.data_as(i32),
        _lib.dptr(cams), cams.shape[0], R, pairs.ctypes.data_as(i32), cfg.ctypes.data_as(i32), _lib.dptr(E), _lib.dptr(F),
        _lib.dptr(H), iptr.ctypes.data_as(i64), m.ctypes.data_as(C.POINTER(C.c_uint32)), _lib.dptr(out.qvec),
        _lib.dptr(out.tvec), _lib.dptr(out.tri_angle), out.config.ctypes.data_as(i32), out.num_points3D.ctypes.data_as(i64),
        out.estimated.ctypes.data_as(C.POINTER(C.c_uint8))), "psfm_two_view_relative_poses")
    out.estimated = out.estimated.astype(bool)
    return out


class RobustRotationEstimatorOptions:
    """RobustRotationEstimator::Options (global/robust_rotation_estimator.h:61-89) with the reference's names and
    defaults, which are what sfm/main_sfm.py runs."""

    def __init__(self, max_num_l1_iterations=5, l1_step_convergence_threshold=0.001, max_num_irls_iterations=100,
                 irls_step_convergence_threshold=0.001, irls_loss_parameter_sigma=np.deg2rad(5.0),
                 rotation_filter_max_degrees=5.0):
        self.max_num_l1_iterations = max_num_l1_iterations
        self.l1_step_convergence_threshold = l1_step_convergence_threshold
        self.max_num_irls_iterations = max_num_irls_iterations
        self.irls_step_convergence_threshold = irls_step_convergence_threshold
        self.irls_loss_parameter_sigma = irls_loss_parameter_sigma
        self.rotation_filter_max_degrees = rotation_filter_max_degrees

    def to_struct(self):
        return _abi.RotationOptions(*(getattr(self, n) for n, _ in _abi.RotationOptions._fields_))


class GlobalRotations:
    """orientations [F][4] (w, x, y, z world-to-camera; zero where has_orientation is False), has_orientation [F]
    bool, pair_kept [R] bool, success (False where the reference returns false: no posed pair, or a failed
    factorisation), summary (dict of psfm_rotation_summary; admm_iterations trimmed to num_l1_rounds)."""

    def __init__(self, orientations, has_orientation, pair_kept, success, summary):
        self.orientations, self.has_orientation, self.pair_kept = orientations, has_orientation, pair_kept
        self.success, self.summary = success, summary


def estimate_global_rotations(num_images, pair_images, qvec, num_correspondences, has_pose=None, options=None):
    """pair_images [R][2] image indices (image 1, image 2; images ordered by id), qvec [R][4] relative rotations 2_R_1
    (w, x, y, z), num_correspondences [R], has_pose [R] (None: every pair), options RobustRotationEstimatorOptions
    (None: the defaults).  Returns GlobalRotations (psfm_estimate_global_rotations, csrc/rotation_averaging.cu).
    From `RelativePoses`: has_pose = poses.estimated, num_correspondences = np.diff(inlier_ptr)."""
    pairs = np.ascontiguousarray(pair_images, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    q = np.ascontiguousarray(qvec, np.float64).reshape(-1, 4)
    nc = np.ascontiguousarray(num_correspondences, np.int32)
    if q.shape[0] != R or nc.shape != (R,):
        raise ValueError("pair_images, qvec and num_correspondences must describe the same pairs")
    hp = None
    if has_pose is not None:
        hp = np.ascontiguousarray(has_pose, np.uint8)
        if hp.shape != (R,):
            raise ValueError("has_pose must have one entry per pair")
    opts = (options or RobustRotationEstimatorOptions()).to_struct()
    F = int(num_images)
    orientations = np.zeros((F, 4))
    has_orientation = np.zeros(F, np.uint8)
    pair_kept = np.zeros(R, np.uint8)
    s = _abi.RotationSummary()
    u8 = C.POINTER(C.c_uint8)
    i32 = C.POINTER(C.c_int32)
    rc = _lib.check(_lib.lib().psfm_estimate_global_rotations(
        F, R, pairs.ctypes.data_as(i32), _lib.dptr(q), nc.ctypes.data_as(i32),
        hp.ctypes.data_as(u8) if hp is not None else None, C.byref(opts), _lib.dptr(orientations),
        has_orientation.ctypes.data_as(u8), pair_kept.ctypes.data_as(u8), C.byref(s)), "psfm_estimate_global_rotations")
    summary = {n: getattr(s, n) for n, _ in _abi.RotationSummary._fields_}
    summary["admm_iterations"] = list(s.admm_iterations)[:s.num_l1_rounds]
    return GlobalRotations(orientations, has_orientation.astype(bool), pair_kept.astype(bool), rc == 0, summary)
