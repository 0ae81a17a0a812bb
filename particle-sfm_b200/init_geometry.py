"""Host mirror of the two batched initialisation ops of SURVEY.md 8(f) row f-4 (csrc/init_geometry.cu).

Names and argument meaning follow the reference:
* `optimize_relative_position_with_known_rotation(points1, points2, rotation1, rotation2)` —
  OptimizeRelativePositionWithKnownRotation, sfm/gmapper/src/global/known_rotation_util.cc:107-196
  (normalised image points, quaternions (w, x, y, z); returns the unit relative position);
* `batch_optimize_relative_position_with_known_rotation(pairs)` — BatchOptimize..., :198-229, every pair in
  one launch instead of one ThreadPool task per pair;
* `triangulate_multi_view_points(tracks)` — the multi-view DLT behind IncrementalTriangulator::Create
  (sfm/incremental_triangulator.cc:463-548), every track in one launch;
* `verify_two_view_geometries(...)` — the geometric verification of `colmap matches_importer --match_type pairs`
  (TwoViewGeometryVerifier -> TwoViewGeometry::EstimateUncalibrated) of every pair in one call: raw matches in, config,
  F, H and inlier matches out, which `TwoViewVerification.to_two_view_geometries` hands to the next step;
* `estimate_relative_poses(...)` — TwoViewGeometry::EstimateRelativePose (estimators/two_view_geometry.cc:172-239)
  of every verified pair in one call, instead of the ThreadPool loop of DatabaseCache::Load
  (base/database_cache.cc:206-228); its inputs are what `handoff.read_two_view_geometries` reads from a database;
* `estimate_global_rotations(...)` — EstimateGlobalRotations (global/robust_rotation_estimator.cc:310-331), the
  first step of the global mapper: pair relative rotations in, one orientation per image out, which
  `batch_optimize_relative_position_with_known_rotation` takes as its rotations;
* `optimize_pairwise_translations(...)` — GlobalMapper::OptimizePairwiseTranslations (sfm/global_mapper.cc:106-109):
  the known-rotation translations of every kept pair, straight from the database arrays;
* `estimate_global_positions(...)` — GlobalMapper::EstimatePositions (sfm/global_mapper.cc:111-132) with the default
  method "lud" and the pose update of RegisterAllImages: camera centres and image tvecs;
* `triangulate_all_points(...)` — GlobalMapper::TriangulateAllPoints (sfm/global_mapper.cc:232-247): the 3D points and
  tracks of every registered image, and `Triangulation.to_reconstruction` the ba.Reconstruction the global BA takes.
There is no CPU fallback: the library raises without a CUDA device."""
import ctypes as C

import numpy as np

from . import _abi, _lib


def _ptr(sizes):
    p = np.zeros(len(sizes) + 1, np.int32)
    np.cumsum(sizes, out=p[1:])
    return p


def _pair_graph(keypoint_ptr, keypoints, image_camera, pair_images, ptr, matches):
    """The image-pair graph the pair stages take, as the library reads it: keypoint_ptr [F + 1] int64, keypoints [K][2]
    float32, image_camera [F] int32, pair_images [R][2] int32, ptr [R + 1] int64 (inlier_ptr or match_ptr) and
    matches [N][2] uint32, all contiguous.  Raises ValueError when the sizes do not describe one graph."""
    kp_ptr = np.ascontiguousarray(keypoint_ptr, np.int64)
    kps = np.ascontiguousarray(keypoints, np.float32).reshape(-1, 2)
    cam_of = np.ascontiguousarray(image_camera, np.int32)
    pairs = np.ascontiguousarray(pair_images, np.int32).reshape(-1, 2)
    ptr = np.ascontiguousarray(ptr, np.int64)
    m = np.ascontiguousarray(matches, np.uint32).reshape(-1, 2)
    if ptr.shape[0] != pairs.shape[0] + 1 or cam_of.shape[0] != kp_ptr.shape[0] - 1:
        raise ValueError("the match pointer must have one entry per pair and one more, image_camera one per image")
    if ptr[-1] != m.shape[0] or kp_ptr[-1] != kps.shape[0]:
        raise ValueError("the match pointer / keypoint_ptr must end at the number of matches / keypoints")
    return kp_ptr, kps, cam_of, pairs, ptr, m


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
    kp_ptr, kps, cam_of, pairs, iptr, m = _pair_graph(keypoint_ptr, keypoints, image_camera, pair_images, inlier_ptr,
                                                      inlier_matches)
    cams = np.ascontiguousarray(cameras, np.float64).reshape(-1, 3)
    cfg = np.ascontiguousarray(config, np.int32)
    R = cfg.shape[0]
    E, F, H = (np.ascontiguousarray(m, np.float64).reshape(R, 9) for m in (E, F, H))
    num_images = kp_ptr.shape[0] - 1
    if pairs.shape[0] != R:
        raise ValueError("pair_images, config, E, F and H must describe the same pairs")
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


def optimize_pairwise_translations(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr, inlier_matches,
                                   orientations, pair_used=None, return_iterations=False):
    """GlobalMapper::OptimizePairwiseTranslations (sfm/global_mapper.cc:106-109): every used pair's translation
    direction re-estimated from all of its inlier matches under the image orientations (OptimizeRelativePositionWith
    KnownRotation per pair, known_rotation_util.cc:195-229).  Images and pairs as `estimate_relative_poses` takes them
    (keypoints normalised on the device with the SIMPLE_PINHOLE camera, (x - cx) / f); orientations [F][4] (w, x, y, z
    world-to-camera, `GlobalRotations.orientations`), pair_used [R] (None: every pair; normally
    `GlobalRotations.pair_kept`).  Returns tvec [R][3] (zeros for unused pairs), and the IRLS iterations [R] with
    return_iterations (psfm_optimize_pairwise_translations, csrc/init_geometry.cu)."""
    kp_ptr, kps, cam_of, pairs, iptr, m = _pair_graph(keypoint_ptr, keypoints, image_camera, pair_images, inlier_ptr,
                                                      inlier_matches)
    cams = np.ascontiguousarray(cameras, np.float64).reshape(-1, 3)
    R = pairs.shape[0]
    q = np.ascontiguousarray(orientations, np.float64).reshape(-1, 4)
    num_images = kp_ptr.shape[0] - 1
    if q.shape[0] != num_images:
        raise ValueError("orientations must have one entry per image")
    used = None
    if pair_used is not None:
        used = np.ascontiguousarray(pair_used, np.uint8)
        if used.shape != (R,):
            raise ValueError("pair_used must have one entry per pair")
    tvec, its = np.zeros((R, 3)), np.zeros(R, np.int32)
    i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    _lib.check(_lib.lib().psfm_optimize_pairwise_translations(
        num_images, kp_ptr.ctypes.data_as(i64), kps.ctypes.data_as(C.POINTER(C.c_float)), cam_of.ctypes.data_as(i32),
        _lib.dptr(cams), cams.shape[0], R, pairs.ctypes.data_as(i32), iptr.ctypes.data_as(i64),
        m.ctypes.data_as(C.POINTER(C.c_uint32)), _lib.dptr(q), used.ctypes.data_as(C.POINTER(C.c_uint8)) if used is not None else None,
        _lib.dptr(tvec), its.ctypes.data_as(i32)), "psfm_optimize_pairwise_translations")
    return (tvec, its) if return_iterations else tvec


class ConstrainedL1SolverOptions:
    """theia::ConstrainedL1Solver::Options, which the reference's LUD estimator constructs with its defaults
    (least_unsquared_deviation_position_estimator.cc:161).  A field left None takes the library's default
    (psfm_lud_default_options; the defaults are recalled, not vendored: csrc/position_recalled.cuh)."""

    def __init__(self, max_num_iterations=None, rho=None, alpha=None, absolute_tolerance=None, relative_tolerance=None):
        self.max_num_iterations = max_num_iterations
        self.rho = rho
        self.alpha = alpha
        self.absolute_tolerance = absolute_tolerance
        self.relative_tolerance = relative_tolerance

    def to_struct(self):
        o = _abi.LudOptions()
        _lib.lib().psfm_lud_default_options(C.byref(o))
        for n, _ in _abi.LudOptions._fields_:
            if getattr(self, n) is not None:
                setattr(o, n, getattr(self, n))
        return o


class GlobalPositions:
    """positions [F][3] camera centres (zero where has_position is False), has_position [F] bool (the images of the
    used pairs), image_tvec [F][3] = -R c (RegisterAllImages), scales [R] (0 for unused pairs), summary (dict of
    psfm_position_summary)."""

    def __init__(self, positions, has_position, image_tvec, scales, summary):
        self.positions, self.has_position, self.image_tvec = positions, has_position, image_tvec
        self.scales, self.summary = scales, summary


def estimate_global_positions(num_images, pair_images, tvec, orientations, has_orientation=None, pair_used=None,
                              options=None):
    """GlobalMapper::EstimatePositions (sfm/global_mapper.cc:111-132) with the default method "lud", then the pose
    update of RegisterAllImages (:140-160).  pair_images [R][2] (image 1, image 2), tvec [R][3] pair translation
    directions (`optimize_pairwise_translations`), orientations [F][4] (w, x, y, z world-to-camera), has_orientation [F]
    (None: every image), pair_used [R] (None: every pair), options ConstrainedL1SolverOptions (None: the defaults).
    The gauge is the smallest image index of the used pairs, at the origin.  Returns GlobalPositions
    (psfm_estimate_global_positions, csrc/position_estimation.cu)."""
    pairs = np.ascontiguousarray(pair_images, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    t = np.ascontiguousarray(tvec, np.float64).reshape(-1, 3)
    q = np.ascontiguousarray(orientations, np.float64).reshape(-1, 4)
    F = int(num_images)
    if t.shape[0] != R or q.shape[0] != F:
        raise ValueError("pair_images and tvec must describe the same pairs, orientations num_images images")
    u8 = C.POINTER(C.c_uint8)
    masks = []
    for name, mask, size in (("has_orientation", has_orientation, F), ("pair_used", pair_used, R)):
        if mask is None:
            masks.append(None)
            continue
        a = np.ascontiguousarray(mask, np.uint8)
        if a.shape != (size,):
            raise ValueError("%s must have one entry per %s" % (name, "image" if size == F else "pair"))
        masks.append(a)
    opts = (options or ConstrainedL1SolverOptions()).to_struct()
    out = GlobalPositions(np.zeros((F, 3)), np.zeros(F, np.uint8), np.zeros((F, 3)), np.zeros(R), None)
    s = _abi.PositionSummary()
    _lib.check(_lib.lib().psfm_estimate_global_positions(
        F, R, pairs.ctypes.data_as(C.POINTER(C.c_int32)), _lib.dptr(t), _lib.dptr(q),
        *(m.ctypes.data_as(u8) if m is not None else None for m in masks), C.byref(opts), _lib.dptr(out.positions),
        out.has_position.ctypes.data_as(u8), _lib.dptr(out.image_tvec), _lib.dptr(out.scales), C.byref(s)),
        "psfm_estimate_global_positions")
    out.has_position = out.has_position.astype(bool)
    out.summary = {n: getattr(s, n) for n, _ in _abi.PositionSummary._fields_}
    return out


class IncrementalTriangulatorOptions:
    """IncrementalTriangulator::Options (sfm/incremental_triangulator.h:46-89): the fields TriangulateImage reads, with
    the reference's names.  A field left None takes the library's default (psfm_triangulator_default_options)."""

    def __init__(self, max_transitivity=None, create_max_angle_error=None, continue_max_angle_error=None, min_angle=None,
                 ignore_two_view_tracks=None, min_focal_length_ratio=None, max_focal_length_ratio=None,
                 max_extra_param=None):
        self.max_transitivity = max_transitivity
        self.create_max_angle_error = create_max_angle_error
        self.continue_max_angle_error = continue_max_angle_error
        self.min_angle = min_angle
        self.ignore_two_view_tracks = ignore_two_view_tracks
        self.min_focal_length_ratio = min_focal_length_ratio
        self.max_focal_length_ratio = max_focal_length_ratio
        self.max_extra_param = max_extra_param

    def to_struct(self):
        o = _abi.TriangulatorOptions()
        _lib.lib().psfm_triangulator_default_options(C.byref(o))
        for n, _ in _abi.TriangulatorOptions._fields_:
            if getattr(self, n) is not None:
                setattr(o, n, int(getattr(self, n)) if n == "ignore_two_view_tracks" else getattr(self, n))
        return o


class Triangulation:
    """Points in the reference's AddPoint3D order (point id = row + 1): xyz [P][3], track_ptr [P + 1], track_image /
    track_point2D [E] (image index, keypoint index in that image) in the reference's track order, point3D_of_keypoint [K]
    (row, -1 without a point), summary (dict of psfm_triangulation_summary).  The poses and cameras it was computed
    with are kept for `to_reconstruction`."""

    def __init__(self, xyz, track_ptr, track_image, track_point2D, point3D_of_keypoint, summary, inputs):
        self.xyz, self.track_ptr = xyz, track_ptr
        self.track_image, self.track_point2D = track_image, track_point2D
        self.point3D_of_keypoint, self.summary = point3D_of_keypoint, summary
        self._inputs = inputs

    def to_reconstruction(self, image_ids, image_names, camera_ids):
        """The ba.Reconstruction that ba.iterative_global_refinement and colmap_io.write_model take: SIMPLE_PINHOLE
        cameras (camera_ids [C]), the registered images (image_ids [F], image_names [F]) with every keypoint as a Point2D
        (point3D_ids -1 where untriangulated), points 1 .. P with their tracks; reg_image_ids in ascending id order."""
        from . import ba
        kp_ptr, kps, cam_of, cams, size, q, t, reg = self._inputs
        cameras = {int(camera_ids[c]): ba.Camera(int(camera_ids[c]), 0, int(size[c, 0]), int(size[c, 1]), cams[c].copy())
                   for c in range(len(cams))}
        images = {}
        for f in np.nonzero(reg)[0]:
            lo, hi = int(kp_ptr[f]), int(kp_ptr[f + 1])
            p3 = self.point3D_of_keypoint[lo:hi]
            images[int(image_ids[f])] = ba.Image(int(image_ids[f]), q[f].copy(), t[f].copy(), int(camera_ids[cam_of[f]]),
                                                 str(image_names[f]), kps[lo:hi].astype(np.float64),
                                                 np.where(p3 >= 0, p3 + 1, -1).astype(np.int64))
        ids = np.asarray(image_ids, np.int64)
        points = {}
        for p in range(self.xyz.shape[0]):
            a, b = self.track_ptr[p], self.track_ptr[p + 1]
            points[p + 1] = ba.Point3D(p + 1, self.xyz[p].copy(), np.zeros(3, np.uint8), 0.0,
                                       ids[self.track_image[a:b]], self.track_point2D[a:b].astype(np.int64))
        return ba.Reconstruction(cameras, images, points, reg_image_ids=sorted(images))


def _triangulation_create(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr, inlier_matches,
                          camera_size, orientations, image_tvec, registered, pair_used=None, options=None):
    """psfm_triangulation_create: returns (handle, P, E, inputs)."""
    kp_ptr, kps, cam_of, pairs, iptr, m = _pair_graph(keypoint_ptr, keypoints, image_camera, pair_images, inlier_ptr,
                                                      inlier_matches)
    cams = np.ascontiguousarray(cameras, np.float64).reshape(-1, 3)
    size = np.ascontiguousarray(camera_size, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    q = np.ascontiguousarray(orientations, np.float64).reshape(-1, 4)
    t = np.ascontiguousarray(image_tvec, np.float64).reshape(-1, 3)
    reg = np.ascontiguousarray(registered, np.uint8)
    F = kp_ptr.shape[0] - 1
    if q.shape[0] != F or t.shape[0] != F or reg.shape != (F,):
        raise ValueError("orientations, image_tvec and registered must have one entry per image")
    if size.shape[0] != cams.shape[0]:
        raise ValueError("camera_size must have one (width, height) per camera")
    used = None
    if pair_used is not None:
        used = np.ascontiguousarray(pair_used, np.uint8)
        if used.shape != (R,):
            raise ValueError("pair_used must have one entry per pair")
    opts = (options or IncrementalTriangulatorOptions()).to_struct()
    L = _lib.lib()
    i32, i64, u8 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
    h = C.c_void_p()
    P, E = C.c_int64(), C.c_int64()
    _lib.check(L.psfm_triangulation_create(
        F, kp_ptr.ctypes.data_as(i64), kps.ctypes.data_as(C.POINTER(C.c_float)), cam_of.ctypes.data_as(i32),
        _lib.dptr(cams), cams.shape[0], size.ctypes.data_as(i32), R, pairs.ctypes.data_as(i32), iptr.ctypes.data_as(i64),
        m.ctypes.data_as(C.POINTER(C.c_uint32)), used.ctypes.data_as(u8) if used is not None else None, _lib.dptr(q),
        _lib.dptr(t), reg.ctypes.data_as(u8), C.byref(opts), C.byref(h), C.byref(P), C.byref(E)),
        "psfm_triangulation_create")
    return h, P.value, E.value, (kp_ptr, kps, cam_of, cams, size, q, t, reg.astype(bool))


def triangulate_all_points(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr, inlier_matches,
                           camera_size, orientations, image_tvec, registered, pair_used=None, options=None):
    """GlobalMapper::TriangulateAllPoints (sfm/global_mapper.cc:232-247): TriangulateImage of every registered image in
    index order (Find, Continue, Create with LO-RANSAC).  Images and pairs as `optimize_pairwise_translations` takes
    them (images in ascending image_id), camera_size [C][2] (width, height), orientations [F][4] and image_tvec [F][3]
    (`estimate_global_rotations` / `estimate_global_positions`), registered [F], pair_used [R] (None: every pair; the
    database cache's pairs, not the rotation stage's pair_kept), options IncrementalTriangulatorOptions.  The pairs
    enter the correspondence graph in array order.  Returns Triangulation (psfm_triangulation_create,
    csrc/triangulation.cu)."""
    h, P, E, inputs = _triangulation_create(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr,
                                            inlier_matches, camera_size, orientations, image_tvec, registered, pair_used,
                                            options)
    L = _lib.lib()
    i32, i64 = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    try:
        xyz, track_ptr = np.zeros((P, 3)), np.zeros(P + 1, np.int64)
        track_image, track_point2D = np.zeros(E, np.int32), np.zeros(E, np.int32)
        p3 = np.zeros(inputs[1].shape[0], np.int64)
        s = _abi.TriangulationSummary()
        _lib.check(L.psfm_triangulation_result(h, _lib.dptr(xyz), track_ptr.ctypes.data_as(i64), track_image.ctypes.data_as(i32),
                                               track_point2D.ctypes.data_as(i32), p3.ctypes.data_as(i64), C.byref(s)),
                   "psfm_triangulation_result")
    finally:
        L.psfm_triangulation_destroy(h)
    summary = {n: getattr(s, n) for n, _ in _abi.TriangulationSummary._fields_}
    return Triangulation(xyz, track_ptr, track_image, track_point2D, p3, summary, inputs)


class ResidentTriangulation:
    """The device result of triangulate_all_points kept on the device (the psfm_triangulation handle), for
    ba.TriangulationSolver: num_points3D, num_track_elements, summary (dict of psfm_triangulation_summary).  close()
    frees it; the solver does not need it once created."""

    def __init__(self, handle, num_points3D, num_track_elements, summary):
        self.handle, self.num_points3D, self.num_track_elements = handle, num_points3D, num_track_elements
        self.summary = summary

    def close(self):
        if self.handle:
            _lib.lib().psfm_triangulation_destroy(self.handle)
            self.handle = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def triangulate_all_points_resident(*args, **kwargs):
    """triangulate_all_points with the same arguments, leaving the points, tracks and point3D_of_keypoint on the
    device: returns a ResidentTriangulation for ba.TriangulationSolver."""
    h, P, E, _ = _triangulation_create(*args, **kwargs)
    s = _abi.TriangulationSummary()
    try:
        _lib.check(_lib.lib().psfm_triangulation_result(h, None, None, None, None, None, C.byref(s)), "psfm_triangulation_result")
    except Exception:
        _lib.lib().psfm_triangulation_destroy(h)
        raise
    return ResidentTriangulation(h, P, E, {n: getattr(s, n) for n, _ in _abi.TriangulationSummary._fields_})


class TwoViewVerificationOptions:
    """TwoViewGeometry::Options with its RANSACOptions, the reference's names.  A field left None takes the library's
    default (psfm_verification_default_options: what sfm/import_feature_matches.py:106-117 runs)."""

    def __init__(self, max_error=None, confidence=None, max_num_trials=None, min_num_trials=None, min_inlier_ratio=None,
                 min_num_inliers=None, dyn_num_trials_multiplier=None, max_H_inlier_ratio=None, detect_watermark=None,
                 watermark_min_inlier_ratio=None, watermark_border_size=None, random_seed=None):
        self.max_error = max_error
        self.confidence = confidence
        self.max_num_trials = max_num_trials
        self.min_num_trials = min_num_trials
        self.min_inlier_ratio = min_inlier_ratio
        self.min_num_inliers = min_num_inliers
        self.dyn_num_trials_multiplier = dyn_num_trials_multiplier
        self.max_H_inlier_ratio = max_H_inlier_ratio
        self.detect_watermark = detect_watermark
        self.watermark_min_inlier_ratio = watermark_min_inlier_ratio
        self.watermark_border_size = watermark_border_size
        self.random_seed = random_seed

    def to_struct(self):
        o = _abi.VerificationOptions()
        _lib.lib().psfm_verification_default_options(C.byref(o))
        for n, _ in _abi.VerificationOptions._fields_:
            if getattr(self, n) is not None:
                setattr(o, n, int(getattr(self, n)) if n == "detect_watermark" else getattr(self, n))
        return o


class TwoViewVerification:
    """Per pair (in the order of the input): config [R] (UNDEFINED 0, DEGENERATE 1, UNCALIBRATED 3,
    PLANAR_OR_PANORAMIC 6, WATERMARK 7), F / E / H [R][3][3] (unit Frobenius norm, largest-magnitude entry positive; E
    zero), inlier_ptr [R + 1], inlier_matches [N][2] uint32 (F's inliers in match order), trials [R][3] (samples drawn
    for F, H and the watermark test), summary (dict of psfm_verification_summary)."""

    def __init__(self, config, F, E, H, inlier_ptr, inlier_matches, trials, summary):
        self.config, self.F, self.E, self.H = config, F, E, H
        self.inlier_ptr, self.inlier_matches = inlier_ptr, inlier_matches
        self.trials, self.summary = trials, summary

    def two_view_rows(self, pair_ids):
        """The two_view_geometries rows (pair_id, inlier matches, config, F, E, H) of every pair, which
        handoff.write_colmap_database stores as `colmap matches_importer` would."""
        return [(int(pid), np.ascontiguousarray(self.inlier_matches[self.inlier_ptr[p]:self.inlier_ptr[p + 1]]),
                 int(self.config[p]), self.F[p], self.E[p], self.H[p]) for p, pid in enumerate(pair_ids)]

    def to_two_view_geometries(self, tables):
        """The handoff.TwoViewGeometries that read_two_view_geometries returns once two_view_rows(tables.pair_ids) are
        written beside `tables` (a handoff.MatchTables): relative_pose_inputs() and triangulate_all_points then run
        without SQLite."""
        from .handoff import TwoViewGeometries
        return TwoViewGeometries(
            image_ids=tables.image_ids, keypoint_ptr=tables.keypoint_ptr, keypoints=tables.keypoints,
            camera_ids=tables.camera_ids, cameras=tables.cameras, image_camera=tables.image_camera,
            pair_ids=tables.pair_ids, pair_images=tables.pair_images, camera_size=tables.camera_size,
            image_names=list(tables.image_names), config=self.config.copy(), F=self.F.copy(), E=self.E.copy(),
            H=self.H.copy(), inlier_ptr=self.inlier_ptr.copy(), inlier_matches=self.inlier_matches.copy())


def verify_two_view_geometries(keypoint_ptr, keypoints, image_camera, camera_size, pair_images, match_ptr, matches,
                               prior_focal_length=None, options=None):
    """The geometric verification of `colmap matches_importer --match_type pairs` (TwoViewGeometryVerifier ->
    EstimateUncalibrated) of every pair at once: keypoint_ptr [F + 1], keypoints [K][2] (as stored in the database),
    image_camera [F], camera_size [C][2] (width, height), pair_images [R][2] (image 1 = the smaller image_id),
    match_ptr [R + 1], matches [M][2] (point2D_idx1, point2D_idx2), prior_focal_length [C] (None: no camera has one),
    options TwoViewVerificationOptions.  handoff.MatchTables.verification_inputs() gives these arguments.  Returns
    TwoViewVerification (psfm_verify_two_view_geometries, csrc/verification.cu)."""
    kp_ptr, kps, cam_of, pairs, mptr, m = _pair_graph(keypoint_ptr, keypoints, image_camera, pair_images, match_ptr, matches)
    size = np.ascontiguousarray(camera_size, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    F = kp_ptr.shape[0] - 1
    prior = None
    if prior_focal_length is not None:
        prior = np.ascontiguousarray(prior_focal_length, np.uint8)
        if prior.shape != (size.shape[0],):
            raise ValueError("prior_focal_length must have one entry per camera")
    i32, i64, u32 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
    return _verify(R, m.shape[0], options, "psfm_verify_two_view_geometries",
                   lambda *out: _lib.lib().psfm_verify_two_view_geometries(
                       F, kp_ptr.ctypes.data_as(i64), kps.ctypes.data_as(C.POINTER(C.c_float)), cam_of.ctypes.data_as(i32),
                       size.shape[0], size.ctypes.data_as(i32),
                       prior.ctypes.data_as(C.POINTER(C.c_uint8)) if prior is not None else None, R,
                       pairs.ctypes.data_as(i32), mptr.ctypes.data_as(i64), m.ctypes.data_as(u32), *out))


def verify_match_table(table, image_camera, camera_size, prior_focal_length=None, options=None):
    """verify_two_view_geometries on a handoff.ResidentMatchTable where it lies on the device (psfm_match_table_verify):
    the same result as verify_two_view_geometries(**table.tables(...).verification_inputs()).  image_camera
    [num_images] in image_id order, camera_size [C][2], prior_focal_length [C] (None: no camera has one)."""
    cam_of = np.ascontiguousarray(image_camera, np.int32)
    size = np.ascontiguousarray(camera_size, np.int32).reshape(-1, 2)
    if cam_of.shape != (table.num_images,):
        raise ValueError("image_camera must have one entry per image of the table")
    prior = None
    if prior_focal_length is not None:
        prior = np.ascontiguousarray(prior_focal_length, np.uint8)
        if prior.shape != (size.shape[0],):
            raise ValueError("prior_focal_length must have one entry per camera")
    i32 = C.POINTER(C.c_int32)
    return _verify(table.num_pairs, table.num_matches, options, "psfm_match_table_verify",
                   lambda *out: _lib.lib().psfm_match_table_verify(
                       table.handle, cam_of.ctypes.data_as(i32), size.shape[0], size.ctypes.data_as(i32),
                       prior.ctypes.data_as(C.POINTER(C.c_uint8)) if prior is not None else None, *out))


def _verify(R, M, options, name, call):
    """Allocate the outputs of R pairs and M raw matches, call(options, outputs...) and wrap them."""
    opts = (options or TwoViewVerificationOptions()).to_struct()
    config, Fm, Em, Hm = np.zeros(R, np.int32), np.zeros((R, 3, 3)), np.zeros((R, 3, 3)), np.zeros((R, 3, 3))
    iptr, out = np.zeros(R + 1, np.int64), np.zeros((M, 2), np.uint32)
    trials = np.zeros((R, 3), np.int32)
    s = _abi.VerificationSummary()
    i32, i64, u32 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint32)
    _lib.check(call(C.byref(opts), config.ctypes.data_as(i32), _lib.dptr(Fm), _lib.dptr(Em), _lib.dptr(Hm),
                    iptr.ctypes.data_as(i64), out.ctypes.data_as(u32), trials.ctypes.data_as(i32), C.byref(s)), name)
    summary = {n: (list(getattr(s, n)) if n.startswith(("num_trials", "num_local", "num_config")) else getattr(s, n))
               for n, _ in _abi.VerificationSummary._fields_}
    return TwoViewVerification(config, Fm, Em, Hm, iptr, np.ascontiguousarray(out[:iptr[-1]]), trials, summary)
