"""CPU restatement (numpy) of the refinement loop AROUND the global bundle adjustment.

TEST INFRASTRUCTURE — the checker for psfm_ba_filter_* / psfm_ba_normalize /
psfm_ba_refine of the CUDA library and for the host mirror in particlesfm_b200/ba.py.
Only tests/, __graft_entry__.smoke() and bench.py's cpu legs import it.

Follows, on the flattened problem (observation arrays + an `alive` mask instead of the
reference's Track / Point2D objects):

  filter_negative_depth      Reconstruction::FilterObservationsWithNegativeDepth
                             base/reconstruction.cc:711-729 + DeleteObservation :300-320
  filter_all_points3d        Reconstruction::FilterAllPoints3D  :697-709
      large reprojection error  FilterPoints3DWithLargeReprojectionError :1383-1434
      small triangulation angle FilterPoints3DWithSmallTriangulationAngle :1321-1381
  normalize                  Reconstruction::Normalize :373-468
  iterative_global_refinement IterativeGlobalRefinement, controllers/global_mapper.cc:245-271,
                             minus the IncrementalTriangulator calls (CompleteAndMergeTracks,
                             Retriangulate: out of scope, they change 0 observations here) and
                             AdjustGlobalBundle :215-243 / sfm/global_mapper.cc:402-448.

COLMAP helpers that are NOT in the reference repository (COLMAP bd84ad6, base/projection.cc,
base/triangulation.cc) are restated from their published source:
  HasPointPositiveDepth(P, X)            = P.row(2) . [X; 1] >= DBL_EPSILON
  CalculateSquaredReprojectionError      = DBL_MAX when (R X + t).z < DBL_EPSILON, else
                                           |f (x/z, y/z) + c - xy|^2
  CalculateTriangulationAngle(c1, c2, X) = law of cosines, min(angle, pi - angle), 0 when a
                                           ray has zero length
The per-point outcomes of the reference's sequential DeleteObservation calls are order
independent and are written here in closed form (see the docstrings).
"""
import numpy as np

EPS = np.finfo(np.float64).eps
DBL_MAX = np.finfo(np.float64).max


def qvec_to_rotmat(q):
    q = np.asarray(q, np.float64)
    w, x, y, z = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    R = np.empty(q.shape[:-1] + (3, 3))
    R[..., 0, 0] = 1 - 2 * (y * y + z * z); R[..., 0, 1] = 2 * (x * y - w * z); R[..., 0, 2] = 2 * (x * z + w * y)
    R[..., 1, 0] = 2 * (x * y + w * z); R[..., 1, 1] = 1 - 2 * (x * x + z * z); R[..., 1, 2] = 2 * (y * z - w * x)
    R[..., 2, 0] = 2 * (x * z - w * y); R[..., 2, 1] = 2 * (y * z + w * x); R[..., 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def _normalized_q(prob):
    return prob.qvec / np.linalg.norm(prob.qvec, axis=1, keepdims=True)


def projection_centers(prob):
    """Image::ProjectionCenter = -R' t."""
    R = qvec_to_rotmat(_normalized_q(prob))
    return -np.einsum("fji,fj->fi", R, prob.tvec)


def camera_points(prob):
    """R X + t per observation."""
    R = qvec_to_rotmat(_normalized_q(prob))
    return np.einsum("mij,mj->mi", R[prob.obs_image], prob.xyz[prob.obs_point]) + prob.tvec[prob.obs_image]


def track_lengths(prob, alive):
    return np.bincount(prob.obs_point[alive], minlength=prob.num_points)


def filter_negative_depth(prob, alive):
    """Returns (alive', num_filtered).  Sequential semantics of the reference: every negative-
    depth observation of a still existing point is one DeleteObservation call; the call that
    finds Track().Length() <= 2 deletes the whole point.  Closed form per point with track
    length L and n negative observations: the point is deleted iff L - n < 2 (all its
    observations go); the number of calls is min(n, max(L - 1, 1))."""
    alive = alive.copy()
    z = camera_points(prob)[:, 2]
    neg = alive & ~(z >= EPS)
    L = track_lengths(prob, alive)
    n = np.bincount(prob.obs_point[neg], minlength=prob.num_points)
    has = n > 0
    delete_point = has & (L - n < 2)
    calls = np.where(has, np.minimum(n, np.maximum(L - 1, 1)), 0)
    alive &= ~neg
    alive &= ~delete_point[prob.obs_point]
    return alive, int(calls.sum())


def squared_reprojection_errors(prob):
    p = camera_points(prob)
    K = prob.cam_params[prob.image_camera[prob.obs_image]]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = K[:, 0] * (p[:, 0] / p[:, 2]) + K[:, 1] - prob.obs_xy[:, 0]     # WorldToImage(hnormalized())
        v = K[:, 0] * (p[:, 1] / p[:, 2]) + K[:, 2] - prob.obs_xy[:, 1]
        e = u * u + v * v
    return np.where(p[:, 2] < EPS, DBL_MAX, e)


def filter_large_reprojection_error(prob, alive, max_reproj_error):
    """Returns (alive', num_filtered, point_error [P], NaN where not set).  Per point with
    track length L and d observations above the threshold: L < 2 or d >= L - 1 -> the point is
    deleted, num_filtered += L; else the d observations go, num_filtered += d and
    Point3D::Error = sum of the kept errors / (L - d)."""
    alive = alive.copy()
    e2 = squared_reprojection_errors(prob)
    bad = alive & (e2 > max_reproj_error * max_reproj_error)
    L = track_lengths(prob, alive)
    d = np.bincount(prob.obs_point[bad], minlength=prob.num_points)
    exists = L > 0
    delete_point = exists & ((L < 2) | (d >= L - 1))
    num = int(np.where(delete_point, L, np.where(exists, d, 0)).sum())
    good = alive & ~bad
    err_sum = np.bincount(prob.obs_point[good], weights=np.sqrt(e2[good]), minlength=prob.num_points)
    err = np.full(prob.num_points, np.nan)
    keep = exists & ~delete_point
    err[keep] = err_sum[keep] / (L - d)[keep]
    alive &= ~bad
    alive &= ~delete_point[prob.obs_point]
    return alive, num, err


def triangulation_angle(c1, c2, X):
    b2 = ((c1 - c2) ** 2).sum(-1)
    r1 = ((X - c1) ** 2).sum(-1)
    r2 = ((X - c2) ** 2).sum(-1)
    den = 2.0 * np.sqrt(r1 * r2)
    with np.errstate(divide="ignore", invalid="ignore"):
        ang = np.abs(np.arccos((r1 + r2 - b2) / den))
    ang = np.minimum(ang, np.pi - ang)
    return np.where(den == 0.0, 0.0, ang)


def filter_small_triangulation_angle(prob, alive, min_tri_angle_deg):
    """Returns (alive', num_filtered = deleted POINTS).  A point is kept iff some pair of its
    track's images sees it under at least the minimum angle (NaN angles compare false)."""
    alive = alive.copy()
    thr = np.deg2rad(min_tri_angle_deg)
    C = projection_centers(prob)
    idx = np.nonzero(alive)[0]
    order = idx[np.argsort(prob.obs_point[idx], kind="stable")]
    pts = prob.obs_point[order]
    bounds = np.nonzero(np.diff(pts))[0] + 1
    starts = np.concatenate([[0], bounds]) if order.size else np.zeros(0, np.int64)
    ends = np.concatenate([bounds, [order.size]]) if order.size else np.zeros(0, np.int64)
    num = 0
    for s, e in zip(starts, ends):
        p = pts[s]
        cs = C[prob.obs_image[order[s:e]]]
        keep = False
        for i1 in range(e - s):
            if i1 == 0:
                continue
            a = triangulation_angle(cs[i1][None, :], cs[:i1], prob.xyz[p][None, :])
            if np.any(a >= thr):
                keep = True
                break
        if not keep:
            num += 1
            alive[order[s:e]] = False
    return alive, num


def filter_all_points3d(prob, alive, max_reproj_error=4.0, min_tri_angle=1.5):
    alive, n1, err = filter_large_reprojection_error(prob, alive, max_reproj_error)
    alive, n2 = filter_small_triangulation_angle(prob, alive, min_tri_angle)
    return alive, n1 + n2, err


def normalize(prob, extent=10.0, p0=0.1, p1=0.9):
    """In place on prob.tvec / prob.xyz (use_images = true, the only form the pipeline calls).
    Per-axis independently sorted FLOAT coordinates of the projection centres; returns
    (translation, scale) or None when fewer than 2 images."""
    F = prob.num_images
    if F < 2:
        return None
    q = _normalized_q(prob)
    R = qvec_to_rotmat(q)
    cen = -np.einsum("fji,fj->fi", R, prob.tvec)
    cs = np.sort(cen.astype(np.float32), axis=0)
    P0 = int(p0 * (F - 1)) if F > 3 else 0
    P1 = int(p1 * (F - 1)) if F > 3 else F - 1
    lo, hi = cs[P0].astype(np.float64), cs[P1].astype(np.float64)
    mean = np.zeros(3)
    for i in range(P0, P1 + 1):                      # sequential, as the reference accumulates
        mean += cs[i].astype(np.float64)
    mean /= (P1 - P0 + 1)
    old_extent = np.linalg.norm(hi - lo)
    scale = 1.0 if old_extent < EPS else extent / old_extent
    cen2 = (cen - mean) * scale
    prob.tvec[:] = np.einsum("fij,fj->fi", R, -cen2)
    prob.xyz[:] = (prob.xyz - mean) * scale
    return mean, scale


def _subproblem(prob, alive):
    from particlesfm_b200._abi import BAProblem
    return BAProblem(prob.qvec, prob.tvec, prob.xyz, prob.cam_params, prob.obs_image[alive], prob.obs_point[alive],
                     prob.obs_xy[alive], prob.image_camera, prob.pose_constant, prob.tvec_constant_mask,
                     prob.camera_constant)


def adjust_global_bundle(prob, alive, opts, ba_solve):
    """GlobalMapper::AdjustGlobalBundle (sfm/global_mapper.cc:402-448) on the flattened problem:
    negative-depth filter, solve (gauge flags are part of `prob`), Normalize.  `ba_solve(problem,
    opts)` solves in place and returns a summary.  Returns (alive', summary or None)."""
    alive, _ = filter_negative_depth(prob, alive)
    sub = _subproblem(prob, alive)
    if sub.num_observations == 0:
        return alive, None
    s = ba_solve(sub, opts)
    prob.qvec[:], prob.tvec[:], prob.cam_params[:] = sub.qvec, sub.tvec, sub.cam_params
    prob.xyz[:] = sub.xyz
    normalize(prob)
    return alive, s


def iterative_global_refinement(prob, alive, opts, ba_solve, max_refinements=5, max_refinement_change=0.0005,
                                max_reproj_error=4.0, min_tri_angle=1.5):
    """One IterativeGlobalRefinement pass.  Returns (alive', report list of dicts)."""
    report = []
    err = np.full(prob.num_points, np.nan)
    for _ in range(max_refinements):
        num_obs = int(alive.sum())
        alive, s = adjust_global_bundle(prob, alive, opts, ba_solve)
        alive, changed_n, err_i = filter_all_points3d(prob, alive, max_reproj_error, min_tri_angle)
        err = np.where(np.isnan(err_i), err, err_i)
        changed = changed_n / num_obs if num_obs else 0.0
        report.append(dict(num_observations=num_obs, changed_observations=changed_n, changed=changed,
                           ba_iterations=(s.num_iterations if s is not None else 0),
                           final_cost=(s.final_cost if s is not None else 0.0)))
        if changed < max_refinement_change:
            break
    return alive, report, err
