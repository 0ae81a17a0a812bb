"""Numpy / scipy restatement of the global position estimation (TEST INFRASTRUCTURE; the product is
csrc/position_estimation.cu) and of the pairwise-translation step that feeds it.

* optimize_pairwise_translations — GlobalMapper::OptimizePairwiseTranslations (sfm/global_mapper.cc:106-109): every used
  pair's points gathered from the database arrays, normalised as (x - cx) / f, then
  init_oracle.optimize_relative_position_with_known_rotation.
* estimate_global_positions — GlobalMapper::EstimatePositions with method "lud"
  (global/least_unsquared_deviation_position_estimator.cc:92-178, use_scale_constraints = false), then the pose update
  of RegisterAllImages (sfm/global_mapper.cc:140-160).  It follows the reference's own formulation: the sparse stacked
  matrix A~ = [A; G] with 3 (V - 1) + R columns (three L1 rows c1 - c2 - s_k d_k per pair, d_k = R2' t_k, one
  inequality row s_k >= 1), scipy.sparse.linalg.splu of A~'A~, and Theia's ConstrainedL1Solver.  The device eliminates
  the scales and works on the Schur complement instead, so agreement checks that reduction independently.

The solver defaults are recalled, not vendored (RECALLED; csrc/position_recalled.cuh keeps the same values).  The
gauge the reference leaves to hash order is defined as in include/psfm_b200.h: the smallest image index of the used
pairs, fixed at the origin."""
import numpy as np
import scipy.sparse
import scipy.sparse.linalg

from . import init_oracle
from .rotation_oracle import invert_quaternion, normalize_quaternion, shrinkage

RECALLED = {
    "max_num_iterations": 1000,     # theia::ConstrainedL1Solver::Options::max_num_iterations
    "rho": 10.0,                    # theia::ConstrainedL1Solver::Options::rho
    "alpha": 1.2,                   # theia::ConstrainedL1Solver::Options::alpha
    "absolute_tolerance": 1e-4,     # theia::ConstrainedL1Solver::Options::absolute_tolerance
    "relative_tolerance": 1e-2,     # theia::ConstrainedL1Solver::Options::relative_tolerance
}
MAX_UNKNOWNS = 8190                 # 3 (V - 1): the dense factor's bound on the device


class InvalidError(ValueError):
    """The device returns PSFM_ERR_INVALID before any launch."""


class OptionsError(InvalidError):
    pass


class UnsupportedError(ValueError):
    """The device returns PSFM_ERR_UNSUPPORTED before any launch."""


def check_options(o):
    """The Check() of psfm_lud_options: max_num_iterations > 0, rho > 0, 0 < alpha < 2, tolerances > 0, all finite."""
    ok = (o["max_num_iterations"] > 0 and np.isfinite(o["rho"]) and o["rho"] > 0 and 0 < o["alpha"] < 2 and
          np.isfinite(o["absolute_tolerance"]) and o["absolute_tolerance"] > 0 and
          np.isfinite(o["relative_tolerance"]) and o["relative_tolerance"] > 0)
    if not ok:
        raise OptionsError("options fail the ConstrainedL1Solver options Check()")


def quaternion_rotate_point(q, p):
    """COLMAP QuaternionRotatePoint: the normalised quaternion applied as Eigen's Quaterniond * Vector3d."""
    q = normalize_quaternion(q)
    v = q[1:]
    uv = np.cross(v, p)
    uv = uv + uv
    return np.asarray(p, np.float64) + q[0] * uv + np.cross(v, uv)


def rotated_translation(q2, t):
    """GetRotatedTranslation (least_unsquared_deviation_position_estimator.cc:61-64): R2' t."""
    return quaternion_rotate_point(invert_quaternion(normalize_quaternion(q2)), t)


def _problem(num_images, pair_images, tvec, orientations, has_orientation, pair_used):
    """The argument rules of psfm_estimate_global_positions; returns (used pairs, views ascending)."""
    F = int(num_images)
    pair_images = np.asarray(pair_images, np.int64).reshape(-1, 2)
    R = pair_images.shape[0]
    keys = set()
    for a, b in pair_images:
        if not (0 <= a < F and 0 <= b < F):
            raise InvalidError("an image index is outside [0, num_images)")
        if a == b:
            raise InvalidError("a pair of an image with itself")
        key = (min(a, b), max(a, b))
        if key in keys:
            raise InvalidError("an unordered image pair is listed twice")
        keys.add(key)
    used = [p for p in range(R) if pair_used is None or pair_used[p]]
    if not used:
        raise InvalidError("no used image pair")
    views = sorted({int(v) for p in used for v in pair_images[p]})
    for f in views:
        if has_orientation is not None and not has_orientation[f]:
            raise InvalidError("a used pair's image has no orientation")
        if not np.all(np.isfinite(orientations[f])):
            raise InvalidError("a non-finite orientation")
    for p in used:
        if not np.all(np.isfinite(tvec[p])):
            raise InvalidError("a non-finite pair tvec")
    parent = {f: f for f in views}

    def find(v):
        while parent[v] != v:
            parent[v] = parent[parent[v]]
            v = parent[v]
        return v

    for p in used:
        ra, rb = find(int(pair_images[p][0])), find(int(pair_images[p][1]))
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    if len({find(f) for f in views}) != 1:
        raise InvalidError("the used pairs do not form one connected graph (S is singular)")
    if 3 * (len(views) - 1) > MAX_UNKNOWNS:
        raise UnsupportedError("more than 2731 views (3 (V - 1) > 8190 unknowns)")
    return used, views


def stacked_system(index, pair_images, d, used):
    """A~ (4R x (3 n_views + R), the gauge's columns dropped: index[f] = -1) and b~ = [0 (3R); 1 (R)]: rows 3k .. 3k + 2
    are c1 - c2 - s_k d_k, row 3R + k is s_k (SetupConstraintMatrix and the geq rows, :147-153, :258-344)."""
    n = 3 * sum(1 for v in index.values() if v >= 0)
    R = len(used)
    rows, cols, vals = [], [], []
    for k, p in enumerate(used):
        a, b = (int(v) for v in pair_images[p])
        for img, sgn in ((a, 1.0), (b, -1.0)):
            if index[img] >= 0:
                for j in range(3):
                    rows.append(3 * k + j)
                    cols.append(3 * index[img] + j)
                    vals.append(sgn)
        for j in range(3):
            rows.append(3 * k + j)
            cols.append(n + k)
            vals.append(-d[k][j])
        rows.append(3 * R + k)
        cols.append(n + k)
        vals.append(1.0)
    A = scipy.sparse.csr_matrix((vals, (rows, cols)), shape=(4 * R, n + R))
    return A, np.concatenate([np.zeros(3 * R), np.ones(R)])


def constrained_l1_solve(A, b, num_l1, options):
    """theia::ConstrainedL1Solver::Solve restated: ADMM on A~ from z = u = 0, shrinkage on the first num_l1 rows and
    max(., 0) on the rest.  Returns (x, iterations, converged, history [(r_norm, primal_eps, s_norm, dual_eps)])."""
    rho, alpha = options["rho"], options["alpha"]
    At = A.T.tocsr()
    lu = scipy.sparse.linalg.splu((At @ A).tocsc())
    z, u = np.zeros(A.shape[0]), np.zeros(A.shape[0])
    b_norm = np.linalg.norm(b)
    primal_abs = np.sqrt(A.shape[0]) * options["absolute_tolerance"]
    dual_abs = np.sqrt(A.shape[1]) * options["absolute_tolerance"]
    rel = options["relative_tolerance"]
    x, history, converged = np.zeros(A.shape[1]), [], False
    for _ in range(options["max_num_iterations"]):
        x = lu.solve(At @ (b + z - u))
        ax = A @ x
        ax_hat = alpha * ax + (1.0 - alpha) * (z + b)
        z_old = z
        v = ax_hat - b + u
        z = np.concatenate([shrinkage(v[:num_l1], 1.0 / rho), np.maximum(v[num_l1:], 0.0)])
        u = u + ax_hat - z - b
        r_norm = np.linalg.norm(ax - z - b)
        s_norm = np.linalg.norm(-rho * (At @ (z - z_old)))
        primal_eps = primal_abs + rel * max(np.linalg.norm(ax), np.linalg.norm(z), b_norm)
        dual_eps = dual_abs + rel * np.linalg.norm(rho * (At @ u))
        history.append((r_norm, primal_eps, s_norm, dual_eps))
        if r_norm < primal_eps and s_norm < dual_eps:
            converged = True
            break
    return x, len(history), converged, history


def schur_x_update(pair_views, d, n_views, rhs):
    """The device's x update: the same solve of A~'A~ x = rhs with the scales eliminated.  pair_views [(va, vb)]
    (column block of each image, -1 for the gauge), d [R][3], rhs = [r_c (3 n_views); r_s (R)].  S = sum_k W_k (x)
    (e1 - e2)(e1 - e2)', W_k = I - d_k d_k' / D_k, D_k = |d_k|^2 + 1; c = S^-1 (r_c - C D^-1 r_s),
    s_k = (r_s,k + d_k'(c1 - c2)) / D_k."""
    n = 3 * n_views
    R = len(pair_views)
    S = np.zeros((n, n))
    r = np.array(rhs[:n], np.float64)
    rs = np.asarray(rhs[n:], np.float64)
    D = (np.asarray(d) ** 2).sum(1) + 1.0
    for k, (va, vb) in enumerate(pair_views):
        W = np.eye(3) - np.outer(d[k], d[k]) / D[k]
        for v, sg in ((va, 1.0), (vb, -1.0)):
            if v >= 0:
                S[3 * v:3 * v + 3, 3 * v:3 * v + 3] += W
                r[3 * v:3 * v + 3] += sg * d[k] * rs[k] / D[k]
        if va >= 0 and vb >= 0:
            S[3 * va:3 * va + 3, 3 * vb:3 * vb + 3] -= W
            S[3 * vb:3 * vb + 3, 3 * va:3 * va + 3] -= W
    c = np.linalg.solve(S, r)
    pos = lambda v: c[3 * v:3 * v + 3] if v >= 0 else np.zeros(3)
    s = np.array([(rs[k] + d[k] @ (pos(va) - pos(vb))) / D[k] for k, (va, vb) in enumerate(pair_views)])
    return np.concatenate([c, s])


def estimate_global_positions(num_images, pair_images, tvec, orientations, has_orientation=None, pair_used=None,
                              options=None, gauge=None):
    """Returns dict(positions [F][3], has_position [F], image_tvec [F][3], scales [R], gauge_image, num_views,
    iterations, converged, history, objective = sum |c1 - c2 - s d|_1, min_scale).  gauge: the image fixed at the
    origin (None: the smallest view, as the device fixes it)."""
    o = dict(RECALLED)
    o.update(options or {})
    check_options(o)
    pair_images = np.asarray(pair_images, np.int64).reshape(-1, 2)
    tvec = np.asarray(tvec, np.float64).reshape(-1, 3)
    orientations = np.asarray(orientations, np.float64).reshape(-1, 4)
    F, R = int(num_images), pair_images.shape[0]
    used, views = _problem(F, pair_images, tvec, orientations, has_orientation, pair_used)
    g = views[0] if gauge is None else int(gauge)
    index, nxt = {}, 0
    for f in views:
        if f == g:
            index[f] = -1
        else:
            index[f] = nxt
            nxt += 1
    d = np.array([rotated_translation(orientations[pair_images[p][1]], tvec[p]) for p in used])
    A, b = stacked_system(index, pair_images, d, used)
    x, its, converged, history = constrained_l1_solve(A, b, 3 * len(used), o)
    n = 3 * (len(views) - 1)
    out = dict(positions=np.zeros((F, 3)), has_position=np.zeros(F, bool), image_tvec=np.zeros((F, 3)),
               scales=np.zeros(R), gauge_image=g, num_views=len(views), iterations=its, converged=converged,
               history=history)
    for f in views:
        c = np.zeros(3) if index[f] < 0 else x[3 * index[f]:3 * index[f] + 3]
        out["positions"][f] = c
        out["has_position"][f] = True
        out["image_tvec"][f] = -quaternion_rotate_point(orientations[f], c)
    out["scales"][used] = x[n:]
    out["objective"] = float(np.abs((A @ x)[:3 * len(used)]).sum())
    out["min_scale"] = float(x[n:].min())
    return out


def optimize_pairwise_translations(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr,
                                   inlier_matches, orientations, pair_used=None):
    """Returns (tvec [R][3], iterations [R]); zeros for unused pairs and pairs without a match."""
    pairs = np.asarray(pair_images, np.int64).reshape(-1, 2)
    iptr = np.asarray(inlier_ptr, np.int64)
    q = np.asarray(orientations, np.float64).reshape(-1, 4)
    R = pairs.shape[0]
    tvec, its = np.zeros((R, 3)), np.zeros(R, np.int32)
    for p in range(R):
        if (pair_used is not None and not pair_used[p]) or iptr[p + 1] == iptr[p]:
            continue
        x1, x2 = normalized_points(keypoint_ptr, keypoints, image_camera, cameras, pairs, iptr, inlier_matches, p)
        a, b = pairs[p]
        tvec[p], its[p] = init_oracle.optimize_relative_position_with_known_rotation(x1, x2, q[a], q[b],
                                                                                    return_iterations=True)
    return tvec, its


def normalized_points(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr, inlier_matches, p):
    """Pair p's normalised points as the device computes them: ((double) x - cx) / f."""
    kps = np.asarray(keypoints, np.float32).reshape(-1, 2).astype(np.float64)
    cams = np.asarray(cameras, np.float64).reshape(-1, 3)
    a, b = (int(v) for v in np.asarray(pair_images).reshape(-1, 2)[p])
    mm = np.asarray(inlier_matches, np.int64).reshape(-1, 2)[inlier_ptr[p]:inlier_ptr[p + 1]]
    ka, kb = cams[image_camera[a]], cams[image_camera[b]]
    return ((kps[keypoint_ptr[a] + mm[:, 0]] - ka[1:]) / ka[0], (kps[keypoint_ptr[b] + mm[:, 1]] - kb[1:]) / kb[0])
