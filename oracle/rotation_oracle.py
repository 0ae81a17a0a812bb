"""Numpy / scipy restatement of EstimateGlobalRotations (TEST INFRASTRUCTURE; the product is
csrc/rotation_averaging.cu).

It follows the reference's own formulation (global/robust_rotation_estimator.cc): the sparse 3R x 3(F-1) matrix A of
+-I blocks, a dense Cholesky of A'A for Theia's L1Solver and of A'WA for every IRLS iteration.  The device uses the
Kronecker reduction A'WA = (B'WB) (x) I3 instead, so agreement checks that reduction independently.

Parts the reference links but does not vendor are restated from memory; their constants are in RECALLED.  The
choices the reference leaves to hash order are defined as in include/psfm_b200.h: the kept component among equally
large ones holds the smallest image index, that image is the gauge and the spanning-tree root, and spanning-tree ties
go by (-num_correspondences, image 1, image 2)."""
import numpy as np
import scipy.linalg
import scipy.sparse

from .two_view_oracle import rotation_matrix_to_quaternion

RECALLED = {
    "admm_rho": 1.0,                 # theia::L1Solver::Options::rho
    "admm_alpha": 1.0,               # theia::L1Solver::Options::alpha
    "admm_absolute_tolerance": 1e-4,  # theia::L1Solver::Options::absolute_tolerance
    "admm_relative_tolerance": 1e-2,  # theia::L1Solver::Options::relative_tolerance
}
DEG_TO_RAD = 0.017453292519943295    # COLMAP DegToRad
DEFAULTS = dict(max_num_l1_iterations=5, l1_step_convergence_threshold=0.001, max_num_irls_iterations=100,
                irls_step_convergence_threshold=0.001, irls_loss_parameter_sigma=5.0 * DEG_TO_RAD,
                rotation_filter_max_degrees=5.0)


class OptionsError(ValueError):
    pass


def check_options(o):
    """RobustRotationEstimator::Options::Check (robust_rotation_estimator.cc:54-62)."""
    for k in DEFAULTS:
        if not o[k] > 0:
            raise OptionsError("%s must be > 0" % k)


# ---- COLMAP / Ceres quaternion helpers, (w, x, y, z) ----------------------------------------------------------------
def quat_mul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def normalize_quaternion(q):
    n = np.linalg.norm(q)
    return np.array([1.0, 0.0, 0.0, 0.0]) if n == 0 else np.asarray(q, np.float64) / n


def concatenate_quaternions(q1, q2):
    """ConcatenateQuaternions(q1, q2): q2 (x) q1, normalised."""
    return normalize_quaternion(quat_mul(normalize_quaternion(q2), normalize_quaternion(q1)))


def invert_quaternion(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def angle_axis_to_quaternion(a):
    t2 = float(np.dot(a, a))
    if t2 > 0:
        t = np.sqrt(t2)
        return np.concatenate([[np.cos(0.5 * t)], np.asarray(a) * (np.sin(0.5 * t) / t)])
    return np.concatenate([[1.0], 0.5 * np.asarray(a)])


def quaternion_to_angle_axis(q):
    s2 = q[1] * q[1] + q[2] * q[2] + q[3] * q[3]
    k = 2.0
    if s2 > 0:
        s, c = np.sqrt(s2), q[0]
        k = 2.0 * (np.arctan2(-s, -c) if c < 0 else np.arctan2(s, c)) / s
    return np.asarray(q[1:], np.float64) * k


def quaternion_to_rotation_matrix(q):
    w, x, y, z = normalize_quaternion(q)
    tx, ty, tz = 2 * x, 2 * y, 2 * z
    return np.array([[1 - (ty * y + tz * z), ty * x - tz * w, tz * x + ty * w],
                     [ty * x + tz * w, 1 - (tx * x + tz * z), tz * y - tx * w],
                     [tz * x - ty * w, tz * y + tx * w, 1 - (tx * x + ty * y)]])


# ---- graph steps ----------------------------------------------------------------------------------------------------
def _find(parent, v):
    while parent[v] != v:
        parent[v] = parent[parent[v]]
        v = parent[v]
    return v


def largest_component(num_images, pair_images, pairs):
    """RemoveDisconnectedViewPairs over `pairs` (indices): (kept pairs, set of the component's images)."""
    parent = list(range(num_images))
    seen = set()
    for p in pairs:
        a, b = (int(v) for v in pair_images[p])
        seen.update((a, b))
        ra, rb = _find(parent, a), _find(parent, b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    comps = {}
    for f in sorted(seen):
        comps.setdefault(_find(parent, f), []).append(f)
    if not comps:
        return [], set()
    best = max(comps.values(), key=lambda c: (len(c), -c[0]))
    imgs = set(best)
    return [p for p in pairs if int(pair_images[p][0]) in imgs], imgs


def spanning_tree_orientations(images, pair_images, qvec, num_correspondences, pairs):
    """OrientationsFromMaximumSpanningTree: Kruskal on (-num_correspondences, image 1, image 2), chained from the
    smallest image (identity) with ComputeOrientation's matrices."""
    parent = {f: f for f in images}

    def find(v):
        while parent[v] != v:
            parent[v] = parent[parent[v]]
            v = parent[v]
        return v

    tree = {f: [] for f in images}
    for p in sorted(pairs, key=lambda p: (-int(num_correspondences[p]), int(pair_images[p][0]), int(pair_images[p][1]))):
        a, b = (int(v) for v in pair_images[p])
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
            tree[a].append(p)
            tree[b].append(p)
    root = min(images)
    orient = {root: np.array([1.0, 0.0, 0.0, 0.0])}
    queue = [root]
    for s in queue:
        Rs = quaternion_to_rotation_matrix(orient[s])
        for p in tree[s]:
            a, b = (int(v) for v in pair_images[p])
            t = b if a == s else a
            if t in orient:
                continue
            Rr = quaternion_to_rotation_matrix(qvec[p])
            orient[t] = rotation_matrix_to_quaternion((Rr if a == s else Rr.T) @ Rs)
            queue.append(t)
    return orient


# ---- the robust estimator, in the reference's 3(F-1) formulation ----------------------------------------------------
def incidence_matrix(index, pair_images, pairs, scalar=False):
    """A (3R x 3n, or the R x n B with scalar=True): -1 at image 1, +1 at image 2, the gauge (index -1) dropped."""
    d = 1 if scalar else 3
    rows, cols, vals = [], [], []
    for r, p in enumerate(pairs):
        for img, sgn in ((int(pair_images[p][0]), -1.0), (int(pair_images[p][1]), 1.0)):
            i = index[img]
            if i >= 0:
                for k in range(d):
                    rows.append(d * r + k)
                    cols.append(d * i + k)
                    vals.append(sgn)
    n = sum(1 for v in index.values() if v >= 0)
    return scipy.sparse.csr_matrix((vals, (rows, cols)), shape=(d * len(pairs), d * n))


def shrinkage(v, kappa):
    return np.maximum(0.0, v - kappa) - np.maximum(0.0, -v - kappa)


def l1_solve(A, factor, b, max_iterations):
    """Theia L1Solver::Solve restated: ADMM from z = u = 0; returns (x, iterations)."""
    rho, alpha = RECALLED["admm_rho"], RECALLED["admm_alpha"]
    abs_tol, rel_tol = RECALLED["admm_absolute_tolerance"], RECALLED["admm_relative_tolerance"]
    At = A.T.tocsr()
    z, u = np.zeros(A.shape[0]), np.zeros(A.shape[0])
    b_norm = np.linalg.norm(b)
    primal_abs, dual_abs = np.sqrt(A.shape[0]) * abs_tol, np.sqrt(A.shape[1]) * abs_tol
    x = np.zeros(A.shape[1])
    it = 0
    for it in range(1, max_iterations + 1):
        x = scipy.linalg.cho_solve(factor, At @ (b + z - u))
        ax = A @ x
        ax_hat = alpha * ax + (1.0 - alpha) * (z + b)
        z_old = z
        z = shrinkage(ax_hat - b + u, 1.0 / rho)
        u = u + ax_hat - z - b
        r_norm = np.linalg.norm(ax - z - b)
        s_norm = np.linalg.norm(-rho * (At @ (z - z_old)))
        primal_eps = primal_abs + rel_tol * max(np.linalg.norm(ax), np.linalg.norm(z), b_norm)
        dual_eps = dual_abs + rel_tol * np.linalg.norm(rho * (At @ u))
        if r_norm < primal_eps and s_norm < dual_eps:
            break
    return x, it


def estimate_global_rotations(num_images, pair_images, qvec, num_correspondences, has_pose=None, options=None):
    """Returns dict(orientations [F][4], has_orientation [F], pair_kept [R], success, l1_rounds, admm_iterations,
    irls_iterations, gauge_image, residual_angles (final |loop| of every pair of the component, radians, -1 elsewhere))."""
    o = dict(DEFAULTS)
    o.update(options or {})
    check_options(o)
    pair_images = np.asarray(pair_images, np.int64).reshape(-1, 2)
    qvec = np.asarray(qvec, np.float64).reshape(-1, 4)
    R, F = pair_images.shape[0], int(num_images)
    out = dict(orientations=np.zeros((F, 4)), has_orientation=np.zeros(F, bool), pair_kept=np.zeros(R, bool),
               success=False, l1_rounds=0, admm_iterations=[], irls_iterations=0, gauge_image=-1,
               residual_angles=np.full(R, -1.0))
    posed = [p for p in range(R) if (has_pose is None or has_pose[p]) and np.all(np.isfinite(qvec[p]))]
    pairs, images = largest_component(F, pair_images, posed)
    if not pairs:
        return out
    images = sorted(images)
    orient = spanning_tree_orientations(images, pair_images, qvec, num_correspondences, pairs)
    gauge = images[0]
    index = {f: i - 1 for i, f in enumerate(images)}
    n = len(images) - 1
    A = incidence_matrix(index, pair_images, pairs)
    At = A.T.tocsr()
    rot = {f: orient[f] for f in images}

    def residuals():
        r = np.zeros(3 * len(pairs))
        for k, p in enumerate(pairs):
            a, b = (int(v) for v in pair_images[p])
            q = concatenate_quaternions(rot[a], qvec[p])
            q = concatenate_quaternions(q, invert_quaternion(rot[b]))
            r[3 * k:3 * k + 3] = quaternion_to_angle_axis(q)
        return r

    def update(x):
        steps = 0.0
        for f in images[1:]:
            xi = x[3 * index[f]:3 * index[f] + 3]
            rot[f] = concatenate_quaternions(angle_axis_to_quaternion(xi), rot[f])
            steps += np.linalg.norm(xi)
        return steps / n

    # SolveL1Regression
    factor = scipy.linalg.cho_factor((At @ A).toarray(), lower=True)
    r = residuals()
    cap = 5
    for _ in range(o["max_num_l1_iterations"]):
        x, its = l1_solve(A, factor, r, cap)
        out["l1_rounds"] += 1
        out["admm_iterations"].append(its)
        step = update(x)
        r = residuals()
        if step <= o["l1_step_convergence_threshold"]:
            break
        cap *= 2
    # SolveIRLS
    sigma = o["irls_loss_parameter_sigma"]
    for _ in range(o["max_num_irls_iterations"]):
        e2 = (r.reshape(-1, 3) ** 2).sum(1)
        w = np.repeat(sigma / (e2 + sigma * sigma) ** 2, 3)
        AtW = At @ scipy.sparse.diags(w)
        x = scipy.linalg.cho_solve(scipy.linalg.cho_factor((AtW @ A).toarray(), lower=True), AtW @ r)
        step = update(x)
        r = residuals()
        out["irls_iterations"] += 1
        if step < o["irls_step_convergence_threshold"]:
            break
    # FilterViewPairsFromOrientation, then RemoveDisconnectedViewPairs
    sq_max = (o["rotation_filter_max_degrees"] * DEG_TO_RAD) ** 2
    kept = []
    for p in pairs:
        a, b = (int(v) for v in pair_images[p])
        loop = concatenate_quaternions(concatenate_quaternions(invert_quaternion(rot[a]), rot[b]), invert_quaternion(qvec[p]))
        aa = quaternion_to_angle_axis(loop)
        out["residual_angles"][p] = np.linalg.norm(aa)
        if aa @ aa <= sq_max:
            kept.append(p)
    final, _ = largest_component(F, pair_images, kept)
    out["pair_kept"][final] = True
    for f in images:
        out["orientations"][f] = rot[f]
        out["has_orientation"][f] = True
    out.update(success=True, gauge_image=gauge)
    return out
