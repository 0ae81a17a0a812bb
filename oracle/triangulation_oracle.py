"""Numpy restatement of GlobalMapper::TriangulateAllPoints (TEST INFRASTRUCTURE; the product is
csrc/triangulation.cu).

A literal restatement of the reference loop (sfm/global_mapper.cc:232-247): the correspondence graph of
CorrespondenceGraph::AddCorrespondences (base/correspondence_graph.cc:153-240) over the used pairs in the caller's
order, then every registered image in index order and every Point2D of it in index order through
IncrementalTriangulator::TriangulateImage (sfm/incremental_triangulator.cc:61-119): Find, Continue, Create with
EstimateTriangulation (LO-RANSAC, CombinationSampler, InlierSupportMeasurer, TriangulationEstimator).  It runs on the
whole graph, not per connected component as the device does, so agreement also checks that decomposition;
`per_component=True` runs the same loop one component at a time for the test that pins that equivalence.

COLMAP's estimator code is not in the reference tree: its constants are recalled (RECALLED; csrc/triangulation_recalled.cuh
keeps the same values).  Every threshold decision records its margin to the threshold (result["margins"]: the
smallest relative margin of each kind), so that a test can require that no decision is close enough for rounding to
flip it."""
import math

import numpy as np

RECALLED = {
    "confidence": 0.9999,                # IncrementalTriangulator::Create's ransac_options.confidence
    "min_inlier_ratio": 0.02,            # ... .min_inlier_ratio
    "max_num_trials": 10000,             # ... .max_num_trials
    "exhaustive_sampling_threshold": 15,  # kExhaustiveSamplingThreshold: min_num_trials = C(m, 2) up to this m
    "dyn_num_trials_multiplier": 3.0,    # RANSACOptions::dyn_num_trials_multiplier default
    "ransac_cap_num_samples": 100000,    # RANSAC constructor: ComputeNumTrials(min_inlier_ratio * 1e5, 1e5, ...)
    "max_num_local_trials": 10,          # LORANSAC kMaxNumLocalTrials
    "min_num_samples": 2,                # TriangulationEstimator::kMinNumSamples
    "depth_epsilon": float(np.finfo(np.float64).eps),   # HasPointPositiveDepth: depth >= epsilon
}
DEFAULTS = {                             # IncrementalTriangulator::Options (sfm/incremental_triangulator.h:46-89)
    "max_transitivity": 1,
    "create_max_angle_error": 2.0,
    "continue_max_angle_error": 2.0,
    "min_angle": 1.5,
    "ignore_two_view_tracks": True,
    "min_focal_length_ratio": 0.1,       # gcolmap overrides (controllers/global_mapper.cc:73-79) with equal values
    "max_focal_length_ratio": 10.0,
    "max_extra_param": 1.0,
}
UNBOUNDED = 2 ** 63 - 1                  # ComputeNumTrials of a support without inliers (the reference casts -inf)


class InvalidError(ValueError):
    """The device returns PSFM_ERR_INVALID before any launch."""


class UnsupportedError(ValueError):
    """The device returns PSFM_ERR_UNSUPPORTED before any launch."""


def check_options(o):
    """IncrementalTriangulator::Options::Check() (incremental_triangulator.cc:40-53) on the fields TriangulateImage
    reads, plus the bogus-camera thresholds' GlobalMapperOptions::Check() rules."""
    ok = (o["max_transitivity"] >= 0 and o["create_max_angle_error"] > 0 and o["continue_max_angle_error"] > 0
          and o["min_angle"] > 0 and o["min_focal_length_ratio"] > 0 and o["max_focal_length_ratio"] > 0
          and o["max_extra_param"] >= 0
          and all(math.isfinite(o[k]) for k in ("create_max_angle_error", "continue_max_angle_error", "min_angle",
                                                "min_focal_length_ratio", "max_focal_length_ratio", "max_extra_param")))
    if not ok:
        raise InvalidError("options fail Check()")
    if o["max_transitivity"] != 1:
        raise UnsupportedError("max_transitivity != 1")


def quat_to_rotmat(q):
    w, x, y, z = np.asarray(q, np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def has_bogus_params(cam, size, o):
    """Camera::HasBogusParams for SIMPLE_PINHOLE (f, cx, cy): the principal point outside [0, w] x [0, h], or
    f / max(w, h) outside [min_focal_length_ratio, max_focal_length_ratio].  SIMPLE_PINHOLE has no extra
    parameter, so max_extra_param never decides."""
    f, cx, cy = cam
    w, h = size
    if cx < 0 or cx > w or cy < 0 or cy > h:
        return True
    r = f / max(w, h)
    return r < o["min_focal_length_ratio"] or r > o["max_focal_length_ratio"]


def angle_between(r1, r2):
    """The angle between rays r1 and r2 ([..., 3]).  The reference takes acos of the normalised dot product; the
    same angle is evaluated here as atan2(|r1 x r2|, r1 . r2), which keeps its relative accuracy near zero, where
    the support comparison of two models with the same inliers is decided (acos loses it there, and returns NaN when
    rounding pushes the dot product past 1)."""
    c = np.cross(r1, r2)
    return np.arctan2(np.sqrt((c * c).sum(-1)), (r1 * r2).sum(-1))


def triangulation_angle(c1, c2, X):
    """CalculateTriangulationAngle (law of cosines, the smaller of the angle and its supplement)."""
    b2 = ((c1 - c2) ** 2).sum(-1)
    r1 = ((X - c1) ** 2).sum(-1)
    r2 = ((X - c2) ** 2).sum(-1)
    den = 2.0 * np.sqrt(r1 * r2)
    with np.errstate(invalid="ignore", divide="ignore"):
        a = np.abs(np.arccos((r1 + r2 - b2) / den))
    a = np.minimum(a, np.pi - a)
    return np.where(den == 0.0, 0.0, a)


def compute_num_trials(num_inliers, num_samples, confidence, multiplier, margins=None):
    """RANSAC::ComputeNumTrials.  A ratio whose square rounds 1 - r^2 to 1 (no inlier) gives log(denom) = 0; the
    reference casts the resulting -inf to size_t, here it is UNBOUNDED."""
    ratio = num_inliers / float(num_samples)
    nom = 1.0 - confidence
    if nom <= 0:
        return UNBOUNDED
    denom = 1.0 - ratio * ratio
    if denom <= 0:
        return 1
    ld = math.log(denom)
    if ld == 0.0:
        return UNBOUNDED
    v = math.log(nom) / ld * multiplier
    if margins is not None and v < 2 ** 62:
        _margin(margins, "num_trials", abs(v - round(v)) / max(v, 1.0))
    n = math.ceil(v)
    return UNBOUNDED if n >= 9.2e18 else int(n)


def max_num_trials_cap():
    """The RANSAC constructor's cap of max_num_trials by min_inlier_ratio."""
    n = RECALLED["ransac_cap_num_samples"]
    return min(RECALLED["max_num_trials"],
               compute_num_trials(int(RECALLED["min_inlier_ratio"] * n), n, RECALLED["confidence"],
                                  RECALLED["dyn_num_trials_multiplier"]))


def combination(t, m):
    """The t-th sample (0-based) of CombinationSampler with 2 of m: (0, 1), (0, 2), ..., (0, m-1), (1, 2), ..."""
    i = 0
    while t >= m - 1 - i:
        t -= m - 1 - i
        i += 1
    return i, i + 1 + t


def _margin(margins, kind, value):
    margins[kind] = min(margins.get(kind, np.inf), float(value))


def two_view_dlt(P1, P2, x1, x2):
    """TriangulatePoint: the right singular vector of the smallest singular value of the 4 x 4 DLT matrix, [B]."""
    A = np.stack([x1[..., 0:1] * P1[..., 2, :] - P1[..., 0, :], x1[..., 1:2] * P1[..., 2, :] - P1[..., 1, :],
                  x2[..., 0:1] * P2[..., 2, :] - P2[..., 0, :], x2[..., 1:2] * P2[..., 2, :] - P2[..., 1, :]], -2)
    v = np.linalg.svd(A)[2][..., 3, :]
    return v[..., :3] / v[..., 3:]


def multi_view_dlt(P, x):
    """TriangulateMultiViewPoint: the eigenvector of the smallest eigenvalue of sum (P - r r' P)' (P - r r' P)."""
    A = np.zeros((4, 4))
    for Pi, xi in zip(P, x):
        r = np.array([xi[0], xi[1], 1.0])
        r /= np.linalg.norm(r)
        T = Pi - np.outer(r, r @ Pi)
        A += T.T @ T
    v = np.linalg.eigh(A)[1][:, 0]
    return v[:3] / v[3]


class _Obs:
    """The PointData / PoseData of one list of observations."""

    def __init__(self, P, C, x):
        self.P, self.C, self.x = P, C, x

    def residuals(self, X, thr, margins):
        """Squared CalculateNormalizedAngularError of every observation (ProjectionMatrix form), [m]."""
        ray = self.P @ np.append(X, 1.0)
        r1 = np.concatenate([self.x, np.ones((len(self.x), 1))], 1)
        r = angle_between(r1, ray) ** 2
        _margin(margins, "inlier", np.min(np.abs(r - thr)) / thr)
        return r

    def depth_ok(self, idx, X, margins):
        d = self.P[idx, 2, :3] @ X + self.P[idx, 2, 3]
        _margin(margins, "depth", np.min(np.abs(d - RECALLED["depth_epsilon"])) / (1.0 + np.linalg.norm(X)))
        return bool((d >= RECALLED["depth_epsilon"]).all())


def _support(r, thr):
    inl = r <= thr
    s = np.cumsum(r[inl])
    return int(inl.sum()), float(s[-1]) if len(s) else 0.0


def _better(s1, s2, margins):
    """InlierSupportMeasurer::Compare: more inliers, then a smaller residual sum."""
    if s1[0] != s2[0]:
        return s1[0] > s2[0]
    if s1[0] > 0:                        # without inliers both sums are exactly 0
        _margin(margins, "support", abs(s1[1] - s2[1]) / max(s1[1], s2[1], 1e-300))
    return s1[1] < s2[1]


def _local_model(obs, inl, min_tri, margins):
    """TriangulationEstimator::Estimate on the inliers (> 2 of them: the multi-view branch)."""
    idx = np.nonzero(inl)[0]
    X = multi_view_dlt(obs.P[idx], obs.x[idx])
    if not obs.depth_ok(idx, X, margins):
        return None
    for a in range(len(idx)):
        for b in range(a):
            ang = triangulation_angle(obs.C[idx[a]], obs.C[idx[b]], X)
            _margin(margins, "tri_angle", abs(ang - min_tri) / min_tri)
            if ang >= min_tri:
                return X
    return None


def estimate_triangulation(obs, o, stats, margins, batch=64):
    """EstimateTriangulation with Create's options: LORANSAC<TriangulationEstimator, TriangulationEstimator,
    InlierSupportMeasurer, CombinationSampler>.  Returns (inlier mask, xyz) or None."""
    m = len(obs.x)
    thr = np.deg2rad(o["create_max_angle_error"]) ** 2
    min_tri = np.deg2rad(o["min_angle"])
    max_trials = min(max_num_trials_cap(), m * (m - 1) // 2)
    min_trials = m * (m - 1) // 2 if m <= RECALLED["exhaustive_sampling_threshold"] else 0
    best, best_X = (0, np.finfo(np.float64).max), None
    dyn = max_trials
    trials = 0
    t = 0
    done = False
    while t < max_trials and not done:
        ts = list(range(t, min(t + batch, max_trials)))
        ij = np.array([combination(u, m) for u in ts])
        Xs = two_view_dlt(obs.P[ij[:, 0]], obs.P[ij[:, 1]], obs.x[ij[:, 0]], obs.x[ij[:, 1]])
        for k, u in enumerate(ts):
            trials += 1
            i, j = ij[k]
            X = Xs[k]
            # TriangulationEstimator::Estimate, two-view branch
            if not obs.depth_ok(np.array([i, j]), X, margins):
                continue
            ang = triangulation_angle(obs.C[i], obs.C[j], X)
            _margin(margins, "tri_angle", abs(ang - min_tri) / min_tri)
            if not ang >= min_tri:
                continue
            r = obs.residuals(X, thr, margins)
            sup = _support(r, thr)
            if _better(sup, best, margins):
                best, best_X = sup, X
                if sup[0] > RECALLED["min_num_samples"]:
                    cur = X
                    for _ in range(RECALLED["max_num_local_trials"]):
                        inl = obs.residuals(cur, thr, margins) <= thr
                        prev = best[0]
                        stats["local_estimates"] += 1
                        Xl = _local_model(obs, inl, min_tri, margins)
                        if Xl is not None:
                            ls = _support(obs.residuals(Xl, thr, margins), thr)
                            if _better(ls, best, margins):
                                best, best_X, cur = ls, Xl, Xl
                        if best[0] <= prev:
                            break
                dyn = compute_num_trials(best[0], m, RECALLED["confidence"], RECALLED["dyn_num_trials_multiplier"],
                                         margins)
            # the trial bound is tested inside the per-model loop: a sample without a model cannot end the loop
            if u >= dyn and u >= min_trials:
                done = True
                break
        t = ts[-1] + 1
    stats["ransac_trials"] += trials
    if best[0] < RECALLED["min_num_samples"]:
        return None
    return obs.residuals(best_X, thr, margins) <= thr, best_X


def build_graph(keypoint_ptr, pair_images, inlier_ptr, inlier_matches, pair_used):
    """CorrespondenceGraph::AddCorrespondences over the used pairs in array order: both points' lists receive the
    match, unless either point already has an accepted correspondence into the other image.  Returns the lists as
    (ptr [K + 1], nbr [..]) in push_back order."""
    K = int(keypoint_ptr[-1])
    src, dst = [], []
    for p in range(len(pair_images)):
        if pair_used is not None and not pair_used[p]:
            continue
        a, b = (int(v) for v in pair_images[p])
        mm = np.asarray(inlier_matches[inlier_ptr[p]:inlier_ptr[p + 1]], np.int64)
        if len(np.unique(mm[:, 0])) == len(mm) and len(np.unique(mm[:, 1])) == len(mm):
            keep = mm
        else:
            seen1, seen2, rows = set(), set(), []
            for i, j in mm.tolist():
                if i in seen1 or j in seen2:
                    continue
                seen1.add(i)
                seen2.add(j)
                rows.append((i, j))
            keep = np.array(rows, np.int64).reshape(-1, 2)
        ka, kb = keypoint_ptr[a] + keep[:, 0], keypoint_ptr[b] + keep[:, 1]
        # push_back order: per match, corrs1 then corrs2 (different lists); a list's entries in pair, then match order
        src.append(np.stack([ka, kb], 1).ravel())
        dst.append(np.stack([kb, ka], 1).ravel())
    src = np.concatenate(src) if src else np.zeros(0, np.int64)
    dst = np.concatenate(dst) if dst else np.zeros(0, np.int64)
    order = np.argsort(src, kind="stable")
    ptr = np.zeros(K + 1, np.int64)
    np.add.at(ptr, src + 1, 1)
    return np.cumsum(ptr), dst[order]


def components(ptr, nbr, img_of, eligible):
    """Connected components of the correspondence graph restricted to eligible images (label = smallest keypoint)."""
    K = len(ptr) - 1
    parent = np.arange(K)

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for k in range(K):
        if not eligible[img_of[k]]:
            continue
        for v in nbr[ptr[k]:ptr[k + 1]]:
            if eligible[img_of[v]]:
                a, b = find(k), find(int(v))
                if a != b:
                    parent[max(a, b)] = min(a, b)
    return np.array([find(k) for k in range(K)])


def triangulate_all_points(keypoint_ptr, keypoints, image_camera, cameras, pair_images, inlier_ptr, inlier_matches,
                           camera_size, orientations, image_tvec, registered, pair_used=None, options=None,
                           per_component=False):
    o = dict(DEFAULTS)
    o.update(options or {})
    check_options(o)
    kp_ptr = np.asarray(keypoint_ptr, np.int64)
    kps = np.asarray(keypoints, np.float32).reshape(-1, 2).astype(np.float64)
    cams = np.asarray(cameras, np.float64).reshape(-1, 3)
    sizes = np.asarray(camera_size, np.float64).reshape(-1, 2)
    cam_of = np.asarray(image_camera, np.int64)
    pairs = np.asarray(pair_images, np.int64).reshape(-1, 2)
    q = np.asarray(orientations, np.float64).reshape(-1, 4)
    tv = np.asarray(image_tvec, np.float64).reshape(-1, 3)
    reg = np.asarray(registered, bool)
    F, K = len(kp_ptr) - 1, int(kp_ptr[-1])
    if (pairs[:, 0] == pairs[:, 1]).any():
        raise InvalidError("a pair of an image with itself")
    if len(np.unique(np.sort(pairs, 1), axis=0)) != len(pairs):
        raise InvalidError("an unordered image pair is listed twice")
    if (sizes <= 0).any():
        raise InvalidError("a camera size <= 0")
    P = np.zeros((F, 3, 4))
    Cc = np.zeros((F, 3))
    for f in np.nonzero(reg)[0]:
        if not (np.isfinite(q[f]).all() and np.isfinite(tv[f]).all()):
            raise InvalidError("a registered image with a non-finite pose")
        R = quat_to_rotmat(q[f])
        P[f] = np.concatenate([R, tv[f][:, None]], 1)
        Cc[f] = -R.T @ tv[f]
    eligible = reg & np.array([not has_bogus_params(cams[cam_of[f]], sizes[cam_of[f]], o) for f in range(F)], bool)
    img_of = np.repeat(np.arange(F), np.diff(kp_ptr))
    xn = np.zeros((K, 2))
    for f in range(F):
        c = cams[cam_of[f]]
        xn[kp_ptr[f]:kp_ptr[f + 1]] = (kps[kp_ptr[f]:kp_ptr[f + 1]] - c[1:]) / c[0]
    used = None if pair_used is None else np.asarray(pair_used, bool)
    ptr, nbr = build_graph(kp_ptr, pairs, np.asarray(inlier_ptr, np.int64), np.asarray(inlier_matches, np.int64).reshape(-1, 2), used)
    label = components(ptr, nbr, img_of, eligible)
    deg_full = np.diff(ptr)
    active = np.zeros(K, bool)
    for k in range(K):
        if eligible[img_of[k]]:
            active[k] = any(eligible[img_of[v]] for v in nbr[ptr[k]:ptr[k + 1]])
    comp_labels, comp_sizes = np.unique(label[active], return_counts=True)

    stats = {"points": 0, "continued": 0, "ransac_trials": 0, "local_estimates": 0}
    margins = {}
    pt_of = np.full(K, -1, np.int64)      # creation index of the keypoint's point
    points = []                            # [creating keypoint, peel, xyz, track list]
    cont_max = np.deg2rad(o["continue_max_angle_error"])

    def is_two_view(k):
        if deg_full[k] != 1:
            return False
        return deg_full[nbr[ptr[k]]] == 1

    def create(lst, ref):
        cur = [k for k in lst if pt_of[k] < 0]
        peel = 0
        while len(cur) >= 2:
            if o["ignore_two_view_tracks"] and len(cur) == 2 and is_two_view(cur[0]):
                break
            idx = np.array(cur)
            res = estimate_triangulation(_Obs(P[img_of[idx]], Cc[img_of[idx]], xn[idx]), o, stats, margins)
            if res is None:
                break
            inl, X = res
            pid = len(points)
            points.append([ref, peel, X, [k for k, b in zip(cur, inl) if b]])
            for k in points[-1][3]:
                pt_of[k] = pid
            cur = [k for k, b in zip(cur, inl) if not b]
            peel += 1

    def cont(ref, lst):
        if pt_of[ref] >= 0:
            return
        f = img_of[ref]
        r1 = np.array([xn[ref, 0], xn[ref, 1], 1.0])
        best, best_k = np.finfo(np.float64).max, -1
        for k in lst:
            if pt_of[k] < 0:
                continue
            X = points[pt_of[k]][2]
            # CalculateAngularError: the qvec / tvec form (QuaternionRotatePoint(q, X) + t)
            err = float(angle_between(r1, P[f, :, :3] @ X + P[f, :, 3]))
            if best_k >= 0 and pt_of[k] != pt_of[best_k]:      # observations of one point tie exactly
                _margin(margins, "continue_order", abs(err - best) / max(err, best, 1e-300))
            if err < best:
                best, best_k = err, k
        if best_k >= 0:
            _margin(margins, "continue", abs(best - cont_max) / cont_max)
        if best_k >= 0 and best <= cont_max:
            points[pt_of[best_k]][3].append(ref)
            pt_of[ref] = pt_of[best_k]
            stats["continued"] += 1

    def triangulate_observation(k):
        lst = [int(v) for v in nbr[ptr[k]:ptr[k + 1]] if eligible[img_of[v]]]
        if not lst:
            return
        ntri = sum(pt_of[v] >= 0 for v in lst)
        if ntri > 0:
            cont(k, lst)
        create(lst + [k], k)

    if per_component:
        for lab in comp_labels:
            for k in np.nonzero(active & (label == lab))[0]:
                triangulate_observation(int(k))
    else:
        for f in range(F):                 # GlobalMapper::TriangulateAllPoints: registered images, ascending
            if not eligible[f]:            # TriangulateImage returns at once for a bogus camera
                continue
            for k in range(kp_ptr[f], kp_ptr[f + 1]):
                triangulate_observation(int(k))

    # AddPoint3D numbers points in creation order: (creating keypoint, peel index) is that order
    order = sorted(range(len(points)), key=lambda i: (points[i][0], points[i][1]))
    new_id = np.empty(len(points), np.int64)
    new_id[order] = np.arange(len(points))
    xyz = np.array([points[i][2] for i in order]).reshape(-1, 3)
    tracks = [points[i][3] for i in order]
    track_ptr = np.concatenate([[0], np.cumsum([len(t) for t in tracks])]).astype(np.int64)
    elems = np.array([k for t in tracks for k in t], np.int64)
    stats["points"] = len(points)
    return {
        "xyz": xyz,
        "track_ptr": track_ptr,
        "track_image": img_of[elems].astype(np.int32) if len(elems) else np.zeros(0, np.int32),
        "track_point2D": (elems - kp_ptr[img_of[elems]]).astype(np.int32) if len(elems) else np.zeros(0, np.int32),
        "point3D_of_keypoint": np.where(pt_of >= 0, new_id[np.maximum(pt_of, 0)] if len(points) else -1, -1),
        "num_components": len(comp_labels),
        "largest_component": int(comp_sizes.max()) if len(comp_sizes) else 0,
        "num_points3D": len(points),
        "num_continued": stats["continued"],
        "num_ransac_trials": stats["ransac_trials"],
        "num_local_estimates": stats["local_estimates"],
        "margins": margins,
    }
