"""Numpy restatement of the two-view geometric verification of `colmap matches_importer --match_type pairs` (TEST
INFRASTRUCTURE; the product is csrc/verification.cu).

Per pair, TwoViewGeometryVerifier skips a pair with fewer raw matches than min_num_inliers (config UNDEFINED) and
runs TwoViewGeometry::EstimateUncalibrated on the others: LORANSAC<seven-point F, eight-point F> with the squared
Sampson error, LORANSAC<normalised DLT H, same> with the squared transfer error, the config rule, F's inliers in match
order, and DetectWatermark with LORANSAC<translation, translation>.  E stays zero.

COLMAP's estimator code is not in the reference tree: its constants are recalled (RECALLED;
csrc/verification_recalled.cuh keeps the same values).  Rules defined here where COLMAP depends on thread scheduling
or on an arbitrary basis, the same way on the device:
* Sampler: each trial's sample is drawn from a SplitMix64 stream keyed by (random_seed, pair, kind, trial) (`sample`);
  the same distribution as COLMAP's RandomSampler, not the same draws.
* The seven-point models come from the real roots of det(lambda a + b) = 0 for an orthonormal basis (a, b) of the
  null space (of det(a + mu b) = 0 when its leading coefficient det(b) is the larger one), solved by `cubic_real_roots`
  with one Newton step per root; a model whose unit-norm form has
  |F(2,2)| < 1e-10 is dropped; the others are scaled to F(2,2) = 1 and ordered by (F(0,0), F(0,1), ...).
* Stored F and H have unit Frobenius norm with the largest-magnitude entry positive (the first one on a tie).
Numpy's SVD stands where COLMAP uses Eigen's.  Every decision that rounding could flip records its margin
(result["margins"], the smallest relative margin of each kind), so that a test can tell a real disagreement from a
rounding tie."""
import math

import numpy as np

RECALLED = {
    "ransac_cap_num_samples": 100000,    # RANSAC constructor: ComputeNumTrials(min_inlier_ratio * 1e5, 1e5, ...)
    "max_num_local_trials": 10,          # LORANSAC kMaxNumLocalTrials
    "seven_point_samples": 7,            # FundamentalMatrixSevenPointEstimator::kMinNumSamples
    "eight_point_samples": 8,            # FundamentalMatrixEightPointEstimator::kMinNumSamples
    "homography_samples": 4,             # HomographyMatrixEstimator::kMinNumSamples
    "translation_samples": 1,            # TranslationTransformEstimator<2>::kMinNumSamples
    "min_f22": 1e-10,                    # the seven-point step drops a model with |F(2,2)| below this
}
DEFAULTS = {                             # what sfm/import_feature_matches.py:106-117 runs; psfm_verification_options
    "max_error": 4.0,
    "confidence": 0.999,
    "max_num_trials": 20000,
    "min_num_trials": 0,
    "min_inlier_ratio": 0.1,
    "min_num_inliers": 15,
    "dyn_num_trials_multiplier": 3.0,
    "max_H_inlier_ratio": 0.8,
    "detect_watermark": 1,
    "watermark_min_inlier_ratio": 0.7,
    "watermark_border_size": 0.1,
    "random_seed": 0,
}
UNDEFINED, DEGENERATE, CALIBRATED, UNCALIBRATED, PLANAR, PANORAMIC, PLANAR_OR_PANORAMIC, WATERMARK = range(8)
KIND_F, KIND_H, KIND_W = 0, 1, 2
UNBOUNDED = 2 ** 63 - 1
DBL_MAX = float(np.finfo(np.float64).max)
M64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15


class InvalidError(ValueError):
    """The device returns PSFM_ERR_INVALID before any launch."""


class UnsupportedError(ValueError):
    """The device returns PSFM_ERR_UNSUPPORTED before any launch."""


def check_options(o):
    """TwoViewGeometry::Options::Check() with RANSACOptions::Check()."""
    ok = (o["max_error"] > 0 and 0 <= o["confidence"] <= 1 and 0 <= o["min_inlier_ratio"] <= 1
          and 0 <= o["min_num_trials"] <= o["max_num_trials"] and o["min_num_inliers"] >= 0
          and o["dyn_num_trials_multiplier"] > 0 and o["max_H_inlier_ratio"] >= 0
          and 0 <= o["watermark_min_inlier_ratio"] <= 1 and 0 <= o["watermark_border_size"] <= 1
          and all(math.isfinite(o[k]) for k in ("max_error", "confidence", "min_inlier_ratio",
                                                "dyn_num_trials_multiplier", "max_H_inlier_ratio",
                                                "watermark_min_inlier_ratio", "watermark_border_size")))
    if not ok:
        raise InvalidError("options fail Check()")


# ---------------------------------------------------------------------------------------------------------- sampler
def mix64(z):
    """SplitMix64's finaliser on a Python int."""
    z ^= z >> 30
    z = (z * 0xBF58476D1CE4E5B9) & M64
    z ^= z >> 27
    z = (z * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def stream_key(seed, pair, kind, trial):
    """The state a trial's stream starts from: mix64(s + GOLDEN (v + 1)) folded over v = pair, kind, trial."""
    s = seed & M64
    for v in (pair, kind, trial):
        s = mix64((s + GOLDEN * (v + 1)) & M64)
    return s


def sample(seed, pair, kind, trial, n, k):
    """k distinct indices of [0, n): the stream's outputs z = mix64(s += GOLDEN) map to (z >> 32) * n >> 32, a
    repeated index is redrawn from the same stream."""
    s = stream_key(seed, pair, kind, trial)
    out = []
    while len(out) < k:
        s = (s + GOLDEN) & M64
        i = ((mix64(s) >> 32) * n) >> 32
        if i not in out:
            out.append(i)
    return out


def compute_num_trials(num_inliers, num_samples, s, confidence, multiplier, margins=None):
    """RANSAC::ComputeNumTrials for an estimator of s samples."""
    ratio = num_inliers / num_samples
    nom = 1.0 - confidence
    if nom <= 0:
        return UNBOUNDED
    denom = 1.0 - ratio ** s
    if denom <= 0:
        return 1
    ld = math.log(denom)
    if ld == 0.0:
        return UNBOUNDED
    v = math.log(nom) / ld * multiplier
    if margins is not None:
        _margin(margins, "num_trials", abs(v - round(v)) / max(1.0, abs(v)) if abs(v - round(v)) > 0 else 1.0)
    n = math.ceil(v)
    return UNBOUNDED if n >= 9.2e18 else int(n)


def _margin(margins, key, value):
    if value < margins.get(key, math.inf):
        margins[key] = value


# ------------------------------------------------------------------------------------------------------- estimators
def _newton_step(c3, c2, c1, c0, x):
    """One Newton step, kept only when it lowers |p| (at a near-multiple root p' is rounding noise)."""
    f = ((c3 * x + c2) * x + c1) * x + c0
    df = (3.0 * c3 * x + 2.0 * c2) * x + c1
    if df == 0.0:
        return x
    y = x - f / df
    g = ((c3 * y + c2) * y + c1) * y + c0
    return y if abs(g) < abs(f) else x


def _stable_quadratic(a, b, c, d):
    """The roots of a x^2 + b x + c (a != 0) for a discriminant d >= 0, without cancellation."""
    h = -0.5 * (b + math.copysign(math.sqrt(d), b))
    return [h / a, c / h if h != 0.0 else 0.0]


def _quadratic_margin(margins, a, b, c, d):
    if margins is not None:
        scale = b * b + abs(4.0 * a * c)
        _margin(margins, "cubic", abs(d) / scale if scale > 0 else 1.0)


def cubic_real_roots(c3, c2, c1, c0, margins=None):
    """Real roots of c3 x^3 + c2 x^2 + c1 x + c0, one Newton step each.  One real root r from the depressed cubic's
    closed form (Cardano with the two cube roots added without cancellation, or the trigonometric form's largest-magnitude
    root); after its Newton step r is deflated out (from the constant term when it is the largest root, from the leading
    term otherwise), and the quadratic left decides whether there are two more real roots and gives them in the stable
    form.  The depressed form yields no other root: once c3 is small its shift -c2 / 3 c3 swamps the moderate roots.
    margins["cubic"]: the relative discriminant of the quadratic that decides the count."""
    c3, c2, c1, c0 = float(c3), float(c2), float(c1), float(c0)
    if c3 == 0.0:
        if c2 == 0.0:
            return [] if c1 == 0.0 else [-c0 / c1]
        d = c1 * c1 - 4.0 * c2 * c0
        _quadratic_margin(margins, c2, c1, c0, d)
        if d < 0:
            return []
        return _stable_quadratic(c2, c1, c0, d)
    b, c, d = c2 / c3, c1 / c3, c0 / c3
    p = c - b * b / 3.0
    q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d
    disc = (q / 2.0) * (q / 2.0) + (p / 3.0) * (p / 3.0) * (p / 3.0)
    shift = -b / 3.0
    r = shift
    if disc > 0:
        A = -math.copysign(float(np.cbrt(abs(q) / 2.0 + math.sqrt(disc))), q)
        r = (A - p / (3.0 * A) if A != 0.0 else 0.0) + shift
    elif p != 0.0:
        rr = 2.0 * math.sqrt(-p / 3.0)
        a = 3.0 * q / (2.0 * p) * math.sqrt(-3.0 / p)
        phi = math.acos(min(1.0, max(-1.0, a))) / 3.0
        r = 0.0
        for k in range(3):
            t = rr * math.cos(phi - 2.0 * math.pi * k / 3.0) + shift
            if abs(t) > abs(r):
                r = t
    r = _newton_step(c3, c2, c1, c0, r)
    if r != 0.0 and abs(c3 * r * r * r) >= abs(c0):         # c3 x^2 + e1 x + e0 = p(x) / (x - r)
        e0 = -c0 / r
        e1 = (e0 - c1) / r
    else:
        e1 = c2 + c3 * r
        e0 = c1 + e1 * r
    dq = e1 * e1 - 4.0 * c3 * e0
    _quadratic_margin(margins, c3, e1, e0, dq)
    if dq < 0:
        return [r]
    x1, x2 = _stable_quadratic(c3, e1, e0, dq)
    return [r, _newton_step(c3, c2, c1, c0, x1), _newton_step(c3, c2, c1, c0, x2)]


def _det3(f):
    return (f[0] * (f[4] * f[8] - f[5] * f[7]) - f[1] * (f[3] * f[8] - f[5] * f[6])
            + f[2] * (f[3] * f[7] - f[4] * f[6]))


def seven_point(x1, x2, margins=None):
    """FundamentalMatrixSevenPointEstimator on raw pixels: the null space of the 7 x 9 system, the real roots of
    det(lambda a + b), models scaled to F(2,2) = 1 and ordered (the rules above).  Returns row-major [k][9]."""
    A = np.stack([x2[:, 0] * x1[:, 0], x2[:, 0] * x1[:, 1], x2[:, 0], x2[:, 1] * x1[:, 0], x2[:, 1] * x1[:, 1],
                  x2[:, 1], x1[:, 0], x1[:, 1], np.ones(7)], axis=1)
    vt = np.linalg.svd(A, full_matrices=True)[2]
    a, b = vt[7], vt[8]
    d0, d1, dm = _det3(b), _det3(a + b), _det3(-a + b)
    c3 = _det3(a)
    c2 = 0.5 * (d1 + dm) - d0
    c1 = 0.5 * (d1 - dm) - c3
    # when |c3| < |d0| the pencil is solved as det(a + mu b), whose leading coefficient d0 is the larger one
    flip = abs(c3) < abs(d0)
    models = []
    for lam in (cubic_real_roots(d0, c1, c2, c3, margins) if flip else cubic_real_roots(c3, c2, c1, d0, margins)):
        F = a + lam * b if flip else lam * a + b
        Fn = F / np.linalg.norm(F)
        if margins is not None:
            _margin(margins, "f22", abs(abs(Fn[8]) - RECALLED["min_f22"]) / RECALLED["min_f22"])
        if abs(Fn[8]) < RECALLED["min_f22"]:
            continue
        models.append(F / F[8])
    models.sort(key=lambda f: tuple(f))
    if margins is not None:
        for u, v in zip(models, models[1:]):
            k = int(np.nonzero(u != v)[0][0]) if np.any(u != v) else 0
            _margin(margins, "order", abs(u[k] - v[k]) / max(abs(u[k]), abs(v[k]), 1e-300))
    return models


def center_and_normalize(x):
    """CenterAndNormalizeImagePoints: centroid to the origin, RMS distance sqrt(2); returns (points, T)."""
    c = x.mean(axis=0)
    rms = math.sqrt(((x - c) ** 2).sum() / x.shape[0])
    s = math.sqrt(2.0) / rms
    T = np.array([[s, 0.0, -s * c[0]], [0.0, s, -s * c[1]], [0.0, 0.0, 1.0]])
    return (x - c) * s, T


def eight_point(x1, x2):
    """FundamentalMatrixEightPointEstimator: normalised points, null vector of the N x 9 system, the smallest singular
    value of F set to zero, denormalised."""
    n1, T1 = center_and_normalize(x1)
    n2, T2 = center_and_normalize(x2)
    o = np.ones(n1.shape[0])
    A = np.stack([n2[:, 0] * n1[:, 0], n2[:, 0] * n1[:, 1], n2[:, 0], n2[:, 1] * n1[:, 0], n2[:, 1] * n1[:, 1],
                  n2[:, 1], n1[:, 0], n1[:, 1], o], axis=1)
    f = np.linalg.svd(A, full_matrices=True)[2][8].reshape(3, 3)
    U, s, Vt = np.linalg.svd(f)
    F = U @ np.diag([s[0], s[1], 0.0]) @ Vt
    return [(T2.T @ F @ T1).ravel()]


def homography_dlt(x1, x2):
    """HomographyMatrixEstimator: normalised DLT, H = T2^-1 H~ T1."""
    n1, T1 = center_and_normalize(x1)
    n2, T2 = center_and_normalize(x2)
    N = n1.shape[0]
    A = np.zeros((2 * N, 9))
    s0, s1, d0, d1 = n1[:, 0], n1[:, 1], n2[:, 0], n2[:, 1]
    A[0::2, 0], A[0::2, 1], A[0::2, 2] = -s0, -s1, -1.0
    A[0::2, 6], A[0::2, 7], A[0::2, 8] = s0 * d0, s1 * d0, d0
    A[1::2, 3], A[1::2, 4], A[1::2, 5] = -s0, -s1, -1.0
    A[1::2, 6], A[1::2, 7], A[1::2, 8] = s0 * d1, s1 * d1, d1
    h = np.linalg.svd(A, full_matrices=True)[2][8].reshape(3, 3)
    return [(np.linalg.inv(T2) @ h @ T1).ravel()]


def translation(x1, x2):
    """TranslationTransformEstimator<2>: mean(dst) - mean(src)."""
    return [x2.mean(axis=0) - x1.mean(axis=0)]


def sampson_error(F, x1, x2):
    """ComputeSquaredSampsonError with F row-major [9]."""
    f = F
    X, Y, U, V = x1[:, 0], x1[:, 1], x2[:, 0], x2[:, 1]
    e0 = f[0] * X + f[1] * Y + f[2]
    e1 = f[3] * X + f[4] * Y + f[5]
    e2 = f[6] * X + f[7] * Y + f[8]
    t0 = f[0] * U + f[3] * V + f[6]
    t1 = f[1] * U + f[4] * V + f[7]
    c = U * e0 + V * e1 + e2
    return c * c / (e0 * e0 + e1 * e1 + t0 * t0 + t1 * t1)


def transfer_error(H, x1, x2):
    """HomographyMatrixEstimator::Residuals: squared transfer error in image 2."""
    h = H
    X, Y = x1[:, 0], x1[:, 1]
    inv = 1.0 / (h[6] * X + h[7] * Y + h[8])
    d0 = x2[:, 0] - (h[0] * X + h[1] * Y + h[2]) * inv
    d1 = x2[:, 1] - (h[3] * X + h[4] * Y + h[5]) * inv
    return d0 * d0 + d1 * d1


def translation_error(t, x1, x2):
    d0 = x2[:, 0] - (x1[:, 0] + t[0])
    d1 = x2[:, 1] - (x1[:, 1] + t[1])
    return d0 * d0 + d1 * d1


ESTIMATORS = {   # kind: (minimal estimator, its sample size, local estimator, its sample size, residual)
    KIND_F: (seven_point, 7, eight_point, 8, sampson_error),
    KIND_H: (homography_dlt, 4, homography_dlt, 4, transfer_error),
    KIND_W: (translation, 1, translation, 1, translation_error),
}


def _evaluate(r, thr, margins):
    with np.errstate(invalid="ignore"):
        ok = r <= thr
        d = np.abs(r - thr) / thr
    d = d[np.isfinite(d)]
    if d.size:
        _margin(margins, "threshold", float(d.min()))
    return int(ok.sum()), float(r[ok].sum()), ok


def _better(a, b, margins):
    if a[0] != b[0]:
        return a[0] > b[0]
    if b[1] != DBL_MAX:
        _margin(margins, "compare", abs(a[1] - b[1]) / max(abs(a[1]), abs(b[1]), 1e-300))
    return a[1] < b[1]


def loransac(kind, x1, x2, o, pair, margins, min_inlier_ratio=None):
    """LORANSAC<Estimator, LocalEstimator>::Estimate with InlierSupportMeasurer and the sampler above.  Returns a dict:
    success, num_trials (samples drawn), num_inliers, residual_sum, model (row-major, None without one), mask (match
    order; None unless success), local_rounds."""
    est, k, local, local_k, residual = ESTIMATORS[kind]
    n = x1.shape[0]
    thr = o["max_error"] ** 2
    rep = dict(success=False, num_trials=0, num_inliers=0, residual_sum=DBL_MAX, model=None, mask=None, local_rounds=0)
    if n < k:
        return rep
    ratio = o["min_inlier_ratio"] if min_inlier_ratio is None else min_inlier_ratio
    cap_n = RECALLED["ransac_cap_num_samples"]
    max_trials = min(o["max_num_trials"], compute_num_trials(int(ratio * cap_n), cap_n, k, o["confidence"],
                                                             o["dyn_num_trials_multiplier"], margins))
    dyn = max_trials
    best, best_model, best_mask = (0, DBL_MAX), None, None
    trials, rounds, abort = 0, 0, False
    for trial in range(max_trials):
        idx = sample(o["random_seed"], pair, kind, trial, n, k)
        trials = trial + 1
        models = est(x1[idx], x2[idx], margins) if kind == KIND_F else est(x1[idx], x2[idx])
        for m in models:
            ni, rs, mask = _evaluate(residual(m, x1, x2), thr, margins)
            if _better((ni, rs), best, margins):
                best, best_model, best_mask = (ni, rs), m, mask
                if ni > k and ni >= local_k:
                    for _ in range(RECALLED["max_num_local_trials"]):
                        prev = best[0]
                        for lm in local(x1[best_mask], x2[best_mask]):
                            li, ls, lmask = _evaluate(residual(lm, x1, x2), thr, margins)
                            if _better((li, ls), best, margins):
                                best, best_model, best_mask = (li, ls), lm, lmask
                        rounds += 1
                        if best[0] <= prev:
                            break
                dyn = compute_num_trials(best[0], n, k, o["confidence"], o["dyn_num_trials_multiplier"], margins)
            if trial >= dyn and trial >= o["min_num_trials"]:
                abort = True
                break
        if abort:
            break
    rep.update(num_trials=trials, num_inliers=best[0], residual_sum=best[1], model=best_model, local_rounds=rounds)
    if best[0] >= k:
        rep.update(success=True, mask=best_mask)
    return rep


def stored(M):
    """The stored form of F or H: unit Frobenius norm, largest-magnitude entry positive (the first on a tie)."""
    if M is None:
        return np.zeros(9)
    M = np.asarray(M, np.float64) / np.linalg.norm(M)
    i = int(np.argmax(np.abs(M)))
    return -M if M[i] < 0 else M


def detect_watermark(x1, x2, size1, size2, F_rep, o, pair, margins):
    """TwoViewGeometry::DetectWatermark on F's inliers; returns (is_watermark, watermark report or None, border count)."""
    if not F_rep["success"] or F_rep["num_inliers"] == 0:
        return False, None, 0
    boxes = []
    for w, h in (size1, size2):
        m = o["watermark_border_size"] * math.sqrt(float(w) * w + float(h) * h)
        boxes.append((m, w - m, m, h - m))
    mask = F_rep["mask"]
    p1, p2 = x1[mask], x2[mask]

    def inside(p, b):
        return (p[:, 0] >= b[0]) & (p[:, 0] <= b[1]) & (p[:, 1] >= b[2]) & (p[:, 1] <= b[3])
    border = int((~inside(p1, boxes[0]) & ~inside(p2, boxes[1])).sum())
    num = F_rep["num_inliers"]
    if border / num < o["watermark_min_inlier_ratio"]:
        return False, None, border
    rep = loransac(KIND_W, p1, p2, o, pair, margins, min_inlier_ratio=o["watermark_min_inlier_ratio"])
    return rep["num_inliers"] / num >= o["watermark_min_inlier_ratio"], rep, border


def verify_pair(x1, x2, size1, size2, o, pair, margins):
    """TwoViewGeometryVerifier + EstimateUncalibrated for one pair; x1, x2 [n][2] float64 matched keypoints."""
    n = x1.shape[0]
    out = dict(config=UNDEFINED, F=np.zeros(9), E=np.zeros(9), H=np.zeros(9), inliers=np.zeros(0, np.int64),
               trials=[0, 0, 0], local_rounds=[0, 0, 0], border=0)
    if n < o["min_num_inliers"]:
        return out
    Fr = loransac(KIND_F, x1, x2, o, pair, margins)
    Hr = loransac(KIND_H, x1, x2, o, pair, margins)
    out.update(F=stored(Fr["model"]), H=stored(Hr["model"]), trials=[Fr["num_trials"], Hr["num_trials"], 0],
               local_rounds=[Fr["local_rounds"], Hr["local_rounds"], 0])
    mi = o["min_num_inliers"]
    if (not Fr["success"] and not Hr["success"]) or (Fr["num_inliers"] < mi and Hr["num_inliers"] < mi):
        out["config"] = DEGENERATE
        return out
    ratio = Hr["num_inliers"] / Fr["num_inliers"] if Fr["num_inliers"] else math.inf
    out["config"] = PLANAR_OR_PANORAMIC if ratio > o["max_H_inlier_ratio"] else UNCALIBRATED
    if Fr["success"]:
        out["inliers"] = np.nonzero(Fr["mask"])[0]
    if o["detect_watermark"]:
        wm, wr, out["border"] = detect_watermark(x1, x2, size1, size2, Fr, o, pair, margins)
        if wr is not None:
            out["trials"][2], out["local_rounds"][2] = wr["num_trials"], wr["local_rounds"]
        if wm:
            out["config"] = WATERMARK
    return out


def verify_two_view_geometries(keypoint_ptr, keypoints, image_camera, camera_size, pair_images, match_ptr, matches,
                               prior_focal_length=None, options=None):
    """psfm_verify_two_view_geometries restated.  Returns a dict: config [R], F / E / H [R][9] (stored form),
    inlier_ptr [R + 1], inlier_matches [N][2] uint32, trials [R][3] (F, H, watermark samples drawn), local_rounds
    [R][3], margins."""
    o = dict(DEFAULTS)
    o.update(options or {})
    check_options(o)
    kp_ptr = np.asarray(keypoint_ptr, np.int64)
    kps = np.asarray(keypoints, np.float32).reshape(-1, 2).astype(np.float64)
    cam_of = np.asarray(image_camera, np.int64)
    size = np.asarray(camera_size, np.int64).reshape(-1, 2)
    pairs = np.asarray(pair_images, np.int64).reshape(-1, 2)
    mptr = np.asarray(match_ptr, np.int64)
    m = np.asarray(matches, np.int64).reshape(-1, 2)
    prior = np.zeros(size.shape[0], bool) if prior_focal_length is None else np.asarray(prior_focal_length, bool)
    F_img = kp_ptr.shape[0] - 1
    R = pairs.shape[0]
    seen = set()
    for p in range(R):
        a, b = int(pairs[p, 0]), int(pairs[p, 1])
        if not (0 <= a < F_img and 0 <= b < F_img) or a == b or (min(a, b), max(a, b)) in seen:
            raise InvalidError("bad pair %d" % p)
        seen.add((min(a, b), max(a, b)))
        if prior[cam_of[a]] and prior[cam_of[b]]:
            raise UnsupportedError("both cameras of pair %d have a prior focal length" % p)
    margins = {}
    res = dict(config=np.zeros(R, np.int32), F=np.zeros((R, 9)), E=np.zeros((R, 9)), H=np.zeros((R, 9)),
               trials=np.zeros((R, 3), np.int64), local_rounds=np.zeros((R, 3), np.int64))
    inl = []
    for p in range(R):
        a, b = int(pairs[p, 0]), int(pairs[p, 1])
        mm = m[mptr[p]:mptr[p + 1]]
        x1 = kps[kp_ptr[a] + mm[:, 0]]
        x2 = kps[kp_ptr[b] + mm[:, 1]]
        r = verify_pair(x1, x2, size[cam_of[a]], size[cam_of[b]], o, p, margins)
        res["config"][p] = r["config"]
        res["F"][p], res["E"][p], res["H"][p] = r["F"], r["E"], r["H"]
        res["trials"][p], res["local_rounds"][p] = r["trials"], r["local_rounds"]
        inl.append(mm[r["inliers"]].astype(np.uint32))
    res["inlier_ptr"] = np.concatenate([[0], np.cumsum([len(i) for i in inl])]).astype(np.int64)
    res["inlier_matches"] = np.concatenate(inl).reshape(-1, 2) if inl else np.zeros((0, 2), np.uint32)
    res["margins"] = margins
    return res
