"""The exact-Schur LM step of every reduced-system path against an extended-precision reference.

The reference assembles the Jacobi-scaled, LM-damped reduced camera system S, its right-hand side
and the per-point blocks H_p in np.longdouble (x86 80-bit) from the oracle's loss-corrected
Jacobians and residuals, and solves it by fp64 Cholesky with longdouble iterative refinement.

The GPU step is judged by measures that do not depend on the conditioning of S:
  * camera step: componentwise (Oettli-Prager) backward error max_k |S x - b|_k / (|S||x| + |b|)_k;
    an error delta in one block of S shows up as about delta in that image's rows;
  * point steps: the same normalisation of H_p y_p + sum_i W_i' y_c(img_i) - g_p;
  * forward error against the reference, bounded by 1e-12 + c kappa_2(S equilibrated) u;
  * inactive slots and unobserved points are exactly 0.0.

The non-GPU tests at the top pin the reference itself against the oracle's exact Schur step and
against a dense solve of the full normal equations.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg

import oracle
from particlesfm_b200 import _abi, synthetic as syn

LD = np.longdouble
U64 = 2.0 ** -53
TILE_ZCAP_ROWS = 27           # NVX2: reduction rows of the fused tile kernel that hold the dense Z


def _opts(rot, focal, loss=_abi.LOSS_SOFT_L1):
    o = oracle.ba_global_options(refine_rotation=rot, refine_focal_length=focal)
    o.linear_solver = _abi.SOLVER_EXACT_SCHUR
    o.loss_function_type = loss
    return o


# ----------------------------------------------------------------------------- the reference

def _active_slots(prob, o):
    """Camera-side slots that are free parameters: the rules of resolve_cfg / the oracle's ctx_init
    (refine flags, pose_constant, tvec_constant_mask, camera_constant, unobserved images / cameras)."""
    F, C = prob.num_images, prob.num_cameras
    act = np.zeros(6 * F + 3 * C, bool)
    img_obs = np.zeros(F, bool)
    img_obs[prob.obs_image] = True
    cam_obs = np.zeros(C, bool)
    cam_obs[prob.image_camera[prob.obs_image]] = True
    for i in range(F):
        if not img_obs[i] or not o.refine_extrinsics or prob.pose_constant[i]:
            continue
        act[6 * i:6 * i + 3] = bool(o.refine_rotation)
        for k in range(3):
            act[6 * i + 3 + k] = not (int(prob.tvec_constant_mask[i]) >> k) & 1
    constant_camera = not (o.refine_focal_length or o.refine_principal_point or o.refine_extra_params)
    for c in range(C):
        if not cam_obs[c] or constant_camera or prob.camera_constant[c]:
            continue
        act[6 * F + 3 * c] = bool(o.refine_focal_length)
        act[6 * F + 3 * c + 1:6 * F + 3 * c + 3] = bool(o.refine_principal_point)
    return act


def _inv3(A):
    """Closed-form inverse of a stack of 3x3 matrices (adjugate / determinant), in A's dtype."""
    a, b, c = A[:, 0, 0], A[:, 0, 1], A[:, 0, 2]
    d, e, f = A[:, 1, 0], A[:, 1, 1], A[:, 1, 2]
    g, h, i = A[:, 2, 0], A[:, 2, 1], A[:, 2, 2]
    adj = np.stack([np.stack([e * i - f * h, c * h - b * i, b * f - c * e], -1),
                    np.stack([f * g - d * i, a * i - c * g, c * d - a * f], -1),
                    np.stack([d * h - e * g, b * g - a * h, a * e - b * d], -1)], 1)
    det = a * adj[:, 0, 0] + b * adj[:, 1, 0] + c * adj[:, 2, 0]
    return adj / det[:, None, None]


class Reference:
    pass


def _reference(prob, o, radius):
    """One exact LM step (Ceres' Jacobi scaling and LM diagonal) in longdouble: S, b, H_p and
    the solution x (camera slots, scaled space) and y_p (points).  The returned step is -x, -y."""
    jc, jp, jk = oracle.ba_jacobians(prob, o)
    _, r, _, _ = oracle.ba_evaluate(prob, o)
    F, P, C = prob.num_images, prob.num_points, prob.num_cameras
    NS = 6 * F + 3 * C
    act = _active_slots(prob, o)
    img = prob.obs_image.astype(np.int64)
    pt = prob.obs_point.astype(np.int64)
    cam = prob.image_camera[img].astype(np.int64)
    cols = np.concatenate([6 * img[:, None] + np.arange(6), 6 * F + 3 * cam[:, None] + np.arange(3)], 1)
    Jc = np.concatenate([jc, jk], 2).astype(LD) * act[cols][:, None, :]
    Jp = jp.astype(LD)
    r = r.astype(LD)
    # Jacobi scaling s = 1 / (1 + ||col||), LM diagonal D^2 = clip(colsq(J s), 1e-6, 1e32) / radius
    csq = np.zeros(NS, LD)
    np.add.at(csq, cols, (Jc * Jc).sum(1))
    psq = np.zeros((P, 3), LD)
    np.add.at(psq, pt, (Jp * Jp).sum(1))
    sc = 1 / (1 + np.sqrt(csq))
    sp = 1 / (1 + np.sqrt(psq))
    Jc = Jc * sc[cols][:, None, :]
    Jp = Jp * sp[pt][:, None, :]
    Dc2 = np.where(act, np.clip(csq * sc * sc, LD(1e-6), LD(1e32)) / LD(radius), LD(0))
    Dp2 = np.clip(psq * sp * sp, LD(1e-6), LD(1e32)) / LD(radius)
    # every sum is formed twice: its value, and the sum of the magnitudes of its terms (|S|, |b|, |H_p|, |W|,
    # |g_p| below) that fp64 rounding of the same sum, or of the data it is summed from, is relative to
    aJc, aJp, ar = np.abs(Jc), np.abs(Jp), np.abs(r)
    S = np.zeros((NS, NS), LD)
    Sa = np.zeros((NS, NS), LD)
    np.add.at(S, (cols[:, :, None], cols[:, None, :]), np.einsum("mki,mkj->mij", Jc, Jc))
    np.add.at(Sa, (cols[:, :, None], cols[:, None, :]), np.einsum("mki,mkj->mij", aJc, aJc))
    S[np.arange(NS), np.arange(NS)] += Dc2
    Sa[np.arange(NS), np.arange(NS)] += Dc2
    g = np.zeros(NS, LD)
    ga = np.zeros(NS, LD)
    np.add.at(g, cols, np.einsum("mki,mk->mi", Jc, r))
    np.add.at(ga, cols, np.einsum("mki,mk->mi", aJc, ar))
    H = np.zeros((P, 3, 3), LD)
    Ha = np.zeros((P, 3, 3), LD)
    np.add.at(H, pt, np.einsum("mki,mkj->mij", Jp, Jp))
    np.add.at(Ha, pt, np.einsum("mki,mkj->mij", aJp, aJp))
    H[:, [0, 1, 2], [0, 1, 2]] += Dp2
    Ha[:, [0, 1, 2], [0, 1, 2]] += Dp2
    gp = np.zeros((P, 3), LD)
    gpa = np.zeros((P, 3), LD)
    np.add.at(gp, pt, np.einsum("mki,mk->mi", Jp, r))
    np.add.at(gpa, pt, np.einsum("mki,mk->mi", aJp, ar))
    W = np.einsum("mki,mkj->mij", Jc, Jp)                        # (M, 9, 3) = Jc' Jp per observation
    Wa = np.einsum("mki,mkj->mij", aJc, aJp)
    Hinv = _inv3(H)
    aHinv = np.abs(Hinv)
    # S -= sum_p W_p H_p^-1 W_p', points grouped by track length
    order = np.argsort(pt, kind="stable")
    cnt = np.bincount(pt, minlength=P)
    start = np.concatenate([[0], np.cumsum(cnt)])
    for L in np.unique(cnt[cnt > 0]):
        pts = np.flatnonzero(cnt == L)
        idx = order[start[pts][:, None] + np.arange(L)]          # (nP, L) observations of each point
        if 9 * L <= 120:
            step = max(1, 2_000_000 // (81 * L * L))
            for a in range(0, len(pts), step):
                p_, i_ = pts[a:a + step], idx[a:a + step]
                Wg = W[i_].reshape(len(p_), 9 * L, 3)
                Wga = Wa[i_].reshape(len(p_), 9 * L, 3)
                cg = cols[i_].reshape(len(p_), 9 * L)
                B = Wg @ Hinv[p_] @ np.swapaxes(Wg, 1, 2)
                np.add.at(S, (cg[:, :, None], cg[:, None, :]), -B)
                np.add.at(Sa, (cg[:, :, None], cg[:, None, :]), Wga @ aHinv[p_] @ np.swapaxes(Wga, 1, 2))
        else:
            for p_, i_ in zip(pts, idx):
                u, inv = np.unique(cols[i_].ravel(), return_inverse=True)
                Wm, Wma = np.zeros((len(u), 3), LD), np.zeros((len(u), 3), LD)
                np.add.at(Wm, inv, W[i_].reshape(-1, 3))
                np.add.at(Wma, inv, Wa[i_].reshape(-1, 3))
                S[np.ix_(u, u)] -= Wm @ Hinv[p_] @ Wm.T
                Sa[np.ix_(u, u)] += Wma @ aHinv[p_] @ Wma.T
    t = np.einsum("mij,mj->mi", Hinv[pt], gp[pt])
    b = g.copy()
    np.add.at(b, cols, -np.einsum("mij,mj->mi", W, t))
    np.add.at(ga, cols, np.einsum("mij,mj->mi", Wa, np.einsum("mij,mj->mi", aHinv[pt], gpa[pt])))
    off = ~act
    for A in (S, Sa):
        A[off, :] = 0
        A[:, off] = 0
        A[off, off] = 1
    b[off] = 0
    ga[off] = 0
    ia = np.flatnonzero(act)
    x = np.zeros(NS, LD)
    if len(ia):
        Sii, bi = S[np.ix_(ia, ia)], b[ia]
        cf = scipy.linalg.cho_factor(Sii.astype(np.float64))
        xa = scipy.linalg.cho_solve(cf, bi.astype(np.float64)).astype(LD)
        for _ in range(3):                                       # mixed-precision iterative refinement
            xa = xa + scipy.linalg.cho_solve(cf, (bi - Sii @ xa).astype(np.float64)).astype(LD)
        x[ia] = xa
    q = gp.copy()
    np.add.at(q, pt, -np.einsum("mij,mi->mj", W, x[cols]))
    R = Reference()
    R.S, R.b, R.x, R.act, R.H, R.W, R.gp, R.cols, R.pt, R.sp = S, b, x, act, H, W, gp, cols, pt, sp
    R.Sa, R.ba, R.Ha, R.Wa, R.gpa = Sa, ga, Ha, Wa, gpa
    R.y = np.einsum("pij,pj->pi", Hinv, q)
    R.observed = cnt > 0
    R.F = F
    return R


# ----------------------------------------------------------------------------- measures

def _slot_name(R, k):
    return f"image {k // 6} slot {k % 6}" if k < 6 * R.F else f"camera {(k - 6 * R.F) // 3} slot {(k - 6 * R.F) % 3}"


def cam_backward_error(R, x):
    """max over active rows of |S x - b| / (|S||x| + |b|), and the worst row.  |S| and |b| are the sums of the
    magnitudes of the terms S and b are formed from (|J|'|J| + D^2 + sum_p |W_p| |H_p^-1| |W_p|', |J|'|r| + ...):
    the measure is the relative perturbation of the Jacobian data that makes x exact.  S itself can be far smaller
    than its terms: an image whose points are observed once loses almost all of J'J to the Schur complement, and
    so does any fp64 formation of S (the oracle's too)."""
    x = np.asarray(x, LD)
    res = np.abs(R.S @ x - R.b)
    den = R.Sa @ np.abs(x) + R.ba
    rows = np.flatnonzero(R.act & (den > 0))
    if len(rows) == 0:
        return 0.0, -1
    be = res[rows] / den[rows]
    k = int(np.argmax(be))
    return float(be[k]), int(rows[k])


def point_backward_error(R, x, y, xyz):
    """max over observed points of |H_p y_p + sum_i W_i' x(img_i) - g_p| / (|H_p||y_p| + sum_i |W_i'||x| + |g_p|)
    (magnitudes as in cam_backward_error).
    A GPU point step is rebuilt as (Xc - X) / s: allowed on top, explicitly, is the residual |H_p| e_p of its
    absolute rounding e_p = 2u (|X_p| / s_p + |y_p|)."""
    x, y = np.asarray(x, LD), np.asarray(y, LD)
    res = np.einsum("pij,pj->pi", R.H, y) - R.gp
    np.add.at(res, R.pt, np.einsum("mij,mi->mj", R.W, x[R.cols]))
    den = np.einsum("pij,pj->pi", R.Ha, np.abs(y)) + R.gpa
    np.add.at(den, R.pt, np.einsum("mij,mi->mj", R.Wa, np.abs(x[R.cols])))
    e = 2 * LD(U64) * (np.abs(np.asarray(xyz, LD)) / R.sp + np.abs(y))
    allow = np.einsum("pij,pj->pi", R.Ha, e)
    ok = R.observed[:, None] & (den > 0)
    be = np.where(ok, np.maximum(np.abs(res) - allow, 0) / np.where(ok, den, 1), 0)
    k = int(np.argmax(be))
    return float(be.flat[k]), k // 3


def forward_error(R, x):
    """||d (x - x_ref)||_2 / ||d x_ref||_2 with d = sqrt(diag S), and kappa_2 of the equilibrated S."""
    ia = np.flatnonzero(R.act)
    if len(ia) == 0:
        return 0.0, 1.0
    d = np.sqrt(np.diag(R.S)[ia])
    Se = (R.S[np.ix_(ia, ia)] / d[:, None] / d[None, :]).astype(np.float64)
    ev = np.linalg.eigvalsh(Se)
    kappa = ev[-1] / max(ev[0], ev[-1] * 1e-300)
    num = np.linalg.norm((d * (np.asarray(x, LD)[ia] - R.x[ia])).astype(np.float64))
    den = np.linalg.norm((d * R.x[ia]).astype(np.float64))
    return float(num / den) if den > 0 else float(num), float(kappa)


# ----------------------------------------------------------------------------- non-GPU: pin the reference

def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("loss", [_abi.LOSS_TRIVIAL, _abi.LOSS_SOFT_L1, _abi.LOSS_CAUCHY])
@pytest.mark.parametrize("rot,focal", [(False, False), (True, True)])
def test_reference_matches_oracle_exact_schur(rot, focal, loss):
    prob, _ = syn.make_ba_problem(9, 250, 5, seed=61, track_len_range=(2, 6))
    o = _opts(rot, focal, loss)
    for radius in (1e4, 1e1):
        R = _reference(prob, o, radius)
        sc0, sp0, _ = oracle.ba_linear_step(prob, o, radius, _abi.SOLVER_EXACT_SCHUR)
        assert _rel(-R.x.astype(np.float64), sc0) < 1e-10, (rot, focal, loss, radius)
        assert _rel(-R.y.astype(np.float64), sp0) < 1e-10, (rot, focal, loss, radius)
        assert np.array_equal(sc0[~R.act], np.zeros((~R.act).sum()))


def _dense_normal_equations_step(prob, o, radius, act):
    """(J'J + D^2) y = J'r over the active columns, solved densely in fp64 (test_oracle_ba's construction)."""
    jc, jp, jk = oracle.ba_jacobians(prob, o)
    _, r, _, _ = oracle.ba_evaluate(prob, o)
    F, P, M = prob.num_images, prob.num_points, prob.num_observations
    NS = 6 * F + 3 * prob.num_cameras
    J = np.zeros((2 * M, NS + 3 * P))
    for i in range(M):
        im, p, c = prob.obs_image[i], prob.obs_point[i], prob.image_camera[prob.obs_image[i]]
        J[2 * i:2 * i + 2, 6 * im:6 * im + 6] = jc[i]
        J[2 * i:2 * i + 2, 6 * F + 3 * c:6 * F + 3 * c + 3] = jk[i]
        J[2 * i:2 * i + 2, NS + 3 * p:NS + 3 * p + 3] = jp[i]
    a = np.concatenate([act, np.ones(3 * P, bool)])
    Js = J[:, a] / (1.0 + np.sqrt((J[:, a] ** 2).sum(0)))
    diag = np.clip((Js ** 2).sum(0), 1e-6, 1e32)
    y = np.linalg.solve(Js.T @ Js + np.diag(diag / radius), Js.T @ r.ravel())
    full = np.zeros(NS + 3 * P)
    full[a] = y
    return full[:NS], full[NS:].reshape(P, 3)


@pytest.mark.parametrize("rot,focal", [(False, False), (True, True), (True, False)])
def test_reference_matches_dense_normal_equations(rot, focal):
    prob, _ = syn.make_ba_problem(5, 40, 4, seed=2)
    o = _opts(rot, focal)
    for radius in (1e4, 3.0):
        R = _reference(prob, o, radius)
        yc, yp = _dense_normal_equations_step(prob, o, radius, R.act)
        assert _rel(R.x.astype(np.float64), yc) < 1e-9
        assert _rel(R.y.astype(np.float64), yp) < 1e-9


def test_measures_see_a_perturbed_block():
    """The backward error of the exact solution of S with one image block perturbed by 1e-9 is ~1e-9 in that
    image's rows, whatever the conditioning (radius 1e12); the reference's own solution scores at rounding level."""
    prob, _ = syn.make_ba_problem(12, 300, 6, seed=62)
    R = _reference(prob, _opts(True, True), 1e12)
    be0, _ = cam_backward_error(R, R.x.astype(np.float64))
    assert be0 < 1e-15
    ia = np.flatnonzero(R.act)
    S2 = R.S.copy()
    S2[6 * 7:6 * 8, 6 * 8:6 * 9] *= LD(1 + 1e-9)
    S2[6 * 8:6 * 9, 6 * 7:6 * 8] *= LD(1 + 1e-9)
    x2 = np.zeros_like(R.x)
    x2[ia] = scipy.linalg.solve(S2[np.ix_(ia, ia)].astype(np.float64), R.b[ia].astype(np.float64))
    x2 = x2.astype(LD)
    for _ in range(3):
        x2[ia] += scipy.linalg.solve(S2[np.ix_(ia, ia)].astype(np.float64), (R.b[ia] - S2[np.ix_(ia, ia)] @ x2[ia]).astype(np.float64))
    be, k = cam_backward_error(R, x2.astype(np.float64))
    assert 1e-11 < be < 1e-8 and k // 6 in (7, 8), (be, _slot_name(R, k))
    bp, _ = point_backward_error(R, R.x.astype(np.float64), R.y.astype(np.float64), prob.xyz)
    assert bp < 1e-15


# ----------------------------------------------------------------------------- fixtures

def _tracks_problem(F, tracks, seed, background=None):
    """Points with the given image lists (observations projected from the ground-truth poses of
    make_ba_problem's helix, + 0.5 px noise, f32-rounded; perturbed start).  `background` =
    (num_points, track_len, first, last) adds video tracks starting in images first..last."""
    base, truth = syn.make_ba_problem(F, 1, 1, seed=seed)
    rng = np.random.default_rng(seed + 1)
    tracks = [np.asarray(t, np.int64) for t in tracks]
    if background is not None:
        n, L, lo, hi = background
        s = rng.integers(lo, hi + 1, n)
        tracks += [np.arange(a, a + L) for a in s]
    P = len(tracks)
    lens = np.array([len(t) for t in tracks])
    img = np.concatenate(tracks)
    pt = np.repeat(np.arange(P), lens)
    X = rng.uniform(-2.5, 2.5, (P, 3))
    Xc = np.einsum("mij,mj->mi", syn.qvec_to_rotmat(truth["qvec"])[img], X[pt]) + truth["tvec"][img]
    f, cx, cy = base.cam_params[0]
    xy = (f * Xc[:, :2] / Xc[:, 2:] + [cx, cy] + rng.normal(0.0, 0.5, (len(img), 2))).astype(np.float32).astype(np.float64)
    perm = rng.permutation(len(img))
    return _abi.BAProblem(base.qvec, base.tvec, X + rng.normal(0.0, 0.05, X.shape), base.cam_params, img[perm], pt[perm],
                          xy[perm], base.image_camera, base.pose_constant, base.tvec_constant_mask, base.camera_constant)


def _mixed_track_problem(frames, long_len, seed, singles=0):
    """(as in test_gpu_ba.py) a few tracks of `long_len` observations, short ones, and `singles`
    points observed once in the last image, which fill whole 512-wide tiles at the end."""
    a, truth = syn.make_ba_problem(frames, 24, long_len, seed=seed)
    b, _ = syn.make_ba_problem(frames, 600, 8, seed=seed + 1)
    rng = np.random.default_rng(seed + 2)
    X = rng.uniform(-2.5, 2.5, (singles, 3))
    Xc = X @ syn.qvec_to_rotmat(truth["qvec"][-1]).T + truth["tvec"][-1]
    f, cx, cy = a.cam_params[0]
    xy = f * Xc[:, :2] / Xc[:, 2:] + [cx, cy] + rng.normal(0.0, 0.5, (singles, 2))
    P = a.num_points + b.num_points
    return _abi.BAProblem(a.qvec, a.tvec, np.concatenate([a.xyz, b.xyz, X + rng.normal(0.0, 0.05, X.shape)]),
                          a.cam_params,
                          np.concatenate([a.obs_image, b.obs_image, np.full(singles, frames - 1)]),
                          np.concatenate([a.obs_point, b.obs_point + a.num_points, P + np.arange(singles)]),
                          np.concatenate([a.obs_xy, b.obs_xy, xy.astype(np.float32).astype(np.float64)]),
                          a.image_camera, a.pose_constant, a.tvec_constant_mask, a.camera_constant)


def _dyn_dup():
    prob, _ = syn.make_ba_problem(30, 1500, 10, seed=64, dynamic_fraction=0.3)
    rng = np.random.default_rng(65)
    n = prob.num_observations // 20
    dup = rng.choice(prob.num_observations, n, replace=False)
    return _abi.BAProblem(prob.qvec, prob.tvec, prob.xyz, prob.cam_params,
                          np.concatenate([prob.obs_image, prob.obs_image[dup]]),
                          np.concatenate([prob.obs_point, prob.obs_point[dup]]),
                          np.concatenate([prob.obs_xy, prob.obs_xy[dup] + rng.normal(0, 0.3, (n, 2))]),
                          prob.image_camera, prob.pose_constant, prob.tvec_constant_mask, prob.camera_constant)


def _gauge():
    """More constant poses, tvec_constant_mask bits, and image 13 without any observation."""
    prob, _ = syn.make_ba_problem(30, 1000, 8, seed=66)
    keep = prob.obs_image != 13
    pc = prob.pose_constant.copy()
    pc[[5, 17]] = 1
    tm = prob.tvec_constant_mask.copy()
    tm[9], tm[22], tm[28] = 0b101, 0b010, 0b111
    return _abi.BAProblem(prob.qvec, prob.tvec, prob.xyz, prob.cam_params, prob.obs_image[keep], prob.obs_point[keep],
                          prob.obs_xy[keep], prob.image_camera, pc, tm, prob.camera_constant)


def _two_cameras():
    """Images 0..11 on camera 0, 12..23 on camera 1 (its own focal length), both constant."""
    prob, truth = syn.make_ba_problem(24, 800, 8, seed=67)
    cams = np.array([prob.cam_params[0], prob.cam_params[0] * [1.05, 1.0, 1.0]])
    ic = (np.arange(24) >= 12).astype(np.int32)
    m = ic[prob.obs_image] == 1
    R = syn.qvec_to_rotmat(truth["qvec"])[prob.obs_image[m]]
    Xc = np.einsum("mij,mj->mi", R, truth["xyz"][prob.obs_point[m]]) + truth["tvec"][prob.obs_image[m]]
    xy = prob.obs_xy.copy()
    xy[m] = (cams[1, 0] * Xc[:, :2] / Xc[:, 2:] + cams[1, 1:]
             + np.random.default_rng(68).normal(0, 0.5, (m.sum(), 2))).astype(np.float32)
    return _abi.BAProblem(prob.qvec, prob.tvec, prob.xyz, cams, prob.obs_image, prob.obs_point, xy, ic,
                          prob.pose_constant, prob.tvec_constant_mask, np.ones(2, np.uint8))


def _fit_limit_256():
    """Tile 0: 22 points over images 1..14 (ns 14, np 22: Z of 6 x 9 = 54 fragment blocks, exactly what the
    27 x 257 reduction rows hold); tile 1: 27 points over images 15..25 (ns 11, np 27: 5 x 11 = 55, one past).
    The next point's length closes each tile (248 + 9 > 256, 243 + 14 > 256)."""
    rng = np.random.default_rng(70)
    t0 = [np.sort(np.concatenate([[1], 2 + rng.choice(13, 11 if k < 6 else 10, replace=False)])) for k in range(22)]
    t0[0] = np.arange(1, 13)                                   # every image of 1..14 is seen
    t0[1] = np.concatenate([[1], np.arange(4, 15)])
    t1 = [np.sort(np.concatenate([[15], 16 + rng.choice(10, 8, replace=False)])) for _ in range(27)]
    t1[0] = np.arange(15, 24)
    t1[1] = np.concatenate([[15], np.arange(18, 26)])
    return _tracks_problem(40, t0 + t1, seed=71, background=(260, 14, 26, 26))


def _fit_limit_512():
    """512-wide tiles (tracks of 297 observations): tile 0 = 288 single observations in image 2 (ns 1, np 288:
    1 x 108 fragment blocks, exactly the 27 x 513 reduction rows), tile 1 = two long tracks filling 512
    observations exactly, tile 2 = 289 single observations in image 5 (1 x 109, one past)."""
    tracks = [[2]] * 288 + [np.arange(3, 300), np.arange(3, 218)] + [[5]] * 289 + [np.arange(6, 300)]
    return _tracks_problem(300, tracks, seed=72, background=(400, 8, 7, 292))


FIXTURES = {
    # name: (builder, expected explicit_fused, expected longest track span or None)
    "band40": (lambda: syn.make_ba_problem(40, 1200, 9, seed=41)[0], 1, 8),        # block-6 band, two CTAs
    "band20": (lambda: syn.make_ba_problem(20, 600, 9, seed=42)[0], 1, 8),         # block-6 band, one CTA
    "span24": (lambda: syn.make_ba_problem(60, 500, 25, seed=43)[0], 1, 24),       # Wb = 25: the 640-thread kernel
    "span25": (lambda: syn.make_ba_problem(40, 400, 26, seed=44)[0], 1, 25),       # dense S + k_chol_blocked
    "dense26": (lambda: syn.make_ba_problem(26, 300, 26, seed=45)[0], 1, 25),      # NS + 1 = 160: whole panels
    "dense27": (lambda: syn.make_ba_problem(27, 300, 27, seed=46)[0], 1, 26),      # NS + 1 = 166
    "f2": (lambda: syn.make_ba_problem(2, 60, 2, seed=47)[0], 1, 1),               # < 3 images: dense S + k_chol_blocked
    "f3": (lambda: syn.make_ba_problem(3, 80, 3, seed=48)[0], 1, 2),
    "span1": (lambda: syn.make_ba_problem(20, 500, 2, seed=49)[0], 1, 1),          # Wb clamped to 3
    "dyn_dup": (_dyn_dup, 1, None),                                                # holes, TILE_PAIRS_DENSE_DUP
    "gauge": (_gauge, 1, 7),                                                       # identity rows in the band
    "two_cams": (_two_cameras, 1, 7),                                              # NS = 6F + 6
    "long300": (lambda: _mixed_track_problem(320, 300, seed=30), 1, None),         # loop tiles, 512 wide
    "singles": (lambda: _mixed_track_problem(320, 300, seed=30, singles=1100), 0, None),  # smem-forced unfused
    "fit256": (_fit_limit_256, 1, 13),
    "fit512": (_fit_limit_512, 1, None),
}

_PROBS, _REFS = {}, {}


def _problem(name):
    if name not in _PROBS:
        _PROBS[name] = FIXTURES[name][0]()
    return _PROBS[name]


def _ref(name, rot, focal, loss, radius):
    key = (name, rot, focal, loss, radius)
    if key not in _REFS:
        _REFS[key] = _reference(_problem(name), _opts(rot, focal, loss), radius)
    return _REFS[key]


def _tile_plan(prob):
    """Mirror of the solver's host tile packing: points by (first image, id), whole points while the tile
    holds <= TILE observations.  Returns the tile width, [(ns, np)] per tile, the pair-task count and the
    longest image span of a track."""
    pt, img = prob.obs_point.astype(np.int64), prob.obs_image.astype(np.int64)
    P = prob.num_points
    cnt = np.bincount(pt, minlength=P)
    first = np.full(P, np.iinfo(np.int64).max)
    np.minimum.at(first, pt, img)
    last = np.full(P, -1)
    np.maximum.at(last, pt, img)
    obs = np.flatnonzero(cnt)
    ids = obs[np.lexsort((obs, first[obs]))]
    tile = 256 if cnt.max() <= 256 else 512
    imgs_of = [set() for _ in range(P)]
    for p, i in zip(pt, img):
        imgs_of[p].add(int(i))
    tiles, cur = [], []
    ncur = 0
    for p in ids:
        if ncur + cnt[p] > tile:
            tiles.append(cur)
            cur, ncur = [], 0
        cur.append(p)
        ncur += cnt[p]
    tiles.append(cur)
    shapes, ntasks = [], 0
    for t in tiles:
        ims = set().union(*(imgs_of[p] for p in t))
        shapes.append((len(ims), len(t)))
        pairs = set()
        for p in t:
            s = sorted(imgs_of[p])
            pairs.update((a, b) for k, a in enumerate(s) for b in s[k:])
        ntasks += len(pairs)
    return tile, shapes, ntasks, int((last[obs] - first[obs]).max())


def _dense_fits(tile, ns, np_):
    """k_tile_pairs_mode's fit test: Z in mma fragment blocks of 16 rows x 8 columns vs the reduction rows."""
    return ((6 * ns + 15) >> 4) * ((3 * np_ + 7) >> 3) * 128 <= TILE_ZCAP_ROWS * (tile + 1)


def test_fixture_shapes():
    """The fixtures reach the shapes they are named for (host-side mirror of the tile packing)."""
    for name, (_, _, span) in FIXTURES.items():
        _, _, _, sp = _tile_plan(_problem(name))
        if span is not None:
            assert sp == span, name
    tile, shapes, _, _ = _tile_plan(_problem("fit256"))
    assert tile == 256 and shapes[0] == (14, 22) and shapes[1] == (11, 27)
    assert _dense_fits(256, 14, 22) and not _dense_fits(256, 11, 27)
    tile, shapes, _, _ = _tile_plan(_problem("fit512"))
    assert tile == 512 and shapes[0] == (1, 288) and shapes[2] == (1, 289)
    assert _dense_fits(512, 1, 288) and not _dense_fits(512, 1, 289)
    assert _problem("gauge").num_images == 30 and not np.any(_problem("gauge").obs_image == 13)


# ----------------------------------------------------------------------------- GPU

def _expected_path(name, arm):
    prob = _problem(name)
    tile, shapes, ntasks, _ = _tile_plan(prob)
    fused = 0 if arm == "unfused" else FIXTURES[name][1]
    dense = sum(_dense_fits(tile, ns, np_) for ns, np_ in shapes) if fused and arm != "loop" else 0
    return fused, dense, ntasks


ARM_ENV = {"default": {}, "loop": {"PSFM_SCHUR_PAIRS": "loop"}, "unfused": {"PSFM_SCHUR_UNFUSED": "1"},
           "no_pipe_schur": {"PSFM_NO_PIPE_SCHUR": "1"}, "no_pipe": {"PSFM_NO_PIPE": "1"},
           "one_sided": {"PSFM_CHOL_ONE_SIDED": "1"}}


def _gpu_step(name, rot, focal, loss, radius):
    """The GPU's exact step and the path its full solve takes, in the current process' environment."""
    from particlesfm_b200 import ba
    prob = _problem(name)
    o = _opts(rot, focal, loss)
    o1 = o.copy()
    o1.max_num_iterations = 1
    s = ba.solve_problem(prob.copy(), o1)
    sc, sp, it = ba.ResidentSolver(prob.copy()).linear_step(o, radius)
    return sc, sp, (s.linear_solver_used, s.explicit_fused, s.explicit_dense_tiles, s.num_pair_tasks, it)


# (camera rows, point rows) thresholds.  Largest backward errors measured on one H100 80GB HBM3 (CUDA 12.9),
# over every arm and option set of the fixture, camera | point rows:
#   band40 1.3e-14 | 2.0e-14   band20 3.2e-15 | 1.1e-14   span24 3.9e-15 | 6.6e-15   span25 1.2e-14 | 1.5e-14
#   dense26 1.4e-14 | 8.7e-15  dense27 2.2e-15 | 4.2e-15  f2 9.0e-17 | 1.1e-14      f3 9.4e-17 | 5.5e-15
#   span1 4.4e-16 | 1.3e-14    dyn_dup 1.8e-15 | 8.2e-15  gauge 1.5e-15 | 4.4e-15   two_cams 1.4e-15 | 1.7e-14
#   long300 1.0e-15 | 1.2e-14  singles 1.0e-15 | 1.3e-12  fit256 2.2e-15 | 5.8e-15   fit512 4.3e-15 | 1.6e-12
# The point rows of `singles` and `fit512` sit higher: their single-observation points have an H_p that only the
# LM diagonal (1e-4 of its scale at radius 1e4) keeps invertible, and the solver stores H_p^-1 explicitly, so
# y_p carries kappa(H_p) u.  Their threshold is the 1e-10 ceiling, 60x above the measurement.
THRESHOLDS = {name: (2e-12, 3e-12) for name in FIXTURES}
THRESHOLDS["singles"] = THRESHOLDS["fit512"] = (2e-12, 1e-10)
FWD_C = 64.0


def _check(name, arm, case, sc, sp, path):
    rot, focal, loss, radius = case
    prob = _problem(name)
    R = _ref(name, rot, focal, loss, radius)
    fused, dense, ntasks = _expected_path(name, arm)
    tag = f"{name}/{arm} rot={rot} focal={focal} loss={loss} radius={radius:g}"
    assert path[0] == _abi.SOLVER_EXACT_SCHUR and path[4] > 0, tag
    assert (path[1], path[2], path[3]) == (fused, dense, ntasks), (tag, path)
    assert np.array_equal(sc[~R.act], np.zeros((~R.act).sum())), tag
    assert np.array_equal(sp[~R.observed], np.zeros(((~R.observed).sum(), 3))), tag
    x, y = -sc, -sp
    tc, tp = THRESHOLDS[name]
    bc, k = cam_backward_error(R, x)
    assert bc <= tc, f"{tag}: camera backward error {bc:.3e} at {_slot_name(R, k)}"
    bp, p = point_backward_error(R, x, y, prob.xyz)
    assert bp <= tp, f"{tag}: point backward error {bp:.3e} at point {p}"
    fe, kappa = forward_error(R, x)
    assert fe <= 1e-12 + FWD_C * kappa * U64, f"{tag}: forward error {fe:.3e}, kappa {kappa:.3e}"
    return bc, bp, fe, kappa


A4, B4 = (False, False, _abi.LOSS_SOFT_L1, 1e4), (True, True, _abi.LOSS_SOFT_L1, 1e4)
EXTREMES = [(True, True, _abi.LOSS_SOFT_L1, 1e-2), (True, True, _abi.LOSS_SOFT_L1, 1e12),
            (True, False, _abi.LOSS_TRIVIAL, 1e4), (True, True, _abi.LOSS_CAUCHY, 1e12),
            (False, False, _abi.LOSS_CAUCHY, 1e-2)]
ROUTE_FIXTURES = ("band40", "span25", "dense26")


def _cases(name):
    return [A4, B4] + (EXTREMES if name in ROUTE_FIXTURES else [])


# (fixture, arm): every fixture runs the default arm; every arm the banded fixture and the route it changes
MATRIX = ([(n, "default") for n in FIXTURES] +
          [("band40", "loop"), ("fit256", "loop"), ("fit512", "loop"), ("dyn_dup", "loop"),
           ("band40", "unfused"), ("dense27", "unfused"), ("dyn_dup", "unfused"), ("two_cams", "unfused"),
           ("band40", "no_pipe_schur"), ("fit256", "no_pipe_schur"),
           ("band40", "no_pipe"), ("long300", "no_pipe"), ("span1", "no_pipe")])
CHILD_MATRIX = [("band40", "one_sided"), ("span24", "one_sided")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,arm", MATRIX, ids=[f"{n}-{a}" for n, a in MATRIX])
def test_exact_step(gpu, monkeypatch, name, arm):
    for k, v in ARM_ENV[arm].items():
        monkeypatch.setenv(k, v)
    for case in _cases(name):
        sc, sp, path = _gpu_step(name, *case)
        _check(name, arm, case, sc, sp, path)


@pytest.mark.gpu
@pytest.mark.parametrize("name,arm", CHILD_MATRIX, ids=[f"{n}-{a}" for n, a in CHILD_MATRIX])
def test_exact_step_cholesky_forms(gpu, tmp_path, name, arm):
    """PSFM_CHOL_ONE_SIDED is read once per process: the GPU step runs in a child."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cases = _cases(name)
    code = ("import sys, numpy as np; sys.path[:0] = [%r, %r]; import test_gpu_exact_step as t;"
            "out = [t._gpu_step(%r, *c) for c in %r];"
            "np.savez(sys.argv[1], *[a for sc, sp, pa in out for a in (sc, sp, np.array(pa))])"
            % (root, os.path.join(root, "tests"), name, cases))
    path = str(tmp_path / "step.npz")
    subprocess.run([sys.executable, "-c", code, path], check=True, cwd=root, env={**os.environ, **ARM_ENV[arm]})
    z = np.load(path)
    for i, case in enumerate(cases):
        _check(name, arm, case, z[f"arr_{3 * i}"], z[f"arr_{3 * i + 1}"], tuple(z[f"arr_{3 * i + 2}"]))
