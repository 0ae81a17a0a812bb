"""The verification's minimal estimators (csrc/verification.cu: seven_point, homography_minimal) and the seven-point
step's cubic (cubic_real_roots), through their test entries psfm_verification_minimal and psfm_verification_cubic,
against references in 50-digit mpmath.  u = 2^-53, C = 32, as in test_gpu_null_vectors, whose double-double and
mpmath helpers and scene geometry this file uses.

The cubic p(x) = c3 x^3 + c2 x^2 + c1 x + c0.  The reference roots come from the closed form at 150 digits.
  * the root count equals the reference's wherever the reference's discriminant is decided: |D| above 1e-12 of the
    sum of the magnitudes of its five terms (the oracle's `cubic` band);
  * every returned root x is backward stable, |p(x)| <= C u sum |c_k| |x|^k;
  * every simple root r is met to its forward bound, |x - r| <= C u sum |c_k| |r|^k / |p'(r)|.

The seven-point step.  A is the 7 x 9 system of the float32 points, exact in double.  The reference takes the 2-D null
space (a, b) from the 50-digit SVD, the real roots of det(lam a + b) (of det(a + mu b) when |det a| < |det b|) and the
models F = lam a + b (a + mu b), and drops a model with |F22| / |F| < 1e-10 as the device does.  Models are compared as
unit-norm matrices up to sign, each reference model against the nearest device model; lambda and the order depend on
the basis and are not compared.  Checks:
  * the model count, where every root's reality and every F22 drop is decided: the chordal distance of any two roots
    of the pencil (rotation of the basis does not change it) above 1e-6, and |F22| / |F| clear of 1e-10;
  * two backward errors that hold whatever the conditioning: |A f| <= C u |A| |f| and |det F| <= C u |F|^3;
  * the forward error <= C u kappa.  kappa is the first-order condition number of the map from (A, det) to the unit
    model f, from implicit differentiation of [A f; det F; (f'f - 1) / 2] = 0: with J = [A; cof(F)'; f'],
    kappa = |J^-1[:, :7]| |A| + |J^-1[:, 7]| (Frobenius norms), for a backward error u |A| in A and u |F|^3 in det F.
A rank-deficient A (duplicated correspondences) has a null space of 3 dimensions: it gets only the backward checks.  A
planar sample, whose null space would have 3 dimensions too, is left just full rank by the float32 rounding of its
points; it gets every check, with its large kappa.

The four-point H: the local-model bound of test_gpu_null_vectors, |H / |H| -+ H* / |H*|| <= 2 kappa_T (e + C u),
with e from the reference's own normalised 8 x 9 system (test_gpu_null_vectors._LocalRef on the four points)."""
import ctypes as C
import functools

import mpmath as mp
import numpy as np
import pytest

from oracle import verification_oracle as vo
from particlesfm_b200 import _lib
from test_gpu_null_vectors import (CU, FLOOR, HEIGHT, NOISES, STEPS, U, WIDTH, _LocalRef, _camera, _dd_add, _dd_mul,
                                   _mp_svd, _project, _scene, _two_prod)

BIG = 100_000                                      # the large batch of each estimator
BATCHES = [1, 127, 128, 129]                       # around k_minimal's and k_cubic's 128-thread block
CUBIC_BAND = 1e-12                                 # test_gpu_verification.BANDS["cubic"]
CHORDAL_BAND = 1e-6
MIN_F22 = vo.RECALLED["min_f22"]


# ---- the cubic -----------------------------------------------------------------------------------------------------

def _cubic_fixtures():
    """(name, [c3, c2, c1, c0]) rows."""
    rng = np.random.default_rng(11)
    out = [("normal", c) for c in rng.standard_normal((1500, 4))]
    for k in range(3, 19):                        # Cardano's cancellation: p^3 / q^2 = +-10^-k
        for sg in (1.0, -1.0):
            for q in (1.0, -2.7, 0.37):
                p = sg * (10.0 ** -k * q * q) ** (1.0 / 3.0)
                out.append(("p3_q2_1e-%d" % k, [1.0, 0.0, p, q]))
                out.append(("p3_q2_1e-%d_shifted" % k, [2.0, -1.2, 2.0 * (p + 0.12), 2.0 * (q + 0.2 * p + 0.016)]))
    for k in range(3, 13):                        # a small leading coefficient: |c3| / max |c_k| = 10^-k
        for _ in range(30):
            c = rng.standard_normal(3)
            c /= np.abs(c).max()
            out.append(("c3_1e-%d" % k, [rng.choice([-1.0, 1.0]) * 10.0 ** -k * rng.uniform(1, 2), *c]))
    out += [("c3_0", [0.0, *rng.standard_normal(3)]) for _ in range(100)]
    out += [("c3_c2_0", [0.0, 0.0, *rng.standard_normal(2)]) for _ in range(30)]
    out += [("c3_c2_0", [0.0, 0.0, 0.0, 1.0]), ("c3_c2_0", [0.0, 0.0, 2.5, 0.0]), ("zero", [0.0, 0.0, 0.0, 0.0])]
    for k in range(2, 17):                        # the quadratic's cancellation: c1^2 / |4 c2 c0| = 10^k
        for s in (1.0, -1.0):
            c2, c0 = rng.uniform(0.5, 2.0), s * rng.uniform(0.5, 2.0)
            c1 = rng.choice([-1.0, 1.0]) * np.sqrt(10.0 ** k * abs(4 * c2 * c0))
            out.append(("quadratic_1e%d" % k, [0.0, c2, c1, c0]))
            out.append(("small_root_1e%d" % k, [rng.uniform(0.5, 2.0), c2, c1, c0]))
    for k in range(2, 13):                        # near-double and near-triple roots, planted
        for r in (1.0, -3.5, 0.02):
            d = 10.0 ** -k
            out.append(("double_1e-%d" % k, np.poly([r, r * (1 + d), -0.7]).tolist()))
            out.append(("triple_1e-%d" % k, np.poly([r, r * (1 + d), r * (1 - d)]).tolist()))
    out += [("triple", [1.0, -3.0, 3.0, -1.0]), ("triple", [2.0, 0.0, 0.0, 0.0]), ("double", [1.0, 0.0, -3.0, 2.0])]
    for roots in ([1e-10, -1.0, -1e9], [3e-7, 2.0, 5e8], [-1e-6, 1e-3, 1e6]):  # roots at both ends of the scale
        out.append(("spread", np.poly(roots).tolist()))
    normal = [c for n, c in out[:200]]
    for e in (60, -60):                           # the whole cubic scaled, and its roots scaled by 2^(e/3)
        out += [("scaled_2^%d" % e, np.ldexp(np.asarray(c, float), e)) for c in normal]
        out += [("roots_scaled_2^%d" % e, np.ldexp(np.asarray(c, float), [0, e // 3, 2 * e // 3, e])) for c in normal]
    return [(n, np.asarray(c, np.float64)) for n, c in out]


def _mp_cubic(c):
    """(real roots as mpf, decided): the roots of c3 x^3 + .. + c0 from the closed form at 150 digits; decided: the
    count is clear of the discriminant band."""
    a, b, cc, d = [mp.mpf(float(x)) for x in c]
    with mp.workdps(150):
        if a == 0:
            if b == 0:
                return ([] if cc == 0 else [-d / cc]), True
            D = cc * cc - 4 * b * d
            scale = cc * cc + abs(4 * b * d)
            decided = abs(D) > CUBIC_BAND * scale
            if D < 0:
                return [], decided
            s = mp.sqrt(D)
            return sorted([(-cc + s) / (2 * b), (-cc - s) / (2 * b)]), decided
        terms = [18 * a * b * cc * d, -4 * b ** 3 * d, b * b * cc * cc, -4 * a * cc ** 3, -27 * a * a * d * d]
        decided = abs(sum(terms)) > CUBIC_BAND * sum(abs(t) for t in terms)
        bb, c1, c0 = b / a, cc / a, d / a
        p = c1 - bb * bb / 3
        q = 2 * bb ** 3 / 27 - bb * c1 / 3 + c0
        s = mp.sqrt(mp.mpc(q * q / 4 + p ** 3 / 27))
        w = -q / 2 + s if abs(-q / 2 + s) >= abs(-q / 2 - s) else -q / 2 - s
        if w == 0:
            roots = [-bb / 3] * 3
        else:
            Cr = mp.root(w, 3)
            om = mp.exp(2j * mp.pi / 3)
            roots = [om ** k * Cr - p / (3 * om ** k * Cr) - bb / 3 for k in range(3)]
        real = [mp.re(r) for r in roots if abs(mp.im(r)) <= mp.mpf(10) ** -45 * (1 + abs(r))]
    return sorted(real), decided


def _cubic_checks(c, x, n):
    """The three checks of one cubic: a list of failures (empty when it passes)."""
    cs = [mp.mpf(float(v)) for v in c]                 # c3, c2, c1, c0
    ref, decided = _mp_cubic(c)
    bad = []
    if decided and n != len(ref):
        bad.append(("count", n, len(ref)))
    xs = sorted(float(v) for v in x[:n])
    for v in xs:
        xm = mp.mpf(v)
        val = ((cs[0] * xm + cs[1]) * xm + cs[2]) * xm + cs[3]
        scale = sum(abs(cs[3 - k]) * abs(xm) ** k for k in range(4))
        if abs(val) > CU * scale:
            bad.append(("backward", v, float(abs(val) / scale / U)))
    if n == len(ref):
        for v, r in zip(xs, ref):
            dp = abs((3 * cs[0] * r + 2 * cs[1]) * r + cs[2])
            if dp == 0:
                continue
            bound = CU * sum(abs(cs[3 - k]) * abs(r) ** k for k in range(4)) / dp
            if abs(mp.mpf(v) - r) > bound:
                bad.append(("forward", v, float(r), float(abs(mp.mpf(v) - r) / bound)))
    return bad


@functools.lru_cache(maxsize=None)
def _cubic_table():
    fx = _cubic_fixtures()
    return [n for n, _ in fx], np.ascontiguousarray(np.stack([c for _, c in fx]))


def _run_cubic(coeffs):
    coeffs = np.ascontiguousarray(coeffs, np.float64)
    x, n = np.full((len(coeffs), 3), np.nan), np.full(len(coeffs), -1, np.int32)
    _lib.check(_lib.lib().psfm_verification_cubic(_lib.dptr(coeffs), len(coeffs), _lib.dptr(x),
                                                  n.ctypes.data_as(C.POINTER(C.c_int32))), "psfm_verification_cubic")
    return x, n


# ---- the seven-point and four-point samples ------------------------------------------------------------------------

def _views(px, depth, step, rotate=True):
    """Correspondences (x1, y1, x2, y2) in float32 of the pixels px [n][2] of camera 1 at the given depths, the second
    camera moved `step` as in test_gpu_null_vectors (rotate=False: the same translation, no rotation)."""
    K, R, t = _camera(step)
    if not rotate:
        R = np.eye(3)
    X = np.c_[px, np.ones(len(px))] @ np.linalg.inv(K).T * np.asarray(depth, float)[:, None]
    return np.c_[_project(K, X), _project(K, X @ R.T - t)].astype(np.float32)


def _design7(P):
    """The seven-point system of float32 points [..][4]: exact in double (products of two floats)."""
    Q = P.astype(np.float64)
    x1, y1, x2, y2 = Q[..., 0], Q[..., 1], Q[..., 2], Q[..., 3]
    return np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, np.ones(x1.shape)], axis=-1)


@functools.lru_cache(maxsize=None)
def _samples(k, n, seed):
    """n samples of k distinct correspondences drawn from the eight scenes (STEPS x NOISES), in turn; [n][k][4]."""
    rng = np.random.default_rng(seed)
    scenes = [_scene(s, z)[0] for s in STEPS for z in NOISES]
    idx = rng.integers(0, len(scenes[0]), (n, k))
    while True:
        s = np.sort(idx, axis=1)
        dup = (s[:, 1:] == s[:, :-1]).any(axis=1)
        if not dup.any():
            break
        idx[dup] = rng.integers(0, len(scenes[0]), (dup.sum(), k))
    which = np.arange(n) % len(scenes)
    out = np.empty((n, k, 4), np.float32)
    for j, P in enumerate(scenes):
        out[which == j] = P[idx[which == j]]
    return out


def _qr_basis(P):
    """seven_point's own null basis (a, b) restated in numpy: null_space_qr, the Householder QR of A' and the last two
    columns of Q.  Used to find fixtures where the device's c3 is small."""
    B = _design7(P).T.copy()
    beta = np.zeros(7)
    for j in range(7):
        nrm = np.sqrt((B[j:, j] ** 2).sum())
        if nrm == 0.0:
            continue
        B[j, j] -= -nrm if B[j, j] >= 0.0 else nrm
        beta[j] = 2.0 / (B[j:, j] ** 2).sum()
        for c in range(j + 1, 7):
            B[j:, c] -= beta[j] * (B[j:, j] @ B[j:, c]) * B[j:, j]
    ns = []
    for k in (7, 8):
        x = np.eye(9)[k]
        for j in range(6, -1, -1):
            x[j:] -= beta[j] * (B[j:, j] @ x[j:]) * B[j:, j]
        ns.append(x)
    return ns


def _qr_pencil(P):
    """The pencil det(lam a + b) = c3 lam^3 + c2 lam^2 + c1 lam + c0 of seven_point's basis: (c3, c2, c1, c0)."""
    a, b = _qr_basis(P)
    d0, d1, dm, c3 = vo._det3(b), vo._det3(a + b), vo._det3(-a + b), vo._det3(a)
    return np.array([c3, 0.5 * (d1 + dm) - d0, 0.5 * (d1 - dm) - c3, d0])


def _qr_seven_point(P, cubic, flip):
    """seven_point restated on its own basis with a given cubic solver, with or without the flip to det(a + mu b)."""
    a, b = _qr_basis(P)
    c3, c2, c1, d0 = _qr_pencil(P)
    f = flip and abs(c3) < abs(d0)
    out = []
    for lam in (cubic(d0, c1, c2, c3) if f else cubic(c3, c2, c1, d0)):
        F = a + lam * b if f else lam * a + b
        if abs(F[8] / np.linalg.norm(F)) >= MIN_F22:
            out.append(F / F[8])
    return np.array(out).reshape(-1, 9)


def _small_c3(P, coord):
    """P with its point-6 coordinate `coord` moved to the float32 value where seven_point's c3 changes sign (the
    leading coefficient of its pencil vanishes), found by bisection."""
    def rel(v):
        Q = P.copy()
        Q[6, coord] = v
        c = _qr_pencil(Q)
        return c[0] / np.abs(c).max()
    span = WIDTH if coord % 2 == 0 else HEIGHT
    grid = np.linspace(0.0, span, 65, dtype=np.float32)
    r = [rel(v) for v in grid]
    i = next((i for i in range(64) if np.sign(r[i]) != np.sign(r[i + 1])), None)
    if i is None:
        return None
    lo, hi = grid[i], grid[i + 1]
    while np.nextafter(lo, hi) != hi:
        mid = np.float32(0.5 * (float(lo) + float(hi)))
        if mid in (lo, hi):
            break
        lo, hi = (mid, hi) if np.sign(rel(mid)) == np.sign(rel(lo)) else (lo, mid)
    Q = P.copy()
    Q[6, coord] = lo if abs(rel(lo)) < abs(rel(hi)) else hi
    return Q


def _special_seven():
    """(name, [7][4]) edge samples."""
    rng = np.random.default_rng(5)
    out = []
    for j, P in enumerate(_samples(7, 80, seed=27)):          # seven_point's c3 near zero
        Q = _small_c3(P, j % 4)
        if Q is not None and abs(_qr_pencil(Q)[0]) < 1e-6 * np.abs(_qr_pencil(Q)).max() and len(out) < 8:
            out.append(("small_c3", Q))
    corners = np.array([[0.0, 0.0], [WIDTH, 0.0], [0.0, HEIGHT], [WIDTH, HEIGHT]])
    for step in STEPS:
        px = np.r_[corners, rng.uniform([0, 0], [WIDTH, HEIGHT], (3, 2))]
        out.append(("corners", _views(px, rng.uniform(2, 40, 7), step)))
        px = rng.uniform([0, 0], [WIDTH, HEIGHT], (7, 2))
        out.append(("translation", _views(px, rng.uniform(2, 40, 7), step, rotate=False)))
        P = _scene(step, 0.0, plane=True)[0]
        out.append(("planar", P[rng.choice(len(P), 7, replace=False)]))
        P = _scene(step, 0.5)[0][rng.choice(200_000, 7, replace=False)]
        P[6] = P[0]
        out.append(("duplicate", P.copy()))
        P[5] = P[1]
        out.append(("duplicate2", P.copy()))
    return out


def _special_four():
    """(name, [4][4]) edge samples of the homography."""
    rng = np.random.default_rng(6)
    out = []
    Hm = _scene(0.02, 0.0, plane=True)[1].reshape(3, 3)

    def through(x1, H):
        y = np.c_[x1, np.ones(len(x1))] @ H.T
        return np.c_[x1, y[:, :2] / y[:, 2:]].astype(np.float32)
    corners = np.array([[0.0, 0.0], [WIDTH, 0.0], [0.0, HEIGHT], [WIDTH, HEIGHT]])
    out.append(("corners", through(corners, Hm)))
    for e in (1e-1, 1e-2, 1e-3, 1e-4):              # three of the points nearly on a line, e px off it
        a, b = rng.uniform([0, 0], [WIDTH, HEIGHT], (2, 2))
        d = (b - a) / np.linalg.norm(b - a)
        c = a + 0.37 * (b - a) + e * np.array([-d[1], d[0]])
        out.append(("collinear_%g" % e, through(np.array([a, b, c, rng.uniform([0, 0], [WIDTH, HEIGHT])]), Hm)))
    for _ in range(4):
        x1 = rng.uniform([0, 0], [WIDTH, HEIGHT], (4, 2))
        out.append(("identity", np.c_[x1, x1 + rng.normal(0, 0.01, x1.shape)].astype(np.float32)))
        c = rng.uniform([10, 10], [WIDTH - 10, HEIGHT - 10])
        out.append(("cluster", through(c + rng.uniform(-2, 2, (4, 2)), Hm)))
    return out


def _run_minimal(kind, samples):
    S = np.ascontiguousarray(samples, np.float32)
    nm = 3 if kind == 0 else 1
    models, n = np.full((len(S), nm, 9), np.nan), np.full(len(S), -1, np.int32)
    _lib.check(_lib.lib().psfm_verification_minimal(kind, S.ctypes.data_as(C.POINTER(C.c_float)), len(S),
                                                    _lib.dptr(models), n.ctypes.data_as(C.POINTER(C.c_int32))),
               "psfm_verification_minimal")
    return models, n


# ---- the seven-point reference -------------------------------------------------------------------------------------

def _mp_det3(F):
    return (F[0] * (F[4] * F[8] - F[5] * F[7]) - F[1] * (F[3] * F[8] - F[5] * F[6])
            + F[2] * (F[3] * F[7] - F[4] * F[6]))


def _cofactor(F):
    M = [[F[3 * r + c] for c in range(3)] for r in range(3)]
    out = []
    for r in range(3):
        for c in range(3):
            rows = [i for i in range(3) if i != r]
            cols = [j for j in range(3) if j != c]
            m = M[rows[0]][cols[0]] * M[rows[1]][cols[1]] - M[rows[0]][cols[1]] * M[rows[1]][cols[0]]
            out.append(m if (r + c) % 2 == 0 else -m)
    return out


def _unit(f):
    """Unit Frobenius norm, the largest-magnitude entry positive (float64 or mpf list in, float64 out)."""
    f = np.array([float(v) for v in f]) if not isinstance(f, np.ndarray) else f.astype(np.float64)
    f = f / np.linalg.norm(f)
    return -f if f[int(np.argmax(np.abs(f)))] < 0 else f


class _SevenRef:
    """The reference seven-point step on one sample P [7][4] float32."""

    def __init__(self, P):
        self.A = _design7(P)
        s, V = _mp_svd(np.r_[self.A, np.zeros((2, 9))])
        self.nA = s[0]
        self.rank_deficient = s[6] <= mp.mpf("1e-30") * s[0]
        self.models, self.kappa, self.f22 = [], [], []
        if self.rank_deficient:
            return
        a, b =[V[k, 7] for k in range(9)], [V[k, 8] for k in range(9)]
        d = lambda lam, mu: _mp_det3([lam * x + mu * y for x, y in zip(a, b)])
        c3, c0 = d(1, 0), d(0, 1)
        c2 = (d(1, 1) + d(-1, 1)) / 2 - c0
        c1 = (d(1, 1) - d(-1, 1)) / 2 - c3
        self.flip = abs(c3) < abs(c0)
        coeffs = [c0, c1, c2, c3] if self.flip else [c3, c2, c1, c0]
        roots = mp.polyroots(coeffs, maxsteps=400, extraprec=400)
        self.chordal = min([abs(x - y) / mp.sqrt((1 + abs(x) ** 2) * (1 + abs(y) ** 2))
                            for i, x in enumerate(roots) for y in roots[i + 1:]])
        for r in roots:
            if abs(mp.im(r)) > mp.mpf(10) ** -40 * (1 + abs(r)):
                continue
            lam = mp.re(r)
            F = [x + lam * y for x, y in zip(a, b)] if self.flip else [lam * x + y for x, y in zip(a, b)]
            nrm = mp.sqrt(sum(v * v for v in F))
            F = [v / nrm for v in F]
            self.f22.append(abs(F[8]))
            if abs(F[8]) < MIN_F22:
                continue
            self.models.append(F)
            J = mp.matrix(9, 9)
            cof = _cofactor(F)
            for j in range(9):
                for i in range(7):
                    J[i, j] = mp.mpf(float(self.A[i, j]))
                J[7, j], J[8, j] = cof[j], F[j]
            Ji = mp.inverse(J)
            k_a = mp.sqrt(sum(Ji[i, j] ** 2 for i in range(9) for j in range(7)))
            k_d = mp.sqrt(sum(Ji[i, 7] ** 2 for i in range(9)))
            self.kappa.append(float(k_a * self.nA + k_d))

    def count_decided(self):
        clear = all(abs(f - MIN_F22) > 0.5 * MIN_F22 + CU * max(self.kappa, default=1.0) for f in self.f22)
        return clear and self.chordal > CHORDAL_BAND

    def forward_errors(self, models):
        """(error, bound) of each reference model against the nearest of `models` (rows, any scale)."""
        out = []
        dev = [_unit(m) for m in models]
        for F, k in zip(self.models, self.kappa):
            f = _unit(F)
            e = min(min(np.linalg.norm(f - g), np.linalg.norm(f + g)) for g in dev) if dev else np.inf
            out.append((e, max(CU * k, FLOOR)))
        return out


def _backward_errors(A, F):
    """|A f| / (|A| |f|) and |det F| / |F|^3 of models F [m][9] for systems A [m][7][9], both exact to about 1e-32
    (double-double): the quantities the C u bounds apply to."""
    Af = _dd_mul((A, np.zeros_like(A)), (F[:, None, :], np.zeros(F[:, None, :].shape)))
    h, lo = Af[0][..., 0], Af[1][..., 0]
    for j in range(1, 9):
        h, lo = _dd_add((h, lo), (Af[0][..., j], Af[1][..., j]))
    nA = np.linalg.norm(A, ord=2, axis=(1, 2))
    nf = np.linalg.norm(F, axis=1)
    ra = np.linalg.norm(h + lo, axis=1) / (nA * nf)

    def m3(i, j, k):
        return _dd_mul(_two_prod(F[:, i], F[:, j]), (F[:, k], np.zeros(len(F))))
    terms = [(m3(0, 4, 8), 1), (m3(0, 5, 7), -1), (m3(1, 3, 8), -1), (m3(1, 5, 6), 1), (m3(2, 3, 7), 1), (m3(2, 4, 6), -1)]
    s = (np.zeros(len(F)), np.zeros(len(F)))
    for (th, tl), sg in terms:
        s = _dd_add(s, (sg * th, sg * tl))
    rd = np.abs(s[0] + s[1]) / nf ** 3
    return ra, rd


# ---- CPU: the reference and the oracle -----------------------------------------------------------------------------

def test_reference_recovers_planted_models():
    """Exact float32 correspondences of a known model: F for y2 = 2 y1 + 3 (F = [0 0 0; 0 0 1; 0 -2 -3]), H for
    x2 = 2 x1 + (3, 5).  The reference finds each to 1e-25."""
    rng = np.random.default_rng(3)
    for _ in range(3):
        x1 = np.round(np.c_[rng.uniform(0, WIDTH, 7), rng.uniform(0, HEIGHT, 7)] * 256) / 256
        P = np.c_[x1, np.round(rng.uniform(0, WIDTH, 7) * 256) / 256, 2 * x1[:, 1] + 3].astype(np.float32)
        assert np.array_equal(P[:, 3].astype(np.float64), 2 * P[:, 1].astype(np.float64) + 3)
        ref = _SevenRef(P)
        F = _unit(np.array([0, 0, 0, 0, 0, 1, 0, -2, -3], float))
        Fm = mp.matrix([0, 0, 0, 0, 0, 1, 0, -2, -3]) / mp.sqrt(14)
        d = min(min(mp.norm(mp.matrix(g) - Fm), mp.norm(mp.matrix(g) + Fm)) for g in ref.models)
        assert d <= mp.mpf("1e-25"), d
        assert np.isfinite(ref.kappa).all() and not ref.rank_deficient
        assert min(e for e, _ in ref.forward_errors([F])) <= 1e-15
        x1 = x1[:4]
        P = np.c_[x1, 2 * x1 + [3.0, 5.0]].astype(np.float32)
        h = _LocalRef("H", P)
        H = mp.matrix([2, 0, 3, 0, 2, 5, 0, 0, 1])
        M = mp.matrix(h.model.tolist())
        Hn, Mn = H / mp.norm(H), M / mp.norm(M)
        assert min(mp.norm(Hn - Mn), mp.norm(Hn + Mn)) <= 1e-15      # the model is rounded to double
        v = mp.matrix(h.v)
        s1, c1x, c1y, s2, c2x, c2y = h.T
        T1 = mp.matrix([[s1, 0, -s1 * c1x], [0, s1, -s1 * c1y], [0, 0, 1]])
        T2 = mp.matrix([[s2, 0, -s2 * c2x], [0, s2, -s2 * c2y], [0, 0, 1]])
        Pn = T2 * mp.matrix([[2, 0, 3], [0, 2, 5], [0, 0, 1]]) * mp.inverse(T1)
        p = mp.matrix([Pn[i // 3, i % 3] for i in range(9)])
        p = p / mp.norm(p)
        assert min(mp.norm(v - p), mp.norm(v + p)) <= mp.mpf("1e-25")


def test_oracle_cubic_meets_the_bounds():
    """The oracle's cubic_real_roots, which the device's restates operation for operation, on every cubic fixture."""
    names, coeffs = _cubic_table()
    bad = []
    for name, c in zip(names, coeffs):
        x = vo.cubic_real_roots(*c)
        f = _cubic_checks(c, np.array(x + [0.0] * (3 - len(x))), len(x))
        if f:
            bad.append((name, c.tolist(), f))
    assert not bad, (len(bad), bad[:10])


def test_cubic_fixtures_cover_the_branches():
    names, coeffs = _cubic_table()
    counts = {0: 0, 1: 0, 2: 0, 3: 0}
    for c in coeffs:
        counts[len(_mp_cubic(c)[0])] += 1
    assert all(v > 0 for v in counts.values()), counts
    for c3, c2, c1, c0 in coeffs[[n == "normal" for n in names]][:200]:
        b, c, d = c2 / c3, c1 / c3, c0 / c3
        p, q = c - b * b / 3, 2 * b ** 3 / 27 - b * c / 3 + d
        counts["disc>0" if q * q / 4 + p ** 3 / 27 > 0 else "disc<0"] = 1
    assert counts.get("disc>0") and counts.get("disc<0")
    assert any(n == "triple" for n in names)           # the p == 0 branch: [1, -3, 3, -1]


def _closed_form_cubic(c3, c2, c1, c0):
    """The cubic seven_point used before, restated: the roots of the depressed cubic in closed form (Cardano's sum of
    two cube roots, the trigonometric form), the quadratic's (-c1 +- s) / 2 c2, one unguarded Newton step each."""
    if c3 == 0.0:
        if c2 == 0.0:
            return [] if c1 == 0.0 else [-c0 / c1]
        d = c1 * c1 - 4.0 * c2 * c0
        if d < 0:
            return []
        s = np.sqrt(d)
        return [(-c1 + s) / (2.0 * c2), (-c1 - s) / (2.0 * c2)]
    b, c, d = c2 / c3, c1 / c3, c0 / c3
    p = c - b * b / 3.0
    q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d
    disc = (q / 2.0) * (q / 2.0) + (p / 3.0) * (p / 3.0) * (p / 3.0)
    if disc > 0:
        s = np.sqrt(disc)
        x = [float(np.cbrt(-q / 2.0 + s) + np.cbrt(-q / 2.0 - s) - b / 3.0)]
    elif p == 0.0:
        x = [-b / 3.0]
    else:
        r, a = 2.0 * np.sqrt(-p / 3.0), 3.0 * q / (2.0 * p) * np.sqrt(-3.0 / p)
        phi = np.arccos(min(1.0, max(-1.0, a))) / 3.0
        x = [r * np.cos(phi - 2.0 * np.pi * k / 3.0) - b / 3.0 for k in range(3)]
    return [vo._newton_step(c3, c2, c1, c0, v) for v in x]


def test_measures_see_the_closed_form_cubic():
    """The cubic seven_point used before fails the bounds on the rows of a small c3, Cardano's cancellation and the
    quadratic's cancellation, and in the seven-point step on the samples whose pencil has a small c3; the current one
    passes them."""
    for c in ([1e-9, 1.0, -3.0, 2.0], [0.0, 1.0, 1e8, 1.0], [1.0, 0.0, 1e-6, 1.0]):
        c = np.array(c)
        x = _closed_form_cubic(*c)
        assert _cubic_checks(c, np.array(x + [0.0] * (3 - len(x))), len(x)), c
        x = vo.cubic_real_roots(*c)
        assert not _cubic_checks(c, np.array(x + [0.0] * (3 - len(x))), len(x)), c
    small = [(n, P, r) for n, P, r in _seven_subset() if n == "small_c3"]
    assert len(small) >= 4
    old = [bool(_seven_checks(n, P, r, m, len(m))) for n, P, r in small for m in [_qr_seven_point(P, _closed_form_cubic, False)]]
    assert sum(old) >= len(small) // 2, old
    for n, P, r in small:
        m = _qr_seven_point(P, vo.cubic_real_roots, True)
        assert not _seven_checks(n, P, r, m, len(m))


@functools.lru_cache(maxsize=None)
def _seven_subset():
    """(name, sample, reference) of the samples the seven-point reference runs on."""
    out = [("scene", P) for P in _samples(7, 48, seed=21)]
    out += _special_seven()
    return [(n, P, _SevenRef(P)) for n, P in out]


@functools.lru_cache(maxsize=None)
def _four_subset():
    out = [("scene", P) for P in _samples(4, 96, seed=22)]
    out += _special_four()
    return [(n, P, _LocalRef("H", np.ascontiguousarray(P))) for n, P in out]


def _seven_checks(name, P, ref, models, n):
    """Failures of one seven-point sample's models [n][9] against its reference."""
    bad = []
    if n:
        ra, rd = _backward_errors(np.repeat(_design7(P)[None], n, 0), np.asarray(models[:n], np.float64))
        bad += [("|A f|", name, float(v / U)) for v in ra if v > CU]
        bad += [("|det F|", name, float(v / U)) for v in rd if v > CU]
    if ref.rank_deficient:
        return bad
    if ref.count_decided() and n != len(ref.models):
        bad.append(("count", name, n, len(ref.models)))
    if n == len(ref.models):
        bad += [("forward", name, e / U, b / U) for e, b in ref.forward_errors(models[:n]) if e > b]
    return bad


def test_oracle_seven_point_meets_the_bounds():
    """The oracle's seven_point (the same pencil, cubic and F22 rule on LAPACK's null space) meets every check, and
    the fixtures have samples with one real root and with three, and rank-deficient ones."""
    bad, roots = [], set()
    for name, P, ref in _seven_subset():
        models = vo.seven_point(P[:, :2].astype(np.float64), P[:, 2:].astype(np.float64))
        bad += _seven_checks(name, P, ref, np.array(models).reshape(-1, 9), len(models))
        if not ref.rank_deficient:
            roots.add(len(ref.f22))
    assert not bad, bad[:10]
    assert roots >= {1, 3}, roots
    assert {n for n, _, r in _seven_subset() if r.rank_deficient} == {"duplicate", "duplicate2"}


def test_oracle_homography_meets_the_bound():
    bad = []
    for name, P, ref in _four_subset():
        H = vo.homography_dlt(P[:, :2].astype(np.float64), P[:, 2:].astype(np.float64))[0]
        if ref.model_error(H) > ref.e_model:
            bad.append((name, ref.model_error(H) / U, ref.e_model / U))
    assert not bad, bad
    ratio = min(float(r.s[7] / r.s[0]) for n, _, r in _four_subset() if n.startswith("collinear"))
    assert ratio < 1e-5, ratio


# ---- GPU -----------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_cubic(gpu):
    names, coeffs = _cubic_table()
    x, n = _run_cubic(coeffs)
    bad = []
    for name, c, xi, ni in zip(names, coeffs, x, n):
        assert 0 <= ni <= 3 and not xi[ni:].any()
        f = _cubic_checks(c, xi, ni)
        if f:
            bad.append((name, c.tolist(), f))
    assert not bad, (len(bad), bad[:10])


@pytest.mark.gpu
def test_seven_point(gpu):
    """The backward checks on a batch of 100,000 samples of the eight scenes; every check on the reference subset."""
    S = _samples(7, BIG, seed=23)
    models, n = _run_minimal(0, S)
    assert ((n >= 0) & (n <= 3)).all() and (n == 3).any() and (n == 1).any()
    for k in range(3):
        assert not models[n <= k, k].any()
    rows = np.concatenate([np.flatnonzero(n > k) for k in range(3)])
    ks = np.concatenate([np.full((n > k).sum(), k) for k in range(3)])
    F = models[rows, ks]
    assert np.isfinite(F).all() and (F[:, 8] == 1.0).all()
    A = np.stack([_design7(P) for P in S])[rows]
    ra, rd = _backward_errors(A, F)
    assert ra.max() <= CU, ra.max() / U
    assert rd.max() <= CU, rd.max() / U
    sub = _seven_subset()
    models, n = _run_minimal(0, np.stack([P for _, P, _ in sub]))
    bad = []
    for (name, P, ref), m, k in zip(sub, models, n):
        bad += _seven_checks(name, P, ref, m, k)
    assert not bad, bad[:10]


@pytest.mark.gpu
def test_homography(gpu):
    sub = _four_subset()
    models, n = _run_minimal(1, np.stack([P for _, P, _ in sub]))
    assert (n == 1).all()
    bad = [(name, ref.model_error(m[0]) / U, ref.e_model / U) for (name, _, ref), m in zip(sub, models)
           if not ref.model_error(m[0]) <= ref.e_model]
    assert not bad, bad
    S = _samples(4, BIG, seed=24)
    models, n = _run_minimal(1, S)
    assert (n == 1).all() and np.isfinite(models).all()
    for i in np.linspace(0, BIG - 1, 12).astype(int):
        ref = _LocalRef("H", np.ascontiguousarray(S[i]))
        assert ref.model_error(models[i, 0]) <= ref.e_model, i


@pytest.mark.gpu
@pytest.mark.parametrize("size", BATCHES)
@pytest.mark.parametrize("entry", ["seven_point", "homography", "cubic"])
def test_batch_indexing(gpu, entry, size):
    """Each item's output is the same bits at every batch size and offset: the first and last `size` items of the
    large batch run alone."""
    if entry == "cubic":
        coeffs = np.random.default_rng(25).standard_normal((BIG, 4))
        x, n = _run_cubic(coeffs)
        for sl in (slice(0, size), slice(BIG - size, BIG)):
            xs, ns = _run_cubic(coeffs[sl])
            assert np.array_equal(ns, n[sl]) and np.array_equal(xs, x[sl])
        return
    kind, k = (0, 7) if entry == "seven_point" else (1, 4)
    S = _samples(k, BIG, seed=26)
    models, n = _run_minimal(kind, S)
    for sl in (slice(0, size), slice(BIG - size, BIG)):
        ms, ns = _run_minimal(kind, S[sl])
        assert np.array_equal(ns, n[sl]) and np.array_equal(ms, models[sl])
