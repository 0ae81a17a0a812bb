"""The small null-vector solvers of the geometry stages (csrc/dlt.cuh) and the verification's local step
(csrc/verification.cu, local_estimate / local_model), through their test entries psfm_null_vectors and
psfm_verification_local_model, against references in 50-digit mpmath.

Every bound scales with the conditioning of the problem, never with a fixed tolerance (u = 2^-53, C = 32):
  * a null vector (or the vector of a simple smallest singular value): sin of its angle to the reference,
    sin(v, v*) <= C u sigma_1 / (sigma_{N-k} - sigma_{N-k+1}) with a floor of 4u, where the reference's k smallest
    singular values are equal (k > 1: a null space of k dimensions, measured by the distance to it);
  * one_sided_jacobi's singular values: relative error <= C u kappa(B), B = A D^-1 with unit columns (the reason it
    works on A: a column-graded A = B D keeps its small singular values), where kappa(B) is finite, and absolute error
    <= C u sigma_1 always; |A V - (A V)_dev| <= C u |A|, |V'V - I| <= C u sqrt(N) (each column of V takes O(N)
    rotations per sweep), |cos| <= C u of any two columns of A V above the rounding level C u N sigma_1;
  * smallest_eigenvector: residual |A v - (v'A v) v| <= C u |A| and sin(v, v*) <= C u |A| / gap (Davis-Kahan), gap
    from the smallest eigenvalue (or cluster of equal ones) to the next;
  * the local step: the null vector as above, with sigma from the reference's own normalised design matrix (the
    device's centroids and scales differ from the exact ones by a few u, a backward perturbation of the rows of the
    same size, which the same bound covers), and the normalisation itself to C u.

The local model.  Let e = the null-vector bound and f* the reference's normalised null vector as a 3 x 3 matrix with
singular values s1 >= s2 >= s3.  F's rank-2 step removes s3 u3 v3'; a perturbation E of f moves s3 by at most |E| and
u3, v3 by at most sqrt(2) |E| / (s2 - s3) each (Wedin), so the rank-2 matrix moves by at most
L |E|, L = 2 + 3 s3 / (s2 - s3) (L = 1 for H, which has no rank-2 step).  Denormalising, F = T2' Fn T1 (H =
T2^-1 Hn T1), multiplies an error of Fn by at most |T2| |T1| in the 2-norm, so relative to |F| by
kappa_T = |T2| |T1| |Fn*| / |F*|.  With the unit-norm forms compared up to sign, the local model's distance is at most
    |F / |F| -+ F* / |F*||  <=  2 kappa_T (L e + C u),
the C u for the rounding of the rank-2 step and the two 3 x 3 products.

The reference for the local step works from the float32 points: centroids, RMS scales and rows as COLMAP defines them
(CenterAndNormalizeImagePoints, the eight-point and DLT rows), the rows and the Gram matrix A'A in numpy double-double
(TwoSum / TwoProd, about 1e-32 relative), then mp.eigsy at 50 digits: forming A'A squares the condition number, which
costs nothing at that precision.  The CPU tests show that the reference recovers planted null vectors to 1e-25, that
LAPACK's SVD of the design matrix meets every bound on every fixture, and that solving the Gram matrix in double (a
literal emulation of the cyclic Jacobi the local step used before it kept R instead) fails the null-vector bound once
the baseline is small."""
import ctypes as C
import functools

import mpmath as mp
import numpy as np
import pytest

from particlesfm_b200 import _lib, synthetic as syn

mp.mp.dps = 50
U = 2.0 ** -53
CU = 32.0 * U
FLOOR = 4 * U
NV = {"jacobi3": 0, "jacobi4": 1, "dlt_point": 2, "eigen3": 3, "eigen4": 4, "jacobi9": 5}
DIM = {"jacobi3": 3, "jacobi4": 4, "dlt_point": 4, "eigen3": 3, "eigen4": 4, "jacobi9": 9}
OUT = {"jacobi3": 18, "jacobi4": 32, "dlt_point": 7, "eigen3": 3, "eigen4": 4, "jacobi9": 171}
BLOCK = 128                      # k_null_vectors' block

# the _mixed_batch geometry of test_gpu_two_view: f = 1228.8, 1024 x 436, points 2 .. 40 away
FOCAL, WIDTH, HEIGHT = 1.2 * 1024, 1024, 436
STEPS = [0.08, 0.02, 0.006, 0.002]
NOISES = [0.0, 0.5]
N_F = [8, 9, 255, 256, 257, 20_000, 200_000]         # 8: the fewest inliers F's local step runs on (flag_lo)
N_H = [5, 9, 255, 256, 257, 20_000, 200_000]         # 5: the same for H
NMAX = 200_000
BANDS_THRESHOLD = 1e-9                                # test_gpu_verification.BANDS["threshold"]


# ---- double-double (TwoSum / TwoProd, vectorised) ------------------------------------------------------------------

def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _quick(a, b):
    s = a + b
    return s, b - (s - a)


def _split(a):
    c = 134217729.0 * a
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _dd_add(x, y):
    s, e = _two_sum(x[0], y[0])
    t, f = _two_sum(x[1], y[1])
    s, e = _quick(s, e + t)
    return _quick(s, e + f)


def _dd_mul(x, y):
    p, e = _two_prod(x[0], y[0])
    return _quick(p, e + (x[0] * y[1] + x[1] * y[0]))


def _dd_sum(x):
    """Pairwise double-double sum along axis 0, as mpf (one per trailing index)."""
    h, lo = np.array(x[0], dtype=np.float64), np.array(x[1], dtype=np.float64)
    while h.shape[0] > 1:
        if h.shape[0] % 2:
            z = np.zeros((1,) + h.shape[1:])
            h, lo = np.concatenate([h, z]), np.concatenate([lo, z])
        h, lo = _dd_add((h[0::2], lo[0::2]), (h[1::2], lo[1::2]))
    h, lo = np.atleast_1d(h[0]), np.atleast_1d(lo[0])
    return [mp.mpf(float(a)) + mp.mpf(float(b)) for a, b in zip(h, lo)]


def _dd(x):
    hi = float(x)
    return hi, float(x - hi)


def _dd_const(x, n):
    hi, lo = _dd(x)
    return np.full(n, hi), np.full(n, lo)


# ---- mpmath helpers ------------------------------------------------------------------------------------------------

def _mp(A):
    return mp.matrix([[mp.mpf(float(x)) for x in row] for row in np.atleast_2d(A)])


def _vec(v):
    return mp.matrix([mp.mpf(float(x)) for x in v])


def _mp_svd(A):
    """Singular values (descending) and the right singular vectors (columns, same order) of a float64 matrix."""
    Um, S, Vt = mp.svd_r(_mp(A))
    s = [S[i] for i in range(len(S))]
    order = sorted(range(len(s)), key=lambda i: -s[i])
    n = Vt.cols
    V = mp.matrix(n, len(s))
    for j, i in enumerate(order):
        for k in range(n):
            V[k, j] = Vt[i, k]
    return [s[i] for i in order], V


def _mp_eig_sym(G):
    """Eigenvalues (ascending) and eigenvectors (columns, same order) of a symmetric mp matrix."""
    E, Q = mp.eigsy(G)
    order = sorted(range(len(E)), key=lambda i: E[i])
    V = mp.matrix(Q.rows, len(E))
    for j, i in enumerate(order):
        for k in range(Q.rows):
            V[k, j] = Q[k, i]
    return [E[i] for i in order], V


def _dist_to_span(v, Q):
    """|v - Q Q' v| / |v| for orthonormal columns Q (mp), v float64."""
    x = _vec(v)
    x = x / mp.norm(x)
    r = x - Q * (Q.T * x)
    return float(mp.norm(r))


def _cluster(vals, lowest, scale):
    """Indices of the values equal to the extreme one (to 1e-40 of scale), and the gap to the next."""
    ref = vals[lowest]
    idx = [i for i in range(len(vals)) if abs(vals[i] - ref) <= mp.mpf("1e-40") * scale]
    rest = [abs(vals[i] - ref) for i in range(len(vals)) if i not in idx]
    return idx, (min(rest) if rest else mp.mpf(0))


def _cols(V, idx):
    Q = mp.matrix(V.rows, len(idx))
    for j, i in enumerate(idx):
        for k in range(V.rows):
            Q[k, j] = V[k, i]
    return Q


def _bound(num, gap):
    return FLOOR if num == 0 else (np.inf if gap == 0 else max(CU * float(num / gap), FLOOR))


def _null_measure(v, s, V):
    """(sin of v to the reference null space of the smallest singular value(s), its bound)."""
    idx, gap = _cluster(s, len(s) - 1, s[0] if s[0] > 0 else 1)
    return _dist_to_span(v, _cols(V, idx)), _bound(s[0], gap)


# ---- the primitives' matrices --------------------------------------------------------------------------------------

def _orth(rng, n):
    q, r = np.linalg.qr(rng.standard_normal((n, n)))
    return q * np.sign(np.diag(r))


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _essential(rng):
    R = syn.axis_angle_to_rotmat(rng.standard_normal((1, 3)) * 0.3)[0]
    return _skew(rng.standard_normal(3)) @ R


def _special(n, symmetric, seed):
    """The edge matrices of one size: (name, matrix)."""
    rng = np.random.default_rng(seed)
    out = []
    for k in range(3):                                  # column-graded: B D, D over 1e-8 .. 1e8
        B = rng.standard_normal((n, n))
        D = np.diag(np.logspace(-8, 8, n)[rng.permutation(n)])
        out.append(("graded", D @ (B @ B.T + n * np.eye(n)) @ D if symmetric else B @ D))
    for r in sorted({n - 1, n - 2, 1} - {0}):           # exact rank deficiency: integer factors, exact products
        Bi = rng.integers(-4, 5, (n, r)).astype(np.float64)
        out.append(("rank%d" % r, Bi @ Bi.T if symmetric else Bi @ rng.integers(-4, 5, (r, n)).astype(np.float64)))
    E = _essential(rng)                                 # sigma_1 = sigma_2 (E), padded for n > 3
    M = np.eye(n) * 0.5
    M[:3, :3] = E
    if n == 9:
        M[3:6, 3:6], M[6:, 6:] = _essential(rng), _essential(rng)
    out.append(("essential", M.T @ M if symmetric else M))
    Q, P = _orth(rng, n), _orth(rng, n)                 # clustered: gaps of 1e-9 at the smallest end and above
    d = np.concatenate([[1.0, 1.0 + 1e-9, 1.0 + 2e-9], 2.0 + np.arange(n - 3)])
    out.append(("clustered", Q @ np.diag(d) @ Q.T if symmetric else Q @ np.diag(d) @ P.T))
    d = rng.uniform(0.5, 4.0, n)
    out.append(("diagonal", np.diag(d)))
    out.append(("diagonal_repeated", np.diag(np.r_[1.0, 1.0, 3.0 + np.arange(n - 2)])))
    out.append(("zero", np.zeros((n, n))))
    return out


def _batch(form, seed=0, n_random=200):
    n = DIM[form]
    symmetric = form.startswith("eigen")
    rng = np.random.default_rng(seed + 100 * n + (7 if symmetric else 0))
    mats = []
    for _ in range(n_random):
        A = rng.standard_normal((n, n))
        mats.append(("random", (A + A.T) / 2.0 if symmetric else A))
    mats += _special(n, symmetric, seed + 1)
    if form == "dlt_point":                             # a point at infinity: the null vector has v[3] = 0 exactly
        v = np.array([1.0, 2.0, -1.0, 0.0])
        B = rng.integers(-4, 5, (4, 4)).astype(np.float64)
        B[:, 0] = -(B[:, 1] * 2.0 - B[:, 2])            # B v = 0
        mats.append(("infinity", B))
    assert len(mats) % BLOCK != 0
    return mats


def _run(form, mats):
    A = np.ascontiguousarray(np.stack([m for _, m in mats]), dtype=np.float64)
    out = np.full((len(mats), OUT[form]), np.nan)
    _lib.check(_lib.lib().psfm_null_vectors(NV[form], _lib.dptr(A), len(mats), _lib.dptr(out)), "psfm_null_vectors")
    return out


# ---- the local step's scenes and reference -------------------------------------------------------------------------

def _camera(step):
    ang = np.array([0.1, 0.5, -0.15]) * step
    R = syn.axis_angle_to_rotmat(ang[None])[0]
    t = np.array([step, 0.2 * step, 0.05 * step])
    K = np.array([[FOCAL, 0.0, WIDTH / 2], [0.0, FOCAL, HEIGHT / 2], [0.0, 0.0, 1.0]])
    return K, R, t


def _project(K, Xc):
    return Xc[:, :2] / Xc[:, 2:] * K[0, 0] + K[:2, 2]


@functools.lru_cache(maxsize=None)
def _scene(step, noise, plane=False, outliers=0.0, seed=0):
    """NMAX correspondences (x1, y1, x2, y2) in float32 and the true model (F for a general scene, H for a plane):
    the second camera X2 = R X - t, moved `step` from the first."""
    rng = np.random.default_rng(seed + int(step * 1e4) + (17 if noise else 0) + (5 if plane else 0))
    K, R, t = _camera(step)
    Ki = np.linalg.inv(K)
    if plane:                                   # the plane n'X = d in front of camera 1
        nrm, dd = np.array([0.1, -0.05, 1.0]), 8.0
        px = np.c_[rng.uniform(0, WIDTH, NMAX), rng.uniform(0, HEIGHT, NMAX), np.ones(NMAX)]
        ray = px @ Ki.T
        X = ray * (dd / (ray @ nrm))[:, None]
        model = K @ (R - np.outer(t, nrm) / dd) @ Ki
    else:
        depth = rng.uniform(2.0, 40.0, NMAX)
        X = np.c_[rng.uniform(-0.6, 0.6, (NMAX, 2)) * depth[:, None], depth]
        model = Ki.T @ _skew(-t) @ R @ Ki
    x1, x2 = _project(K, X), _project(K, X @ R.T - t)
    x1 = x1 + rng.normal(0.0, noise, x1.shape) if noise else x1
    x2 = x2 + rng.normal(0.0, noise, x2.shape) if noise else x2
    bad = rng.random(NMAX) < outliers
    x2[bad] = np.c_[rng.uniform(0, WIDTH, bad.sum()), rng.uniform(0, HEIGHT, bad.sum())]
    return np.ascontiguousarray(np.c_[x1, x2].astype(np.float32)), model.reshape(9)


def _residuals(kind, f, P):
    """verification.cu's residual<KIND> in float64 (the squared Sampson error of F, the squared transfer error of H)."""
    X, Y, Uu, V = (P[:, k].astype(np.float64) for k in range(4))
    if kind == "F":
        e0, e1, e2 = f[0] * X + f[1] * Y + f[2], f[3] * X + f[4] * Y + f[5], f[6] * X + f[7] * Y + f[8]
        t0, t1 = f[0] * Uu + f[3] * V + f[6], f[1] * Uu + f[4] * V + f[7]
        c = Uu * e0 + V * e1 + e2
        return c * c / (e0 * e0 + e1 * e1 + t0 * t0 + t1 * t1)
    inv = 1.0 / (f[6] * X + f[7] * Y + f[8])
    d0, d1 = Uu - (f[0] * X + f[1] * Y + f[2]) * inv, V - (f[3] * X + f[4] * Y + f[5]) * inv
    return d0 * d0 + d1 * d1


def _normalisation(P):
    """CenterAndNormalizeImagePoints of both images in high precision: [s1, c1x, c1y, s2, c2x, c2y] as mpf."""
    n = len(P)
    sums = _dd_sum((P.astype(np.float64), np.zeros((n, 4))))
    c = [x / n for x in sums]
    out = []
    for img in range(2):
        cx, cy = c[2 * img], c[2 * img + 1]
        dx = _dd_add((P[:, 2 * img].astype(np.float64), np.zeros(n)), _dd_const(-cx, n))
        dy = _dd_add((P[:, 2 * img + 1].astype(np.float64), np.zeros(n)), _dd_const(-cy, n))
        r = _dd_add(_dd_mul(dx, dx), _dd_mul(dy, dy))
        rms = _dd_sum((r[0][:, None], r[1][:, None]))[0]
        out += [mp.sqrt(2) / mp.sqrt(rms / n), cx, cy]
    return out


def _rows(kind, P, T):
    """The normalised design matrix's rows in double-double: (hi [m][9], lo [m][9])."""
    n = len(P)
    s1, c1x, c1y, s2, c2x, c2y = T

    def coord(k, c, s):
        d = _dd_add((P[:, k].astype(np.float64), np.zeros(n)), _dd_const(-c, n))
        return _dd_mul(d, _dd_const(s, n))

    a0, a1, d0, d1 = coord(0, c1x, s1), coord(1, c1y, s1), coord(2, c2x, s2), coord(3, c2y, s2)
    one, zero = (np.ones(n), np.zeros(n)), (np.zeros(n), np.zeros(n))
    neg = lambda x: (-x[0], -x[1])
    if kind == "F":
        rows = [[_dd_mul(d0, a0), _dd_mul(d0, a1), d0, _dd_mul(d1, a0), _dd_mul(d1, a1), d1, a0, a1, one]]
    else:
        rows = [[neg(a0), neg(a1), neg(one), zero, zero, zero, _dd_mul(a0, d0), _dd_mul(a1, d0), d0],
                [zero, zero, zero, neg(a0), neg(a1), neg(one), _dd_mul(a0, d1), _dd_mul(a1, d1), d1]]
    hi = np.concatenate([np.stack([r[0] for r in rr], axis=1) for rr in rows])
    lo = np.concatenate([np.stack([r[1] for r in rr], axis=1) for rr in rows])
    return hi, lo


def _gram(hi, lo):
    """A'A of the double-double rows, as a symmetric mp matrix."""
    iu, ju = np.triu_indices(9)
    p = _dd_mul((hi[:, iu], lo[:, iu]), (hi[:, ju], lo[:, ju]))
    vals = _dd_sum(p)
    G = mp.matrix(9, 9)
    for k, (i, j) in enumerate(zip(iu, ju)):
        G[i, j] = G[j, i] = vals[k]
    return G


def _denormalise(kind, f, T):
    """The local model from the normalised null vector (mp): F = T2' rank2(Fn) T1, H = T2^-1 Hn T1.  Also returns
    kappa_T and L of the module docstring."""
    s1, c1x, c1y, s2, c2x, c2y = T
    T1 = mp.matrix([[s1, 0, -s1 * c1x], [0, s1, -s1 * c1y], [0, 0, 1]])
    T2 = mp.matrix([[s2, 0, -s2 * c2x], [0, s2, -s2 * c2y], [0, 0, 1]])
    Fn = mp.matrix(3, 3)
    for i in range(9):
        Fn[i // 3, i % 3] = f[i]
    if kind == "F":
        Um, S, Vt = mp.svd_r(Fn)
        sv = sorted([S[i] for i in range(3)], reverse=True)
        L = 2 + 3 * sv[2] / (sv[1] - sv[2]) if sv[1] > sv[2] else mp.inf
        D = mp.diag([S[i] if S[i] != min(S[i] for i in range(3)) else 0 for i in range(3)])
        Fn2 = Um * D * Vt
        M, left = T2.T * Fn2 * T1, T2
    else:
        L, Fn2 = mp.mpf(1), Fn
        left = mp.inverse(T2)
        M = left * Fn2 * T1
    two = lambda A: max(mp.svd_r(A, compute_uv=False))
    kappa = two(left) * two(T1) * mp.mnorm(Fn2, "f") / mp.mnorm(M, "f")
    return np.array([float(M[i // 3, i % 3]) for i in range(9)]), float(kappa), float(L)


class _LocalRef:
    """The reference local step on the inliers P (float32 [n][4]) of one kind."""

    def __init__(self, kind, P):
        self.kind = kind
        self.T = _normalisation(P)
        self.hi, self.lo = _rows(kind, P, self.T)
        lam, Q = _mp_eig_sym(_gram(self.hi, self.lo))
        self.s = [mp.sqrt(max(x, 0)) for x in reversed(lam)]            # descending
        self.V = mp.matrix(9, 9)
        for j in range(9):
            for k in range(9):
                self.V[k, j] = Q[k, 8 - j]
        self.v = [self.V[k, 8] for k in range(9)]
        self.model, self.kappa_T, self.L = _denormalise(kind, self.v, self.T)
        idx, gap = _cluster(self.s, 8, self.s[0])
        assert idx == [8], "a fixture with a null space of more than one dimension"
        self.e_v = _bound(self.s[0], gap)
        self.e_model = 2.0 * self.kappa_T * (self.L * self.e_v + CU)

    def null_error(self, v):
        return _dist_to_span(v, _cols(self.V, [8]))

    def model_error(self, m):
        a, b = m / np.linalg.norm(m), self.model / np.linalg.norm(self.model)
        return min(np.linalg.norm(a - b), np.linalg.norm(a + b))

    def normalisation_error(self, T, P):
        """max over the six values of |T - T*| / scale: s relative to itself, the centroids to the largest |x|."""
        big = [float(np.abs(P[:, k]).max()) for k in range(4)]
        scale = [float(self.T[0]), big[0], big[1], float(self.T[3]), big[2], big[3]]
        return max(abs(float(T[i] - self.T[i])) / scale[i] for i in range(6))


def _fixture(kind, step, noise, n):
    P, _ = _scene(step, noise)
    return np.ascontiguousarray(P[:n])


@functools.lru_cache(maxsize=None)
def _reference(kind, step, noise, n):
    return _LocalRef(kind, _fixture(kind, step, noise, n))


def _design64(kind, P):
    """The normalised design matrix in float64, the centroids and scales as np.mean / np.sqrt compute them."""
    Q = P.astype(np.float64)
    T = []
    for img in range(2):
        c = Q[:, 2 * img:2 * img + 2].mean(axis=0)
        s = np.sqrt(2.0) / np.sqrt(((Q[:, 2 * img:2 * img + 2] - c) ** 2).sum(axis=1).mean())
        T += [s, c[0], c[1]]
    a0, a1 = (Q[:, 0] - T[1]) * T[0], (Q[:, 1] - T[2]) * T[0]
    d0, d1 = (Q[:, 2] - T[4]) * T[3], (Q[:, 3] - T[5]) * T[3]
    one, zero = np.ones(len(Q)), np.zeros(len(Q))
    if kind == "F":
        A = np.stack([d0 * a0, d0 * a1, d0, d1 * a0, d1 * a1, d1, a0, a1, one], axis=1)
    else:
        A = np.concatenate([np.stack([-a0, -a1, -one, zero, zero, zero, a0 * d0, a1 * d0, d0], axis=1),
                            np.stack([zero, zero, zero, -a0, -a1, -one, a0 * d1, a1 * d1, d1], axis=1)])
    return A, T


def _lapack_local(kind, P):
    """The local step in float64 with LAPACK's SVD of the design matrix itself (COLMAP's route)."""
    A, T = _design64(kind, P)
    v = np.linalg.svd(A, full_matrices=len(A) < 9)[2][8]
    s1, c1x, c1y, s2, c2x, c2y = T
    T1 = np.array([[s1, 0, -s1 * c1x], [0, s1, -s1 * c1y], [0, 0, 1]])
    T2 = np.array([[s2, 0, -s2 * c2x], [0, s2, -s2 * c2y], [0, 0, 1]])
    M = v.reshape(3, 3)
    if kind == "F":
        Uu, S, Vt = np.linalg.svd(M)
        M = T2.T @ (Uu @ np.diag([S[0], S[1], 0.0]) @ Vt) @ T1
    else:
        M = np.linalg.inv(T2) @ M @ T1
    return v, T, M.reshape(9)


def _gram_jacobi(G):
    """A literal numpy emulation of the cyclic Jacobi eigen-solver the local step used on the Gram matrix."""
    A, n = G.copy(), G.shape[0]
    V = np.eye(n)
    for _ in range(30):
        off = sum(A[i, j] ** 2 for i in range(n) for j in range(i + 1, n))
        if not off > 1e-34 * sum(A[i, i] ** 2 for i in range(n)):
            break
        for p in range(n - 1):
            for q in range(p + 1, n):
                apq = A[p, q]
                if apq == 0.0:
                    continue
                th = (A[q, q] - A[p, p]) / (2.0 * apq)
                t = (1.0 if th >= 0 else -1.0) / (abs(th) + np.sqrt(th * th + 1.0))
                c = 1.0 / np.sqrt(t * t + 1.0)
                s = t * c
                ap, aq = A[:, p].copy(), A[:, q].copy()
                A[:, p], A[:, q] = c * ap - s * aq, s * ap + c * aq
                ap, aq = A[p, :].copy(), A[q, :].copy()
                A[p, :], A[q, :] = c * ap - s * aq, s * ap + c * aq
                vp, vq = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = c * vp - s * vq, s * vp + c * vq
    return V[:, int(np.argmin(np.diag(A)))]


def _local_step(kind, P, best, thr):
    v, T, m = np.full(9, np.nan), np.full(6, np.nan), np.full(9, np.nan)
    Pc = np.ascontiguousarray(P, dtype=np.float32)
    rc = _lib.lib().psfm_verification_local_model(0 if kind == "F" else 1, Pc.ctypes.data_as(C.POINTER(C.c_float)),
                                                  len(Pc), _lib.dptr(np.ascontiguousarray(best, dtype=np.float64)),
                                                  thr, _lib.dptr(v), _lib.dptr(T), _lib.dptr(m))
    _lib.check(rc, "psfm_verification_local_model")
    return v, T, m


LOCAL_CASES = [(k, s, z, n) for k, ns in (("F", N_F), ("H", N_H)) for s in STEPS for z in NOISES for n in ns]


def _id(c):
    return "%s-step%g-noise%g-n%d" % c


# ---- CPU: the reference and the measures ---------------------------------------------------------------------------

def test_reference_recovers_planted_null_vectors():
    """F: the second image differs from the first by a horizontal shift only (y2 = y1 exactly), whose F has one free
    entry pair; H: x2 = 2 x1 + (3, 5) exactly in float32.  The normalised null vector is T2^-T F T1^-1 (T2 H T1^-1),
    computed in mp from the reference's own normalisation."""
    rng = np.random.default_rng(3)
    n = 3000
    x1 = np.round(np.c_[rng.uniform(0, WIDTH, n), rng.uniform(0, HEIGHT, n)] * 256) / 256
    cases = {"F": (np.c_[x1, rng.uniform(0, WIDTH, n), x1[:, 1]], np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]])),
             "H": (np.c_[x1, 2 * x1 + [3.0, 5.0]], np.array([[2, 0, 3], [0, 2, 5], [0, 0, 1]]))}
    for kind, (P, M) in cases.items():
        P = P.astype(np.float32)
        assert np.array_equal(P.astype(np.float64)[:, 2:] if kind == "H" else P[:, 3],
                              (2 * P.astype(np.float64)[:, :2] + [3.0, 5.0]) if kind == "H" else P[:, 1])
        ref = _LocalRef(kind, P)
        s1, c1x, c1y, s2, c2x, c2y = ref.T
        T1 = mp.matrix([[s1, 0, -s1 * c1x], [0, s1, -s1 * c1y], [0, 0, 1]])
        T2 = mp.matrix([[s2, 0, -s2 * c2x], [0, s2, -s2 * c2y], [0, 0, 1]])
        Mm = mp.matrix(M.tolist())
        Pn = mp.inverse(T2).T * Mm * mp.inverse(T1) if kind == "F" else T2 * Mm * mp.inverse(T1)
        p = mp.matrix([Pn[i // 3, i % 3] for i in range(9)])
        p = p / mp.norm(p)
        v = mp.matrix(ref.v)
        d = min(mp.norm(v - p), mp.norm(v + p))
        assert d <= mp.mpf("1e-25"), (kind, d)
        assert ref.s[8] ** 2 <= mp.mpf("1e-25") * ref.s[0] ** 2, (kind, ref.s[8])      # sigma_9^2: an eigenvalue of A'A
    # and a primitive's planted null space: an integer 4 x 4 of rank 3 with null vector (1, 2, -1, 3)
    B = rng.integers(-5, 6, (4, 4)).astype(np.float64)
    B[:, 0] = -(2 * B[:, 1] - B[:, 2] + 3 * B[:, 3])
    s, V = _mp_svd(B)
    d, _ = _null_measure(np.array([1.0, 2.0, -1.0, 3.0]), s, V)
    assert d <= 1e-25 and s[3] <= mp.mpf("1e-40"), (d, s[3])


@pytest.mark.parametrize("case", LOCAL_CASES, ids=_id)
def test_lapack_meets_every_bound(case):
    kind, step, noise, n = case
    P = _fixture(*case)
    ref = _reference(*case)
    v, T, m = _lapack_local(kind, P)
    assert ref.null_error(v) <= ref.e_v, (ref.null_error(v) / U, ref.e_v / U)
    assert ref.normalisation_error(T, P) <= CU
    assert ref.model_error(m) <= ref.e_model, (ref.model_error(m) / U, ref.e_model / U)


GRAM_TABLE = [(0.08, 0.0), (0.02, 0.5), (0.006, 0.5), (0.002, 0.0)]


@pytest.mark.parametrize("step,noise", GRAM_TABLE)
def test_measures_see_the_gram_route(step, noise):
    """The eight-point null vector of 2,000 correspondences through the Gram matrix in double and the cyclic Jacobi:
    the error grows with kappa^2 and fails the bound once step <= 0.006; LAPACK's SVD of A passes it everywhere."""
    P = _fixture("F", step, noise, 2000)
    ref = _LocalRef("F", P)
    A, _ = _design64("F", P)
    g = ref.null_error(_gram_jacobi(A.T @ A))
    lap = ref.null_error(np.linalg.svd(A, full_matrices=len(A) < 9)[2][8])
    kappa = float(ref.s[0] / ref.s[7])
    print("step %g noise %g: kappa %.0f, LAPACK %.1e, Gram %.1e, u kappa %.1e, bound %.1e"
          % (step, noise, kappa, lap, g, U * kappa, ref.e_v))
    assert lap <= ref.e_v
    if step <= 0.006:
        assert g > ref.e_v, (g, ref.e_v)
        assert g > 100 * lap


def test_measures_see_a_perturbed_vector():
    ref = _reference("F", 0.02, 0.5, 2000)
    v = np.array([float(x) for x in ref.v])
    w = np.random.default_rng(0).standard_normal(9)
    w -= (w @ v) * v
    bad = v + 4 * ref.e_v * w / np.linalg.norm(w)
    assert ref.null_error(bad) > ref.e_v


# ---- GPU: the primitives -------------------------------------------------------------------------------------------

def _svd_checks(name, A, AV, V):
    n = A.shape[0]
    s, Vr = _mp_svd(A)
    nA = float(s[0])
    sig = np.sort(np.linalg.norm(AV, axis=0))[::-1]
    sref = np.array([float(x) for x in s])
    assert np.all(np.abs(sig - sref) <= CU * nA), (name, sig, sref)
    cn = np.linalg.norm(A, axis=0)
    if (cn > 0).all():
        Bs = _mp_svd(A / cn)[0]
        kB = float(Bs[0] / Bs[-1]) if Bs[-1] > mp.mpf("1e-30") else np.inf
        if kB < 1e15:
            assert np.all(np.abs(sig - sref) <= CU * kB * sref), (name, (np.abs(sig - sref) / sref / U).max(), kB)
    assert np.abs(A @ V - AV).max() <= CU * max(nA, np.abs(A).max()) * n, name
    assert np.abs(V.T @ V - np.eye(n)).max() <= CU * np.sqrt(n), name
    nrm = np.linalg.norm(AV, axis=0)
    nz = nrm > CU * n * nA                              # columns at the rounding level have no direction
    Cc = (AV[:, nz] / nrm[nz]).T @ (AV[:, nz] / nrm[nz])
    assert np.abs(Cc - np.eye(nz.sum())).max() <= CU, name
    v = V[:, int(np.argmin(np.linalg.norm(AV, axis=0)))]
    d, b = _null_measure(v, s, Vr)
    assert d <= b, (name, d / U, b / U)
    return v


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["jacobi3", "jacobi4", "jacobi9"])
def test_one_sided_jacobi(gpu, form):
    mats = _batch(form)
    out = _run(form, mats)
    n = DIM[form]
    for (name, A), o in zip(mats, out):
        AV, V = o[:n * n].reshape(n, n), o[n * n:2 * n * n].reshape(n, n)
        if name == "zero":
            assert not AV.any() and np.array_equal(V, np.eye(n)), form
            continue
        v = _svd_checks(name, A, AV, V)
        if form == "jacobi9":
            assert np.array_equal(o[162:], v), name


@pytest.mark.gpu
def test_dlt_point(gpu):
    mats = _batch("dlt_point")
    out = _run("dlt_point", mats)
    for (name, A), o in zip(mats, out):
        X, v = o[:3], o[3:]
        if name == "zero" or name == "infinity":
            assert not np.isfinite(X).all() or np.abs(X).max() > 1e12, (name, X)
            continue
        s, V = _mp_svd(A)
        d, b = _null_measure(v, s, V)
        assert d <= b and abs(np.linalg.norm(v) - 1.0) <= CU, (name, d / U, b / U)
        with np.errstate(divide="ignore", invalid="ignore"):
            assert np.array_equal(X, v[:3] / v[3], equal_nan=True), name


@pytest.mark.gpu
@pytest.mark.parametrize("form", ["eigen3", "eigen4"])
def test_smallest_eigenvector(gpu, form):
    mats = _batch(form)
    out = _run(form, mats)
    for (name, A), v in zip(mats, out):
        assert abs(np.linalg.norm(v) - 1.0) <= CU, (name, v)
        lam, Q = _mp_eig_sym(_mp(A))
        nA = float(max(abs(lam[0]), abs(lam[-1])))
        r = np.linalg.norm(A @ v - (v @ A @ v) * v)
        assert r <= CU * max(nA, 1e-300) or (nA == 0 and r == 0), (name, r / U, nA)
        idx, gap = _cluster(lam, 0, nA if nA else 1)
        d = _dist_to_span(v, _cols(Q, idx))
        assert d <= _bound(nA, gap), (name, d / U, _bound(nA, gap) / U)


# ---- GPU: the local step -------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("case", LOCAL_CASES, ids=_id)
def test_local_step(gpu, case):
    """Every point an inlier (threshold 1e300): the device's null vector, normalisation and local model against the
    reference."""
    kind, step, noise, n = case
    P = _fixture(*case)
    best = _scene(step, noise)[1] if kind == "F" else np.eye(3).reshape(9)
    v, T, m = _local_step(kind, P, best, 1e300)
    ref = _reference(*case)
    assert abs(np.linalg.norm(v) - 1.0) <= CU
    assert ref.normalisation_error(T, P) <= CU, ref.normalisation_error(T, P) / U
    ev, em = ref.null_error(v), ref.model_error(m)
    assert ev <= ref.e_v, ("null vector", ev / U, ref.e_v / U)
    assert em <= ref.e_model, ("local model", em / U, ref.e_model / U)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["F", "H"])
def test_local_step_with_outliers_and_a_threshold(gpu, kind):
    """20 % outliers and the stage's threshold 4 px (16 squared), every inlier decision clear of rounding by the
    verification tests' margin; the inliers the reference solves are the ones residual<KIND> keeps.  Two calls give
    the same bits."""
    P, model = _scene(0.006, 0.5, plane=kind == "H", outliers=0.2, seed=1)
    P = P[:20_000]
    thr = 16.0
    r = _residuals(kind, model, P)
    clear = np.abs(r - thr) > BANDS_THRESHOLD * thr
    P = np.ascontiguousarray(P[clear])
    inl = _residuals(kind, model, P) <= thr
    assert 0.6 * len(P) < inl.sum() < 0.95 * len(P)
    v, T, m = _local_step(kind, P, model, thr)
    ref = _LocalRef(kind, np.ascontiguousarray(P[inl]))
    assert ref.normalisation_error(T, P[inl]) <= CU
    assert ref.null_error(v) <= ref.e_v, (ref.null_error(v) / U, ref.e_v / U)
    assert ref.model_error(m) <= ref.e_model, (ref.model_error(m) / U, ref.e_model / U)
    again = _local_step(kind, P, model, thr)
    for a, b in zip((v, T, m), again):
        assert np.array_equal(a, b)
