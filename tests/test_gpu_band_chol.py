"""The single-CTA register-window band(+arrow) Cholesky of the exact-Schur mode
(csrc/ba_band_chol.cuh) against numpy on random SPD systems, through the C ABI."""
import ctypes as C

import numpy as np
import pytest

from particlesfm_b200 import _lib

pytestmark = pytest.mark.gpu


def _system(nb, bw, seed, arrow=True):
    rng = np.random.default_rng(seed)
    n = nb + 3
    B = rng.standard_normal((n, n))
    A = B @ B.T
    i, j = np.indices((n, n))
    A[(np.abs(i - j) > bw) & (i < nb) & (j < nb)] = 0.0
    if not arrow:                       # inactive intrinsics: identity rows, as k_band_assemble writes them
        A[nb:, :] = 0.0
        A[:, nb:] = 0.0
    A += np.eye(n) * (np.abs(A).sum(axis=1).max() + 1.0)
    b = rng.standard_normal(n)
    if not arrow:
        A[nb:, nb:] = np.eye(3)
        b[nb:] = 0.0
    return A, b


def _solve(A, b, nb, bw):
    x = np.zeros_like(b)
    rc = _lib.lib().psfm_ba_band_solve(_lib.dptr(np.ascontiguousarray(A)), _lib.dptr(b), nb, bw, _lib.dptr(x))
    return rc, x


# (nb, bw), grouped by the instantiation of the block-6 kernel they launch (threads, tile of a worker thread)
CASES = [
    # 512, 3 x 3: window of 3 blocks (also clamped up from bw = 5 on a two-sided matrix), window = matrix (bw clamped
    # to nb - 1), one CTA, two CTAs, the two-sided threshold F = 4 Wb (162: one CTA, 168: two), identity padding rows
    # past the matrix (nb not a multiple of 8), and the widest window of this instantiation (12 blocks: the bench's
    # reduced system, 6 * 200 images with tracks spanning 11)
    (30, 9), (18, 17), (18, 40), (36, 17), (36, 35), (78, 17), (90, 59), (900, 35), (2400, 23), (2400, 5),
    (162, 35), (168, 35), (1206, 40), (1200, 65),
    # 384, 3 x 6: two CTAs
    (1200, 71), (1200, 77), (3000, 71),
    # 512, 6 x 6: two CTAs, up to the widest window of this instantiation (22 blocks)
    (1200, 83), (1200, 95), (1200, 125),
    # 640, 6 x 6: window of 23 blocks, the widest window (25 blocks) as the whole matrix and on a long matrix (two CTAs)
    (600, 127), (150, 149), (1200, 143)]


@pytest.mark.parametrize("nb,bw", CASES)
def test_band_solve_matches_numpy(gpu, nb, bw):
    A, b = _system(nb, bw, seed=nb + bw)
    rc, x = _solve(A, b, nb, bw)
    assert rc == 0, _lib.lib().psfm_last_error()
    ref = np.linalg.solve(A, b)
    assert np.abs(x - ref).max() <= 1e-11 * np.abs(ref).max()


def test_band_solve_inactive_arrow_and_failure(gpu):
    A, b = _system(120, 35, seed=1, arrow=False)
    rc, x = _solve(A, b, 120, 35)
    assert rc == 0
    ref = np.linalg.solve(A, b)
    assert np.abs(x - ref).max() <= 1e-11 * np.abs(ref).max()
    assert np.array_equal(x[120:], np.zeros(3))
    A[57, 57] = -1.0                    # not positive definite -> reported, no garbage accepted
    rc, _ = _solve(A, b, 120, 35)
    assert rc == -1
    rc, _ = _solve(A, b, 120, 400)      # clamped to nb - 1 = 119: a window of the whole matrix, still a solvable shape
    assert rc == -1
    # PSFM_ERR_UNSUPPORTED: nb not a multiple of 6 (400 with a window of 51 blocks, 100), a window of
    # (149 + 5) / 6 + 1 = 26 blocks on a 200-block matrix
    for nb, bw in ((400, 300), (100, 31), (1200, 149)):
        A2, b2 = _system(nb, bw, seed=2)
        rc, _ = _solve(A2, b2, nb, bw)
        assert rc == -4, (nb, bw)


def test_block6_forms_agree(gpu, tmp_path):
    """Two-sided (default) vs one-sided (PSFM_CHOL_ONE_SIDED) on two long matrices: a different but fixed elimination
    order, so the solutions agree to rounding and are not the same bits.  The switch is read once per process: each
    form runs in a child process."""
    import os
    import subprocess
    import sys
    code = ("import numpy as np, sys; sys.path[:0] = [%r, %r]; from test_gpu_band_chol import _system, _solve;"
            "A, b = _system(%d, %d, seed=11); rc, x = _solve(A, b, %d, %d); assert rc == 0; np.save(sys.argv[1], x)")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for nb, bw in ((1200, 71), (1200, 95)):
        out = {}
        for name, env in (("two", {}), ("one", {"PSFM_CHOL_ONE_SIDED": "1"})):
            path = str(tmp_path / f"_band_{nb}_{bw}_{name}.npy")
            subprocess.run([sys.executable, "-c", code % (root, os.path.join(root, "tests"), nb, bw, nb, bw), path],
                           check=True, env={**os.environ, **env}, cwd=root)
            out[name] = np.load(path)
        assert np.abs(out["two"] - out["one"]).max() <= 1e-12 * np.abs(out["one"]).max(), (nb, bw)
        assert not np.array_equal(out["two"], out["one"]), (nb, bw)


@pytest.mark.parametrize("bad", [0, 57, 281, 282, 299, 317, 318, 450, 599])
def test_block6_two_sided_form_reports_a_bad_pivot_wherever_it_is(gpu, bad):
    """nb = 600, bw = 35: block-6 kernel, window of 6 image blocks, two CTAs (top-down 47 blocks, bottom-up 47, 6 in
    the middle).  A negative diagonal on either side or in the middle must come back as an error, never as a hang or
    a silent solve."""
    A, b = _system(600, 35, seed=5)
    rc, x = _solve(A, b, 600, 35)
    assert rc == 0
    ref = np.linalg.solve(A, b)
    assert np.abs(x - ref).max() <= 1e-11 * np.abs(ref).max()
    A[bad, bad] = -1.0
    rc, _ = _solve(A, b, 600, 35)
    assert rc == -1
