"""The C-ABI library loads on a machine without a GPU, exports every symbol that
include/psfm_b200.h declares, and fails loudly (no CPU fallback) when asked to compute."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from particlesfm_b200 import _abi, _lib, synthetic as syn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_exported():
    hdr = open(os.path.join(ROOT, "include", "psfm_b200.h")).read()
    declared = set(re.findall(r"\b(psfm_[a-z_]+)\s*\(", hdr))
    L = _lib.lib()
    assert declared, "no declarations parsed"
    for name in sorted(declared):
        assert hasattr(L, name), f"{name} declared in psfm_b200.h but not exported"
    assert set(_lib.EXPORTS) == declared
    assert L.psfm_abi_version() == 2


def test_struct_layouts_match_defaults():
    L = _lib.lib()
    o = _abi.BAOptions()
    L.psfm_ba_global_options(C.byref(o))
    # controllers/global_mapper.cc:41-71
    assert (o.function_tolerance, o.gradient_tolerance, o.parameter_tolerance) == (1e-6, 1.0, 1e-8)
    assert (o.max_num_iterations, o.max_linear_solver_iterations) == (50, 100)
    assert o.loss_function_type == _abi.LOSS_SOFT_L1 and o.refine_rotation == 0 and o.refine_focal_length == 0
    assert o.max_num_consecutive_invalid_steps == 10 and o.jacobi_scaling == 1 and o.eta == 0.1
    t = _abi.TrajOptions()
    L.psfm_traj_default_options(C.byref(t))
    # trajectory_optimize.cpp:74-79 + Ceres defaults
    assert t.max_num_iterations == 200 and t.function_tolerance == 1e-6 and t.gradient_tolerance == 1e-10
    assert t.parameter_tolerance == 1e-8 and t.initial_trust_region_radius == 1e4


def test_oracle_and_product_defaults_agree():
    import oracle
    a, b = _abi.BAOptions(), _abi.BAOptions()
    _lib.lib().psfm_ba_global_options(C.byref(a))
    oracle.lib().psfm_oracle_ba_global_options(C.byref(b))
    b.exact_r_tolerance = a.exact_r_tolerance
    assert bytes(a) == bytes(b)
    ta, tb = _abi.TrajOptions(), _abi.TrajOptions()
    _lib.lib().psfm_traj_default_options(C.byref(ta))
    oracle.lib().psfm_oracle_traj_default_options(C.byref(tb))
    assert bytes(ta) == bytes(tb)


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_no_cpu_fallback():
    from particlesfm_b200 import ba, traj
    uv12, r1, r2, sc, f12 = syn.make_traj_inputs(10, 32, 32, seed=0)
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        traj.optimize_location(uv12, r1, r2, sc, f12, 10, 32, 32)
    prob, _ = syn.make_ba_problem(3, 10, 2, seed=0)
    o = _abi.BAOptions()
    _lib.lib().psfm_ba_global_options(C.byref(o))
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        ba.solve_problem(prob, o)


def _dense_chol_entries(A, b, ns, nb, bw, max_ctas, only=None):
    """The three dense-Cholesky test entries (those named in `only`, default all) on the same arguments: (name,
    status, psfm_last_error).  The outputs are sized for A; a call with a larger ns must be refused before it reads
    or writes anything."""
    L = _lib.lib()
    m = max(A.shape[0] if A is not None else ns, 1)
    x, X3, Xi = np.zeros(m), np.zeros((m, 3)), np.zeros((m, m))
    B = None if b is None else np.ascontiguousarray(np.repeat(b[:, None], 3, axis=1))
    out = []
    for name, call in (
            ("psfm_blocked_cholesky_solve",
             lambda: L.psfm_blocked_cholesky_solve(_lib.dptr(A), _lib.dptr(b), ns, nb, bw, max_ctas, _lib.dptr(x))),
            ("psfm_laplacian_solve", lambda: L.psfm_laplacian_solve(_lib.dptr(A), _lib.dptr(B), ns, _lib.dptr(X3))),
            ("psfm_spd_inverse", lambda: L.psfm_spd_inverse(_lib.dptr(A), ns, _lib.dptr(Xi)))):
        if only is None or name in only:
            rc = call()
            out.append((name, rc, L.psfm_last_error().decode()))
    return out


# (change to the good arguments A = I4, b = 1, ns = nb = bw = 4, max_ctas = 0; the entries that must refuse it)
DENSE_CHOL_BAD = {
    "null_A": (dict(A=None), {"psfm_blocked_cholesky_solve", "psfm_laplacian_solve", "psfm_spd_inverse"}),
    "null_b": (dict(b=None), {"psfm_blocked_cholesky_solve", "psfm_laplacian_solve"}),
    "n0": (dict(ns=0, nb=0), {"psfm_blocked_cholesky_solve", "psfm_laplacian_solve", "psfm_spd_inverse"}),
    "nb0": (dict(nb=0), {"psfm_blocked_cholesky_solve"}),
    "nb_above_ns": (dict(nb=5), {"psfm_blocked_cholesky_solve"}),
    "bw_negative": (dict(bw=-1), {"psfm_blocked_cholesky_solve"}),
    "max_ctas_negative": (dict(max_ctas=-1), {"psfm_blocked_cholesky_solve"}),
    # above the position stage's 8,190 unknowns, the rotation stage's 8,191, and the solver entry's 32,767
    "n8191": (dict(ns=8191, nb=8191, bw=8191), {"psfm_spd_inverse"}),
    "n8192": (dict(ns=8192, nb=8192, bw=8192), {"psfm_laplacian_solve", "psfm_spd_inverse"}),
    "n32768": (dict(ns=32768, nb=32768, bw=32768),
               {"psfm_blocked_cholesky_solve", "psfm_laplacian_solve", "psfm_spd_inverse"}),
}


@pytest.mark.parametrize("case", list(DENSE_CHOL_BAD))
def test_dense_chol_entries_check_arguments_before_the_device(case):
    """Bad arguments are PSFM_ERR_INVALID, named in psfm_last_error, on any machine and before any launch."""
    args = dict(A=np.eye(4), b=np.ones(4), ns=4, nb=4, bw=4, max_ctas=0)
    change, refused = DENSE_CHOL_BAD[case]
    args.update(change)
    n0 = _lib.lib().psfm_launch_count()
    too_large = case in ("n8191", "n8192", "n32768")       # only the entries that must refuse the size are called
    for name, rc, msg in _dense_chol_entries(**args, only=refused if too_large else None):
        if name in refused:
            assert rc == _abi.PSFM_ERR_INVALID and msg.startswith(name + ":"), (name, rc, msg)
        else:
            assert rc in (_abi.PSFM_OK, _abi.PSFM_ERR_NO_DEVICE), (name, rc, msg)
    if _lib.lib().psfm_device_count() == 0:
        assert _lib.lib().psfm_launch_count() == n0


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_no_cpu_fallback_of_the_dense_chol_entries():
    for name, rc, msg in _dense_chol_entries(np.eye(4), np.ones(4), 4, 4, 4, 0):
        assert rc == _abi.PSFM_ERR_NO_DEVICE and "no CUDA device" in msg, (name, rc, msg)
    for name, rc, msg in _dense_chol_entries(np.eye(40), np.ones(40), 40, 37, 5, 2):      # the band route too
        if name == "psfm_blocked_cholesky_solve":
            assert rc == _abi.PSFM_ERR_NO_DEVICE, (rc, msg)


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_no_cpu_fallback_of_the_initialisation_ops():
    """SURVEY.md 8(f) f-4 ops: host-side argument checks come first, then the library refuses without a device."""
    import numpy as np
    from particlesfm_b200 import init_geometry as ig
    p = np.zeros((5, 2))
    q = np.array([1.0, 0.0, 0.0, 0.0])
    with pytest.raises(ValueError):
        ig.batch_optimize_relative_position_with_known_rotation([(p, p[:-1], q, q)])
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        ig.optimize_relative_position_with_known_rotation(p, p, q, q)
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        ig.triangulate_multi_view_points([(np.zeros((2, 3, 4)), np.zeros((2, 2)))])
    assert ig.batch_optimize_relative_position_with_known_rotation([]).shape == (0, 3)      # nothing to do: no device needed
    assert ig.triangulate_multi_view_points([]).shape == (0, 3)


def _null_vector_entries(form=0, A=np.eye(3), count=1, kind=0, n=8, best=np.eye(3).reshape(9), thr=16.0,
                         points=np.zeros((8, 4), np.float32), out=True, only=None):
    """The null-vector and minimal-solver test entries on the same kind of arguments: (name, status,
    psfm_last_error).  The outputs are sized for one good call; a call with more is refused before it reads or writes
    anything."""
    L = _lib.lib()
    o = np.zeros(171) if out else None
    v, T, m = (np.zeros(9), np.zeros(6), np.zeros(9)) if out else (None, None, None)
    nums = np.zeros(1, np.int32)
    num = nums.ctypes.data_as(C.POINTER(C.c_int32)) if out else None
    pts = None if points is None else points.ctypes.data_as(C.POINTER(C.c_float))
    res = []
    for name, call in (("psfm_null_vectors", lambda: L.psfm_null_vectors(form, _lib.dptr(A), count, _lib.dptr(o))),
                       ("psfm_verification_local_model",
                        lambda: L.psfm_verification_local_model(kind, pts, n, _lib.dptr(best), thr, _lib.dptr(v),
                                                                _lib.dptr(T), _lib.dptr(m))),
                       ("psfm_verification_minimal",
                        lambda: L.psfm_verification_minimal(kind, pts, count, _lib.dptr(o), num)),
                       ("psfm_verification_cubic", lambda: L.psfm_verification_cubic(_lib.dptr(A), count, _lib.dptr(o), num))):
        if only is None or name in only:
            rc = call()
            res.append((name, rc, L.psfm_last_error().decode()))
    return res


NULL_VECTOR_BAD = {
    "null_input": (dict(A=None, points=None), {"psfm_null_vectors", "psfm_verification_local_model",
                                               "psfm_verification_minimal", "psfm_verification_cubic"}),
    "null_output": (dict(out=False), {"psfm_null_vectors", "psfm_verification_local_model", "psfm_verification_minimal",
                                      "psfm_verification_cubic"}),
    "null_best": (dict(best=None), {"psfm_verification_local_model"}),
    "form_negative": (dict(form=-1), {"psfm_null_vectors"}),
    "form_unknown": (dict(form=6), {"psfm_null_vectors"}),
    "count0": (dict(count=0), {"psfm_null_vectors", "psfm_verification_minimal", "psfm_verification_cubic"}),
    "count_above_2e24": (dict(count=(1 << 24) + 1), {"psfm_null_vectors", "psfm_verification_minimal",
                                                      "psfm_verification_cubic"}),
    "kind_negative": (dict(kind=-1), {"psfm_verification_local_model", "psfm_verification_minimal"}),
    "kind_watermark": (dict(kind=2), {"psfm_verification_local_model", "psfm_verification_minimal"}),
    "n0": (dict(n=0), {"psfm_verification_local_model"}),
    "n2e31": (dict(n=1 << 31), {"psfm_verification_local_model"}),
    "threshold_negative": (dict(thr=-1.0), {"psfm_verification_local_model"}),
    "threshold_nan": (dict(thr=float("nan")), {"psfm_verification_local_model"}),
}


@pytest.mark.parametrize("case", list(NULL_VECTOR_BAD))
def test_null_vector_entries_check_arguments_before_the_device(case):
    """Bad arguments are PSFM_ERR_INVALID, named in psfm_last_error, on any machine and before any launch."""
    change, refused = NULL_VECTOR_BAD[case]
    n0 = _lib.lib().psfm_launch_count()
    for name, rc, msg in _null_vector_entries(**change, only=refused):
        assert rc == _abi.PSFM_ERR_INVALID and msg.startswith(name + ":"), (name, rc, msg)
    if _lib.lib().psfm_device_count() == 0:
        assert _lib.lib().psfm_launch_count() == n0


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_no_cpu_fallback_of_the_null_vector_entries():
    for name, rc, msg in _null_vector_entries():
        assert rc == _abi.PSFM_ERR_NO_DEVICE and "no CUDA device" in msg, (name, rc, msg)
    for form in range(6):
        A = np.zeros((1, 81))
        name, rc, msg = _null_vector_entries(form=form, A=A, only={"psfm_null_vectors"})[0]
        assert rc == _abi.PSFM_ERR_NO_DEVICE, (form, rc, msg)
