"""psfm_estimate_global_positions and psfm_optimize_pairwise_translations at the C ABI: argument errors are decided on
the host before any launch, so they hold on a machine without a GPU; everything else needs the device."""
import ctypes as C

import numpy as np
import pytest

from oracle import position_oracle as po
from particlesfm_b200 import _abi, _lib, init_geometry, launch_count

PAIRS = np.array([[0, 1], [1, 2], [2, 3]], np.int32)
TVEC = np.tile([1.0, 0.0, 0.0], (3, 1))
ORIENT = np.tile([1.0, 0.0, 0.0, 0.0], (4, 1))


def _call(num_images=4, pairs=PAIRS, tvec=TVEC, orient=ORIENT, has_orientation=None, pair_used=None, opts=None):
    pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    t = np.ascontiguousarray(tvec, np.float64).reshape(-1, 3)
    q = np.ascontiguousarray(orient, np.float64).reshape(-1, 4)
    F = max(num_images, 1)
    pos, tv, has, sc = np.zeros((F, 3)), np.zeros((F, 3)), np.zeros(F, np.uint8), np.zeros(max(R, 1))
    u8 = C.POINTER(C.c_uint8)
    mask = lambda m: None if m is None else np.ascontiguousarray(m, np.uint8).ctypes.data_as(u8)
    s = _abi.PositionSummary()
    rc = _lib.lib().psfm_estimate_global_positions(
        num_images, R, pairs.ctypes.data_as(C.POINTER(C.c_int32)), _lib.dptr(t), _lib.dptr(q), mask(has_orientation),
        mask(pair_used), C.byref(opts) if opts is not None else None, _lib.dptr(pos), has.ctypes.data_as(u8),
        _lib.dptr(tv), _lib.dptr(sc), C.byref(s))
    return rc, _lib.lib().psfm_last_error().decode()


def test_default_options_match_recalled():
    o = _abi.LudOptions()
    _lib.lib().psfm_lud_default_options(C.byref(o))
    py = init_geometry.ConstrainedL1SolverOptions(rho=3.0).to_struct()
    for name, _ in _abi.LudOptions._fields_:
        assert getattr(o, name) == po.RECALLED[name], name
        assert getattr(py, name) == (3.0 if name == "rho" else po.RECALLED[name]), name


@pytest.mark.parametrize("change, why", [
    (dict(pair_used=np.zeros(3)), "no used image pair"),
    (dict(pairs=np.array([[0, 1], [1, 2], [2, 4]])), "outside"),
    (dict(pairs=np.array([[0, 1], [1, 2], [-1, 3]])), "outside"),
    (dict(pairs=np.array([[0, 1], [1, 1], [2, 3]])), "with itself"),
    (dict(pairs=np.array([[0, 1], [1, 0], [2, 3]])), "listed twice"),
    (dict(has_orientation=np.array([1, 1, 0, 1])), "no orientation"),
    (dict(orient=np.array([[1.0, 0, 0, 0]] * 3 + [[np.nan, 0, 0, 0]])), "non-finite orientation"),
    (dict(tvec=np.array([[1.0, 0, 0], [np.inf, 0, 0], [1.0, 0, 0]])), "non-finite pair tvec"),
    (dict(pairs=np.array([[0, 1], [2, 3], [0, 2]]), pair_used=np.array([1, 1, 0])), "connected"),
])
def test_bad_arguments_are_invalid_before_any_launch(change, why):
    n0 = launch_count()
    rc, msg = _call(**change)
    assert rc == _abi.PSFM_ERR_INVALID
    assert why in msg and msg.startswith("psfm_estimate_global_positions:")
    assert launch_count() == n0


@pytest.mark.parametrize("field, value", [("max_num_iterations", 0), ("rho", 0.0), ("alpha", 0.0), ("alpha", 2.0),
                                          ("absolute_tolerance", 0.0), ("relative_tolerance", -1.0)])
def test_each_check_violation_is_invalid(field, value):
    o = _abi.LudOptions()
    _lib.lib().psfm_lud_default_options(C.byref(o))
    setattr(o, field, value)
    n0 = launch_count()
    rc, msg = _call(opts=o)
    assert rc == _abi.PSFM_ERR_INVALID and "Check()" in msg
    assert launch_count() == n0


def test_too_many_views_are_unsupported_before_any_launch():
    F = 2732
    pairs = np.stack([np.arange(F - 1), np.arange(1, F)], 1)
    n0 = launch_count()
    rc, msg = _call(F, pairs, np.tile([1.0, 0, 0], (F - 1, 1)), np.tile([1.0, 0, 0, 0], (F, 1)))
    assert rc == _abi.PSFM_ERR_UNSUPPORTED and "2731" in msg
    assert launch_count() == n0


def _pairwise(kp_ptr, match):
    kps = np.zeros((int(kp_ptr[-1]), 2), np.float32)
    q = np.tile([1.0, 0, 0, 0], (2, 1))
    out, its = np.zeros((1, 3)), np.zeros(1, np.int32)
    i64, i32 = C.POINTER(C.c_int64), C.POINTER(C.c_int32)
    kp = np.ascontiguousarray(kp_ptr, np.int64)
    m = np.ascontiguousarray(match, np.uint32).reshape(-1, 2)
    pairs, cam_of, iptr = np.array([[0, 1]], np.int32), np.zeros(2, np.int32), np.array([0, len(m)], np.int64)
    cams = np.array([[500.0, 10.0, 10.0]])
    rc = _lib.lib().psfm_optimize_pairwise_translations(
        2, kp.ctypes.data_as(i64), kps.ctypes.data_as(C.POINTER(C.c_float)), cam_of.ctypes.data_as(i32), _lib.dptr(cams),
        1, 1, pairs.ctypes.data_as(i32), iptr.ctypes.data_as(i64), m.ctypes.data_as(C.POINTER(C.c_uint32)), _lib.dptr(q),
        None, _lib.dptr(out), its.ctypes.data_as(i32))
    return rc, _lib.lib().psfm_last_error().decode()


def test_pairwise_keypoint_out_of_range_is_invalid_before_any_launch():
    n0 = launch_count()
    rc, msg = _pairwise([0, 3, 5], [[0, 0], [2, 2]])
    assert rc == _abi.PSFM_ERR_INVALID and "keypoint index" in msg and msg.startswith("psfm_optimize_pairwise_translations:")
    assert launch_count() == n0


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_no_cpu_fallback_of_position_estimation():
    assert _call()[0] == _abi.PSFM_ERR_NO_DEVICE
    assert _pairwise([0, 3, 5], [[0, 0], [2, 1]])[0] == _abi.PSFM_ERR_NO_DEVICE
    with pytest.raises(_lib.PsfmError):
        init_geometry.estimate_global_positions(4, PAIRS, TVEC, ORIENT)
