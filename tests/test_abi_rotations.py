"""psfm_estimate_global_rotations at the C ABI: argument errors and the no-pair failure are decided on the host
before any launch, so they hold on a machine without a GPU; everything else needs the device."""
import ctypes as C

import numpy as np
import pytest

from particlesfm_b200 import _abi, _lib, init_geometry, launch_count

PAIRS = np.array([[0, 1], [1, 2], [0, 2]], np.int32)
QVEC = np.tile([1.0, 0.0, 0.0, 0.0], (3, 1))
NC = np.array([10, 10, 10], np.int32)


def _call(num_images=3, pairs=PAIRS, qvec=QVEC, nc=NC, has_pose=None, opts=None):
    pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
    R = pairs.shape[0]
    q = np.ascontiguousarray(qvec, np.float64).reshape(-1, 4)
    nc = np.ascontiguousarray(nc, np.int32)
    out = np.zeros((max(num_images, 1), 4))
    has_o, kept = np.zeros(max(num_images, 1), np.uint8), np.zeros(max(R, 1), np.uint8)
    s = _abi.RotationSummary()
    u8, i32 = C.POINTER(C.c_uint8), C.POINTER(C.c_int32)
    hp = None if has_pose is None else np.ascontiguousarray(has_pose, np.uint8).ctypes.data_as(u8)
    rc = _lib.lib().psfm_estimate_global_rotations(
        num_images, R, pairs.ctypes.data_as(i32), _lib.dptr(q), nc.ctypes.data_as(i32), hp,
        C.byref(opts) if opts is not None else None, _lib.dptr(out), has_o.ctypes.data_as(u8), kept.ctypes.data_as(u8),
        C.byref(s))
    return rc, s


def test_default_options_match_the_reference():
    o = _abi.RotationOptions()
    _lib.lib().psfm_rotation_default_options(C.byref(o))
    py = init_geometry.RobustRotationEstimatorOptions()
    for name, _ in _abi.RotationOptions._fields_:
        assert getattr(o, name) == pytest.approx(getattr(py, name), rel=1e-15), name
    assert o.irls_loss_parameter_sigma == np.deg2rad(5.0)


@pytest.mark.parametrize("pairs, why", [
    (np.array([[0, 3]]), "an image index is outside"),
    (np.array([[-1, 0]]), "an image index is outside"),
    (np.array([[1, 1]]), "with itself"),
    (np.array([[0, 1], [1, 0]]), "listed twice"),
])
def test_bad_pairs_are_invalid_before_any_launch(pairs, why):
    n0 = launch_count()
    rc, _ = _call(pairs=pairs, qvec=np.tile([1.0, 0, 0, 0], (len(pairs), 1)), nc=np.ones(len(pairs), np.int32))
    assert rc == _abi.PSFM_ERR_INVALID
    assert why in _lib.lib().psfm_last_error().decode()
    assert launch_count() == n0


@pytest.mark.parametrize("field", [n for n, _ in _abi.RotationOptions._fields_])
def test_each_check_violation_is_invalid(field):
    o = _abi.RotationOptions()
    _lib.lib().psfm_rotation_default_options(C.byref(o))
    setattr(o, field, 0)
    rc, _ = _call(opts=o)
    assert rc == -1 and "Check()" in _lib.lib().psfm_last_error().decode()


def test_too_many_l1_rounds_are_unsupported():
    o = _abi.RotationOptions()
    _lib.lib().psfm_rotation_default_options(C.byref(o))
    o.max_num_l1_iterations = _abi.ROTATION_MAX_L1_ROUNDS + 1
    assert _call(opts=o)[0] == -4


@pytest.mark.parametrize("case", ["no pairs", "none posed", "nan qvec"])
def test_no_posed_pair_fails_without_a_launch(case):
    n0 = launch_count()
    if case == "no pairs":
        rc, s = _call(pairs=np.zeros((0, 2)), qvec=np.zeros((0, 4)), nc=np.zeros(0))
    elif case == "none posed":
        rc, s = _call(has_pose=np.zeros(3))
    else:
        rc, s = _call(qvec=np.full((3, 4), np.nan))
    assert rc == _abi.NO_ROTATIONS
    assert s.num_l1_rounds == 0 and s.gauge_image == -1 and s.num_launches == 0
    assert launch_count() == n0
    r = init_geometry.estimate_global_rotations(3, np.zeros((0, 2)), np.zeros((0, 4)), np.zeros(0))
    assert not r.success and not r.has_orientation.any()


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_no_cpu_fallback_of_rotation_averaging():
    assert _call()[0] == -2
    with pytest.raises(_lib.PsfmError):
        init_geometry.estimate_global_rotations(3, PAIRS, QVEC, NC)
