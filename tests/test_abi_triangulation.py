"""psfm_triangulation_create at the C ABI: argument errors are decided on the host before any launch, so they hold on a
machine without a GPU; everything else needs the device."""
import ctypes as C

import numpy as np
import pytest

from oracle import triangulation_oracle as to
from particlesfm_b200 import _abi, _lib, device_count, init_geometry, launch_count
from test_oracle_triangulation import micro


def _db():
    db, _ = micro(np.array([[0.1, 0.0, 0.2], [0.0, 0.3, -0.1]]), [[0, 1, 2], [0, 1, 2]], 3)
    return db


def _call(db, opts=None):
    i32, i64, u8 = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint8)
    a = {k: np.ascontiguousarray(v) for k, v in db.items()}
    kp_ptr = a["keypoint_ptr"].astype(np.int64)
    kps = a["keypoints"].astype(np.float32)
    cam_of, size = a["image_camera"].astype(np.int32), a["camera_size"].astype(np.int32)
    cams, pairs = a["cameras"].astype(np.float64), a["pair_images"].astype(np.int32)
    iptr, m = a["inlier_ptr"].astype(np.int64), a["inlier_matches"].astype(np.uint32)
    q, t, reg = a["orientations"].astype(np.float64), a["image_tvec"].astype(np.float64), a["registered"].astype(np.uint8)
    h, P, E = C.c_void_p(), C.c_int64(), C.c_int64()
    rc = _lib.lib().psfm_triangulation_create(
        len(kp_ptr) - 1, kp_ptr.ctypes.data_as(i64), kps.ctypes.data_as(C.POINTER(C.c_float)), cam_of.ctypes.data_as(i32),
        _lib.dptr(cams), len(cams), size.ctypes.data_as(i32), len(pairs), pairs.ctypes.data_as(i32),
        iptr.ctypes.data_as(i64), m.ctypes.data_as(C.POINTER(C.c_uint32)), None, _lib.dptr(q), _lib.dptr(t),
        reg.ctypes.data_as(u8), C.byref(opts) if opts is not None else None, C.byref(h), C.byref(P), C.byref(E))
    if h.value:
        _lib.lib().psfm_triangulation_destroy(h)
    return rc, _lib.lib().psfm_last_error().decode()


def test_default_options_match_the_header_and_recalled():
    o = _abi.TriangulatorOptions()
    _lib.lib().psfm_triangulator_default_options(C.byref(o))
    py = init_geometry.IncrementalTriangulatorOptions(min_angle=3.0).to_struct()
    for name, _ in _abi.TriangulatorOptions._fields_:
        assert getattr(o, name) == to.DEFAULTS[name], name
        assert getattr(py, name) == (3.0 if name == "min_angle" else to.DEFAULTS[name]), name
    assert to.RECALLED["max_num_trials"] == 10000 and to.RECALLED["confidence"] == 0.9999
    # the recalled constants of the library are the oracle's (csrc/triangulation_recalled.cuh)
    import os
    src = open(os.path.join(os.path.dirname(_lib.__file__), "csrc", "triangulation_recalled.cuh")).read()
    for name, value in (("kConfidence", "0.9999"), ("kMinInlierRatio", "0.02"), ("kMaxNumTrials", "10000"),
                        ("kExhaustiveSamplingThreshold", "15"), ("kDynNumTrialsMultiplier", "3.0"),
                        ("kCapNumSamples", "100000"), ("kMaxNumLocalTrials", "10"), ("kMinNumSamples", "2")):
        assert (name + " = " + value + ";") in src, name


def _bad(name):
    db = _db()
    if name == "image index":
        db["pair_images"] = np.array([[0, 1], [0, 3], [1, 2]])
    elif name == "camera index":
        db["image_camera"] = np.array([0, 1, 0])
    elif name == "keypoint index":
        db["inlier_matches"] = db["inlier_matches"].copy()
        db["inlier_matches"][0, 0] = 7
    elif name == "with itself":
        db["pair_images"] = np.array([[0, 1], [1, 1], [1, 2]])
    elif name == "listed twice":
        db["pair_images"] = np.array([[0, 1], [1, 0], [1, 2]])
    elif name == "non-finite pose":
        db["image_tvec"] = db["image_tvec"].copy()
        db["image_tvec"][1, 0] = np.nan
    elif name == "camera size":
        db["camera_size"] = np.array([[640, 0]])
    return db


@pytest.mark.parametrize("why", ["image index", "camera index", "keypoint index", "with itself", "listed twice",
                                 "non-finite pose", "camera size"])
def test_bad_arguments_are_invalid_before_any_launch(why):
    n0 = launch_count()
    rc, msg = _call(_bad(why))
    assert rc == _abi.PSFM_ERR_INVALID, msg
    assert why in msg and msg.startswith("psfm_triangulation_create:")
    assert launch_count() == n0


def test_an_unregistered_image_may_have_a_non_finite_pose():
    db = _bad("non-finite pose")
    db["registered"] = np.array([1, 0, 1], bool)
    rc, msg = _call(db)
    assert rc in (_abi.PSFM_OK, _abi.PSFM_ERR_NO_DEVICE), msg


def test_options_check_and_unsupported_transitivity():
    o = init_geometry.IncrementalTriangulatorOptions(min_angle=0.0).to_struct()
    n0 = launch_count()
    assert _call(_db(), o)[0] == _abi.PSFM_ERR_INVALID
    o = init_geometry.IncrementalTriangulatorOptions(max_transitivity=2).to_struct()
    rc, msg = _call(_db(), o)
    assert rc == _abi.PSFM_ERR_UNSUPPORTED and "max_transitivity" in msg
    assert launch_count() == n0


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_no_device_is_refused():
    rc, msg = _call(_db())
    assert rc == _abi.PSFM_ERR_NO_DEVICE and "no CUDA device" in msg
    with pytest.raises(_lib.PsfmError):
        init_geometry.triangulate_all_points(**_db())
