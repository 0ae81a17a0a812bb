"""psfm_convert_create / psfm_convert_result at the C ABI and the host checks of particlesfm_b200.convert: every bad
argument is refused on the host before any launch, so these hold on a machine without a GPU."""
import ctypes as C

import numpy as np
import pytest

from particlesfm_b200 import _abi, _lib, convert, device_count, launch_count
from test_oracle_convert import one_image, random_model

i64p, ip, u8p = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


def _create(a, budget=1 << 20):
    F = len(a["image_ids"])
    size = np.ascontiguousarray(a["camera_size"], np.int32)
    cam = np.ascontiguousarray(a["image_camera"], np.int32)
    ptr = np.ascontiguousarray(a["keypoint_ptr"], np.int64)
    q, t = np.ascontiguousarray(a["qvec"], np.float64), np.ascontiguousarray(a["tvec"], np.float64)
    kp, xyz = np.ascontiguousarray(a["keypoints"], np.float64), np.ascontiguousarray(a["xyz"], np.float64)
    row = np.ascontiguousarray(a["row"], np.int32)
    lut = convert.binary_lut()
    valid, bptr, h = np.zeros(F, np.int64), np.zeros(F + 1, np.int32), C.c_void_p()
    rc = _lib.lib().psfm_convert_create(len(size), size.ctypes.data_as(ip), F, _lib.dptr(q), _lib.dptr(t),
                                        cam.ctypes.data_as(ip), ptr.ctypes.data_as(i64p), _lib.dptr(kp),
                                        row.ctypes.data_as(ip), len(xyz), _lib.dptr(xyz), lut.ctypes.data_as(u8p), budget,
                                        C.byref(h), valid.ctypes.data_as(i64p), bptr.ctypes.data_as(ip), None)
    if rc == 0:
        _lib.lib().psfm_convert_destroy(h)
    return rc


def _args(why):
    a = random_model(3)
    a["row"] = np.where(a["point3D_ids"] >= 0, 0, -1)
    budget = 1 << 20
    if why == "camera size":
        a["camera_size"] = np.array([[64, 48], [40, 0]])
    elif why == "camera index":
        a["image_camera"] = np.array([0, 1, 2, 0])
    elif why == "point row":
        a["row"] = a["row"].copy()
        a["row"][5] = len(a["xyz"])
    elif why == "point row below -1":
        a["row"] = a["row"].copy()
        a["row"][5] = -2
    elif why == "keypoint_ptr":
        a["keypoint_ptr"] = a["keypoint_ptr"].copy()
        a["keypoint_ptr"][2] = a["keypoint_ptr"][1] - 1
    elif why == "memory_budget":
        budget = 0
    return a, budget


@pytest.mark.parametrize("why", ["camera size", "camera index", "point row", "point row below -1", "keypoint_ptr",
                                 "memory_budget"])
def test_bad_arguments_are_invalid_before_any_launch(why):
    n0 = launch_count()
    a, budget = _args(why)
    assert _create(a, budget) == _abi.PSFM_ERR_INVALID
    msg = _lib.lib().psfm_last_error().decode()
    assert why.split()[0] in msg, msg
    assert launch_count() == n0


def test_result_of_a_null_handle_is_invalid():
    assert _lib.lib().psfm_convert_result(None, 0, 0, None, None, None) == _abi.PSFM_ERR_INVALID


@pytest.mark.parametrize("why", ["path separator", "camera model", "missing point"])
def test_host_refusals_of_the_python_layer_come_before_the_library(tmp_path, why):
    a = random_model(4)
    n0 = launch_count()
    if why == "path separator":
        a["image_names"][1] = "sub/frame.jpg"
        err = ValueError
    elif why == "camera model":
        a["camera_model"] = np.array([0, 4])
        a["image_camera"] = np.array([0, 1, 1, 0])
        err = NotImplementedError
    else:
        a["point3D_ids"] = a["point3D_ids"].copy()
        a["point3D_ids"][3] = 10 ** 9
        err = KeyError
    with pytest.raises(err):
        convert.save_depth_pose_arrays(str(tmp_path / "out"), **a)
    assert launch_count() == n0 and not (tmp_path / "out").exists()


def test_text_model_and_missing_model_are_refused(tmp_path):
    for n in ("cameras", "images", "points3D"):
        (tmp_path / (n + ".txt")).write_text("")
    with pytest.raises(ValueError, match="text COLMAP model"):
        convert.write_depth_pose_from_colmap_format(str(tmp_path), str(tmp_path / "out"))
    with pytest.raises(FileNotFoundError):
        convert.write_depth_pose_from_colmap_format(str(tmp_path / "nothing"), str(tmp_path / "out"))


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_no_device_is_refused(tmp_path):
    a = one_image([[1, 1]], [2.0])
    a["row"] = np.array([0])
    assert _create(a) == _abi.PSFM_ERR_NO_DEVICE
    assert "no CUDA device" in _lib.lib().psfm_last_error().decode()
    with pytest.raises(_lib.PsfmError) as e:
        convert.save_depth_pose_arrays(str(tmp_path / "out"), **one_image([[1, 1]], [2.0]))
    assert e.value.code == _abi.PSFM_ERR_NO_DEVICE and not (tmp_path / "out").exists()
