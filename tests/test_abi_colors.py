"""psfm_colors_create / psfm_colors_add_images at the C ABI and the host checks of particlesfm_b200.colors: every bad
argument is refused before any launch.  The create refusals and the Python layer's hold without a GPU; the
add_images refusals need a handle, so they run on the device."""
import ctypes as C

import numpy as np
import pytest

from particlesfm_b200 import _abi, _lib, colors, device_count, launch_count

i64p, ip, u8p = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)


def _create(ptr, kp, rows, P):
    ptr = np.ascontiguousarray(ptr, np.int64)
    kp, rows = np.ascontiguousarray(kp, np.float64), np.ascontiguousarray(rows, np.int32)
    h = C.c_void_p()
    rc = _lib.lib().psfm_colors_create(len(ptr) - 1, ptr.ctypes.data_as(i64p), _lib.dptr(kp), rows.ctypes.data_as(ip),
                                       P, C.byref(h), None)
    return rc, h


def _model():
    return np.array([0, 3, 5, 8]), np.arange(16, dtype=np.float64).reshape(8, 2), np.array([0, -1, 2, 1, 0, -1, 2, 3])


@pytest.mark.parametrize("why", ["point row", "point row below -1", "keypoint_ptr", "keypoint_ptr start"])
def test_create_refusals_are_invalid_before_any_launch(why):
    ptr, kp, rows = _model()
    if why == "point row":
        rows[4] = 4
    elif why == "point row below -1":
        rows[4] = -2
    elif why == "keypoint_ptr":
        ptr[2] = 2
    else:
        ptr[0] = 1
    n0 = launch_count()
    rc, _ = _create(ptr, kp, rows, 4)
    assert rc == _abi.PSFM_ERR_INVALID
    msg = _lib.lib().psfm_last_error().decode()
    assert why.split()[0] in msg and "psfm_colors_create" in msg, msg
    assert launch_count() == n0


def test_add_images_and_result_of_a_null_handle_are_invalid():
    L = _lib.lib()
    assert L.psfm_colors_add_images(None, 0, 0, None, None, None) == _abi.PSFM_ERR_INVALID
    assert L.psfm_colors_result(None, None, None) == _abi.PSFM_ERR_INVALID


@pytest.mark.parametrize("mode", ["I;16", "CMYK", "I", "F", "1"])
def test_unsupported_modes_are_refused_before_any_launch(tmp_path, mode):
    from PIL import Image
    (tmp_path / "sub").mkdir()
    Image.fromarray(np.full((6, 5, 3), 100, np.uint8)).save(tmp_path / "a.png")
    ext = ".tif" if mode in ("I", "F") else (".jpg" if mode == "CMYK" else ".png")
    Image.new(mode, (5, 6)).save(tmp_path / "sub" / ("b" + ext))
    ptr, kp, rows = _model()
    n0 = launch_count()
    with pytest.raises(ValueError, match=r"image 'sub/b%s'.*mode %s" % (ext.replace(".", r"\."), mode.replace(";", ";"))):
        colors.extract_colors_for_all_images(str(tmp_path), ["a.png", "sub/b" + ext, "missing.png"], ptr, kp, rows, 4)
    assert launch_count() == n0


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_no_device_is_refused(tmp_path):
    ptr, kp, rows = _model()
    rc, _ = _create(ptr, kp, rows, 4)
    assert rc == _abi.PSFM_ERR_NO_DEVICE
    assert "psfm_colors_create: no CUDA device" in _lib.lib().psfm_last_error().decode()
    with pytest.raises(_lib.PsfmError) as e:
        colors.extract_colors_for_all_images(str(tmp_path), ["a.png", "b.png", "c.png"], ptr, kp, rows, 4)
    assert e.value.code == _abi.PSFM_ERR_NO_DEVICE


def _add(h, first, sizes):
    w = np.array([s[0] for s in sizes], np.int32)
    hh = np.array([s[1] for s in sizes], np.int32)
    px = np.zeros(max(1, sum(3 * max(a, 0) * max(b, 0) for a, b in sizes)), np.uint8)
    return _lib.lib().psfm_colors_add_images(h, first, len(sizes), w.ctypes.data_as(ip), hh.ctypes.data_as(ip),
                                             px.ctypes.data_as(u8p))


@pytest.mark.gpu
@pytest.mark.parametrize("why", ["image index", "negative image index", "given twice", "zero width", "zero height"])
def test_add_images_refusals_are_invalid_before_any_launch(gpu, why):
    ptr, kp, rows = _model()
    rc, h = _create(ptr, kp, rows, 4)
    assert rc == 0
    L = _lib.lib()
    try:
        assert _add(h, 0, [(4, 3)]) == 0
        n0 = launch_count()
        if why == "image index":
            rc = _add(h, 2, [(4, 3), (4, 3)])
        elif why == "negative image index":
            rc = _add(h, -1, [(4, 3)])
        elif why == "given twice":
            rc = _add(h, 0, [(4, 3)])
        elif why == "zero width":
            rc = _add(h, 1, [(4, 3), (0, 3)])
        else:
            rc = _add(h, 1, [(4, 0)])
        assert rc == _abi.PSFM_ERR_INVALID
        msg = L.psfm_last_error().decode()
        assert ("image index" if why in ("image index", "negative image index", "given twice") else "image size") in msg, msg
        assert launch_count() == n0
        # the refused call added nothing: images 1 and 2 can still be added, and the result runs
        assert _add(h, 1, [(4, 3), (4, 3)]) == 0
        rgb = np.zeros((4, 3), np.uint8)
        assert L.psfm_colors_result(h, rgb.ctypes.data_as(u8p), None) == 0
    finally:
        L.psfm_colors_destroy(h)
