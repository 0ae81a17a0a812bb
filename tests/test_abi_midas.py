"""The depth entries of the C ABI (csrc/midas.cu): bad arguments are PSFM_ERR_INVALID before any launch, valid ones are
PSFM_ERR_NO_DEVICE without a GPU."""
import ctypes as C

import pytest

from particlesfm_b200 import _abi, _lib, device_count, launch_count

P = C.c_void_p(256)        # never dereferenced: every call below is refused before the device is touched
ENTRIES = ["psfm_depth_prepare", "psfm_depth_upsample", "psfm_depth_quantize"]


def _calls(L, h=40, w=192, n=2, net=(64, 384), half=0, p=P):
    return {
        "psfm_depth_prepare": lambda: L.psfm_depth_prepare(p, n, h, w, net[0], net[1], half, p, None),
        "psfm_depth_upsample": lambda: L.psfm_depth_upsample(p, n, net[0], net[1], half, h, w, p, p, None),
        "psfm_depth_quantize": lambda: L.psfm_depth_quantize(p, n, h, w, p, p, None),
    }


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("why", ["null", "size", "count", "net", "half"])
def test_bad_arguments_are_invalid_before_any_launch(entry, why):
    L = _lib.lib()
    if why == "null":
        call = _calls(L, p=None)[entry]
    elif why == "size":
        call = _calls(L, h=0)[entry]
    elif why == "count":
        call = _calls(L, n=0)[entry]
    elif why == "net":
        if entry == "psfm_depth_quantize":
            pytest.skip("no network size")
        call = _calls(L, net=(64, 0))[entry]
    else:
        if entry == "psfm_depth_quantize":
            pytest.skip("float32 maps only")
        call = _calls(L, half=2)[entry]
    n0 = launch_count()
    assert call() == _abi.PSFM_ERR_INVALID
    assert entry in L.psfm_last_error().decode()
    assert launch_count() == n0


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
@pytest.mark.parametrize("entry", ENTRIES)
def test_no_device_is_refused(entry):
    L = _lib.lib()
    assert _calls(L)[entry]() == _abi.PSFM_ERR_NO_DEVICE
    assert "%s: no CUDA device" % entry in L.psfm_last_error().decode()
