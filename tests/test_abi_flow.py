"""The optical-flow entries of the C ABI (csrc/optical_flow.cu): bad arguments are PSFM_ERR_INVALID before any launch,
valid ones are PSFM_ERR_NO_DEVICE without a GPU."""
import ctypes as C

import pytest

from particlesfm_b200 import _abi, _lib, device_count, launch_count

P = C.c_void_p(256)        # never dereferenced: every call below is refused before the device is touched
PAD = (C.c_int32 * 4)(1, 2, 2, 3)


def _calls(L, h=16, w=17, n=2, pad=PAD, p=P):
    return {
        "psfm_corr_pyramids": lambda: L.psfm_corr_pyramids(p, p, h, w, None),
        "psfm_corr_lookup": lambda: L.psfm_corr_lookup(p, n, h, w, p, p, None),
        "psfm_flow_upsample": lambda: L.psfm_flow_upsample(p, p, n, h, w, pad, p, None),
        "psfm_flow_to_image": lambda: L.psfm_flow_to_image(p, n, h, w, p, None),
    }


@pytest.mark.parametrize("entry", ["psfm_corr_pyramids", "psfm_corr_lookup", "psfm_flow_upsample", "psfm_flow_to_image"])
@pytest.mark.parametrize("why", ["null", "size", "count", "pad"])
def test_bad_arguments_are_invalid_before_any_launch(entry, why):
    L = _lib.lib()
    if why == "null":
        call = _calls(L, p=None)[entry]
    elif why == "size":
        call = _calls(L, h=0 if entry in ("psfm_flow_upsample", "psfm_flow_to_image") else 7)[entry]
    elif why == "count":
        if entry == "psfm_corr_pyramids":
            pytest.skip("one pair per call")
        call = _calls(L, n=0)[entry]
    else:
        if entry != "psfm_flow_upsample":
            pytest.skip("no padding argument")
        call = _calls(L, pad=(C.c_int32 * 4)(1, 8, 0, 0))[entry]
    n0 = launch_count()
    assert call() == _abi.PSFM_ERR_INVALID
    assert entry in L.psfm_last_error().decode()
    assert launch_count() == n0


def test_pyramid_size():
    L = _lib.lib()
    assert L.psfm_corr_pyramid_floats(16, 17) == 272 * (16 * 17 + 8 * 8 + 4 * 4 + 2 * 2)
    assert L.psfm_corr_pyramid_floats(7, 17) == _abi.PSFM_ERR_INVALID


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
@pytest.mark.parametrize("entry", ["psfm_corr_pyramids", "psfm_corr_lookup", "psfm_flow_upsample", "psfm_flow_to_image"])
def test_no_device_is_refused(entry):
    L = _lib.lib()
    assert _calls(L)[entry]() == _abi.PSFM_ERR_NO_DEVICE
    assert "%s: no CUDA device" % entry in L.psfm_last_error().decode()
