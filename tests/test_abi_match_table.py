"""The database match table's C entries refuse a missing handle or output before touching a device."""
import ctypes as C

from particlesfm_b200 import _abi, _lib


def _err():
    return _lib.lib().psfm_last_error().decode()


def test_null_handles_are_refused():
    L = _lib.lib()
    out, n = C.c_void_p(), C.c_int64()
    assert L.psfm_matches_table(None, None, C.byref(out), C.byref(n), C.byref(n), C.byref(n)) == _abi.PSFM_ERR_INVALID
    assert "psfm_matches_table" in _err() and not out.value
    assert L.psfm_match_table_result(None, None, None, None, None, None) == _abi.PSFM_ERR_INVALID
    assert "psfm_match_table_result" in _err()
    assert L.psfm_match_table_verify(None, None, 0, None, None, None, None, None, None, None, None, None, None,
                                     None) == _abi.PSFM_ERR_INVALID
    assert "psfm_match_table_verify" in _err()
    L.psfm_match_table_destroy(None)
