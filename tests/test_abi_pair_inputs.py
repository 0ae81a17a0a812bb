"""The image-pair graph checks the pair stages share (csrc/pair_inputs.cu), at the C ABI.  Every check runs on the host
before the device check and before any launch, so these hold on a machine without a GPU: for each stage and each
shared fault it checks, the status and the full psfm_last_error text, and no launch.  Without a device, every entry
point that needs no handle refuses with PSFM_ERR_NO_DEVICE and a message that starts with its own name."""
import ctypes as C

import numpy as np
import pytest

from particlesfm_b200 import _abi, _lib, device_count, launch_count

i32p, i64p, u8p, u32p = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint8), C.POINTER(C.c_uint32)


def _graph():
    """Three images of one camera with 4, 5 and 6 keypoints, pairs (0, 1) and (1, 2) with 3 and 2 matches."""
    return dict(num_images=3, num_pairs=2,
                keypoint_ptr=np.array([0, 4, 9, 15], np.int64),
                keypoints=np.arange(30, dtype=np.float32).reshape(15, 2),
                image_camera=np.zeros(3, np.int32),
                cameras=np.array([[500.0, 320.0, 240.0]]),
                camera_size=np.array([[640, 480]], np.int32),
                pair_images=np.array([[0, 1], [1, 2]], np.int32),
                ptr=np.array([0, 3, 5], np.int64),
                matches=np.array([[0, 1], [1, 2], [3, 4], [4, 5], [2, 0]], np.uint32))


def _c(a, dtype):
    return np.ascontiguousarray(a, dtype)


def _two_view(g):
    R = len(g["pair_images"])
    out = [np.zeros((R, 4)), np.zeros((R, 3)), np.zeros(R), np.zeros(R, np.int32), np.zeros(R, np.int64), np.zeros(R, np.uint8)]
    E = np.tile(np.eye(3).reshape(1, 9), (R, 1))
    return _lib.lib().psfm_two_view_relative_poses(
        g["num_images"], _c(g["keypoint_ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["keypoints"], np.float32).ctypes.data_as(C.POINTER(C.c_float)), _c(g["image_camera"], np.int32).ctypes.data_as(i32p),
        _lib.dptr(_c(g["cameras"], np.float64)), len(g["cameras"]), g["num_pairs"],
        _c(g["pair_images"], np.int32).ctypes.data_as(i32p), np.full(R, 2, np.int32).ctypes.data_as(i32p), _lib.dptr(E),
        _lib.dptr(E), _lib.dptr(E), _c(g["ptr"], np.int64).ctypes.data_as(i64p), _c(g["matches"], np.uint32).ctypes.data_as(u32p),
        _lib.dptr(out[0]), _lib.dptr(out[1]), _lib.dptr(out[2]), out[3].ctypes.data_as(i32p), out[4].ctypes.data_as(i64p),
        out[5].ctypes.data_as(u8p))


def _pairwise(g):
    R = len(g["pair_images"])
    q = np.tile([1.0, 0.0, 0.0, 0.0], (len(g["image_camera"]), 1))
    tvec, its = np.zeros((R, 3)), np.zeros(R, np.int32)
    return _lib.lib().psfm_optimize_pairwise_translations(
        g["num_images"], _c(g["keypoint_ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["keypoints"], np.float32).ctypes.data_as(C.POINTER(C.c_float)), _c(g["image_camera"], np.int32).ctypes.data_as(i32p),
        _lib.dptr(_c(g["cameras"], np.float64)), len(g["cameras"]), g["num_pairs"],
        _c(g["pair_images"], np.int32).ctypes.data_as(i32p), _c(g["ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["matches"], np.uint32).ctypes.data_as(u32p), _lib.dptr(q), None, _lib.dptr(tvec), its.ctypes.data_as(i32p))


def _rotations(g):
    R, F = len(g["pair_images"]), len(g["image_camera"])
    q = np.tile([1.0, 0.0, 0.0, 0.0], (R, 1))
    nc = np.full(R, 100, np.int32)
    orient, has_o, kept = np.zeros((F, 4)), np.zeros(F, np.uint8), np.zeros(R, np.uint8)
    return _lib.lib().psfm_estimate_global_rotations(
        g["num_images"], g["num_pairs"], _c(g["pair_images"], np.int32).ctypes.data_as(i32p), _lib.dptr(q),
        nc.ctypes.data_as(i32p), None, None, _lib.dptr(orient), has_o.ctypes.data_as(u8p), kept.ctypes.data_as(u8p), None)


def _positions(g):
    R, F = len(g["pair_images"]), len(g["image_camera"])
    t = np.tile([1.0, 0.0, 0.0], (R, 1))
    q = np.tile([1.0, 0.0, 0.0, 0.0], (F, 1))
    pos, has_p, tv, sc = np.zeros((F, 3)), np.zeros(F, np.uint8), np.zeros((F, 3)), np.zeros(R)
    return _lib.lib().psfm_estimate_global_positions(
        g["num_images"], g["num_pairs"], _c(g["pair_images"], np.int32).ctypes.data_as(i32p), _lib.dptr(t), _lib.dptr(q),
        None, None, None, _lib.dptr(pos), has_p.ctypes.data_as(u8p), _lib.dptr(tv), _lib.dptr(sc), None)


def _triangulation(g):
    F = len(g["image_camera"])
    q = np.tile([1.0, 0.0, 0.0, 0.0], (F, 1))
    t = np.tile([0.0, 0.0, 1.0], (F, 1)) * np.arange(F)[:, None]
    reg = np.ones(F, np.uint8)
    h, P, E = C.c_void_p(), C.c_int64(), C.c_int64()
    rc = _lib.lib().psfm_triangulation_create(
        g["num_images"], _c(g["keypoint_ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["keypoints"], np.float32).ctypes.data_as(C.POINTER(C.c_float)), _c(g["image_camera"], np.int32).ctypes.data_as(i32p),
        _lib.dptr(_c(g["cameras"], np.float64)), len(g["cameras"]), _c(g["camera_size"], np.int32).ctypes.data_as(i32p),
        g["num_pairs"], _c(g["pair_images"], np.int32).ctypes.data_as(i32p), _c(g["ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["matches"], np.uint32).ctypes.data_as(u32p), None, _lib.dptr(q), _lib.dptr(t), reg.ctypes.data_as(u8p), None,
        C.byref(h), C.byref(P), C.byref(E))
    if h.value:
        _lib.lib().psfm_triangulation_destroy(h)
    return rc


def _verification(g):
    R = len(g["pair_images"])
    config, F, E, H = np.zeros(R, np.int32), np.zeros((R, 9)), np.zeros((R, 9)), np.zeros((R, 9))
    iptr, out, trials = np.zeros(R + 1, np.int64), np.zeros((len(g["matches"]), 2), np.uint32), np.zeros((R, 3), np.int32)
    return _lib.lib().psfm_verify_two_view_geometries(
        g["num_images"], _c(g["keypoint_ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["keypoints"], np.float32).ctypes.data_as(C.POINTER(C.c_float)), _c(g["image_camera"], np.int32).ctypes.data_as(i32p),
        len(g["camera_size"]), _c(g["camera_size"], np.int32).ctypes.data_as(i32p), None, g["num_pairs"],
        _c(g["pair_images"], np.int32).ctypes.data_as(i32p), _c(g["ptr"], np.int64).ctypes.data_as(i64p),
        _c(g["matches"], np.uint32).ctypes.data_as(u32p), None, config.ctypes.data_as(i32p), _lib.dptr(F), _lib.dptr(E),
        _lib.dptr(H), iptr.ctypes.data_as(i64p), out.ctypes.data_as(u32p), trials.ctypes.data_as(i32p), None)


# entry -> (call, name of its match pointer, the shared faults it checks)
_COMMON = ["negative size", "too many pairs", "image index"]
_GRAPH = ["keypoint_ptr[0]", "keypoint_ptr order", "camera index", "ptr[0]", "ptr order", "keypoint index"]
_DISTINCT = ["with itself", "listed twice"]
STAGES = {
    "psfm_two_view_relative_poses": (_two_view, "inlier_ptr", _COMMON + _GRAPH),
    "psfm_optimize_pairwise_translations": (_pairwise, "inlier_ptr", _COMMON + _GRAPH),
    "psfm_estimate_global_rotations": (_rotations, None, _COMMON + _DISTINCT),
    "psfm_estimate_global_positions": (_positions, None, _COMMON + _DISTINCT),
    "psfm_triangulation_create": (_triangulation, "inlier_ptr", _COMMON + _GRAPH + _DISTINCT + ["camera size"]),
    "psfm_verify_two_view_geometries": (_verification, "match_ptr", _COMMON + _GRAPH + _DISTINCT + ["camera size"]),
}


def _fault(g, fault, ptr_name):
    """Apply one fault to the valid graph g; returns the message the entry point must give."""
    if fault == "negative size":
        g["num_images"] = -1
        return "negative size"
    if fault == "too many pairs":
        g["num_pairs"] = 1 << 31
        return "more than 2^31 - 1 pairs"
    if fault == "keypoint_ptr[0]":
        g["keypoint_ptr"] = np.array([1, 4, 9, 15], np.int64)
        return "keypoint_ptr[0] must be 0"
    if fault == "keypoint_ptr order":
        g["keypoint_ptr"] = np.array([0, 4, 3, 15], np.int64)
        return "keypoint_ptr must be non-decreasing"
    if fault == "camera index":
        g["image_camera"] = np.array([0, 1, 0], np.int32)
        return "a camera index is outside [0, num_cameras)"
    if fault == "camera size":
        g["camera_size"] = np.array([[640, 0]], np.int32)
        return "a camera size <= 0"
    if fault == "ptr[0]":
        g["ptr"] = np.array([1, 3, 5], np.int64)
        return ptr_name + "[0] must be 0"
    if fault == "ptr order":
        g["ptr"] = np.array([0, 3, 2], np.int64)
        return ptr_name + " must be non-decreasing"
    if fault == "image index":
        g["pair_images"] = np.array([[0, 1], [1, 3]], np.int32)
        return "an image index is outside [0, num_images)"
    if fault == "with itself":
        g["pair_images"] = np.array([[0, 1], [2, 2]], np.int32)
        return "a pair of an image with itself"
    if fault == "listed twice":
        g["pair_images"] = np.array([[0, 1], [1, 0]], np.int32)
        return "an unordered image pair is listed twice"
    assert fault == "keypoint index"
    g["matches"] = g["matches"].copy()
    g["matches"][1, 0] = 4              # image 0 has 4 keypoints
    return "a keypoint index is outside its image's keypoints"


@pytest.mark.parametrize("entry,fault", [(e, f) for e, (_, _, faults) in STAGES.items() for f in faults])
def test_a_single_fault_is_named_before_any_launch(entry, fault):
    call, ptr_name, _ = STAGES[entry]
    g = _graph()
    why = _fault(g, fault, ptr_name)
    n0 = launch_count()
    rc = call(g)
    assert (rc, _lib.lib().psfm_last_error().decode()) == (_abi.PSFM_ERR_INVALID, "%s: %s" % (entry, why))
    assert launch_count() == n0


def _raised(fn):
    """Status and psfm_last_error of a Python wrapper that raises PsfmError."""
    with pytest.raises(_lib.PsfmError) as e:
        fn()
    return e.value.code, _lib.lib().psfm_last_error().decode()


def _no_device_calls():
    from particlesfm_b200 import ba, handoff, init_geometry as ig, synthetic as syn, traj
    from test_abi import _dense_chol_entries, _null_vector_entries
    from test_abi_convert import _args, _create
    L = _lib.lib()
    calls = {name: (lambda c=call: (c(_graph()), L.psfm_last_error().decode())) for name, (call, _, _) in STAGES.items()}

    def ba_solve():
        prob, _ = syn.make_ba_problem(3, 10, 2, seed=0)
        o = _abi.BAOptions()
        L.psfm_ba_global_options(C.byref(o))
        return _raised(lambda: ba.solve_problem(prob, o))

    def traj_optimize():
        uv12, r1, r2, sc, f12 = syn.make_traj_inputs(10, 32, 32, seed=0)
        return _raised(lambda: traj.optimize_location(uv12, r1, r2, sc, f12, 10, 32, 32))

    def known_rotation():
        p, q = np.zeros((5, 2)), np.array([1.0, 0.0, 0.0, 0.0])
        return _raised(lambda: ig.optimize_relative_position_with_known_rotation(p, p, q, q))

    def matches_create():
        tracks = syn.make_track_arrays(50, 10, 300, seed=4)
        return _raised(lambda: handoff.traj_to_matches_device(tracks, 10))

    def tracker_create():
        h = C.c_void_p()
        return L.psfm_tracker_create(36, 52, 2, 7, None, C.byref(h)), L.psfm_last_error().decode()

    def convert_create():
        a, budget = _args(None)
        return _create(a, budget), L.psfm_last_error().decode()

    calls.update({
        "psfm_ba_solve": ba_solve,
        "psfm_traj_optimize": traj_optimize,
        "psfm_known_rotation_translations": known_rotation,
        "psfm_triangulate_tracks": lambda: _raised(lambda: ig.triangulate_multi_view_points([(np.zeros((2, 3, 4)),
                                                                                                np.zeros((2, 2)))])),
        "psfm_matches_create": matches_create,
        "psfm_tracker_create": tracker_create,
        "psfm_convert_create": convert_create,
    })
    for name in ("psfm_blocked_cholesky_solve", "psfm_laplacian_solve", "psfm_spd_inverse"):
        calls[name] = lambda n=name: _dense_chol_entries(np.eye(4), np.ones(4), 4, 4, 4, 0, only={n})[0][1:]
    for name in ("psfm_null_vectors", "psfm_verification_local_model", "psfm_verification_minimal",
                 "psfm_verification_cubic"):
        calls[name] = lambda n=name: _null_vector_entries(only={n})[0][1:]
    return calls


NO_DEVICE_ENTRIES = list(STAGES) + ["psfm_ba_solve", "psfm_traj_optimize", "psfm_known_rotation_translations",
                                    "psfm_triangulate_tracks", "psfm_matches_create", "psfm_tracker_create",
                                    "psfm_convert_create", "psfm_blocked_cholesky_solve", "psfm_laplacian_solve",
                                    "psfm_spd_inverse", "psfm_null_vectors", "psfm_verification_local_model",
                                    "psfm_verification_minimal", "psfm_verification_cubic"]


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
@pytest.mark.parametrize("entry", NO_DEVICE_ENTRIES)
def test_no_device_is_refused_under_the_entry_name(entry):
    n0 = launch_count()
    rc, msg = _no_device_calls()[entry]()
    assert rc == _abi.PSFM_ERR_NO_DEVICE, (rc, msg)
    assert msg == entry + ": no CUDA device available (this library has no CPU path)", msg
    assert launch_count() == n0
