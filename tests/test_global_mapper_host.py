"""The global mapper's host side without a GPU: the database cache's pair rules, the vectorised model writer against
write_model, the command line sfm/main_sfm.py runs, the refusal of unbuilt paths before any device call, and the
argument checks of the new ABI entries."""
import ctypes as C
import os
import sqlite3

import numpy as np
import pytest

from particlesfm_b200 import _abi, _lib, ba, colmap_io, device_count, global_mapper as gm, handoff, launch_count

W, H = 640, 480


def _database(path, num_images, keypoints_per_image=40):
    db = sqlite3.connect(path)
    db.execute("CREATE TABLE cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, "
               "width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL)")
    db.execute("CREATE TABLE images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, "
               "camera_id INTEGER NOT NULL)")
    db.execute("INSERT INTO cameras VALUES (1, 0, ?, ?, ?, 0)", (W, H, np.array([500.0, W / 2, H / 2]).tobytes()))
    for i in range(1, num_images + 1):
        db.execute("INSERT INTO images (image_id, name, camera_id) VALUES (?, ?, 1)", (i, "%05d.png" % i))
    db.commit()
    db.close()
    rng = np.random.default_rng(0)
    return [(i, (rng.random((keypoints_per_image, 2)) * [W, H]).astype(np.float32)) for i in range(1, num_images + 1)]


def _row(a, b, n, config):
    m = np.stack([np.arange(n), np.arange(n)], 1).astype(np.uint32)
    eye = np.eye(3)
    return (handoff.image_ids_to_pair_id(a, b), m, config, eye, eye, eye)


def _cache_db(tmp_path):
    path = str(tmp_path / "database.db")
    kps = _database(path, 5)
    rows = [_row(1, 2, 15, 3),           # 15 inliers: kept
            _row(1, 3, 14, 3),           # 14: below min_num_matches
            _row(2, 3, 20, 7),           # WATERMARK
            _row(3, 4, 20, 0),           # UNDEFINED
            _row(4, 5, 5, 3)]            # image 5's only pair, too few matches
    handoff.write_colmap_database(path, handoff.DatabaseRows(kps, [], rows))
    return path


def test_cache_rules(tmp_path):
    path = _cache_db(tmp_path)
    g, used = handoff.load_database_cache(path)
    ref = handoff.read_two_view_geometries(path)
    assert used.tolist() == [True, False, True, False, False]
    assert np.array_equal(g.pair_images, ref.pair_images) and np.array_equal(g.inlier_ptr, ref.inlier_ptr)
    assert g.image_ids.tolist() == [1, 2, 3, 4, 5] and g.keypoint_ptr[-1] == 5 * 40    # every image stays
    _, used = handoff.load_database_cache(path, ignore_watermarks=True)
    assert used.tolist() == [True, False, False, False, False]
    _, used = handoff.load_database_cache(path, min_num_matches=14)
    assert used.tolist() == [True, True, True, False, False]
    _, used = handoff.load_database_cache(path, min_num_matches=5)
    assert used.tolist() == [True, True, True, False, True]
    # no used pair touches image 5 (index 4) at the default threshold, so no stage can register it
    g, used = handoff.load_database_cache(path)
    assert not np.isin(4, g.pair_images[used])


def test_cache_after_relative_pose_drops_undefined():
    class Poses:
        config = np.array([3, 0, 4, 5])
    assert handoff.cache_after_relative_pose([True, True, False, True], Poses).tolist() == [True, False, False, True]


def _random_model(seed):
    """A Reconstruction as apply_observation_mask leaves it (deleted points, -1 entries) and the same model as arrays."""
    rng = np.random.default_rng(seed)
    cams = {1: ba.Camera(1, 0, W, H, np.array([510.0, 320.5, 239.5])), 3: ba.Camera(3, 0, 800, 600, np.array([700.0, 400.0, 300.0]))}
    image_ids, names, cam_of, nk = [2, 5, 6, 9], ["a.png", "bb.png", "c/c.png", "d.png"], [0, 1, 0, 0], [7, 0, 11, 5]
    kp_ptr = np.concatenate([[0], np.cumsum(nk)])
    K = kp_ptr[-1]
    xys = rng.random((K, 2)) * 500
    P = 9
    p3 = np.where(rng.random(K) < 0.6, rng.integers(1, P + 1, K), -1)
    deleted = {2, 7}
    p3[np.isin(p3, list(deleted))] = -1
    images = {}
    for f, i in enumerate(image_ids):
        lo, hi = kp_ptr[f], kp_ptr[f + 1]
        images[i] = ba.Image(i, rng.standard_normal(4), rng.standard_normal(3), [1, 3][cam_of[f]], names[f], xys[lo:hi].copy(),
                             p3[lo:hi].astype(np.int64))
    img_of = np.repeat(np.arange(len(image_ids)), nk)
    points, tp, ti, t2 = {}, [0], [], []
    for pid in range(1, P + 1):
        if pid in deleted:
            continue
        ks = np.nonzero(p3 == pid)[0]
        tid = np.array(image_ids)[img_of[ks]].astype(np.int32)
        t2d = (ks - kp_ptr[img_of[ks]]).astype(np.int32)
        points[pid] = ba.Point3D(pid, rng.standard_normal(3), np.zeros(3, np.uint8), float(rng.random()), tid, t2d)
        tp.append(tp[-1] + len(ks))
        ti.append(tid)
        t2.append(t2d)
    rec = ba.Reconstruction(cams, images, points)
    ids = sorted(points)
    arrays = dict(camera_ids=np.array([1, 3]), camera_size=np.array([[W, H], [800, 600]]),
                  cam_params=np.stack([cams[1].params, cams[3].params]), image_ids=np.array(image_ids),
                  image_names=names, image_camera=np.array(cam_of), qvec=np.stack([images[i].qvec for i in image_ids]),
                  tvec=np.stack([images[i].tvec for i in image_ids]), keypoint_ptr=kp_ptr, keypoints=xys, point3D_ids=p3,
                  point_ids=np.array(ids), xyz=np.stack([points[p].xyz for p in ids]),
                  error=np.array([points[p].error for p in ids]), track_ptr=np.array(tp),
                  track_image_ids=np.concatenate(ti), track_point2D=np.concatenate(t2))
    return rec, arrays


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_write_model_arrays_is_byte_identical_to_write_model(tmp_path, seed):
    rec, arrays = _random_model(seed)
    colmap_io.write_model(rec, str(tmp_path / "a"))
    colmap_io.write_model_arrays(str(tmp_path / "b"), **arrays)
    for name in ("cameras.bin", "images.bin", "points3D.bin"):
        assert open(tmp_path / "a" / name, "rb").read() == open(tmp_path / "b" / name, "rb").read(), name
    back = colmap_io.read_model(str(tmp_path / "b"))
    assert sorted(back.points3D) == sorted(rec.points3D)


@pytest.mark.parametrize("chunk", [1, 2, 3])
def test_write_model_arrays_across_point_chunks(tmp_path, monkeypatch, chunk):
    monkeypatch.setattr(colmap_io, "_PT_CHUNK", chunk)
    rec, arrays = _random_model(4)
    colmap_io.write_model(rec, str(tmp_path / "a"))
    colmap_io.write_model_arrays(str(tmp_path / "b"), **arrays)
    assert open(tmp_path / "a" / "points3D.bin", "rb").read() == open(tmp_path / "b" / "points3D.bin", "rb").read()


def test_write_model_arrays_without_points(tmp_path):
    rec, arrays = _random_model(3)
    rec.points3D = {}
    for im in rec.images.values():
        im.point3D_ids[:] = -1
    arrays.update(point3D_ids=np.full_like(arrays["point3D_ids"], -1), point_ids=np.zeros(0, np.int64), xyz=np.zeros((0, 3)),
                  error=np.zeros(0), track_ptr=np.zeros(1, np.int64), track_image_ids=np.zeros(0, np.int32),
                  track_point2D=np.zeros(0, np.int32))
    colmap_io.write_model(rec, str(tmp_path / "a"))
    colmap_io.write_model_arrays(str(tmp_path / "b"), **arrays)
    for name in ("cameras.bin", "images.bin", "points3D.bin"):
        assert open(tmp_path / "a" / name, "rb").read() == open(tmp_path / "b" / name, "rb").read(), name


# sfm/main_sfm.py's gcolmap call, with gcolmap_path pointed at this module
MAIN_SFM_ARGS = ["--database_path", "DB", "--image_path", "IMAGES", "--output_path", "MODEL", "--GlobalMapper.num_threads",
                 "64", "--random_seed", "100", "--GlobalMapper.min_num_matches", "20",
                 "--GlobalMapper.ba_refine_principal_point", "0", "--GlobalMapper.ba_refine_extra_params", "0"]


def test_main_sfm_arguments_parse():
    args = gm.build_parser().parse_args(MAIN_SFM_ARGS)
    assert gm.unsupported(args) is None
    o = gm.options_from_args(args)
    assert (args.database_path, args.image_path, args.output_path, args.random_seed) == ("DB", "IMAGES", "MODEL", 100)
    assert o.num_threads == 64 and o.min_num_matches == 20
    assert o.ba_refine_principal_point is False and o.ba_refine_extra_params is False and o.ba_refine_focal_length is True
    d = gm.GlobalMapperOptions()
    assert (d.min_num_matches, d.ignore_watermarks, d.ba_refine_extra_params, d.ba_global_max_refinements,
            d.ba_global_max_refinement_change, d.filter_max_reproj_error) == (15, False, True, 5, 0.0005, 4.0)


@pytest.mark.parametrize("flags", [["--GlobalMapper.filter_with_1dsfm", "1"], ["--GlobalMapper.position_method", "nonlinear"],
                                   ["--GlobalMapper.lud_use_scale_constraints", "1"]])
def test_unbuilt_paths_exit_non_zero_before_any_device_call(tmp_path, monkeypatch, capsys, flags):
    path = _cache_db(tmp_path)

    def no_device_call(*a, **k):
        raise AssertionError("the mapper ran")
    monkeypatch.setattr(gm, "global_mapper", no_device_call)
    n0 = launch_count()
    rc = gm.main(["--database_path", path, "--output_path", str(tmp_path / "out")] + flags)
    assert rc != 0 and "is not supported" in capsys.readouterr().err
    assert launch_count() == n0 and not os.path.exists(tmp_path / "out")
    # the same refusal when called as gcolmap is, with the subcommand first
    assert gm.main(["global_mapper", "--database_path", path, "--output_path", str(tmp_path / "out")] + flags) != 0


# ---- the ABI entries: argument checks first, then the device check


def _dummy():
    """A non-null handle that the entries must not dereference before they find a device."""
    buf = C.create_string_buffer(256)
    return buf, C.cast(buf, C.c_void_p)


def _create(tri, q=True):
    x = np.zeros(12)
    u8 = np.zeros(3, np.uint8)
    h = C.c_void_p()
    p = C.POINTER(C.c_uint8)
    rc = _lib.lib().psfm_ba_create_from_triangulation(tri, _lib.dptr(x) if q else None, _lib.dptr(x), _lib.dptr(x),
                                                      u8.ctypes.data_as(p), None, None, C.byref(h), None, None, None)
    return rc, _lib.lib().psfm_last_error().decode()


def _get_model(S, complete=True):
    x, i64, i32 = np.zeros(64), np.zeros(8, np.int64), np.zeros(8, np.int32)
    ip, lp = C.POINTER(C.c_int32), C.POINTER(C.c_int64)
    rc = _lib.lib().psfm_ba_get_model(S, _lib.dptr(x), _lib.dptr(x), _lib.dptr(x), _lib.dptr(x), i64.ctypes.data_as(lp),
                                      i32.ctypes.data_as(ip), i32.ctypes.data_as(ip), i64.ctypes.data_as(lp) if complete else None)
    return rc, _lib.lib().psfm_last_error().decode()


def test_new_entries_check_arguments_first():
    _keep, d = _dummy()
    assert _create(None)[0] == _abi.PSFM_ERR_INVALID
    rc, msg = _create(d, q=False)
    assert rc == _abi.PSFM_ERR_INVALID and msg.startswith("psfm_ba_create_from_triangulation: null argument")
    assert _get_model(None)[0] == _abi.PSFM_ERR_INVALID
    rc, msg = _get_model(d, complete=False)
    assert rc == _abi.PSFM_ERR_INVALID and msg.startswith("psfm_ba_get_model: null argument")
    assert _lib.lib().psfm_ba_get_observations(None, None, None, None, None) == _abi.PSFM_ERR_INVALID


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_new_entries_without_a_device():
    _keep, d = _dummy()
    rc, msg = _create(d)
    assert rc == _abi.PSFM_ERR_NO_DEVICE and "no CUDA device" in msg
    rc, msg = _get_model(d)
    assert rc == _abi.PSFM_ERR_NO_DEVICE and "no CUDA device" in msg
    p = np.zeros(4, np.int32).ctypes.data_as(C.POINTER(C.c_int32))
    assert _lib.lib().psfm_ba_get_observations(d, p, None, None, p) == _abi.PSFM_ERR_NO_DEVICE


def _positions_raise(monkeypatch, tmp_path, code):
    """The mapper on the cache database with every stage before the positions stubbed, and the positions raising
    `code`."""
    from particlesfm_b200 import init_geometry

    class Rot:
        success, orientations = True, np.tile([1.0, 0, 0, 0], (5, 1))
        has_orientation, pair_kept, summary = np.ones(5, bool), np.ones(5, bool), {}

    class Poses:
        config, estimated, qvec = np.full(5, 3), np.ones(5, bool), np.zeros((5, 4))

    def raise_code(*a, **k):
        raise _lib.PsfmError("psfm_estimate_global_positions failed with status %d: why" % code, code)
    monkeypatch.setattr(init_geometry, "estimate_relative_poses", lambda **k: Poses)
    monkeypatch.setattr(init_geometry, "estimate_global_rotations", lambda *a, **k: Rot)
    monkeypatch.setattr(init_geometry, "optimize_pairwise_translations", lambda *a, **k: np.zeros((5, 3)))
    monkeypatch.setattr(init_geometry, "estimate_global_positions", raise_code)
    out = str(tmp_path / "out")
    return gm.main(["--database_path", _cache_db(tmp_path), "--output_path", out]), out


def test_a_failed_position_stage_writes_nothing_and_exits_0(tmp_path, monkeypatch, capsys):
    rc, out = _positions_raise(monkeypatch, tmp_path, _abi.PSFM_ERR_INVALID)
    assert rc == 0 and not os.path.exists(os.path.join(out, "0"))
    err = capsys.readouterr().err
    assert "Global position failed" in err and "why" in err


@pytest.mark.parametrize("code", [_abi.PSFM_ERR_CUDA, _abi.PSFM_ERR_UNSUPPORTED, _abi.PSFM_ERR_NO_DEVICE])
def test_other_position_errors_are_errors_of_the_run(tmp_path, monkeypatch, capsys, code):
    rc, out = _positions_raise(monkeypatch, tmp_path, code)
    assert rc != 0 and not os.path.exists(os.path.join(out, "0"))
    assert "status %d" % code in capsys.readouterr().err
