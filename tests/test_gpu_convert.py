"""The model conversion on the device (csrc/convert.cu, particlesfm_b200.convert) against the numpy restatement
(oracle/convert_oracle.py): depth maps bit for bit, display images pixel for pixel, text files byte for byte."""
import io
import os
import sqlite3
import subprocess
import sys

import numpy as np
import pytest

from oracle import convert_oracle as co
from particlesfm_b200 import ba, colmap_io, convert, global_mapper as gm, handoff, init_geometry, synthetic as syn
from test_oracle_convert import random_model, read_png_rgba

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W, H = 1024, 436


def write_model(path, a):
    """a (save_depth_pose_arrays' keyword arguments) as a binary COLMAP model through colmap_io.write_model."""
    models = np.broadcast_to(np.asarray(a.get("camera_model", 0)), (len(a["camera_ids"]),))
    cams = {int(c): ba.Camera(int(c), int(m), int(s[0]), int(s[1]), np.asarray(p[:4 if m == 2 else 3], np.float64))
            for c, m, s, p in zip(a["camera_ids"], models, a["camera_size"], a["cam_params"])}
    ptr = a["keypoint_ptr"]
    ims = {int(i): ba.Image(int(i), np.asarray(a["qvec"][j]), np.asarray(a["tvec"][j]),
                            int(a["camera_ids"][a["image_camera"][j]]), a["image_names"][j],
                            np.asarray(a["keypoints"][ptr[j]:ptr[j + 1]]), np.asarray(a["point3D_ids"][ptr[j]:ptr[j + 1]]))
           for j, i in enumerate(a["image_ids"])}
    pts = {int(p): ba.Point3D(int(p), np.asarray(x), np.zeros(3, np.uint8), 0.0, np.zeros(0, np.int32), np.zeros(0, np.int32))
           for p, x in zip(a["point_ids"], a["xyz"])}
    colmap_io.write_model(ba.Reconstruction(cams, ims, pts), path)


def edge_model():
    """Images of three sizes and both camera models: a shared pixel (last wins), x.5 keypoints, clipped keypoints,
    depth -1 and negative depths, a keypoint without a point, and an image whose valid values are all equal."""
    imgs = [  # (camera, keypoints, depths)
        (0, [[2.2, 1.1], [1.9, 0.8], [2.4, 1.4], [2.5, 0.5], [3.5, 1.5], [-7.2, 2.0], [20, 40], [-0.5, 5.5], [6, 4]],
         [3.0, 2.0, 4.0, 1.0, 2.5, 3.0, 4.0, 5.0, None]),
        (1, [[0, 0], [1, 0], [2, 0], [3, 0], [4, 0]], [-2.0, -1.0, 1.0, 2.0, -0.5]),
        (2, [[0, 0], [3, 2], [5, 4], [6, 1]], [2.0, 2.0, 2.0, None]),
    ]
    xyz, p3, kps, ptr = [], [], [], [0]
    for _, xy, z in imgs:
        for v in z:
            if v is None:
                p3.append(-1)
            else:
                xyz.append([0.0, 0.0, v])
                p3.append(100 + len(xyz))
        kps += xy
        ptr.append(len(kps))
    return dict(camera_ids=np.array([3, 1, 2]), camera_size=np.array([[8, 6], [5, 3], [7, 5]]),
                cam_params=np.array([[10.0, 4, 3, 0.0], [11.0, 2.5, 1.5, 0.02], [12.0, 3.5, 2.5, 0.0]]),
                camera_model=np.array([0, 2, 0]), image_ids=np.array([7, 3, 5]),
                image_names=["e0.png", "e1.jpg", "e2"], image_camera=np.array([c for c, _, _ in imgs]),
                qvec=np.tile([1.0, 0, 0, 0], (3, 1)), tvec=np.zeros((3, 3)), keypoint_ptr=np.array(ptr),
                keypoints=np.array(kps, np.float64), point3D_ids=np.array(p3), point_ids=np.array(p3)[np.array(p3) >= 0],
                xyz=np.array(xyz))


def savetxt_bytes(a):
    buf = io.BytesIO()
    np.savetxt(buf, a)
    return buf.getvalue()


def check_output(out, a):
    """Every file under out against the oracle for the model arrays a."""
    vec, ref = co.depth_maps(a), co.depth_maps_loop(a)
    scale = 16 * np.abs(a["qvec"]).max() ** 2 * (np.abs(a["xyz"]).max() + 1)
    models = np.broadcast_to(np.asarray(a.get("camera_model", 0)), (len(a["camera_ids"]),))
    assert sorted(os.listdir(out)) == ["depths", "intrinsics", "poses"]
    for i, name in enumerate(a["image_names"]):
        stem = os.path.splitext(name)[0]
        d = np.load(os.path.join(out, "depths", stem + ".npy"))
        assert d.dtype == np.float64 and np.array_equal(d, vec[i]), name
        assert np.all(np.abs(d - ref[i]) <= 4 * np.finfo(float).eps * scale), name
        assert np.array_equal(read_png_rgba(os.path.join(out, "depths", stem + ".png")), co.display_rgba(d)), name
        c = a["image_camera"][i]
        f, cx, cy = a["cam_params"][c][:3]
        assert models[c] in (0, 2)
        K = np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]])
        assert open(os.path.join(out, "intrinsics", stem + ".txt"), "rb").read() == savetxt_bytes(K)
        Rt = np.concatenate([co.qvec2rotmat(np.asarray(a["qvec"][i])), np.expand_dims(np.asarray(a["tvec"][i]), -1)], -1)
        assert open(os.path.join(out, "poses", stem + ".txt"), "rb").read() == savetxt_bytes(Rt)
    assert len(os.listdir(os.path.join(out, "poses"))) == len(a["image_names"])


def test_edge_cases_match_the_oracle(tmp_path, gpu):
    a = edge_model()
    write_model(str(tmp_path / "m"), a)
    rep = convert.write_depth_pose_from_colmap_format(str(tmp_path / "m"), str(tmp_path / "out"))
    assert list(rep.valid_count) == [6, 2, 3] and rep.written == 3
    check_output(str(tmp_path / "out"), a)
    d = np.load(str(tmp_path / "out" / "depths" / "e0.npy"))
    assert d[1, 2] == 4.0 and d[0, 2] == 1.0 and d[2, 4] == 2.5 and d[5, 7] == 4.0 and d[5, 0] == 5.0
    rgba = read_png_rgba(str(tmp_path / "out" / "depths" / "e2.png"))
    assert (rgba[np.load(str(tmp_path / "out" / "depths" / "e2.npy")) > 0, :3] == 0).all()      # NaN: black


@pytest.mark.parametrize("seed", range(4))
def test_random_models_match_the_oracle(tmp_path, gpu, seed):
    a = random_model(seed, num_images=6, keypoints=(100, 3000))
    write_model(str(tmp_path / "m"), a)
    rep = convert.write_depth_pose_from_colmap_format(str(tmp_path / "m"), str(tmp_path / "out"), memory_budget=40000)
    assert rep.num_batches > 1
    check_output(str(tmp_path / "out"), a)
    # the arrays entry writes the same files
    convert.save_depth_pose_arrays(str(tmp_path / "arr"), **a)
    for sub in ("depths", "poses", "intrinsics"):
        for f in os.listdir(tmp_path / "out" / sub):
            assert (tmp_path / "out" / sub / f).read_bytes() == (tmp_path / "arr" / sub / f).read_bytes(), f


def sintel_model(num_images=12, keypoints=20000, seed=0):
    rng = np.random.default_rng(seed)
    P = keypoints * 2
    xyz = rng.uniform([-3, -1.5, 2], [3, 1.5, 12], size=(P, 3))
    ptr, kps, p3 = [0], [], []
    for i in range(num_images):
        xy = rng.uniform([-2, -2], [W + 1, H + 1], size=(keypoints, 2))
        xy[: keypoints // 10] = np.round(xy[: keypoints // 10] * 2) / 2
        kps.append(xy)
        p3.append(np.where(rng.random(keypoints) < 0.6, rng.integers(0, P, keypoints) + 1, -1))
        ptr.append(ptr[-1] + keypoints)
    q = np.column_stack([np.ones(num_images), rng.normal(0, 0.02, (num_images, 3))])
    return dict(camera_ids=np.array([1]), camera_size=np.array([[W, H]]), cam_params=np.array([[900.0, W / 2, H / 2]]),
                image_ids=np.arange(1, num_images + 1), image_names=["frame_%04d.png" % i for i in range(num_images)],
                image_camera=np.zeros(num_images, np.int64), qvec=q, tvec=rng.normal(0, 0.1, (num_images, 3)),
                keypoint_ptr=np.array(ptr), keypoints=np.concatenate(kps), point3D_ids=np.concatenate(p3),
                point_ids=np.arange(1, P + 1), xyz=xyz)


def test_sintel_shape_across_batch_and_host_chunk_boundaries(tmp_path, gpu):
    a = sintel_model()
    px = W * H
    rep = convert.save_depth_pose_arrays(str(tmp_path / "out"), **a, memory_budget=2 * (16 * 3 * px + 32 * 60000),
                                         host_budget=12 * 5 * px)
    assert rep.num_batches == 4
    check_output(str(tmp_path / "out"), a)


def test_an_image_without_a_valid_pixel_writes_nothing(tmp_path, gpu):
    a = random_model(1)
    p3 = a["point3D_ids"].copy()
    p3[a["keypoint_ptr"][2]:a["keypoint_ptr"][3]] = -1
    a["point3D_ids"] = p3
    with pytest.raises(IndexError, match="frame_002"):
        convert.save_depth_pose_arrays(str(tmp_path / "out"), **a)
    assert not (tmp_path / "out").exists()
    write_model(str(tmp_path / "m"), a)
    (tmp_path / "empty").mkdir()
    with pytest.raises(IndexError, match="frame_002"):
        convert.write_depth_pose_from_colmap_format(str(tmp_path / "m"), str(tmp_path / "empty"))
    assert os.listdir(tmp_path / "empty") == []


def test_model_subdirectory_fallback_and_command_line(tmp_path, gpu):
    a = random_model(5)
    write_model(str(tmp_path / "sfm" / "model"), a)
    convert.write_depth_pose_from_colmap_format(str(tmp_path / "sfm"), str(tmp_path / "api"))
    check_output(str(tmp_path / "api"), a)
    r = subprocess.run([sys.executable, "-m", "particlesfm_b200.convert", "--input_dir", str(tmp_path / "sfm"),
                        "--output_dir", str(tmp_path / "cli")], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert r.stdout.splitlines() == ["num_cameras: 2", "num_images: 4", "num_points3D: 300", str(tmp_path / "cli")]
    for sub in ("depths", "poses", "intrinsics"):
        assert sorted(os.listdir(tmp_path / "cli" / sub)) == sorted(os.listdir(tmp_path / "api" / sub))
        for f in os.listdir(tmp_path / "api" / sub):
            assert (tmp_path / "cli" / sub / f).read_bytes() == (tmp_path / "api" / sub / f).read_bytes(), f


# ----------------------------------------------------------------------------- the mapper's hand-off


def _scene_db(path, n_frames=10, seed=7, noise_px=0.0):
    """A helix video through traj_to_matches, geometric verification and write_colmap_database: the database
    build_database leaves for the mapper, keypoints with Gaussian noise of noise_px.  Returns the true poses."""
    tracks, qvec, tvec, cam = syn.make_two_view_scene(1500, n_frames, 9000, seed=seed, step=0.08, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, n_frames))
    mt = handoff.MatchTables.from_rows(rows, ids, names, cam, (W, H))
    if noise_px:
        mt.keypoints = syn.corrupt_keypoints(mt.keypoints, 0.0, seed=seed, noise_px=noise_px)[0]
        k = dict(rows.keypoints)
        rows.keypoints = [(i, mt.keypoints[mt.keypoint_ptr[r]:mt.keypoint_ptr[r + 1]].reshape(k[i].shape[0], 2))
                          for r, i in enumerate(mt.image_ids.tolist())]
    ver = init_geometry.verify_two_view_geometries(**mt.verification_inputs())
    db = sqlite3.connect(path)
    db.execute("CREATE TABLE cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, "
               "width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL)")
    db.execute("CREATE TABLE images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, "
               "camera_id INTEGER NOT NULL)")
    db.execute("INSERT INTO cameras VALUES (1, 0, ?, ?, ?, 0)", (W, H, np.asarray(cam, np.float64).tobytes()))
    for i, n in zip(ids, names):
        db.execute("INSERT INTO images (image_id, name, camera_id) VALUES (?, ?, 1)", (i, n))
    db.commit()
    db.close()
    handoff.write_colmap_database(path, handoff.DatabaseRows(rows.keypoints, rows.matches, ver.two_view_rows(mt.pair_ids)))
    return qvec, tvec


def test_mapper_convert_path_equals_converting_the_written_model(tmp_path, gpu):
    db = str(tmp_path / "database.db")
    qvec, tvec = _scene_db(db, n_frames=10, seed=7)
    rep = gm.global_mapper(db, str(tmp_path / "sfm"), gm.GlobalMapperOptions(ba_refine_extra_params=False),
                           convert_path=str(tmp_path / "A"))
    assert rep.success and rep.seconds("convert") > 0
    convert.write_depth_pose_from_colmap_format(rep.output, str(tmp_path / "B"))
    for sub in ("depths", "poses", "intrinsics"):
        names = sorted(os.listdir(tmp_path / "A" / sub))
        assert names == sorted(os.listdir(tmp_path / "B" / sub)) and names
        for f in names:
            assert (tmp_path / "A" / sub / f).read_bytes() == (tmp_path / "B" / sub / f).read_bytes(), f
    # the ATE from poses/*.txt is the ATE from the model
    m = colmap_io.read_model(rep.output)
    ids = sorted(m.images)
    truth = syn.camera_centres(qvec, tvec)[np.array(ids) - 1]
    est = syn.camera_centres(np.array([m.images[i].qvec for i in ids]), np.array([m.images[i].tvec for i in ids]))
    from_txt = []
    for i in ids:
        Rt = np.loadtxt(str(tmp_path / "A" / "poses" / (os.path.splitext(m.images[i].name)[0] + ".txt")))
        from_txt.append(-Rt[:, :3].T @ Rt[:, 3])
    ate_model, ate_txt = syn.umeyama_ate(est, truth), syn.umeyama_ate(np.array(from_txt), truth)
    extent = np.linalg.norm(truth - truth.mean(0), axis=1).max()
    assert abs(ate_model - ate_txt) <= 1e-9 * extent and ate_model <= 0.05 * extent


def test_a_batch_holds_at_most_65535_images(gpu):
    """Many tiny images under a large budget: the planner starts a new batch after 65,535 images (grid.y of the
    launches), and both batches return their maps."""
    import ctypes as C
    from particlesfm_b200 import _lib
    F = 65535 + 7
    i64p, ip, u8p = C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_uint8)
    size = np.array([[2, 2]], np.int32)
    cam = np.zeros(F, np.int32)
    q, t = np.tile([1.0, 0, 0, 0], (F, 1)), np.zeros((F, 3))
    ptr = np.arange(F + 1, dtype=np.int64)
    kp = np.tile([1.0, 0.0], (F, 1))                            # pixel (x 1, y 0)
    row = np.arange(F, dtype=np.int32)
    xyz = np.column_stack([np.zeros(F), np.zeros(F), 1.0 + np.arange(F)])
    lut = convert.binary_lut()
    valid, bptr, h = np.zeros(F, np.int64), np.zeros(F + 1, np.int32), C.c_void_p()
    L = _lib.lib()
    _lib.check(L.psfm_convert_create(1, size.ctypes.data_as(ip), F, _lib.dptr(q), _lib.dptr(t), cam.ctypes.data_as(ip),
                                     ptr.ctypes.data_as(i64p), _lib.dptr(kp), row.ctypes.data_as(ip), F, _lib.dptr(xyz),
                                     lut.ctypes.data_as(u8p), 1 << 30, C.byref(h), valid.ctypes.data_as(i64p),
                                     bptr.ctypes.data_as(ip), None), "psfm_convert_create")
    try:
        assert (valid == 1).all() and list(bptr[:3]) == [0, 65535, F]
        depth, rgba = np.empty(4 * F), np.empty(16 * F, np.uint8)
        _lib.check(L.psfm_convert_result(h, 0, 2, _lib.dptr(depth), rgba.ctypes.data_as(u8p), None), "psfm_convert_result")
    finally:
        L.psfm_convert_destroy(h)
    d = depth.reshape(F, 2, 2)
    assert np.array_equal(d[:, 0, 1], xyz[:, 2]) and (d.reshape(F, 4)[:, [0, 2, 3]] == 0).all()
    ref = co.display_rgba(d[-1])
    assert np.array_equal(rgba.reshape(F, 2, 2, 4)[-1], ref) and np.array_equal(rgba.reshape(F, 2, 2, 4)[0], co.display_rgba(d[0]))
