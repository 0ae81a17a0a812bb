"""Known answers of the numpy restatement of the two-view geometric verification (oracle/verification_oracle.py), the
database round trip of its rows, and handoff.read_matches / MatchTables.from_rows.  No GPU needed."""
import sqlite3

import numpy as np
import pytest

from oracle import verification_oracle as vo
from particlesfm_b200 import handoff, synthetic as syn

W, H = 1024, 436


def scene_tables(num_trajs, num_frames, num_obs, seed, step=0.02, path="line", outliers=0.0, noise_px=0.0):
    """MatchTables of a synthetic video: make_two_view_scene -> traj_to_matches -> database rows, with a seeded share
    of keypoints moved 20 .. 60 px and Gaussian noise."""
    tracks, _, _, cam = syn.make_two_view_scene(num_trajs, num_frames, num_obs, seed=seed, step=step, path=path)
    names, ids = ["%05d.png" % i for i in range(num_frames)], list(range(1, num_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches(tracks, num_frames))
    mt = handoff.MatchTables.from_rows(rows, ids, names, cam, (W, H))
    if outliers or noise_px:
        mt.keypoints = syn.corrupt_keypoints(mt.keypoints, outliers, seed=seed, noise_px=noise_px)[0]
    return mt


def pair_tables(pairs):
    """MatchTables of independent pairs: pair p is images 2p and 2p + 1 with keypoints x1 / x2 [n][2], match i = (i, i)."""
    kps, mptr, ms = [], [0], []
    for x1, x2 in pairs:
        kps += [np.asarray(x1, np.float32).reshape(-1, 2), np.asarray(x2, np.float32).reshape(-1, 2)]
        n = len(x1)
        ms.append(np.stack([np.arange(n), np.arange(n)], 1).astype(np.uint32))
        mptr.append(mptr[-1] + n)
    F = len(kps)
    return handoff.MatchTables(
        image_ids=np.arange(1, F + 1), image_names=["%d.png" % i for i in range(F)],
        keypoint_ptr=np.concatenate([[0], np.cumsum([k.shape[0] for k in kps])]).astype(np.int64),
        keypoints=np.concatenate(kps), camera_ids=np.array([1]), cameras=np.array([[500.0, W / 2, H / 2]]),
        image_camera=np.zeros(F, np.int32), camera_size=np.array([[W, H]]), prior_focal_length=np.zeros(1, bool),
        pair_ids=np.array([handoff.image_ids_to_pair_id(2 * p + 1, 2 * p + 2) for p in range(len(pairs))]),
        pair_images=np.array([[2 * p, 2 * p + 1] for p in range(len(pairs))], np.int32),
        match_ptr=np.array(mptr, np.int64), matches=np.concatenate(ms).reshape(-1, 2))


def two_views(n, seed, plane=False, rotation_only=False):
    """n exact correspondences of two calibrated views (f 500, image W x H); returns x1, x2, F, H (plane / rotation)."""
    rng = np.random.default_rng(seed)
    K = np.array([[500.0, 0, W / 2], [0, 500.0, H / 2], [0, 0, 1]])
    R = syn.axis_angle_to_rotmat(np.array([[0.02, -0.05, 0.01]]))[0]
    t = np.zeros(3) if rotation_only else np.array([0.3, 0.05, 0.02])
    px = rng.random((n, 2)) * [W, H]
    depth = np.full(n, 5.0) if plane else 3.0 + 10.0 * rng.random(n)
    X = np.concatenate([(px - K[:2, 2]) / 500.0, np.ones((n, 1))], 1) * depth[:, None]
    Y = X @ R.T + t
    x2 = Y[:, :2] / Y[:, 2:] * 500.0 + K[:2, 2]
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Ki = np.linalg.inv(K)
    Fm = Ki.T @ tx @ R @ Ki
    Hm = K @ (R + np.outer(t, [0, 0, 1.0]) / 5.0) @ Ki
    return px, x2, Fm, Hm


def _same_up_to_scale(a, b):
    a, b = vo.stored(np.ravel(a)), vo.stored(np.ravel(b))
    return np.abs(a - b).max()


def test_seven_point_recovers_f():
    x1, x2, Fm, _ = two_views(7, 1)
    models = vo.seven_point(x1, x2)
    assert 1 <= len(models) <= 3
    assert min(_same_up_to_scale(m, Fm) for m in models) < 1e-6
    assert all(m[8] == 1.0 for m in models) and [tuple(m) for m in models] == sorted(tuple(m) for m in models)


def test_eight_point_recovers_f():
    x1, x2, Fm, _ = two_views(40, 2)
    assert _same_up_to_scale(vo.eight_point(x1, x2)[0], Fm) < 1e-9


@pytest.mark.parametrize("kind", ["plane", "rotation"])
def test_dlt_recovers_h(kind):
    x1, x2, _, Hm = two_views(30, 3, plane=kind == "plane", rotation_only=kind == "rotation")
    assert _same_up_to_scale(vo.homography_dlt(x1, x2)[0], Hm) < 1e-9
    assert _same_up_to_scale(vo.homography_dlt(x1[:4], x2[:4])[0], Hm) < 1e-8


def test_sampson_error():
    x1, x2, Fm, _ = two_views(10, 4)
    assert np.abs(vo.sampson_error(Fm.ravel(), x1, x2)).max() < 1e-18
    F = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0.0]]).ravel()       # pure x translation: epipolar lines y = const
    r = vo.sampson_error(F, np.array([[10.0, 20.0]]), np.array([[30.0, 23.0]]))
    assert r[0] == pytest.approx(9.0 / 2.0)                              # (y2 - y1)^2 / 2


def test_sampler():
    a = vo.sample(7, 3, 1, 11, 50, 7)
    assert len(set(a)) == 7 and all(0 <= i < 50 for i in a) and a == vo.sample(7, 3, 1, 11, 50, 7)
    assert a != vo.sample(7, 3, 1, 12, 50, 7) and a != vo.sample(7, 3, 0, 11, 50, 7)
    # a plain restatement with Python ints
    M, G = 2 ** 64, 0x9E3779B97F4A7C15

    def mix(z):
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9 % M
        z = (z ^ (z >> 27)) * 0x94D049BB133111EB % M
        return z ^ (z >> 31)
    s = 7
    for v in (3, 1, 11):
        s = mix((s + G * (v + 1)) % M)
    out = []
    while len(out) < 7:
        s = (s + G) % M
        i = (mix(s) >> 32) * 50 >> 32
        if i not in out:
            out.append(i)
    assert out == a
    assert len(set(vo.sample(0, 0, 0, 0, 7, 7))) == 7


def test_compute_num_trials():
    n = vo.compute_num_trials
    assert n(10000, 100000, 7, 0.999, 3.0) > 20000 and n(10000, 100000, 4, 0.999, 3.0) == 207223
    assert n(70000, 100000, 1, 0.999, 3.0) == 18                       # the watermark cap
    assert n(90, 100, 7, 0.999, 3.0) == 32 and n(50, 100, 4, 0.999, 3.0) == 322
    assert n(100, 100, 7, 0.999, 3.0) == 1 and n(0, 100, 4, 0.999, 3.0) == vo.UNBOUNDED


def _verify(mt, **o):
    return vo.verify_two_view_geometries(**mt.verification_inputs(), options=o)


def test_configs():
    x1p, x2p, _, _ = two_views(60, 5, plane=True)
    x1, x2, _, _ = two_views(60, 6)
    rng = np.random.default_rng(0)
    few = rng.random((14, 2)) * [W, H]
    junk1, junk2 = rng.random((40, 2)) * [W, H], rng.random((40, 2)) * [W, H]
    border = np.concatenate([rng.random((30, 1)) * 90, rng.random((30, 1)) * H], 1)
    mt = pair_tables([(x1p, x2p), (x1, x2), (few, few + 1), (junk1, junk2), (border, border + [4.0, -2.0])])
    r = _verify(mt)
    assert r["config"].tolist() == [vo.PLANAR_OR_PANORAMIC, vo.UNCALIBRATED, vo.UNDEFINED, vo.DEGENERATE, vo.WATERMARK]
    n = np.diff(r["inlier_ptr"])
    assert n[0] == 60 and n[1] == 60 and n[2] == 0 and n[3] == 0 and n[4] == 30
    assert r["trials"][2].tolist() == [0, 0, 0] and 1 <= r["trials"][4][2] <= 18
    assert np.all(r["E"] == 0)
    # without the watermark test the border pair is an ordinary planar pair
    assert _verify(mt, detect_watermark=0)["config"][4] == vo.PLANAR_OR_PANORAMIC


def test_video_scene_and_outliers():
    r = _verify(scene_tables(300, 5, 1500, seed=3, step=0.08, path="helix", outliers=0.2, noise_px=0.5))
    assert (r["config"] == vo.UNCALIBRATED).sum() >= 8
    assert (r["local_rounds"][:, 0] > 0).all()


def test_options_check():
    with pytest.raises(vo.InvalidError):
        _verify(pair_tables([two_views(20, 1)[:2]]), max_error=0.0)
    mt = pair_tables([two_views(20, 1)[:2]])
    mt.prior_focal_length = np.ones(1, bool)
    with pytest.raises(vo.UnsupportedError):
        _verify(mt)


def _database(path, mt, cam):
    db = sqlite3.connect(path)
    db.execute("CREATE TABLE cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, "
               "width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL)")
    db.execute("CREATE TABLE images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, "
               "camera_id INTEGER NOT NULL)")
    db.execute("INSERT INTO cameras VALUES (1, 0, ?, ?, ?, 0)", (W, H, np.asarray(cam, np.float64).tobytes()))
    for i, n in zip(mt.image_ids, mt.image_names):
        db.execute("INSERT INTO images (image_id, name, camera_id) VALUES (?, ?, 1)", (int(i), n))
    db.commit()
    db.close()


def test_read_matches_equals_from_rows_and_round_trip(tmp_path):
    nf = 5
    tracks, _, _, cam = syn.make_two_view_scene(300, nf, 1500, seed=3, step=0.08, path="helix")
    names, ids = ["%05d.png" % i for i in range(nf)], [nf - i for i in range(nf)]
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches(tracks, nf))
    mt = handoff.MatchTables.from_rows(rows, ids, names, cam, (W, H))
    path = str(tmp_path / "database.db")
    _database(path, mt, cam)
    handoff.write_colmap_database(path, rows)
    back = handoff.read_matches(path)
    for k in ("image_ids", "keypoint_ptr", "keypoints", "image_camera", "camera_ids", "cameras", "camera_size",
              "prior_focal_length", "pair_ids", "pair_images", "match_ptr", "matches"):
        assert np.array_equal(getattr(back, k), getattr(mt, k)), k
    assert back.image_names == mt.image_names
    # the oracle's rows through the database equal to_two_view_geometries' arrays
    r = vo.verify_two_view_geometries(**mt.verification_inputs())
    verified = handoff.DatabaseRows([], [], [(int(pid), r["inlier_matches"][r["inlier_ptr"][p]:r["inlier_ptr"][p + 1]],
                                             int(r["config"][p]), r["F"][p], r["E"][p], r["H"][p])
                                            for p, pid in enumerate(mt.pair_ids)])
    handoff.write_colmap_database(path, verified)
    g = handoff.read_two_view_geometries(path)
    assert np.array_equal(g.config, r["config"]) and np.array_equal(g.inlier_ptr, r["inlier_ptr"])
    assert np.array_equal(g.inlier_matches, r["inlier_matches"])
    assert np.array_equal(g.F.reshape(-1, 9), r["F"]) and np.array_equal(g.H.reshape(-1, 9), r["H"])
    assert np.array_equal(g.pair_images, mt.pair_images) and np.array_equal(g.keypoints, mt.keypoints)
