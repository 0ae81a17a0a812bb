"""The relative pose of every verified pair on the GPU (init_geometry.estimate_relative_poses, csrc/two_view.cu)
against the numpy restatement (oracle/two_view_oracle.py), whose known answers tests/test_oracle_two_view.py pins."""
import sqlite3

import numpy as np
import pytest

from oracle import two_view_oracle as tv
from particlesfm_b200 import _lib, handoff, init_geometry, synthetic as syn

CAMS = np.array([[520.0, 320.0, 240.0], [480.0, 300.0, 250.0]])
NUM_IMAGES = 6
BIG = 210_000


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _mixed_batch(seed=0):
    """Six images of BIG static points (images 3 .. 5 with 0.5 px noise), the camera moving 0.02 per frame while the
    points are 2 .. 40 away: adjacent frames see points on both sides of max_depth.  Every point is a keypoint of
    every image, in a per-image shuffled order.  Pairs: E, F and H configs, 20 % outliers, 0 / 1 / 2 inliers, E = I,
    a pure-rotation H, configs that pass through, and one pair of BIG inliers."""
    rng = np.random.default_rng(seed)
    f = np.arange(NUM_IMAGES, dtype=np.float64)
    Rs = syn.axis_angle_to_rotmat(np.stack([0.002 * f, 0.01 * f, -0.003 * f], axis=1))
    ts = -np.einsum("fij,fj->fi", Rs, np.stack([0.02 * f, 0.004 * f, 0.001 * f], axis=1))
    depth = rng.uniform(2.0, 40.0, BIG)
    X = np.c_[rng.uniform(-0.6, 0.6, (BIG, 2)) * depth[:, None], depth]
    cam_of = np.arange(NUM_IMAGES) % 2
    perm = [rng.permutation(BIG) for _ in range(NUM_IMAGES)]
    kps = []
    for i in range(NUM_IMAGES):
        Xc = X @ Rs[i].T + ts[i]
        xy = CAMS[cam_of[i], 0] * Xc[:, :2] / Xc[:, 2:] + CAMS[cam_of[i], 1:]
        if i >= 3:
            xy += rng.normal(0.0, 0.5, xy.shape)
        k = np.empty_like(xy)
        k[perm[i]] = xy                                          # point j is keypoint perm[i][j] of image i
        kps.append(k.astype(np.float32))
    K = [tv.calibration(CAMS[c]) for c in cam_of]

    def rel(a, b):
        R = Rs[b] @ Rs[a].T
        return R, ts[b] - R @ ts[a]

    pairs = []

    def add(a, b, config, n, E=None, F=None, H=None, outliers=0.0):
        pts = rng.choice(BIG, n, replace=False) if n < BIG else np.arange(BIG)
        m = np.stack([perm[a][pts], perm[b][pts]], axis=1)
        bad = rng.random(n) < outliers
        m[bad, 1] = rng.integers(0, BIG, int(bad.sum()))
        R, t = rel(a, b)
        E = _skew(t) @ R if E is None else E
        F = np.linalg.inv(K[b]).T @ _skew(t) @ R @ np.linalg.inv(K[a]) * 3.0 if F is None else F
        if H is None:
            nrm = np.array([0.05, -0.1, 1.0])
            H = K[b] @ (R + np.outer(t, nrm / np.linalg.norm(nrm)) / 8.0) @ np.linalg.inv(K[a])
        pairs.append((a, b, config, E, F, H, m.astype(np.uint32)))

    add(0, 1, 2, 4000)
    add(1, 2, 3, 4000)
    add(0, 2, 6, 3000)
    add(3, 4, 2, 4000, outliers=0.2)
    add(4, 5, 4, 3000, outliers=0.2)
    add(2, 3, 5, 2000)
    add(3, 5, 3, 3000, outliers=0.2)
    add(0, 3, 2, 2000, E=np.eye(3))
    R, _ = rel(1, 4)
    add(1, 4, 6, 2000, H=K[4] @ R @ np.linalg.inv(K[1]))
    add(0, 4, 2, 0)
    add(1, 5, 2, 1)
    add(2, 5, 6, 2)
    add(2, 4, 3, 2)
    for cfg in (0, 1, 7):
        add(0, 5, cfg, 50)
    add(0, 1, 2, BIG)
    kp_ptr = np.arange(NUM_IMAGES + 1, dtype=np.int64) * BIG
    counts = [p[6].shape[0] for p in pairs]
    return dict(keypoint_ptr=kp_ptr, keypoints=np.concatenate(kps), image_camera=cam_of.astype(np.int32), cameras=CAMS,
                pair_images=np.array([p[:2] for p in pairs], np.int32), config=np.array([p[2] for p in pairs], np.int32),
                E=np.array([p[3] for p in pairs]), F=np.array([p[4] for p in pairs]), H=np.array([p[5] for p in pairs]),
                inlier_ptr=np.concatenate([[0], np.cumsum(counts)]).astype(np.int64),
                inlier_matches=np.concatenate([p[6] for p in pairs]))


def _compare(dev, ref, min_kept_pairs=1):
    """Device result against the oracle's per-pair dicts; returns the number of pairs whose kept sets were compared
    through their median angle."""
    compared = 0
    for p, r in enumerate(ref):
        assert bool(dev.estimated[p]) == r["estimated"], p
        assert dev.config[p] == r["config"], p
        if not r["estimated"]:
            assert not dev.qvec[p].any() and not dev.tvec[p].any() and dev.tri_angle[p] == 0 and dev.num_points3D[p] == 0
            continue
        # the chosen candidate: its rotation (through the quaternion) and translation
        np.testing.assert_allclose(dev.qvec[p], r["qvec"], rtol=0, atol=1e-12, err_msg="pair %d" % p)
        np.testing.assert_allclose(dev.tvec[p], r["t"], rtol=0, atol=1e-12, err_msg="pair %d" % p)
        c = r["candidate"]
        near = int((r["margin"][:, c].min(axis=1) < 1e-9).sum()) if r["margin"].shape[1] else 0
        assert abs(int(dev.num_points3D[p]) - r["num_points3D"]) <= near, (p, dev.num_points3D[p], r["num_points3D"], near)
        if near == 0:
            assert dev.num_points3D[p] == r["num_points3D"]
            assert np.isclose(dev.tri_angle[p], r["tri_angle"], rtol=0, atol=1e-12, equal_nan=True), \
                (p, dev.tri_angle[p], r["tri_angle"])
            compared += r["num_points3D"] >= min_kept_pairs
    return compared


@pytest.mark.gpu
def test_device_equals_oracle_on_a_mixed_batch(gpu):
    args = _mixed_batch()
    dev = init_geometry.estimate_relative_poses(**args)
    ref = tv.estimate_relative_poses(**args)
    assert [r["candidate"] for r in ref][9] == 3                   # the pair without inliers: four tied candidates
    assert ref[8]["config"] == 5 and ref[8]["num_points3D"] == 0   # the pure rotation
    assert ref[-1]["num_points3D"] > 100_000
    # adjacent frames: points on both sides of max_depth
    assert 0 < ref[0]["num_points3D"] < 4000 and 0 < ref[-1]["num_points3D"] < BIG
    assert _compare(dev, ref) >= 8


@pytest.mark.gpu
def test_device_is_deterministic(gpu):
    args = _mixed_batch(seed=1)
    a = init_geometry.estimate_relative_poses(**args)
    b = init_geometry.estimate_relative_poses(**args)
    for k in ("qvec", "tvec", "tri_angle", "config", "num_points3D", "estimated"):
        assert np.array_equal(getattr(a, k), getattr(b, k), equal_nan=k in ("tri_angle",)), k


@pytest.mark.gpu
def test_device_launches_nothing_without_pairs_and_only_per_pair_kernels_without_inliers(gpu):
    L = _lib.lib()
    args = _mixed_batch()
    n0 = L.psfm_launch_count()
    empty = {**args, "pair_images": np.zeros((0, 2), np.int32), "config": np.zeros(0, np.int32), "E": np.zeros((0, 3, 3)),
             "F": np.zeros((0, 3, 3)), "H": np.zeros((0, 3, 3)), "inlier_ptr": np.zeros(1, np.int64),
             "inlier_matches": np.zeros((0, 2), np.uint32)}
    r = init_geometry.estimate_relative_poses(**empty)
    assert r.qvec.shape == (0, 4) and L.psfm_launch_count() == n0
    sel = [9, 0, 2, 13]                                          # no inliers, E, H, config 0
    no_inliers = {**args, "pair_images": args["pair_images"][sel], "config": args["config"][sel], "E": args["E"][sel],
                  "F": args["F"][sel], "H": args["H"][sel], "inlier_ptr": np.zeros(len(sel) + 1, np.int64),
                  "inlier_matches": np.zeros((0, 2), np.uint32)}
    dev = init_geometry.estimate_relative_poses(**no_inliers)
    assert L.psfm_launch_count() == n0 + 2
    _compare(dev, tv.estimate_relative_poses(**no_inliers))
    assert list(dev.estimated) == [True, True, True, False] and not dev.num_points3D.any() and not dev.tri_angle.any()


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["image", "camera", "keypoint"])
def test_device_refuses_out_of_range_indices(gpu, what):
    args = _mixed_batch()
    if what == "image":
        args["pair_images"] = args["pair_images"].copy()
        args["pair_images"][3, 1] = NUM_IMAGES
    elif what == "camera":
        args["image_camera"] = args["image_camera"].copy()
        args["image_camera"][2] = -1
    else:
        args["inlier_matches"] = args["inlier_matches"].copy()
        args["inlier_matches"][-1, 0] = BIG
    n0 = _lib.lib().psfm_launch_count()
    with pytest.raises(_lib.PsfmError, match="psfm_two_view_relative_poses: an? %s index" % what):
        init_geometry.estimate_relative_poses(**args)
    assert _lib.lib().psfm_launch_count() == n0


@pytest.mark.gpu
def test_database_end_to_end(gpu, tmp_path):
    """Synthetic scene -> tracks -> traj_to_matches_device -> import_keypoints_matches_arrays -> write_colmap_database,
    E of every pair from the true poses; read back, device against oracle."""
    nf = 8
    tracks, qvec, tvec, cam = syn.make_two_view_scene(3000, nf, 18000, seed=3)
    names = ["%05d.png" % i for i in range(nf)]
    ids = [nf - i for i in range(nf)]
    path = str(tmp_path / "database.db")
    db = sqlite3.connect(path)
    db.execute("CREATE TABLE cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, "
               "width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL)")
    db.execute("CREATE TABLE images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, "
               "camera_id INTEGER NOT NULL, prior_qw REAL, prior_qx REAL, prior_qy REAL, prior_qz REAL, prior_tx REAL, "
               "prior_ty REAL, prior_tz REAL)")
    db.execute("INSERT INTO cameras VALUES (1, 0, 1024, 436, ?, 0)", (np.asarray(cam, np.float64).tobytes(),))
    for n, i in zip(names, ids):
        db.execute("INSERT INTO images (image_id, name, camera_id) VALUES (?, ?, 1)", (i, n))
    db.commit()
    db.close()
    m = handoff.traj_to_matches_device(tracks, nf)
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), m, skip_geometric_verification=True)
    handoff.write_colmap_database(path, rows)
    db = sqlite3.connect(path)
    frame = {i: k for k, i in enumerate(ids)}
    for pid, in db.execute("SELECT pair_id FROM two_view_geometries").fetchall():
        a, b = handoff.pair_id_to_image_ids(pid)
        db.execute("UPDATE two_view_geometries SET E = ? WHERE pair_id = ?",
                   (syn.relative_essential(qvec, tvec, frame[a], frame[b]).tobytes(), pid))
    db.commit()
    db.close()
    g = handoff.read_two_view_geometries(path)
    assert g.inlier_matches.shape[0] == sum(x.shape[0] for _, x in rows.two_view)
    inputs = g.relative_pose_inputs()
    dev = init_geometry.estimate_relative_poses(**inputs)
    ref = tv.estimate_relative_poses(**inputs)
    assert dev.estimated.all() and (dev.num_points3D > 0).all()
    assert _compare(dev, ref) >= len(ref) // 2
    # the same arrays without the database round trip
    direct = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    d2 = init_geometry.estimate_relative_poses(**direct)
    order = np.argsort([pid for pid, _ in rows.matches])          # the database lists its pairs by pair_id
    assert np.array_equal(d2.num_points3D[order], dev.num_points3D) and np.array_equal(d2.qvec[order], dev.qvec)
