"""Known-answer tests of the relative-pose restatement (oracle/two_view_oracle.py), the database reader
(handoff.read_two_view_geometries) and the argument checks of psfm_two_view_relative_poses.  No GPU needed."""
import sqlite3

import numpy as np
import pytest

from oracle import two_view_oracle as tv
from particlesfm_b200 import _lib, handoff, init_geometry, synthetic as syn

CAM1 = np.array([520.0, 320.0, 240.0])
CAM2 = np.array([480.0, 300.0, 250.0])


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _scene(n=60, seed=0, baseline=(0.3, -0.05, 0.1)):
    rng = np.random.default_rng(seed)
    R = syn.axis_angle_to_rotmat(np.array([0.05, -0.12, 0.03]))
    t = np.array(baseline, np.float64)
    X = np.c_[rng.uniform(-2, 2, (n, 2)), rng.uniform(4, 10, n)]
    return R, t, X


def _project(cam, X):
    return cam[0] * X[:, :2] / X[:, 2:] + cam[1:]


def _views(R, t, X):
    return _project(CAM1, X), _project(CAM2, X @ R.T + t)


def test_essential_matrix_recovers_the_pose_and_keeps_every_point():
    R, t, X = _scene()
    xy1, xy2 = _views(R, t, X)
    r = tv.estimate_relative_pose(2, _skew(t) @ R, np.eye(3), np.eye(3), CAM1, CAM2, xy1, xy2)
    assert r["estimated"] and r["config"] == 2
    np.testing.assert_allclose(r["R"], R, atol=1e-12)
    np.testing.assert_allclose(r["t"], t / np.linalg.norm(t), atol=1e-12)
    assert r["num_points3D"] == len(X) and r["counts"].max() == len(X) and (r["counts"] == len(X)).sum() == 1
    np.testing.assert_allclose(r["qvec"], syn.rotmat_to_qvec(R), atol=1e-12)
    ang = np.arccos(np.einsum("ij,ij->i", X, X - (-R.T @ t)) / np.linalg.norm(X, axis=1) / np.linalg.norm(X + R.T @ t, axis=1))
    assert abs(r["tri_angle"] - np.median(np.minimum(ang, np.pi - ang))) < 1e-12


def test_fundamental_matrix_goes_through_the_calibrations():
    R, t, X = _scene(seed=1)
    xy1, xy2 = _views(R, t, X)
    K1, K2 = tv.calibration(CAM1), tv.calibration(CAM2)
    F = np.linalg.inv(K2).T @ _skew(t) @ R @ np.linalg.inv(K1)
    r = tv.estimate_relative_pose(3, np.zeros((3, 3)), F * 7.0, np.eye(3), CAM1, CAM2, xy1, xy2)
    assert r["config"] == 3 and r["num_points3D"] == len(X)
    np.testing.assert_allclose(r["R"], R, atol=1e-12)
    np.testing.assert_allclose(r["t"], t / np.linalg.norm(t), atol=1e-12)


def test_plane_induced_homography_recovers_the_pose():
    R, t, _ = _scene()
    rng = np.random.default_rng(3)
    nrm = np.array([0.1, -0.2, 1.0])
    nrm /= np.linalg.norm(nrm)
    d = 6.0
    uv = rng.uniform(-2, 2, (50, 2))
    X = np.c_[uv, (d - uv @ nrm[:2]) / nrm[2]]                      # n' X = d
    xy1, xy2 = _views(R, t, X)
    K1, K2 = tv.calibration(CAM1), tv.calibration(CAM2)
    H = K2 @ (R + np.outer(t, nrm) / d) @ np.linalg.inv(K1)
    r = tv.estimate_relative_pose(6, np.eye(3), np.eye(3), H * 0.3, CAM1, CAM2, xy1, xy2)
    assert r["config"] == 4 and r["num_points3D"] == len(X)
    np.testing.assert_allclose(r["R"], R, atol=1e-12)
    np.testing.assert_allclose(r["t"], t / d, atol=1e-12)
    assert r["tri_angle"] > 0


def test_pure_rotation_homography_is_panoramic_with_candidate_zero():
    R, _, X = _scene()
    xy1, xy2 = _views(R, np.zeros(3), X)
    H = tv.calibration(CAM2) @ R @ np.linalg.inv(tv.calibration(CAM1))
    for cfg, out_cfg in ((6, 5), (4, 4), (5, 5)):
        r = tv.estimate_relative_pose(cfg, np.eye(3), np.eye(3), H, CAM1, CAM2, xy1, xy2)
        assert r["config"] == out_cfg and r["candidate"] == 0 and list(r["counts"]) == [0]
        np.testing.assert_allclose(r["R"], R, atol=1e-12)
        assert not r["t"].any() and r["tri_angle"] == 0.0 and r["num_points3D"] == 0


def test_skip_verification_pair_with_identity_e():
    """write_colmap_database's skip-verification rows: config 2, E = I.  Candidates W, W', +-e3."""
    c = tv.decompose_essential_matrix(np.eye(3))
    e3 = np.array([0.0, 0.0, 1.0])
    for (R, t), (R0, t0) in zip(c, [(tv.W, e3), (tv.W.T, e3), (tv.W, -e3), (tv.W.T, -e3)]):
        assert np.array_equal(R, R0) and np.array_equal(t, t0)
    R, t, X = _scene(n=30)
    xy1, xy2 = _views(R, t, X)
    r = tv.estimate_relative_pose(2, np.eye(3), np.eye(3), np.eye(3), CAM1, CAM2, xy1, xy2)
    best = int(np.nonzero(r["counts"] == r["counts"].max())[0][-1])            # ties: the later candidate
    assert r["candidate"] == best and r["num_points3D"] == r["counts"].max()
    assert np.array_equal(r["R"], c[best][0]) and np.array_equal(r["t"], c[best][1])


def test_essential_candidate_order_does_not_depend_on_the_svd_signs():
    R, t, _ = _scene()
    E = _skew(t) @ R
    ref = tv.decompose_essential_matrix(E)
    for s in (-1.0, 5.0, -0.01):
        for (Ra, ta), (Rb, tb) in zip(tv.decompose_essential_matrix(E * s), ref):
            np.testing.assert_allclose(Ra, Rb, atol=1e-12)
            np.testing.assert_allclose(ta, tb, atol=1e-12)
    assert np.trace(ref[0][0]) >= np.trace(ref[1][0])
    assert ref[0][1][np.argmax(np.abs(ref[0][1]))] > 0


def test_ties_and_empty_pairs():
    R, t, _ = _scene()
    empty = np.zeros((0, 2))
    r = tv.estimate_relative_pose(2, _skew(t) @ R, None, None, CAM1, CAM2, empty, empty)
    assert r["candidate"] == 3 and r["num_points3D"] == 0 and r["tri_angle"] == 0.0   # >=: the last of four ties
    H = tv.calibration(CAM2) @ (R + np.outer(t, [0, 0, 1.0]) / 5.0) @ np.linalg.inv(tv.calibration(CAM1))
    r = tv.estimate_relative_pose(6, None, None, H, CAM1, CAM2, empty, empty)
    assert r["candidate"] == 0 and r["config"] == 4 and r["tri_angle"] == 0.0         # nothing kept: candidate 0


@pytest.mark.parametrize("values,expected", [([3.0], 3.0), ([5.0, 1.0, 3.0], 3.0), ([4.0, 1.0], 2.5),
                                             ([9.0, 1.0, 4.0, 2.0], 3.0), ([2.0, 2.0, 7.0, 1.0, 0.5, 3.0], 2.0)])
def test_median_odd_and_even(values, expected):
    assert tv.median(values) == expected


@pytest.mark.parametrize("axis_angle", [(0.1, 0.2, -0.3),            # trace > 0
                                        (np.pi * 0.9, 0, 0),          # i = 0
                                        (0, np.pi * 0.9, 0.1),        # i = 1
                                        (0.1, 0, np.pi * 0.9),        # i = 2
                                        (np.pi, 0, 0), (0, 0, np.pi)])
def test_quaternion_every_branch(axis_angle):
    R = syn.axis_angle_to_rotmat(np.array(axis_angle, np.float64))
    q = tv.rotation_matrix_to_quaternion(R)
    np.testing.assert_allclose(np.abs(q), np.abs(syn.rotmat_to_qvec(R)), atol=1e-12)
    np.testing.assert_allclose(syn.qvec_to_rotmat(q), R, atol=1e-12)


@pytest.mark.parametrize("config", [0, 1, 7, 8])
def test_other_configs_pass_through(config):
    R, t, X = _scene(n=10)
    xy1, xy2 = _views(R, t, X)
    r = tv.estimate_relative_pose(config, _skew(t) @ R, np.eye(3), np.eye(3), CAM1, CAM2, xy1, xy2)
    assert not r["estimated"] and r["config"] == config and not r["qvec"].any() and r["num_points3D"] == 0


def test_margins_flag_points_near_max_depth():
    R, t, _ = _scene()
    t = t / np.linalg.norm(t)
    X = np.array([[0.1, 0.2, 999.0], [0.0, 0.0, 5.0], [0.3, -0.1, 1000.0 * (1 + 1e-12)]])
    xy1, xy2 = tv.image_to_world(CAM1, _project(CAM1, X)), tv.image_to_world(CAM2, _project(CAM2, X @ R.T + t))
    kept, _, margin = tv.check_cheirality(R, t, xy1, xy2)
    assert kept[1] and margin[1].min() > 1e-3
    assert margin[2].min() < 1e-9


def _write_database(path, num_images=6):
    """A database as the pipeline fills it: cameras and images (COLMAP's schema), then write_colmap_database."""
    rng = np.random.default_rng(7)
    names = ["%05d.png" % i for i in range(num_images)]
    ids = [num_images - i + 3 for i in range(num_images)]
    db = sqlite3.connect(path)
    db.execute("CREATE TABLE cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, "
               "width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL)")
    db.execute("CREATE TABLE images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, "
               "camera_id INTEGER NOT NULL, prior_qw REAL, prior_qx REAL, prior_qy REAL, prior_qz REAL, prior_tx REAL, "
               "prior_ty REAL, prior_tz REAL)")
    db.execute("INSERT INTO cameras VALUES (?, ?, ?, ?, ?, ?)", (3, 0, 640, 480, CAM1.tobytes(), 0))
    db.execute("INSERT INTO cameras VALUES (?, ?, ?, ?, ?, ?)", (9, 0, 640, 480, CAM2.tobytes(), 0))
    for i, (n, k) in enumerate(zip(names, ids)):
        db.execute("INSERT INTO images (image_id, name, camera_id) VALUES (?, ?, ?)", (k, n, 3 if i % 2 else 9))
    db.commit()
    db.close()
    tracks = syn.make_track_arrays(300, num_images, 1200, seed=5)
    tracks.xy = rng.random(tracks.xy.shape) * 600
    m = handoff.traj_to_matches(tracks, num_images)
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), m, skip_geometric_verification=True)
    handoff.write_colmap_database(path, rows)
    return rows, ids


def test_database_reads_back_as_written(tmp_path):
    path = str(tmp_path / "db.sqlite")
    rows, ids = _write_database(path)
    g = handoff.read_two_view_geometries(path)
    assert list(g.image_ids) == sorted(ids) and list(g.camera_ids) == [3, 9]
    np.testing.assert_array_equal(g.cameras, np.stack([CAM1, CAM2]))
    kp = dict(rows.keypoints)
    for f, i in enumerate(g.image_ids):
        assert np.array_equal(g.keypoints[g.keypoint_ptr[f]:g.keypoint_ptr[f + 1]], kp[int(i)])
    by_pair = dict(rows.two_view)
    assert list(g.pair_ids) == sorted(by_pair)
    for p, pid in enumerate(g.pair_ids):
        a, b = g.image_ids[g.pair_images[p]]
        assert a < b and handoff.image_ids_to_pair_id(int(a), int(b)) == pid
        assert np.array_equal(g.inlier_matches[g.inlier_ptr[p]:g.inlier_ptr[p + 1]], by_pair[int(pid)])
    assert (g.config == 2).all() and all((m == np.eye(3)).all() for m in (*g.E, *g.F, *g.H))
    assert g.inlier_matches.dtype == np.uint32 and g.keypoints.dtype == np.float32
    # image -> camera follows the images table
    cam_of = {k: (3 if i % 2 else 9) for i, k in enumerate(ids)}
    assert [int(g.camera_ids[c]) for c in g.image_camera] == [cam_of[int(i)] for i in g.image_ids]
    assert set(g.relative_pose_inputs()) == set(handoff.TwoViewGeometries.FIELDS)


def test_oracle_batch_matches_single_pair_calls(tmp_path):
    path = str(tmp_path / "db.sqlite")
    _write_database(path)
    g = handoff.read_two_view_geometries(path)
    res = tv.estimate_relative_poses(**g.relative_pose_inputs())
    assert len(res) == len(g.pair_ids) and all(r["estimated"] for r in res)


def test_abi_checks_arguments_then_refuses_without_a_device():
    if _lib.lib().psfm_device_count() > 0:
        pytest.skip("a CUDA device is present: tests/test_gpu_two_view.py covers the call")
    R, t, X = _scene(n=8)
    xy1, xy2 = _views(R, t, X)
    args = dict(keypoint_ptr=[0, 8, 16], keypoints=np.r_[xy1, xy2], image_camera=[0, 0], cameras=[CAM1],
                pair_images=[[0, 1]], config=[2], E=[_skew(t) @ R], F=[np.eye(3)], H=[np.eye(3)], inlier_ptr=[0, 8],
                inlier_matches=np.c_[np.arange(8), np.arange(8)])
    with pytest.raises(_lib.PsfmError, match="status -2"):
        init_geometry.estimate_relative_poses(**args)
    for key, bad, what in (("pair_images", [[0, 2]], "image index"), ("image_camera", [0, 1], "camera index"),
                           ("inlier_matches", np.c_[np.arange(8), np.arange(1, 9)], "keypoint index")):
        with pytest.raises(_lib.PsfmError, match="psfm_two_view_relative_poses: .*" + what):
            init_geometry.estimate_relative_poses(**{**args, key: bad})
