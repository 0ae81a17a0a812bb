"""Known answers for the numpy restatement of GlobalMapper::TriangulateAllPoints (oracle/triangulation_oracle.py), which
tests/test_gpu_triangulation.py compares the device against."""
import math

import numpy as np
import pytest

from oracle import triangulation_oracle as to
from particlesfm_b200 import handoff, synthetic as syn

FOCAL, W, H = 500.0, 640, 480


def ring_poses(F, radius=4.0, arc=1.2):
    """F cameras on an arc around the origin, looking at it (world-to-camera qvec / tvec)."""
    q, t = np.zeros((F, 4)), np.zeros((F, 3))
    for f in range(F):
        a = arc * (f / max(F - 1, 1) - 0.5)
        c = np.array([radius * math.sin(a), 0.1 * f, -radius * math.cos(a)])
        z = -c / np.linalg.norm(c)
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        q[f] = syn.rotmat_to_qvec(R)
        t[f] = -R @ c
    return q, t


def micro(X, seen, F, pairs=None, qt=None, shift=None):
    """Images 0 .. F-1 on a ring; point j is keypoint n of image f for every f in seen[j] (in point order); every pair
    of images (or `pairs`, in that order) matches the points both see.  shift: {(j, f): (dx, dy)} moves observations."""
    q, t = qt if qt is not None else ring_poses(F)
    kps = [[] for _ in range(F)]
    index = {}
    for j, fs in enumerate(seen):
        for f in fs:
            R = syn.qvec_to_rotmat(q[f])
            p = R @ X[j] + t[f]
            uv = FOCAL * p[:2] / p[2] + [W / 2, H / 2] + np.asarray((shift or {}).get((j, f), (0.0, 0.0)))
            index[(j, f)] = len(kps[f])
            kps[f].append(uv)
    pairs = pairs if pairs is not None else [(a, b) for a in range(F) for b in range(a + 1, F)]
    m, ptr = [], [0]
    for a, b in pairs:
        rows = [(index[(j, a)], index[(j, b)]) for j in range(len(seen)) if (j, a) in index and (j, b) in index]
        m.extend(rows)
        ptr.append(len(m))
    return dict(keypoint_ptr=np.concatenate([[0], np.cumsum([len(k) for k in kps])]).astype(np.int64),
                keypoints=np.array([u for k in kps for u in k], np.float32).reshape(-1, 2),
                image_camera=np.zeros(F, np.int32), cameras=np.array([[FOCAL, W / 2, H / 2]]),
                pair_images=np.array(pairs, np.int32).reshape(-1, 2), inlier_ptr=np.array(ptr, np.int64),
                inlier_matches=np.array(m, np.uint32).reshape(-1, 2), camera_size=np.array([[W, H]]), orientations=q,
                image_tvec=t, registered=np.ones(F, bool)), index


def scene(n_traj=300, n_frames=25, n_obs=4000, seed=3, noise_px=0.0, outliers=0.0, step=0.02):
    """make_two_view_scene on a helix through the hand-off: ParticleSfM's graph shape (one component per trajectory,
    anchor structure for trajectories longer than sample_k = 20), true poses."""
    tracks, qvec, tvec, cam = syn.make_two_view_scene(n_traj, n_frames, n_obs, seed=seed, step=step, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches(tracks, n_frames))
    a = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    db = {k: a[k] for k in ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr",
                            "inlier_matches")}
    if noise_px or outliers:
        db["keypoints"], _ = syn.corrupt_keypoints(db["keypoints"], outliers, seed=seed + 5, noise_px=noise_px)
    db.update(camera_size=np.array([[1024, 436]]), orientations=qvec, image_tvec=tvec, registered=np.ones(n_frames, bool))
    return db


def random_graph(seed=0, F=8, n_points=60):
    """A general graph: random visibility, several keypoints of one image in one component (points joined by shared
    keypoints across pairs), a few gross outliers."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1.0, 1.0, (n_points, 3))
    seen = [sorted(rng.choice(F, rng.integers(2, F + 1), replace=False).tolist()) for _ in range(n_points)]
    shift = {(j, f): tuple(rng.uniform(-40, 40, 2)) for j in range(n_points) for f in seen[j] if rng.random() < 0.08}
    db, index = micro(X, seen, F, shift=shift)
    # join points j and j + 1 through a wrong match between an image only j sees and one only j + 1 sees: their
    # components merge, with several keypoints of one image in the merged component
    pairs, ptr, m = db["pair_images"], db["inlier_ptr"], db["inlier_matches"].tolist()
    rows = [m[ptr[p]:ptr[p + 1]] for p in range(len(pairs))]
    for j in range(0, n_points - 1, 3):
        only_a = [f for f in seen[j] if f not in seen[j + 1]]
        only_b = [f for f in seen[j + 1] if f not in seen[j]]
        if only_a and only_b:
            a, b = only_a[0], only_b[0]
            p = [tuple(x) for x in pairs.tolist()].index((min(a, b), max(a, b)))
            ka, kb = index[(j, a)], index[(j + 1, b)]
            rows[p].append([ka, kb] if a < b else [kb, ka])
    db["inlier_matches"] = np.array([r for rr in rows for r in rr], np.uint32).reshape(-1, 2)
    db["inlier_ptr"] = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    return db, X


def reprojection_angles(db, ref):
    """Angular error of every track element against its point (true poses)."""
    kp = db["keypoints"].astype(np.float64)
    out = []
    for p in range(len(ref["xyz"])):
        for e in range(ref["track_ptr"][p], ref["track_ptr"][p + 1]):
            f, j = ref["track_image"][e], ref["track_point2D"][e]
            R = syn.qvec_to_rotmat(db["orientations"][f])
            r2 = R @ ref["xyz"][p] + db["image_tvec"][f]
            x = (kp[db["keypoint_ptr"][f] + j] - db["cameras"][0, 1:]) / db["cameras"][0, 0]
            out.append(float(to.angle_between(np.append(x, 1.0), r2)))
    return np.array(out)


def test_noise_free_tracks_give_one_point_each_at_the_truth():
    X = np.random.default_rng(1).uniform(-1, 1, (20, 3))
    db, _ = micro(X, [list(range(6))] * 20, 6)
    ref = to.triangulate_all_points(**db)
    assert ref["num_points3D"] == 20 and np.array_equal(np.diff(ref["track_ptr"]), np.full(20, 6))
    assert np.abs(ref["xyz"] - X).max() <= 1e-4            # float32 keypoints
    assert (ref["point3D_of_keypoint"] >= 0).all() and ref["num_continued"] == 0


def test_a_corrupted_observation_is_left_out_or_peeled_into_a_second_point():
    X = np.array([[0.1, 0.2, 0.3]])
    db, index = micro(X, [list(range(6))], 6, shift={(0, 3): (30.0, 0.0)})
    ref = to.triangulate_all_points(**db)
    # the five good observations form point 1; the corrupted one is alone and stays untriangulated
    assert ref["num_points3D"] == 1 and ref["track_ptr"][1] == 5 and 3 not in ref["track_image"].tolist()
    assert ref["point3D_of_keypoint"][db["keypoint_ptr"][3] + index[(0, 3)]] == -1
    # two corrupted observations that agree with each other become a second point (peel index 1)
    db, _ = micro(X, [list(range(8))], 8, qt=ring_poses(8, arc=2.0), shift={(0, 3): (40.0, 0.0), (0, 6): (40.0, 0.0)})
    ref = to.triangulate_all_points(**db, options={"ignore_two_view_tracks": False})
    assert ref["num_points3D"] >= 1 and ref["track_ptr"][1] == 6


def test_two_view_tracks_are_ignored_and_kept_with_the_option_off():
    X = np.array([[0.0, 0.0, 0.0], [0.3, -0.2, 0.1]])
    db, _ = micro(X, [[0, 5], [0, 3, 5]], 6)
    ref = to.triangulate_all_points(**db)
    assert ref["num_points3D"] == 1 and ref["track_ptr"][1] == 3
    ref = to.triangulate_all_points(**db, options={"ignore_two_view_tracks": False})
    assert ref["num_points3D"] == 2


def test_continue_attaches_below_its_bound_and_not_above_it():
    # image 1's observation creates the point from images 1 .. 4; image 5 matches only image 4, so its observation
    # finds a triangulated correspondence and continues the point when its error is within 2 degrees
    X = np.array([[0.1, 0.0, 0.2]])
    pairs = [(1, 2), (1, 3), (1, 4), (2, 3), (2, 4), (3, 4), (4, 5)]
    for dx, expect in ((5.0, 1), (40.0, 0)):            # 5 px ~ 0.57 deg, 40 px ~ 4.6 deg at f = 500
        db, _ = micro(X, [list(range(6))], 6, pairs=pairs, shift={(0, 5): (dx, 0.0)})
        ref = to.triangulate_all_points(**db)
        assert ref["num_continued"] == expect, dx


def test_unregistered_and_bogus_camera_images_are_skipped():
    X = np.random.default_rng(2).uniform(-1, 1, (5, 3))
    db, _ = micro(X, [list(range(5))] * 5, 5)
    db["registered"] = np.array([1, 1, 0, 1, 1], bool)
    ref = to.triangulate_all_points(**db)
    assert 2 not in ref["track_image"].tolist() and ref["track_ptr"][1] == 4
    # a second, bogus camera (principal point outside the image) for image 1
    db["image_camera"] = np.array([0, 1, 0, 0, 0], np.int32)
    db["cameras"] = np.array([[FOCAL, W / 2, H / 2], [FOCAL, W + 10.0, H / 2]])
    db["camera_size"] = np.array([[W, H], [W, H]])
    ref = to.triangulate_all_points(**db)
    assert not {1, 2} & set(ref["track_image"].tolist()) and ref["track_ptr"][1] == 3
    assert to.has_bogus_params([FOCAL, W / 2, H / 2], [W, H], to.DEFAULTS) is False
    assert to.has_bogus_params([0.05 * W, W / 2, H / 2], [W, H], to.DEFAULTS) is True
    assert to.has_bogus_params([11.0 * W, W / 2, H / 2], [W, H], to.DEFAULTS) is True


def test_duplicate_matches_follow_the_correspondence_graph_rule():
    kp_ptr = np.array([0, 3, 6])
    ptr, nbr = to.build_graph(kp_ptr, np.array([[0, 1]]), np.array([0, 4]),
                              np.array([[0, 0], [0, 1], [1, 1], [1, 0]]), None)
    # (0, 1) repeats point 0 of image 0: dropped, so it does not block (1, 1); (1, 0) repeats both: dropped
    assert ptr.tolist() == [0, 1, 2, 2, 3, 4, 4] and nbr.tolist() == [3, 4, 0, 1]
    ptr, nbr = to.build_graph(kp_ptr, np.array([[0, 1]]), np.array([0, 2]), np.array([[0, 0], [1, 2]]), np.array([0]))
    assert ptr[-1] == 0


def test_trial_counts_exhaustive_and_compute_num_trials():
    assert to.compute_num_trials(10, 10, 0.9999, 3.0) == 1
    assert to.compute_num_trials(0, 10, 0.9999, 3.0) == to.UNBOUNDED
    r = 0.5
    assert to.compute_num_trials(5, 10, 0.9999, 3.0) == math.ceil(math.log(1e-4) / math.log(1 - r * r) * 3.0)
    assert to.max_num_trials_cap() == 10000
    assert [to.combination(t, 4) for t in range(6)] == [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    X = np.array([[0.1, 0.0, 0.2]])
    for m in (3, 6, 15, 16):
        db, _ = micro(X, [list(range(m))], m, qt=ring_poses(m, arc=2.0))
        ref = to.triangulate_all_points(**db)
        if m <= 15:
            assert ref["num_ransac_trials"] == m * (m - 1) // 2, m
        else:        # every observation an inlier: ComputeNumTrials = 1, the loop stops after trial index 1
            assert ref["num_ransac_trials"] == 2, m


def test_point_ids_follow_creation_order():
    X = np.random.default_rng(4).uniform(-1, 1, (6, 3))
    seen = [[2, 3, 4], [0, 1, 2], [1, 3, 4], [0, 2, 4], [3, 4, 5], [0, 5, 1]]
    db, index = micro(X, seen, 6)
    ref = to.triangulate_all_points(**db)
    creators = [min(int(db["keypoint_ptr"][f]) + index[(j, f)] for f in seen[j]) for j in range(6)]
    order = np.argsort(creators)
    assert ref["num_points3D"] == 6
    assert np.abs(ref["xyz"] - X[order]).max() <= 1e-4


def test_per_component_replay_equals_the_global_pass():
    db, _ = random_graph(seed=5)
    a = to.triangulate_all_points(**db)
    b = to.triangulate_all_points(**db, per_component=True)
    assert a["num_points3D"] > 10
    assert a["largest_component"] > 8          # more observations than images: joined points
    for k in ("xyz", "track_ptr", "track_image", "track_point2D", "point3D_of_keypoint"):
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("change, exc", [
    (dict(options={"create_max_angle_error": 0.0}), to.InvalidError),
    (dict(options={"max_transitivity": 2}), to.UnsupportedError),
    (dict(camera_size=np.array([[0, 480]])), to.InvalidError),
])
def test_argument_rules(change, exc):
    db, _ = micro(np.zeros((1, 3)), [[0, 1, 2]], 3)
    db.update(change)
    with pytest.raises(exc):
        to.triangulate_all_points(**db)


def test_database_read_gives_camera_sizes_and_image_names(tmp_path):
    from test_oracle_two_view import _write_database
    path = str(tmp_path / "db.sqlite")
    _, ids = _write_database(path)
    g = handoff.read_two_view_geometries(path)
    assert g.camera_size.tolist() == [[640, 480], [640, 480]]
    # image_id k was written with name %05d of its position; read back in image_id order
    names = {k: "%05d.png" % i for i, k in enumerate(ids)}
    assert g.image_names == [names[int(i)] for i in g.image_ids]
    assert set(handoff.TwoViewGeometries.FIELDS) <= set(vars(g))
