"""psfm_verify_two_view_geometries on the device against the numpy restatement (oracle/verification_oracle.py): equal
configs, inlier matches and trial counts, F and H to 1e-9, with every oracle decision clear of rounding; determinism;
and the device chain from matches to a refined model without a colmap call."""
import numpy as np
import pytest

from oracle import verification_oracle as vo
from particlesfm_b200 import ba, colmap_io, handoff, init_geometry, synthetic as syn
from test_oracle_verification import pair_tables, scene_tables, two_views, W, H

pytestmark = pytest.mark.gpu

# the smallest relative margin each kind of oracle decision must keep, so that the device's rounding cannot flip it
BANDS = {"threshold": 1e-9, "compare": 1e-9, "cubic": 1e-12, "num_trials": 1e-13, "f22": 1e-6, "order": 1e-9}


def _compare(mt, f_not_unique=(), **o):
    """f_not_unique: the pairs whose points lie on a plane or only translate in the image, where F's null space has
    more than one dimension and any F of it is as good; only F's inlier decisions are compared there (the local step's
    rounds depend on which F it takes, so their count is not compared either)."""
    ref = vo.verify_two_view_geometries(**mt.verification_inputs(), options=o)
    for k, v in ref["margins"].items():
        assert v > BANDS[k], (k, v)
    dev = init_geometry.verify_two_view_geometries(**mt.verification_inputs(),
                                                   options=init_geometry.TwoViewVerificationOptions(**o))
    assert np.array_equal(dev.config, ref["config"])
    assert np.array_equal(dev.inlier_ptr, ref["inlier_ptr"]) and np.array_equal(dev.inlier_matches, ref["inlier_matches"])
    assert np.array_equal(dev.trials, ref["trials"])
    for name in ("F", "H"):
        d, r = dev.__dict__[name].reshape(-1, 9), ref[name]
        if name == "F":
            keep = np.setdiff1d(np.arange(len(r)), f_not_unique)
            d, r = d[keep], r[keep]
        if len(r):
            assert np.abs(d - r).max() <= 1e-9, (name, np.abs(d - r).max(axis=1))
    assert not dev.E.any()
    s = dev.summary
    assert s["num_trials"] == ref["trials"].sum(0).tolist() and s["num_trials_scored"] == s["num_trials"]
    if not len(f_not_unique):
        assert s["num_local_rounds"] == ref["local_rounds"].sum(0).tolist()
    assert s["num_config"] == np.bincount(ref["config"], minlength=8).tolist() and s["num_launches"] == 3
    return dev, ref


def test_line_path(gpu):
    _, ref = _compare(scene_tables(300, 5, 1500, seed=3))
    assert (ref["config"] == vo.PLANAR_OR_PANORAMIC).all()


def test_helix_path(gpu):
    _, ref = _compare(scene_tables(300, 5, 1500, seed=3, step=0.08, path="helix", noise_px=0.5))
    assert (ref["config"] == vo.UNCALIBRATED).sum() >= 8


def test_planar_scene(gpu):
    _, ref = _compare(pair_tables([two_views(200, s, plane=True)[:2] for s in range(4)]), f_not_unique=range(4))
    assert (ref["config"] == vo.PLANAR_OR_PANORAMIC).all()


@pytest.mark.parametrize("fraction", [0.1, 0.3])
def test_outliers(gpu, fraction):
    _, ref = _compare(scene_tables(400, 5, 2000, seed=5, step=0.08, path="helix", outliers=fraction, noise_px=0.5))
    assert (ref["local_rounds"][:, 0] > 0).any()


def test_mixed_batch_and_determinism(gpu):
    rng = np.random.default_rng(0)
    few = rng.random((14, 2)) * [W, H]
    border = np.concatenate([rng.random((40, 1)) * 90, rng.random((40, 1)) * H], 1)
    x1, x2, _, _ = two_views(80, 6)
    mt = pair_tables([(few, few + 1), (np.zeros((0, 2)), np.zeros((0, 2))), (border, border + [4.0, -2.0]), (x1, x2)])
    dev, ref = _compare(mt, f_not_unique=[2])
    assert ref["config"].tolist() == [vo.UNDEFINED, vo.UNDEFINED, vo.WATERMARK, vo.UNCALIBRATED]
    again = init_geometry.verify_two_view_geometries(**mt.verification_inputs())
    for k in ("config", "F", "H", "inlier_ptr", "inlier_matches", "trials"):
        assert np.array_equal(getattr(again, k), getattr(dev, k)), k
    big = scene_tables(400, 6, 2400, seed=9, step=0.08, path="helix", outliers=0.2, noise_px=0.5)
    a = init_geometry.verify_two_view_geometries(**big.verification_inputs())
    b = init_geometry.verify_two_view_geometries(**big.verification_inputs())
    for k in ("config", "F", "H", "inlier_ptr", "inlier_matches", "trials"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k


def test_chain_from_matches_to_a_refined_model(gpu, tmp_path):
    n_frames = 10
    tracks, qvec, tvec, cam = syn.make_two_view_scene(1500, n_frames, 9000, seed=7, step=0.08, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, n_frames))
    mt = handoff.MatchTables.from_rows(rows, ids, names, cam, (1024, 436))
    mt.keypoints = syn.corrupt_keypoints(mt.keypoints, 0.1, seed=7, noise_px=0.3)[0]
    ver = init_geometry.verify_two_view_geometries(**mt.verification_inputs())
    assert (ver.config != vo.DEGENERATE).all()
    g = ver.to_two_view_geometries(mt)
    poses = init_geometry.estimate_relative_poses(**g.relative_pose_inputs())
    rot = init_geometry.estimate_global_rotations(n_frames, g.pair_images, poses.qvec, np.diff(g.inlier_ptr),
                                                  has_pose=poses.estimated)
    db = {k: getattr(g, k) for k in ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr",
                                     "inlier_matches")}
    t = init_geometry.optimize_pairwise_translations(**db, orientations=rot.orientations, pair_used=rot.pair_kept)
    pos = init_geometry.estimate_global_positions(n_frames, g.pair_images, t, rot.orientations,
                                                  has_orientation=rot.has_orientation, pair_used=rot.pair_kept)
    tri = init_geometry.triangulate_all_points(**db, camera_size=g.camera_size, orientations=rot.orientations,
                                               image_tvec=pos.image_tvec, registered=pos.has_position)
    assert tri.summary["num_points3D"] > 100
    rec = tri.to_reconstruction(g.image_ids, g.image_names, g.camera_ids)
    ba.iterative_global_refinement(rec, False)
    ba.iterative_global_refinement(rec, True)
    truth = syn.camera_centres(qvec, tvec)[pos.has_position]
    q = np.array([rec.images[i].qvec for i in ids if i in rec.images])
    tv = np.array([rec.images[i].tvec for i in ids if i in rec.images])
    extent = np.linalg.norm(truth - truth.mean(0), axis=1).max()
    assert syn.umeyama_ate(syn.camera_centres(q, tv), truth) <= 0.05 * extent
    colmap_io.write_model(rec, str(tmp_path))
    back = colmap_io.read_model(str(tmp_path))
    assert sorted(back.images) == sorted(rec.images) and sorted(back.points3D) == sorted(rec.points3D)
