"""TriangulateAllPoints on the GPU (init_geometry.triangulate_all_points, csrc/triangulation.cu) against the numpy
restatement of the reference loop (oracle/triangulation_oracle.py, pinned by tests/test_oracle_triangulation.py), and
the device chain from database rows to a refined model."""
import numpy as np
import pytest

from oracle import triangulation_oracle as to
from particlesfm_b200 import ba, colmap_io, handoff, init_geometry, launch_count, synthetic as syn
from test_oracle_triangulation import random_graph, scene

pytestmark = pytest.mark.gpu

COUNTS = ("num_components", "largest_component", "num_points3D", "num_continued", "num_ransac_trials",
          "num_local_estimates")


def _fixture(name):
    if name == "scene":
        return scene(300, 25, 4000, seed=3)
    if name == "noise_outliers":
        return scene(300, 25, 4000, seed=4, noise_px=0.5, outliers=0.05)
    if name == "unregistered_bogus":
        db = scene(250, 26, 3500, seed=5, noise_px=0.5, outliers=0.05)
        db["registered"] = db["registered"].copy()
        db["registered"][[3, 11]] = False
        db["orientations"] = db["orientations"].copy()
        db["orientations"][11] = np.nan                # an unregistered image's pose is never read
        db["image_camera"] = np.where(np.arange(26) == 7, 1, 0).astype(np.int32)
        db["cameras"] = np.array([db["cameras"][0], [db["cameras"][0][0], 1100.0, 218.0]])     # cx > width: bogus
        db["camera_size"] = np.array([[1024, 436], [1024, 436]])
        return db
    if name == "far_points":                            # short baselines: most tracks stay below min_angle
        return scene(300, 30, 5000, seed=6, noise_px=0.3, step=0.006)
    if name == "random_graph":
        return random_graph(seed=5, F=10, n_points=150)[0]
    raise KeyError(name)


def _assert_margins(ref):
    """Every threshold decision of the restatement is decided with margin, so rounding cannot flip it on the device."""
    for kind, m in ref["margins"].items():
        assert m > 1e-7, (kind, m)


def _compare(dev, ref, db):
    assert dev.xyz.shape[0] == ref["num_points3D"]
    assert np.array_equal(dev.point3D_of_keypoint, ref["point3D_of_keypoint"])
    for k in ("track_ptr", "track_image", "track_point2D"):
        assert np.array_equal(getattr(dev, k), ref[k]), k
    if ref["num_points3D"]:
        reg = np.asarray(db["registered"], bool)
        R = np.array([syn.qvec_to_rotmat(q) for q in np.asarray(db["orientations"])[reg]])
        centres = -np.einsum("fji,fj->fi", R, np.asarray(db["image_tvec"])[reg])
        extent = max(np.linalg.norm(ref["xyz"] - centres.mean(0), axis=1).max(),
                     np.linalg.norm(centres - centres.mean(0), axis=1).max())
        assert np.abs(dev.xyz - ref["xyz"]).max() <= 1e-9 * extent
    for k in COUNTS:
        assert dev.summary[k] == ref[k], (k, dev.summary[k], ref[k])


@pytest.mark.parametrize("name", ["scene", "noise_outliers", "unregistered_bogus", "far_points", "random_graph"])
def test_device_matches_the_restatement(gpu, name):
    db = _fixture(name)
    ref = to.triangulate_all_points(**db)
    _assert_margins(ref)
    assert ref["num_points3D"] > 5
    if name in ("scene", "noise_outliers"):
        assert ref["largest_component"] > 20          # trajectories longer than sample_k: anchor structure
    n0 = launch_count()
    dev = init_geometry.triangulate_all_points(**db)
    assert dev.summary["num_launches"] == launch_count() - n0
    _compare(dev, ref, db)
    again = init_geometry.triangulate_all_points(**db)
    for k in ("xyz", "track_ptr", "track_image", "track_point2D", "point3D_of_keypoint"):
        assert np.array_equal(getattr(again, k), getattr(dev, k)), k
    assert again.summary["num_launches"] == dev.summary["num_launches"]


def test_unused_pairs_leave_the_graph(gpu):
    db = scene(200, 25, 3000, seed=8, noise_px=0.5)
    used = np.arange(len(db["pair_images"])) % 5 != 1
    ref = to.triangulate_all_points(**db, pair_used=used)
    _assert_margins(ref)
    dev = init_geometry.triangulate_all_points(**db, pair_used=used)
    _compare(dev, ref, db)


DB = ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr", "inlier_matches")


def test_chain_from_database_rows_to_a_refined_model(gpu, tmp_path):
    n_frames = 10
    tracks, qvec, tvec, cam = syn.make_two_view_scene(1500, n_frames, 9000, seed=7, step=0.08, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, n_frames))
    args = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    poses = init_geometry.estimate_relative_poses(**args)
    rot = init_geometry.estimate_global_rotations(n_frames, args["pair_images"], poses.qvec, np.diff(args["inlier_ptr"]),
                                                  has_pose=poses.estimated)
    db = {k: args[k] for k in DB}
    t = init_geometry.optimize_pairwise_translations(**db, orientations=rot.orientations, pair_used=rot.pair_kept)
    pos = init_geometry.estimate_global_positions(n_frames, args["pair_images"], t, rot.orientations,
                                                  has_orientation=rot.has_orientation, pair_used=rot.pair_kept)
    tri = init_geometry.triangulate_all_points(**db, camera_size=np.array([[1024, 436]]), orientations=rot.orientations,
                                               image_tvec=pos.image_tvec, registered=pos.has_position)
    assert tri.summary["num_points3D"] > 100
    rec = tri.to_reconstruction(ids, names, [1])
    assert rec.RegImageIds() == sorted(rec.images) and sorted(rec.points3D) == list(range(1, tri.xyz.shape[0] + 1))
    truth = syn.camera_centres(qvec, tvec)
    have = pos.has_position

    def ate():
        q = np.array([rec.images[i].qvec for i in ids if i in rec.images])
        tv = np.array([rec.images[i].tvec for i in ids if i in rec.images])
        return syn.umeyama_ate(syn.camera_centres(q, tv), truth[have])
    before = ate()
    ba.iterative_global_refinement(rec, False)
    ba.iterative_global_refinement(rec, True)
    after = ate()
    extent = np.linalg.norm(truth - truth.mean(0), axis=1).max()
    assert after <= 0.02 * extent and after <= before + 1e-9 * extent, (before, after, extent)
    colmap_io.write_model(rec, str(tmp_path))
    back = colmap_io.read_model(str(tmp_path))
    imgs, pts = back.images, back.points3D
    assert sorted(imgs) == sorted(rec.images) and sorted(pts) == sorted(rec.points3D)
    for pid in list(rec.points3D)[:50]:
        assert np.array_equal(pts[pid].xyz, rec.points3D[pid].xyz)
        assert np.array_equal(pts[pid].image_ids, rec.points3D[pid].image_ids)
