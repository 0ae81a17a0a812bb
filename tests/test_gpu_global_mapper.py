"""The global mapper on the device: the triangulation -> bundle-adjustment hand-off against ba.flatten of
Triangulation.to_reconstruction, the mapper's model against the Python route (the same stages with the database cache,
then to_reconstruction and ba.iterative_global_refinement), and the command line from a real SQLite database to
OUT/0."""
import os
import sqlite3

import numpy as np
import pytest

from particlesfm_b200 import ba, colmap_io, global_mapper as gm, handoff, init_geometry, synthetic as syn

pytestmark = pytest.mark.gpu

W, H = 1024, 436


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


@pytest.fixture(scope="module")
def scene(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("mapper") / "database.db")
    qvec, tvec = _scene_db(path)
    return path, qvec, tvec


def _stages(path, o):
    g, used = handoff.load_database_cache(path, o.min_num_matches, o.ignore_watermarks)
    staged = gm.poses_and_points(g, used, o, gm.MapperReport())
    assert staged is not None
    return (g,) + staged


def _triangulation_args(g, used, rot, image_tvec, registered):
    db = {k: getattr(g, k) for k in ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr",
                                     "inlier_matches")}
    return dict(db, camera_size=g.camera_size, orientations=rot.orientations, image_tvec=image_tvec, registered=registered,
                pair_used=used)


def _check_handoff(g, used, rot, image_tvec, registered):
    args = _triangulation_args(g, used, rot, image_tvec, registered)
    tri = init_geometry.triangulate_all_points(**args)
    rec = tri.to_reconstruction(g.image_ids, g.image_names, g.camera_ids)
    cfg = ba.BundleAdjustmentConfig()
    for i in rec.RegImageIds():
        cfg.AddImage(i)
    prob, maps = ba.flatten(rec, cfg)
    res = init_geometry.triangulate_all_points_resident(**args)
    try:
        S = ba.TriangulationSolver(res, rot.orientations, image_tvec, g.cameras)
    finally:
        res.close()
    try:
        img, pt, xy, p2d = S.observations()
    finally:
        S.close()
    assert S.num_observations == prob.num_observations and S.num_images == prob.num_images
    assert np.array_equal(img, prob.obs_image) and np.array_equal(pt, prob.obs_point)
    assert np.array_equal(xy, prob.obs_xy) and np.array_equal(p2d, maps["obs_point2D_idx"])
    return tri


def test_handoff_equals_flatten(gpu, scene):
    g, used, rot, pos, res = _stages(scene[0], gm.GlobalMapperOptions())
    res.close()
    tri = _check_handoff(g, used, rot, pos.image_tvec, pos.has_position)
    assert tri.summary["num_points3D"] > 100


def test_handoff_with_unregistered_images_and_untriangulated_keypoints(gpu, scene):
    g, used, rot, pos, res = _stages(scene[0], gm.GlobalMapperOptions())
    res.close()
    reg = pos.has_position.copy()
    reg[[2, 5]] = False
    tri = _check_handoff(g, used, rot, pos.image_tvec, reg)
    f = np.repeat(np.arange(len(reg)), np.diff(g.keypoint_ptr))
    assert (tri.point3D_of_keypoint[reg[f]] < 0).any() and (tri.point3D_of_keypoint[~reg[f]] < 0).all()


def test_model_of_filtered_observations_equals_apply_observation_mask(gpu, tmp_path):
    """psfm_ba_get_model after point filters that delete single observations and whole points, against
    apply_observation_mask of the same alive mask on flatten's container: tracks, point3D_ids and positions bit for
    bit."""
    path = str(tmp_path / "noisy.db")
    _scene_db(path, seed=8, noise_px=0.5)
    g, used, rot, pos, res = _stages(path, gm.GlobalMapperOptions())
    res.close()
    args = _triangulation_args(g, used, rot, pos.image_tvec, pos.has_position)
    tri = init_geometry.triangulate_all_points(**args)
    rec = tri.to_reconstruction(g.image_ids, g.image_names, g.camera_ids)
    cfg = ba.BundleAdjustmentConfig()
    for i in rec.RegImageIds():
        cfg.AddImage(i)
    prob, maps = ba.flatten(rec, cfg)
    res = init_geometry.triangulate_all_points_resident(**args)
    try:
        S = ba.TriangulationSolver(res, rot.orientations, pos.image_tvec, g.cameras)
    finally:
        res.close()
    try:
        S.filter_points(max_reproj_error=0.5, min_tri_angle=3.0)
        alive, err = S.observation_mask(), S.point_errors()
        model = S.get_model(len(g.keypoints))
        assert S.num_alive() == alive.sum()
    finally:
        S.close()
    lengths = np.diff(model.track_ptr)
    assert (~alive).any() and (lengths == 0).any() and ((lengths > 0) & (lengths < np.diff(tri.track_ptr))).any()
    ba.apply_observation_mask(prob, maps, rec, alive, err)
    assert sorted(rec.points3D) == (np.nonzero(lengths)[0] + 1).tolist()
    for p, pt in rec.points3D.items():
        a, b = model.track_ptr[p - 1], model.track_ptr[p]
        assert np.array_equal(g.image_ids[model.track_image[a:b]], pt.image_ids), p
        assert np.array_equal(model.track_point2D[a:b], pt.point2D_idxs), p
        assert np.array_equal(model.xyz[p - 1], pt.xyz) and model.error[p - 1] == pt.error, p
    for f in np.nonzero(pos.has_position)[0]:
        p3 = model.point3D_of_keypoint[g.keypoint_ptr[f]:g.keypoint_ptr[f + 1]]
        assert np.array_equal(np.where(p3 >= 0, p3 + 1, -1), rec.images[int(g.image_ids[f])].point3D_ids), f


def _python_route(path, o):
    """The chain of test_gpu_verification with the cache applied: stages 1-7, then the hand-off and write-back through
    the Python containers."""
    g, used, rot, pos, res = _stages(path, o)
    res.close()
    tri = init_geometry.triangulate_all_points(**_triangulation_args(g, used, rot, pos.image_tvec, pos.has_position),
                                               options=o.triangulator_options())
    rec = tri.to_reconstruction(g.image_ids, g.image_names, g.camera_ids)
    kw = dict(ba_refine_focal_length=o.ba_refine_focal_length, ba_refine_principal_point=o.ba_refine_principal_point,
              ba_refine_extra_params=o.ba_refine_extra_params)
    ba.iterative_global_refinement(rec, False, **kw)
    ba.iterative_global_refinement(rec, True, **kw)
    return rec


def test_model_equals_the_python_route(gpu, scene, tmp_path):
    o = gm.GlobalMapperOptions(ba_refine_principal_point=False, ba_refine_extra_params=False)
    rep = gm.global_mapper(scene[0], str(tmp_path), o)
    assert rep.success and rep.output == os.path.join(str(tmp_path), "0")
    m = colmap_io.read_model(rep.output)
    r = _python_route(scene[0], o)
    assert sorted(m.images) == sorted(r.images) and sorted(m.points3D) == sorted(r.points3D) and len(m.points3D) > 100
    rel = lambda a, b: np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)
    worst, identical = 0.0, True
    for i in r.images:
        a, b = m.images[i], r.images[i]
        assert np.array_equal(a.point3D_ids, b.point3D_ids) and a.name == b.name and np.array_equal(a.xys, b.xys)
        for x, y in ((a.qvec, b.qvec), (a.tvec, b.tvec)):
            worst, identical = max(worst, rel(x, y)), identical and np.array_equal(x, y)
    for p in r.points3D:
        a, b = m.points3D[p], r.points3D[p]
        assert np.array_equal(a.image_ids, b.image_ids) and np.array_equal(a.point2D_idxs, b.point2D_idxs)
        worst, identical = max(worst, rel(a.xyz, b.xyz)), identical and np.array_equal(a.xyz, b.xyz)
        assert abs(a.error - b.error) <= 1e-9 * max(b.error, 1.0)
    for c in r.cameras:
        worst, identical = max(worst, rel(m.cameras[c].params, r.cameras[c].params)), \
            identical and np.array_equal(m.cameras[c].params, r.cameras[c].params)
    print("mapper vs Python route: worst relative difference %.3g, bit-identical: %s" % (worst, identical))
    assert worst <= 1e-9
    for name in ("database_cache", "relative_poses", "rotations", "pairwise_translations", "positions", "triangulation",
                 "handoff", "refinement_A", "refinement_B", "model", "write"):
        assert rep.seconds(name) > 0, name
    assert set(rep.not_run) == {"CompleteAndMergeTracks", "Retriangulate", "FilterImages", "ExtractColors"}


def test_command_line_end_to_end(gpu, scene, tmp_path):
    path, qvec, tvec = scene
    outs = []
    for k in range(2):
        out = str(tmp_path / ("model%d" % k))
        assert gm.main(["global_mapper", "--database_path", path, "--image_path", "images", "--output_path", out,
                        "--GlobalMapper.num_threads", "64", "--random_seed", "100",
                        "--GlobalMapper.ba_refine_principal_point", "0", "--GlobalMapper.ba_refine_extra_params", "0",
                        "--quiet"]) == 0
        outs.append(os.path.join(out, "0"))
    m = colmap_io.read_model(outs[0])
    ids = sorted(m.images)
    truth = syn.camera_centres(qvec, tvec)[np.array(ids) - 1]
    est = syn.camera_centres(np.array([m.images[i].qvec for i in ids]), np.array([m.images[i].tvec for i in ids]))
    extent = np.linalg.norm(truth - truth.mean(0), axis=1).max()
    assert len(ids) >= 8 and syn.umeyama_ate(est, truth) <= 0.05 * extent
    # the bundle adjustment's reductions are not in a fixed order (DESIGN.md section 3.2), so two runs agree in every
    # id, track and name, and in their values to rounding
    b = colmap_io.read_model(outs[1])
    assert sorted(b.images) == ids and sorted(b.points3D) == sorted(m.points3D)
    for i in ids:
        assert np.array_equal(b.images[i].point3D_ids, m.images[i].point3D_ids) and b.images[i].name == m.images[i].name
        assert np.abs(b.images[i].tvec - m.images[i].tvec).max() <= 1e-9 * max(np.abs(m.images[i].tvec).max(), 1.0)
    for p in m.points3D:
        assert np.array_equal(b.points3D[p].image_ids, m.points3D[p].image_ids)
        assert np.array_equal(b.points3D[p].point2D_idxs, m.points3D[p].point2D_idxs)
        assert np.abs(b.points3D[p].xyz - m.points3D[p].xyz).max() <= 1e-9 * max(np.abs(m.points3D[p].xyz).max(), 1.0)
    assert abs(b.cameras[1].params[0] - m.cameras[1].params[0]) <= 1e-9 * m.cameras[1].params[0]


def test_no_pair_above_min_num_matches_writes_nothing(gpu, scene, tmp_path):
    out = str(tmp_path / "model")
    assert gm.main(["--database_path", scene[0], "--output_path", out, "--GlobalMapper.min_num_matches", "1000000000",
                    "--quiet"]) == 0
    assert not os.path.exists(os.path.join(out, "0"))
    rep = gm.global_mapper(scene[0], out, gm.GlobalMapperOptions(min_num_matches=10 ** 9))
    assert not rep.success and rep.failed_stage == "rotations"
