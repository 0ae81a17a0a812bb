"""The SfM driver on the device (particlesfm_b200.sfm, DESIGN.md §4.12): the resident match table against the host route
(import_keypoints_matches_arrays, then MatchTables.from_rows) bit for bit, its verification against the host entry bit
for bit, and the whole step from track.npy and PNG frames to the converted poses against the step-by-step route."""
import os
import sqlite3
import threading

import numpy as np
import pytest
from PIL import Image

from particlesfm_b200 import _abi, _lib, colmap_io, convert, global_mapper as gm, handoff, init_geometry, sfm
from particlesfm_b200 import synthetic as syn
from test_handoff import GOLD, _tracks
from test_import_matches import IMP

pytestmark = pytest.mark.gpu

W, H = 1024, 436
CAM = np.array([1.2 * W, W / 2.0, H / 2.0])


def _host_route(tracks, names, ids, remove_dynamic=True):
    """import_keypoints_matches_arrays on the host traj_to_matches, image ids in get_image_ids order (name order, as
    import_small.npz records it), then MatchTables.from_rows: (rows, tables)."""
    tm = handoff.traj_to_matches(tracks, len(names), remove_dynamic)
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), tm)
    return rows, handoff.MatchTables.from_rows(rows, ids, names, CAM, (W, H))


def _assert_tables_equal(a, b):
    for k in ("image_ids", "keypoint_ptr", "keypoints", "camera_ids", "cameras", "image_camera", "camera_size",
              "prior_focal_length", "pair_ids", "pair_images", "match_ptr", "matches"):
        x, y = getattr(a, k), getattr(b, k)
        assert x.dtype == y.dtype and x.shape == y.shape, k
        assert x.tobytes() == y.tobytes(), k
    assert list(a.image_names) == list(b.image_names)


def _shapes():
    g = np.load(GOLD)
    n = int(g["num_images"])
    small = _tracks(g)
    helix = syn.make_two_view_scene(3000, 50, 60000, seed=11, step=0.08, path="helix", focal=1.2 * W)[0].to_dict()
    out = []
    for name, tracks, frames in (("small", small, n), ("helix50", helix, 50)):
        for remove_dynamic in ((True, False) if name == "small" else (True,)):
            for order in ("names", "reversed"):
                ids = list(range(1, frames + 1)) if order == "names" else list(range(frames, 0, -1))
                out.append(pytest.param(tracks, frames, ids, remove_dynamic, id=f"{name}-{remove_dynamic}-{order}"))
    return out


SHAPES = _shapes()


@pytest.mark.parametrize("tracks,frames,ids,remove_dynamic", SHAPES)
def test_device_table_equals_host_route(gpu, tracks, frames, ids, remove_dynamic):
    names = ["%05d.png" % i for i in range(frames)]
    rows, host = _host_route(tracks, names, ids, remove_dynamic)
    with handoff.ResidentMatchTable(handoff._flatten(tracks, remove_dynamic), ids) as t:
        dev = t.tables(names, CAM, (W, H))
        assert (t.num_keypoints, t.num_pairs, t.num_matches) == (len(dev.keypoints), len(dev.pair_ids), len(dev.matches))
        # the ordered pair list the handle keeps for image_match_pairs.txt
        tm = handoff.traj_to_matches(tracks, frames, remove_dynamic)
        assert np.array_equal(t.pairs.pair_images, tm.pair_images) and np.array_equal(t.pairs.pair_ptr, tm.pair_ptr)
    _assert_tables_equal(dev, host)
    kps, ms = dev.rows()
    assert [(i, k.tobytes()) for i, k in kps] == sorted((i, k.tobytes()) for i, k in rows.keypoints)
    assert [(p, m.tobytes()) for p, m in ms] == sorted((p, m.tobytes()) for p, m in rows.matches)


def test_device_rows_equal_the_reference_database(gpu):
    """The reference's import_keypoints_matches on handoff_small.npz with ids against the name order."""
    gi = np.load(IMP, allow_pickle=True)
    g = np.load(GOLD)
    n = int(g["num_images"])
    names = ["%05d.png" % i for i in range(n)]
    idmap = {str(k): int(v) for k, v in zip(gi["image_names"], gi["image_id_values"])}
    ids = [idmap[nm] for nm in names]
    with handoff.ResidentMatchTable(handoff._flatten(_tracks(g), True), ids) as t:
        kps, ms = t.tables(names, CAM, (W, H)).rows()
    assert sorted((int(i), int(r), int(c), bytes(b)) for i, r, c, b in gi["verify_keypoints"]) == \
        [(i, k.shape[0], 2, k.tobytes()) for i, k in kps]
    assert sorted((int(i), int(r), int(c), bytes(b)) for i, r, c, b in gi["verify_matches"]) == \
        [(p, m.shape[0], 2, m.tobytes()) for p, m in ms]


@pytest.mark.parametrize("tracks,frames,ids,remove_dynamic", SHAPES)
def test_resident_verification_equals_host_entry(gpu, tracks, frames, ids, remove_dynamic):
    names = ["%05d.png" % i for i in range(frames)]
    _, host = _host_route(tracks, names, ids, remove_dynamic)
    ref = init_geometry.verify_two_view_geometries(**host.verification_inputs())
    with handoff.ResidentMatchTable(handoff._flatten(tracks, remove_dynamic), ids) as t:
        tables = t.tables(names, CAM, (W, H))
        dev = init_geometry.verify_match_table(t, tables.image_camera, tables.camera_size)
    for k in ("config", "F", "E", "H", "inlier_ptr", "inlier_matches", "trials"):
        x, y = getattr(dev, k), getattr(ref, k)
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), k
    for k in ("num_trials", "num_local_rounds", "num_config", "num_launches"):
        assert dev.summary[k] == ref.summary[k], k


def test_unverified_geometries_equal_the_skip_database(gpu, tmp_path):
    g = np.load(GOLD)
    n = int(g["num_images"])
    names, ids = ["%05d.png" % i for i in range(n)], list(range(1, n + 1))
    tm = handoff.traj_to_matches(_tracks(g), n)
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), tm, skip_geometric_verification=True)
    path = str(tmp_path / "database.db")
    db = sqlite3.connect(path)
    images = sfm.ImageSet(names, W, H)
    sfm.write_schema(db, images)
    db.close()
    handoff.write_colmap_database(path, rows)
    ref = handoff.read_two_view_geometries(path)
    with handoff.ResidentMatchTable(handoff._flatten(_tracks(g), True), ids) as t:
        got = t.tables(names, images.camera, (W, H)).unverified_two_view_geometries()
    _assert_geometries_equal(got, ref)


def _assert_geometries_equal(a, b):
    for k in ("image_ids", "keypoint_ptr", "keypoints", "camera_ids", "cameras", "image_camera", "pair_ids", "pair_images",
              "camera_size", "config", "F", "E", "H", "inlier_ptr", "inlier_matches"):
        x, y = np.asarray(getattr(a, k)), np.asarray(getattr(b, k))
        assert x.shape == y.shape and np.array_equal(x, y), k
        assert x.dtype == y.dtype, k
    assert list(a.image_names) == list(b.image_names)


# ------------------------------------------------------------------------------------------------ end to end

def _video(root, n_frames=12, seed=7):
    """A helix video: PNG frames of W x H and OUT/trajectories_labeled/track.npy, a labelled dict whose static samples
    carry 0.5 px of noise, plus dynamic samples (labels 1) at random places.  Returns (image dir, out dir, tracks,
    true qvec, true tvec)."""
    tracks, qvec, tvec, _ = syn.make_two_view_scene(1500, n_frames, 9000, seed=seed, step=0.08, path="helix",
                                                    focal=1.2 * W)
    rng = np.random.default_rng(seed)
    d = tracks.to_dict()
    for t in d.values():
        xy = np.asarray(t["locations"]) + rng.normal(0, 0.5, (len(t["locations"]), 2))
        lab = rng.random(len(xy)) < 0.03
        xy[lab] = rng.random((lab.sum(), 2)) * [W, H]
        t["locations"], t["labels"] = list(xy), lab.astype(int).tolist()
    for k in range(200):                                   # whole dynamic trajectories
        f0 = int(rng.integers(0, n_frames - 3))
        d[10 ** 6 + k] = {"frame_ids": list(range(f0, f0 + 3)), "locations": list(rng.random((3, 2)) * [W, H]),
                          "labels": [1, 1, 1]}
    img, out = os.path.join(root, "images"), os.path.join(root, "out")
    os.makedirs(img)
    yy, xx = np.mgrid[0:H, 0:W]
    for i in range(n_frames):
        f = np.stack([127 + 120 * np.sin(xx / (37.0 + i) + c) * np.cos(yy / 23.0 - c * i) for c in range(3)], -1)
        Image.fromarray(np.clip(f, 0, 255).astype(np.uint8)).save(os.path.join(img, "%05d.png" % i))
    os.makedirs(os.path.join(out, "trajectories_labeled"))
    np.save(os.path.join(out, "trajectories_labeled", "track.npy"), d, allow_pickle=True)
    return img, out, d, qvec, tvec


def _tables_of(path):
    con = sqlite3.connect(path)
    names = [r[0] for r in con.execute("SELECT name FROM sqlite_master WHERE type = 'table' ORDER BY name")]
    out = {t: con.execute(f"SELECT * FROM {t} ORDER BY rowid").fetchall() for t in names if t != "sqlite_sequence"}
    con.close()
    return out


@pytest.fixture(scope="module")
def video(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("sfm"))
    img, out, tracks, qvec, tvec = _video(root)
    rep = sfm.sfm_reconstruction(img, out, os.path.join(out, "trajectories_labeled"))
    # the step-by-step route into its own database
    names = sorted(os.listdir(img))
    ids = list(range(1, len(names) + 1))
    tm = handoff.traj_to_matches_device(tracks, len(names))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), tm)
    mt = handoff.MatchTables.from_rows(rows, ids, names, CAM, (W, H))
    ver = init_geometry.verify_two_view_geometries(**mt.verification_inputs())
    ref_db = os.path.join(root, "step", "database.db")
    os.makedirs(os.path.dirname(ref_db))
    db = sqlite3.connect(ref_db)
    sfm.write_schema(db, sfm.read_image_set(img))
    db.close()
    handoff.write_colmap_database(ref_db, handoff.DatabaseRows(rows.keypoints, rows.matches, ver.two_view_rows(mt.pair_ids)))
    return dict(root=root, img=img, out=out, tracks=tracks, qvec=qvec, tvec=tvec, rep=rep, ref_db=ref_db, names=names)


def test_database_equals_step_by_step_route(gpu, video):
    assert video["rep"].success, video["rep"].failed_stage
    got, ref = _tables_of(os.path.join(video["out"], "sfm", "database.db")), _tables_of(video["ref_db"])
    assert sorted(got) == sorted(ref) == ["cameras", "descriptors", "images", "keypoints", "matches",
                                          "two_view_geometries"]
    for t in ref:
        assert got[t] == ref[t], t
    assert len(got["two_view_geometries"]) == len(got["matches"]) > 0


def test_database_holds_what_the_mapper_was_given(gpu, video):
    names = video["names"]
    ids = list(range(1, len(names) + 1))
    with handoff.ResidentMatchTable(handoff._flatten(video["tracks"], True), ids) as t:
        tables = t.tables(names, CAM, (W, H))
        g = init_geometry.verify_match_table(t, tables.image_camera, tables.camera_size).to_two_view_geometries(tables)
    _assert_geometries_equal(handoff.read_two_view_geometries(os.path.join(video["out"], "sfm", "database.db")), g)


def test_pair_list_equals_host_traj_to_matches(gpu, video, tmp_path):
    ref = str(tmp_path / "pairs.txt")
    handoff.traj_to_matches(video["tracks"], len(video["names"])).write_pair_list(ref, video["names"])
    assert open(os.path.join(video["out"], "sfm", "image_match_pairs.txt")).read() == open(ref).read()


def test_model_equals_global_mapper_on_the_database(gpu, video):
    sfm_dir = os.path.join(video["out"], "sfm")
    ref_rep = gm.global_mapper(os.path.join(sfm_dir, "database.db"), os.path.join(video["root"], "ref_model"),
                               sfm.mapper_options(), image_path=video["img"])
    assert ref_rep.success
    a, b = colmap_io.read_model(os.path.join(sfm_dir, "model")), colmap_io.read_model(ref_rep.output)
    for name in ("cameras.bin", "images.bin", "points3D.bin"):       # SFM/model/ holds copies of SFM/model/0/
        assert open(os.path.join(sfm_dir, "model", name), "rb").read() == \
            open(os.path.join(sfm_dir, "model", "0", name), "rb").read()
    # ids, tracks and observations exactly; the bundle adjustment's reductions are not in a fixed order (DESIGN.md
    # §3.2), so poses, points and the focal length agree to rounding
    assert list(a.images) == list(b.images) and list(a.points3D) == list(b.points3D)
    rel = lambda x, y: np.abs(np.asarray(x) - np.asarray(y)).max() / max(np.abs(np.asarray(y)).max(), 1.0)
    assert rel(a.cameras[1].params, b.cameras[1].params) <= 1e-9
    for i in a.images:
        x, y = a.images[i], b.images[i]
        assert x.name == y.name and np.array_equal(x.point3D_ids, y.point3D_ids) and np.array_equal(x.xys, y.xys)
        assert rel(x.qvec, y.qvec) <= 1e-9 and rel(x.tvec, y.tvec) <= 1e-9
    for p in a.points3D:
        x, y = a.points3D[p], b.points3D[p]
        assert np.array_equal(x.image_ids, y.image_ids) and np.array_equal(x.point2D_idxs, y.point2D_idxs)
        assert rel(x.xyz, y.xyz) <= 1e-9
    # stats: a numpy restatement of model_analyzer's numbers on the read-back model
    s = video["rep"].stats
    obs = sum(len(p.image_ids) for p in a.points3D.values())
    err = np.array([p.error for p in a.points3D.values()])
    assert s["num_reg_images"] == len(a.images) and s["num_sparse_points"] == len(a.points3D)
    assert s["num_observations"] == obs
    assert s["mean_track_length"] == obs / len(a.points3D) and s["num_observations_per_image"] == obs / len(a.images)
    assert abs(s["mean_reproj_error"] - err[err != -1].mean()) <= 1e-12 * err.mean()
    # the poses recover the truth after a similarity alignment
    ids = sorted(a.images)
    truth = syn.camera_centres(video["qvec"], video["tvec"])[np.array(ids) - 1]
    est = syn.camera_centres(np.array([a.images[i].qvec for i in ids]), np.array([a.images[i].tvec for i in ids]))
    ate = syn.umeyama_ate(est, truth) / np.linalg.norm(truth - truth.mean(0), axis=1).max()
    assert len(ids) >= 10 and ate <= 0.05, (len(ids), ate)


def test_converted_output_equals_convert_of_the_model(gpu, video, tmp_path):
    ref = str(tmp_path / "converted")
    convert.write_depth_pose_from_colmap_format(os.path.join(video["out"], "sfm"), ref)
    got = os.path.join(video["out"], "colmap_outputs_converted")
    for sub in ("depths", "poses", "intrinsics"):
        files = sorted(os.listdir(os.path.join(ref, sub)))
        assert files == sorted(os.listdir(os.path.join(got, sub))) and files
        for f in files:
            x, y = os.path.join(got, sub, f), os.path.join(ref, sub, f)
            if f.endswith(".npy"):
                assert np.array_equal(np.load(x), np.load(y)), f
            elif f.endswith(".txt"):
                assert open(x, "rb").read() == open(y, "rb").read(), f


def _layout(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def test_cli_writes_the_same_layout(gpu, video, tmp_path, capsys):
    out = str(tmp_path / "out")
    os.makedirs(os.path.join(out, "trajectories_labeled"))
    os.link(os.path.join(video["out"], "trajectories_labeled", "track.npy"),
            os.path.join(out, "trajectories_labeled", "track.npy"))
    assert sfm.main(["--image_dir", video["img"], "--output_dir", out]) == 0
    text = capsys.readouterr().out
    assert "num_reg_images" in text and "verification" in text
    assert _layout(out) == _layout(video["out"])


def test_failed_position_stage_writes_no_model(gpu, video, tmp_path, monkeypatch, capsys):
    """A position stage that fails (as on a disconnected view graph): the database is complete, nothing else."""
    def fail(*a, **k):
        raise _lib.PsfmError("psfm_estimate_global_positions failed with status -1: the view graph is not connected",
                             _abi.PSFM_ERR_INVALID)
    monkeypatch.setattr(init_geometry, "estimate_global_positions", fail)
    out = str(tmp_path / "out")
    rc = sfm.main(["--image_dir", video["img"], "--output_dir", out, "--traj_dir",
                   os.path.join(video["out"], "trajectories_labeled"), "--quiet"])
    err = capsys.readouterr().err
    assert rc == 1 and "positions" in err and "Could not find binary or text COLMAP model" in err
    assert _tables_of(os.path.join(out, "sfm", "database.db")) == _tables_of(video["ref_db"])
    assert os.listdir(os.path.join(out, "sfm", "model")) == []
    assert not os.path.exists(os.path.join(out, "colmap_outputs_converted"))
    with pytest.raises(FileNotFoundError):
        sfm.sfm_reconstruction(video["img"], str(tmp_path / "again"), os.path.join(video["out"], "trajectories_labeled"))
    assert _tables_of(os.path.join(str(tmp_path / "again"), "sfm", "database.db")) == _tables_of(video["ref_db"])


def test_no_thread_outlives_a_call_that_raised(gpu, video, tmp_path, monkeypatch):
    def boom(*a, **k):
        raise RuntimeError("raised inside the mapper")
    monkeypatch.setattr(init_geometry, "estimate_relative_poses", boom)
    before = set(threading.enumerate())
    with pytest.raises(RuntimeError, match="inside the mapper"):
        sfm.main_global_sfm(str(tmp_path / "sfm"), video["img"], video["tracks"])
    assert set(threading.enumerate()) == before
    assert _tables_of(str(tmp_path / "sfm" / "database.db")) == _tables_of(video["ref_db"])
