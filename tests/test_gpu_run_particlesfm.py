"""The whole-pipeline command on the device (particlesfm_b200.run_particlesfm, DESIGN.md §4.15): the match table built
from the resident tracker against the one built from its host arrays bit for bit, the command's track set against the
staged commands on the flow directory it keeps, and the whole route on a rigid room clip with exact flows against the
staged route (flows as .flo files, point_trajectory, sfm)."""
import ctypes as C
import os
import shutil
import sys

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import raft_oracle as ro
from particlesfm_b200 import _abi, _lib, colmap_io, handoff, optical_flow as of, point_trajectory as pt
from particlesfm_b200 import run_particlesfm as rp, sfm, synthetic as syn, tracker

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gpu_sfm import _assert_tables_equal, _tables_of   # noqa: E402
from test_gpu_tracker_stage import _same   # noqa: E402

pytestmark = pytest.mark.gpu

# the room clip of tests 3 and 4: 24 frames of 224 x 160
ROOM = dict(n_frames=24, h=160, w=224, seed=3)
# ATE of the room clip's reconstruction over the extent of the true centres: 1.27e-6 measured on an H100 80GB HBM3 (see
# DESIGN.md §4.15); the bound leaves headroom above it
ROOM_ATE = 1e-4


# ------------------------------------------------------------------------------------------------ 1. the entry

def _finished_tracker(n, h, w, seed, pc, min_len, flows=None):
    fw, fb, f2, b2 = flows or syn.make_flow_sequence(n, h, w, seed=seed)
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    trk = tracker._ResidentTracker(h, w, 2, n, path_consistency=pc)
    prev = None
    for t in range(n - 1):
        g2, h2 = (dev(f2[t - 1]), dev(b2[t - 1])) if pc and t >= 1 else (None, None)
        f = dev(fw[t])
        trk.advance(t, f, dev(fb[t]), prev, g2, h2)
        prev = f
    return trk, trk.finish(min_len)


def _cases():
    out = []
    for pc in (True, False):
        out.append(pytest.param(dict(n=9, h=48, w=64, seed=4, pc=pc, min_len=3), id="seeded-pc%d" % pc))
    out.append(pytest.param(dict(n=6, h=40, w=56, seed=5, pc=True, min_len=50), id="min_len-drops-all"))
    out.append(pytest.param(dict(n=5, h=40, w=56, seed=6, pc=False, min_len=2, away=True), id="empty"))
    out.append(pytest.param(dict(n=5, h=40, w=56, seed=6, pc=False, min_len=1, away=True), id="singletons"))
    return out


@pytest.mark.parametrize("case", _cases())
@pytest.mark.parametrize("side_stream", [False, True])
def test_tracker_table_equals_the_host_array_table(gpu, case, side_stream):
    case = dict(case)
    n, h, w = case["n"], case["h"], case["w"]
    flows = None
    if case.pop("away", False):          # every particle leaves the frame at once: trajectories of one sample
        away = [np.full((h, w, 2), 1e3, np.float32)] * (n - 1)
        flows = (away, away, away[:n - 2], away[:n - 2])
    stream = torch.cuda.Stream() if side_stream else torch.cuda.current_stream()
    F = n + 2                            # more images than frames is allowed
    names = ["%05d.png" % i for i in range(F)]
    ids = np.arange(F, 0, -1)
    cam, size = np.array([1.2 * w, w / 2, h / 2]), (w, h)
    with torch.cuda.stream(stream):
        trk, arrays = _finished_tracker(n, h, w, case["seed"], case["pc"], case["min_len"], flows)
        try:
            if case["min_len"] >= 50 or case["min_len"] == 2:
                assert arrays.frame_ids.shape[0] == 0
            # the entry's handle against psfm_matches_create's on the host arrays
            ref = handoff.traj_to_matches_device(arrays, F)
            handle, npairs, nmatches = trk.matches(F, handoff.SAMPLE_K)
            try:
                L = _lib.lib()
                i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
                kp_ptr, kxy = np.empty(F + 1, np.int64), np.empty((arrays.frame_ids.shape[0], 2))
                pair_images, pair_ptr = np.empty((npairs, 2), np.int64), np.empty(npairs + 1, np.int64)
                matches = np.empty((nmatches, 2), np.int64)
                _lib.check(L.psfm_matches_result(handle, i64(kp_ptr), _lib.dptr(kxy), i64(pair_images), i64(pair_ptr),
                                                 i64(matches)), "psfm_matches_result")
            finally:
                _lib.lib().psfm_matches_destroy(handle)
            assert np.array_equal(np.concatenate([[0], np.cumsum([k.shape[0] for k in ref.keypoints])]), kp_ptr)
            assert np.concatenate(ref.keypoints).tobytes() == kxy.tobytes()
            for k, v in (("pair_images", pair_images), ("pair_ptr", pair_ptr), ("matches", matches)):
                assert np.array_equal(getattr(ref, k), v), k
            # the resident tables
            a = handoff.ResidentMatchTable(handoff._flatten(arrays, False), ids)
            b = handoff.ResidentMatchTable.from_tracker(trk, ids)
            try:
                for k in ("pair_images", "pair_ptr"):
                    x, y = getattr(a.pairs, k), getattr(b.pairs, k)
                    assert x.dtype == y.dtype and x.tobytes() == y.tobytes(), k
                _assert_tables_equal(a.tables(names, cam, size), b.tables(names, cam, size))
            finally:
                a.close()
                b.close()
        finally:
            trk.close()
    stream.synchronize()


def test_entry_refusals(gpu):
    trk = tracker._ResidentTracker(32, 40, 2, 3)
    try:
        with pytest.raises(_lib.PsfmError, match="finish") as e:
            trk.matches(3, 20)
        assert e.value.code == _abi.PSFM_ERR_INVALID
        fw, fb, f2, b2 = syn.make_flow_sequence(3, 32, 40, seed=1)
        dev = lambda a: torch.from_numpy(a).cuda()
        trk.advance(0, dev(fw[0]), dev(fb[0]))
        trk.advance(1, dev(fw[1]), dev(fb[1]), dev(fw[0]), dev(f2[0]), dev(b2[0]))
        trk.finish(3, result=False)
        for args, needle in (((2, 20), "number of frames"), ((3, 0), "sample_k")):
            with pytest.raises(_lib.PsfmError, match=needle) as e:
                trk.matches(*args)
            assert e.value.code == _abi.PSFM_ERR_INVALID
        handle, _, _ = trk.matches(3, 20)          # still usable after the refusals
        _lib.lib().psfm_matches_destroy(handle)
    finally:
        trk.close()


# ------------------------------------------------------------------------------------------------ 2. seeded RAFT

@pytest.fixture(scope="module")
def seeded(tmp_path_factory):
    root = tmp_path_factory.mktemp("seeded")
    img = str(root / "images")
    os.makedirs(img)
    # frames and weights whose flows keep particles alive through every frame: with path consistency a frame
    # without a 3-observation particle stops the reference (optimize_buffer's np.stack([])), and the command with it
    for i, f in enumerate(ro.seeded_frames(5, 123, 125, seed=9)):
        Image.fromarray(f).save(os.path.join(img, "%05d.png" % i))
    weights = str(root / "w.pth")
    torch.save(ro.seeded_state_dict(4), weights)
    return str(root), img, weights


@pytest.mark.parametrize("skip_pc", [False, True])
def test_kept_track_npy_equals_the_staged_commands_on_the_kept_flows(gpu, seeded, skip_pc):
    root, img, weights = seeded
    out = os.path.join(root, "keep%d" % skip_pc)
    rep = rp.particlesfm(img, out, weights, skip_path_consistency=skip_pc, skip_sfm=True, keep_intermediate=True)
    assert [n for n, _ in rep.stages] == ["flows_trajectories", "track_npy"] and rep.sfm is None
    subs = ["flow_b", "flow_f", "flow_imgs"] + ([] if skip_pc else ["flow_b2", "flow_f2", "flow_imgs2"])
    assert sorted(os.listdir(os.path.join(out, "optical_flows"))) == sorted(subs)
    staged = os.path.join(root, "staged%d" % skip_pc)
    pt.main_connect_point_trajectories(os.path.join(out, "optical_flows"), staged, skip_path_consistency=skip_pc)
    load = lambda d: np.load(os.path.join(d, "track.npy"), allow_pickle=True).item().as_dict()
    got, ref = load(os.path.join(out, "trajectories")), load(staged)
    assert len(got) > 0
    _same(got, ref)
    # without --keep_intermediate only the track set is written
    lean = os.path.join(root, "lean%d" % skip_pc)
    rp.particlesfm(img, lean, weights, skip_path_consistency=skip_pc, skip_sfm=True)
    assert os.listdir(lean) == ["trajectories"] and os.listdir(os.path.join(lean, "trajectories")) == ["track.npy"]
    _same(load(os.path.join(lean, "trajectories")), ref)


def test_command_line_skip_sfm(gpu, seeded, capsys):
    root, img, weights = seeded
    out = os.path.join(root, "cli")
    assert rp.main(["--model", weights, "-i", img, "-o", out, "--assume_static", "--skip_sfm"]) == 0
    text = capsys.readouterr().out
    assert "[ParticleSfM] Connecting (optimization enabled)" in text and "flows_trajectories" in text
    assert os.listdir(out) == ["trajectories"]


# ------------------------------------------------------------------------------------------------ 3. the room clip

def _write_room(root, frames):
    img = os.path.join(root, "images")
    os.makedirs(img)
    for i, f in enumerate(frames):
        Image.fromarray(f).save(os.path.join(img, "%05d.png" % i))
    return img


@pytest.fixture(scope="module")
def room(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("room"))
    frames, flows, qvec, tvec = syn.make_room_sequence(**ROOM)
    img = _write_room(root, frames)
    out = os.path.join(root, "fused")
    rep = rp.particlesfm(img, out, flow_source=rp.array_flow_source(flows), quiet=True)
    # the staged route: the same flows as .flo files, then point_trajectory, then sfm
    staged = os.path.join(root, "staged")
    flow_dir = os.path.join(staged, "optical_flows")
    paths = sorted(os.path.join(img, n) for n in os.listdir(img))
    of.make_flow_dirs(flow_dir, True)
    files = of.flow_files(paths, flow_dir)
    for (t, s), (f, b) in flows.items():
        ff, fb, _ = files(t, s)
        of.write_flo(ff, f)
        of.write_flo(fb, b)
    traj = os.path.join(staged, "trajectories")
    pt.main_connect_point_trajectories(flow_dir, traj)
    srep = sfm.sfm_reconstruction(img, staged, traj, assume_static=True)
    return dict(root=root, img=img, out=out, rep=rep, staged=staged, srep=srep, qvec=qvec, tvec=tvec, flows=flows)


def _assert_models_equal(a_dir, b_dir):
    a, b = colmap_io.read_model(a_dir), colmap_io.read_model(b_dir)
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
    return a


def test_room_clip_equals_the_staged_route(gpu, room):
    rep, out, staged = room["rep"], room["out"], room["staged"]
    assert rep.success and room["srep"].success, (rep.sfm.failed_stage, rep.sfm.reason)
    assert [n for n, _ in rep.stages] == ["flows_trajectories", "sfm"]
    assert sorted(os.listdir(out)) == ["colmap_outputs_converted", "sfm"]       # no intermediate written
    got, ref = _tables_of(os.path.join(out, "sfm", "database.db")), _tables_of(os.path.join(staged, "sfm", "database.db"))
    assert sorted(got) == sorted(ref)
    for t in ref:
        assert got[t] == ref[t], t
    pairs = lambda d: open(os.path.join(d, "sfm", "image_match_pairs.txt"), "rb").read()
    assert pairs(out) == pairs(staged) and len(pairs(out)) > 0
    a = _assert_models_equal(os.path.join(out, "sfm", "model"), os.path.join(staged, "sfm", "model"))
    assert len(a.images) == ROOM["n_frames"]
    ids = sorted(a.images)
    truth = syn.camera_centres(room["qvec"], room["tvec"])[np.array(ids) - 1]
    est = syn.camera_centres(np.array([a.images[i].qvec for i in ids]), np.array([a.images[i].tvec for i in ids]))
    ate = syn.umeyama_ate(est, truth) / np.linalg.norm(truth - truth.mean(0), axis=1).max()
    print("room clip: %d images, %d points, ATE %.3g of the extent" % (len(ids), len(a.points3D), ate))
    assert ate <= ROOM_ATE
    for d in ("depths", "poses"):
        assert sorted(os.listdir(os.path.join(out, "colmap_outputs_converted", d))) == \
            sorted(os.listdir(os.path.join(staged, "colmap_outputs_converted", d)))


# ------------------------------------------------------------------------------------------------ 4. --skip_exists

def test_skip_exists_reads_the_existing_track_set(gpu, room):
    out = os.path.join(room["root"], "reuse")
    os.makedirs(os.path.join(out, "trajectories"))
    shutil.copy(os.path.join(room["staged"], "trajectories", "track.npy"), os.path.join(out, "trajectories"))

    def no_flows(*a):
        raise AssertionError("the flow source was called")

    rep = rp.particlesfm(room["img"], out, flow_source=no_flows, skip_exists=True, quiet=True)
    assert rep.success and [n for n, _ in rep.stages] == ["sfm"]
    got, ref = _tables_of(os.path.join(out, "sfm", "database.db")), _tables_of(os.path.join(room["out"], "sfm", "database.db"))
    for t in ref:
        assert got[t] == ref[t], t
    _assert_models_equal(os.path.join(out, "sfm", "model"), os.path.join(room["out"], "sfm", "model"))


# ------------------------------------------------------------------------------------------------ 5. --root_dir

@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 or more GPUs")
def test_root_dir_equals_workspace_runs(gpu, room, seeded, tmp_path):
    weights = seeded[2]
    root = tmp_path / "root"
    for k in range(2):
        frames, flows, _, _ = syn.make_room_sequence(**dict(ROOM, seed=10 + k))
        ws = str(root / ("seq%d" % k))
        _write_room(ws, frames)
        # the track set from the exact flows, reused through --skip_exists by every run below
        trk, _ = _finished_tracker(ROOM["n_frames"], ROOM["h"], ROOM["w"], 0, True, 3,
                                   ([flows[(t, 1)][0] for t in range(ROOM["n_frames"] - 1)],
                                    [flows[(t, 1)][1] for t in range(ROOM["n_frames"] - 1)],
                                    [flows[(t, 2)][0] for t in range(ROOM["n_frames"] - 2)],
                                    [flows[(t, 2)][1] for t in range(ROOM["n_frames"] - 2)]))
        os.makedirs(os.path.join(ws, "trajectories"))
        with trk.track_npy_body() as body:
            pt.write_track_npy(os.path.join(ws, "trajectories", "track.npy"), body.view())
        trk.close()
        single = str(tmp_path / ("single%d" % k))
        shutil.copytree(ws, single)
        assert rp.main(["--model", weights, "--workspace_dir", single, "--assume_static", "--skip_exists"]) == 0
    lines = []
    args = rp.build_parser().parse_args(["--model", weights, "--root_dir", str(root), "--assume_static", "--skip_exists"])
    assert rp.run_root(args, out=lines.append) == 0
    devices = {line.split(" on device ")[1].split()[0] for line in lines if " on device " in line}
    assert len(devices) == 2, lines
    for k in range(2):
        a, b = str(root / ("seq%d" % k)), str(tmp_path / ("single%d" % k))
        got, ref = _tables_of(os.path.join(a, "sfm", "database.db")), _tables_of(os.path.join(b, "sfm", "database.db"))
        for t in ref:
            assert got[t] == ref[t], t
        _assert_models_equal(os.path.join(a, "sfm", "model"), os.path.join(b, "sfm", "model"))
