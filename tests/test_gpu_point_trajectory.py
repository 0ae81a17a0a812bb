"""The point-trajectory command on the GPU (particlesfm_b200.point_trajectory): .flo directories to track.npy, with
and without path consistency, against the reference's own track sets (tests/golden/tracker_small.npz,
track_small.npz) and the host path bit for bit; the device emitter of the file's state (csrc/track_npy.cu) byte for
byte against the numpy oracle."""
import os
import sys

import numpy as np
import pytest

from oracle import track_npy_oracle as tno
from particlesfm_b200 import _lib, handoff, point_trajectory as pt, synthetic as syn, tracker

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gpu_tracker_stage import _golden_filtered, _same   # noqa: E402
from test_point_trajectory_host import crafted_track_arrays, empty_track_arrays, same_set, write_flow_dir, _bad_arrays  # noqa: E402
from test_tracker import _compare, _load   # noqa: E402

TRACK_GOLD = os.path.join(HERE, "golden", "track_small.npz")


def _loaded(traj_dir):
    return np.load(os.path.join(traj_dir, "track.npy"), allow_pickle=True).item().as_dict()


def _host_skip(fw, fb, ratio, min_len):
    _, occ = tracker.flow_check(fw, fb, 1.0)
    return tracker.track(fw, occ, ratio, traj_min_len=min_len)


@pytest.mark.gpu
def test_command_reproduces_the_reference_track_sets(gpu, tmp_path):
    g, fw, fb, f2, b2, occ, occ2 = _load()
    d = write_flow_dir(str(tmp_path / "flows"), fw, fb, f2, b2)
    assert pt.main(["--flow_dir", d, "--traj_dir", str(tmp_path / "pc")]) == 0
    _golden_filtered(_loaded(str(tmp_path / "pc")), g, 3)
    gs = np.load(TRACK_GOLD)
    assert pt.main(["--flow_dir", d, "--traj_dir", str(tmp_path / "skip"), "--skip_path_consistency", "--traj_min_len", "0"]) == 0
    _compare(_loaded(str(tmp_path / "skip")), gs)
    arrays = pt.main_connect_point_trajectories(d, str(tmp_path / "skip3"), skip_path_consistency=True)
    _golden_filtered(_loaded(str(tmp_path / "skip3")), gs, 3)
    _golden_filtered(arrays.to_dict(), gs, 3)
    _compare(tracker.track(fw, occ, 2, device=True), gs)


@pytest.mark.gpu
@pytest.mark.parametrize("skip", [False, True], ids=["path_consistency", "skip_path_consistency"])
@pytest.mark.parametrize("n_frames,h,w,ratio", [(11, 436, 1024, 2), (4, 480, 854, 1), (6, 101, 157, 3)])
def test_command_equals_host_path(gpu, tmp_path, n_frames, h, w, ratio, skip):
    fw, fb, f2, b2 = syn.make_flow_sequence(n_frames, h, w, seed=n_frames + ratio)
    d = write_flow_dir(str(tmp_path / "flows"), fw, fb, None if skip else f2, None if skip else b2)
    if skip:
        host = _host_skip(fw, fb, ratio, 0)
    else:
        host = tracker.main_connect_point_trajectories(fw, fb, f2, b2, ratio, 1.0, 0)
    traj = str(tmp_path / "traj")
    arrays = pt.main_connect_point_trajectories(d, traj, ratio, 1.0, 0, skip_path_consistency=skip)
    assert np.diff(arrays.lengths()).any() and arrays.frame_ids.max() == n_frames - 1
    _same(arrays.to_dict(), host)
    same_set(np.load(os.path.join(traj, "track.npy"), allow_pickle=True).item(), arrays)
    with tracker.track_npy_body_device(arrays) as body:
        assert open(os.path.join(traj, "track.npy"), "rb").read().find(bytes(body.view())) > 0


@pytest.mark.gpu
def test_frame_where_every_particle_dies(gpu, tmp_path):
    """Skip mode runs through a frame without survivors (re-seeding by the (y + 1)^2 + x^2 > r^2 rule) to the end,
    as the host track does; with path consistency the host path and the command raise the same ValueError."""
    g, fw, fb, f2, b2, occ, occ2 = _load()
    fw = [f.copy() for f in fw]
    fw[2] += 1000.0                                     # every particle leaves the image at frame 2
    d = write_flow_dir(str(tmp_path / "flows"), fw, fb, f2, b2)
    host = _host_skip(fw, fb, 2, 0)
    assert min(v["frame_ids"][0] for v in host.values() if v["frame_ids"][-1] > 3) == 3
    arrays = pt.main_connect_point_trajectories(d, str(tmp_path / "skip"), 2, 1.0, 0, skip_path_consistency=True)
    _same(arrays.to_dict(), host)
    assert arrays.frame_ids.max() == len(fw)
    same_set(np.load(str(tmp_path / "skip" / "track.npy"), allow_pickle=True).item(), arrays)
    with pytest.raises(ValueError, match="need at least one array to stack"):
        tracker.main_connect_point_trajectories(fw, fb, f2, b2, 2, 1.0, 0)
    with pytest.raises(ValueError, match="need at least one array to stack"):
        pt.main_connect_point_trajectories(d, str(tmp_path / "pc"), 2, 1.0, 0)
    assert not os.path.exists(str(tmp_path / "pc" / "track.npy"))


@pytest.mark.gpu
@pytest.mark.parametrize("skip", [False, True], ids=["path_consistency", "skip_path_consistency"])
def test_device_emitter_equals_the_oracle_for_the_tracker_result(gpu, skip):
    import torch
    g, fw, fb, f2, b2, occ, occ2 = _load()
    dv = lambda a, dt: tracker._on_device(a, dt)
    trk = tracker._ResidentTracker(36, 52, 2, len(fw) + 1, path_consistency=not skip)
    try:
        for t in range(len(fw)):
            f = dv(fw[t], torch.float32)
            if skip or t == 0:
                assert trk.step(f, dv(occ[t], torch.uint8)) == 0
            else:
                trk.optimize_buffer(trk.step(f, dv(occ[t], torch.uint8), prev, dv(f2[t - 1], torch.float32),
                                             dv(occ2[t - 1], torch.uint8)), None, None)
            prev = f
        arrays = trk.finish(2)
        with trk.track_npy_body() as body:
            dev = bytes(body.view())
    finally:
        trk.close()
    assert dev == tno.encode_body(arrays.ids, arrays.ptr, arrays.frame_ids, arrays.xy)


@pytest.mark.gpu
def test_device_emitter_equals_the_oracle_on_crafted_arrays(gpu):
    rng = np.random.default_rng(3)
    big_ptr = np.concatenate([[0], np.cumsum(rng.integers(1, 90, 5000))])
    big = tracker.TrackArrays(np.arange(5000, dtype=np.int64) * 997, big_ptr,
                              rng.integers(0, 70000, big_ptr[-1]).astype(np.int32), rng.normal(0, 300, (big_ptr[-1], 2)))
    for arrays in (crafted_track_arrays(), empty_track_arrays(), big):
        with tracker.track_npy_body_device(arrays) as body:
            assert bytes(body.view()) == tno.encode_body(arrays.ids, arrays.ptr, arrays.frame_ids, arrays.xy)
    for bad in _bad_arrays():
        with pytest.raises(_lib.PsfmError) as e:
            tracker.track_npy_body_device(bad)
        assert e.value.code == -1


@pytest.mark.gpu
def test_returned_arrays_and_the_file_feed_the_same_handoff(gpu, tmp_path):
    g, fw, fb, f2, b2, occ, occ2 = _load()
    d = write_flow_dir(str(tmp_path / "flows"), fw, fb, f2, b2)
    arrays = pt.main_connect_point_trajectories(d, str(tmp_path / "traj"))
    loaded = np.load(str(tmp_path / "traj" / "track.npy"), allow_pickle=True).item()
    n = len(fw) + 1
    ma, mf = handoff.traj_to_matches(arrays, n), handoff.traj_to_matches(loaded, n)
    assert all(np.array_equal(a, b) for a, b in zip(ma.keypoints, mf.keypoints))
    for k in ("pair_images", "pair_ptr", "matches"):
        assert np.array_equal(getattr(ma, k), getattr(mf, k))
    assert ma.matches.shape[0] > 0
