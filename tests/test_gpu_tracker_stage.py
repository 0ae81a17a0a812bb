"""The tracker stage resident on the GPU (tracker.track_optimize_device / main_connect_point_trajectories_device,
csrc/tracker.cu psfm_tracker_*): the same track set, bit for bit, as the host path (device=False with the library's
HP1) and as the golden set made from the reference (tests/golden/tracker_small.npz)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from particlesfm_b200 import _lib, handoff, synthetic as syn, tracker

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_tracker import _compare, _load, _oracle_opt   # noqa: E402


def _same(a, b):
    """Two track-set dicts are identical: keys and their order, types, frame ids, every double, labels."""
    assert list(a.keys()) == list(b.keys())
    for k in a:
        ta, tb = a[k], b[k]
        assert type(k) is int and list(ta.keys()) == list(tb.keys()) == ["frame_ids", "locations", "labels"]
        assert ta["frame_ids"] == tb["frame_ids"] and all(type(f) is int for f in ta["frame_ids"])
        assert ta["labels"] == tb["labels"] and not any(ta["labels"])
        assert len(ta["locations"]) == len(tb["locations"])
        for la, lb in zip(ta["locations"], tb["locations"]):
            assert la.dtype == lb.dtype == np.float64 and la.shape == lb.shape == (2,)
            assert np.array_equal(la, lb)


def _golden_filtered(res, g, min_len):
    ids, lens = g["ids"], g["lens"]
    off = np.concatenate([[0], np.cumsum(lens)])
    keep = [k for k in range(ids.shape[0]) if lens[k] >= min_len]
    assert list(res.keys()) == [int(ids[k]) for k in keep]
    for k in keep:
        t = res[int(ids[k])]
        assert t["frame_ids"] == g["frames"][off[k]:off[k + 1]].tolist()
        assert np.array_equal(np.stack(t["locations"]), g["locs"][off[k]:off[k + 1]])


@pytest.mark.gpu
def test_resident_stage_reproduces_the_golden_track_set(gpu):
    g, fw, fb, f2, b2, occ, occ2 = _load()
    arrays = tracker.track_optimize_device(fw, f2, occ, occ2, 2)
    assert isinstance(arrays, tracker.TrackArrays)
    _compare(arrays.to_dict(), g)
    _compare(tracker.track_optimize(fw, f2, occ, occ2, 2, device=True), g)
    res3 = tracker.main_connect_point_trajectories(fw, fb, f2, b2, 2, 1.0, 3, device=True)
    _golden_filtered(res3, g, 3)
    assert list(tracker.main_connect_point_trajectories_device(fw, fb, f2, b2, 2, 1.0, 3).ids) == list(res3.keys())


@pytest.mark.gpu
def test_custom_optimiser_through_the_buffer_callback(gpu):
    """A host optimiser (the CPU oracle) gets the buffered set through get/set buffer and gives the golden set."""
    g, fw, fb, f2, b2, occ, occ2 = _load()
    _compare(tracker.track_optimize(fw, f2, occ, occ2, 2, optimize_fn=_oracle_opt, device=True), g)
    _golden_filtered(tracker.main_connect_point_trajectories(fw, fb, f2, b2, 2, 1.0, 3, optimize_fn=_oracle_opt, device=True), g, 3)


def test_synthetic_sequence_is_the_golden_recipe():
    g, fw, fb, f2, b2, _, _ = _load()
    s = syn.make_flow_sequence(7, 36, 52, seed=11)
    for mine, gold in zip(s, (fw, fb, f2, b2)):
        assert len(mine) == len(gold) and all(np.array_equal(a, b) for a, b in zip(mine, gold))


@pytest.mark.gpu
@pytest.mark.parametrize("n_frames,h,w,ratio", [(11, 436, 1024, 2), (4, 480, 854, 1), (6, 101, 157, 3)])
def test_resident_stage_equals_host_path(gpu, n_frames, h, w, ratio):
    fw, fb, f2, b2 = syn.make_flow_sequence(n_frames, h, w, seed=n_frames + ratio)
    host = tracker.main_connect_point_trajectories(fw, fb, f2, b2, ratio, 1.0, 0)
    dev = tracker.main_connect_point_trajectories_device(fw, fb, f2, b2, ratio, 1.0, 0)
    assert dev.ptr[-1] == dev.xy.shape[0] == dev.frame_ids.shape[0]
    assert np.diff(dev.lengths()).any() and dev.frame_ids.max() == n_frames - 1       # particles died and were re-seeded
    _same(dev.to_dict(), host)
    _same(tracker.main_connect_point_trajectories(fw, fb, f2, b2, ratio, 1.0, 3, device=True),
          {k: v for k, v in host.items() if len(v["frame_ids"]) >= 3})


def _host_steps(flows, occs, h, w, ratio):
    """The host path's first frames without optimize_buffer (its selection is empty on them)."""
    import torch
    trajs = tracker.BatchedTrajectorySet(len(flows) + 1, h, w, ratio, None)
    for t, (flow, occ) in enumerate(zip(flows, occs)):
        trajs.new_traj_all(t, trajs.sample_candidates)
        cur = trajs.get_cur_pos()
        nxt = cur + tracker.grid_sample(torch.from_numpy(flow).permute(2, 0, 1).float(), cur)
        o = tracker.grid_sample(torch.from_numpy(occ).unsqueeze(0).float(), cur) > 0.1
        valid = (nxt[:, 0] > 0) * (nxt[:, 0] < w - 1) * (nxt[:, 1] > 0) * (nxt[:, 1] < h - 1)
        trajs.extend_all(nxt, t + 1, valid * (1.0 - np.squeeze(o, axis=-1)))
    trajs.clear_active()
    return trajs.full_trajs(0)


@pytest.mark.gpu
@pytest.mark.parametrize("ratio", [1, 2, 3])
def test_frame_where_every_particle_dies(gpu, ratio):
    """No survivor: the host path re-seeds from scipy's distance transform of an occupancy map without an occupied
    pixel; the resident stage seeds the same points."""
    import torch
    g, fw, fb, f2, b2, occ, occ2 = _load()
    h, w = occ[0].shape
    dead = np.ones((h, w), bool)
    host = _host_steps([fw[0], fw[1]], [dead, occ[1]], h, w, ratio)
    trk = tracker._ResidentTracker(h, w, ratio, 3)
    try:
        dv = lambda a, dt: tracker._on_device(a, dt)
        f0 = dv(fw[0], torch.float32)
        assert trk.step(f0, dv(dead, torch.uint8)) == 0
        assert trk.step(dv(fw[1], torch.float32), dv(occ[1], torch.uint8), f0, dv(f2[0], torch.float32),
                        dv(occ2[0], torch.uint8)) == 0
        dev = trk.finish(0)
    finally:
        trk.close()
    assert min(len(v["frame_ids"]) for v in host.values()) == 1 and max(v["frame_ids"][0] for v in host.values()) == 1
    _same(dev.to_dict(), host)
    # and the full stage then finds nothing to optimise, on both paths
    for at in (0, 1, 2):
        occ_dead = [dead if i == at else o for i, o in enumerate(occ)]
        with pytest.raises(ValueError, match="need at least one array to stack"):
            tracker.track_optimize(fw, f2, occ_dead, occ2, ratio)
        with pytest.raises(ValueError, match="need at least one array to stack"):
            tracker.track_optimize(fw, f2, occ_dead, occ2, ratio, device=True)


@pytest.mark.gpu
def test_cuda_tensor_inputs(gpu):
    import torch
    g, fw, fb, f2, b2, occ, occ2 = _load()
    cu = lambda xs: [torch.from_numpy(x).cuda() for x in xs]
    a = tracker.track_optimize_device(fw, f2, occ, occ2, 2)
    b = tracker.track_optimize_device(cu(fw), cu(f2), cu(occ), cu(occ2), 2)
    assert all(np.array_equal(getattr(a, k), getattr(b, k)) for k in ("ids", "ptr", "frame_ids", "xy"))
    c = tracker.main_connect_point_trajectories_device(cu(fw), cu(fb), cu(f2), cu(b2), 2, 1.0, 3)
    _golden_filtered(c.to_dict(), g, 3)
    _compare(tracker.track_optimize(cu(fw), cu(f2), cu(occ), cu(occ2), 2, optimize_fn=_oracle_opt, device=True), g)


@pytest.mark.gpu
def test_track_arrays_feed_the_handoff(gpu):
    g, fw, fb, f2, b2, occ, occ2 = _load()
    arrays = tracker.main_connect_point_trajectories_device(fw, fb, f2, b2, 2, 1.0, 3)
    d = arrays.to_dict()
    _same(d, tracker.main_connect_point_trajectories(fw, fb, f2, b2, 2, 1.0, 3))
    for x, y in zip(handoff.tracks_to_observations(arrays), handoff.tracks_to_observations(d)):
        if isinstance(x, list):
            assert x == y
        else:
            assert x.dtype == y.dtype and np.array_equal(x, y)
    n = len(fw) + 1
    ma, md = handoff.traj_to_matches(arrays, n), handoff.traj_to_matches(d, n)
    assert all(np.array_equal(a, b) for a, b in zip(ma.keypoints, md.keypoints))
    for k in ("pair_images", "pair_ptr", "matches"):
        assert np.array_equal(getattr(ma, k), getattr(md, k))
    assert ma.matches.shape[0] > 0


def test_track_arrays_to_dict_and_handoff_without_a_device():
    """TrackArrays is plain host data: its dict and hand-off equal those of the equivalent dict."""
    ids = np.array([0, 2, 5], np.int64)
    ptr = np.array([0, 3, 5, 9], np.int64)
    frame_ids = np.array([0, 1, 2, 1, 2, 0, 1, 2, 3], np.int32)
    xy = np.random.default_rng(0).uniform(0, 50, (9, 2))
    d = {int(i): {"frame_ids": frame_ids[s:e].astype(np.int64).tolist(), "locations": [xy[k].copy() for k in range(s, e)],
                  "labels": [False] * int(e - s)} for i, s, e in zip(ids, ptr[:-1], ptr[1:])}
    arrays = tracker.TrackArrays(ids, ptr, frame_ids, xy)
    out = arrays.to_dict()
    _same(out, d)
    out[0]["locations"][0][0] = -1.0
    assert xy[0, 0] != -1.0                                                  # the dict does not alias the arrays
    for x, y in zip(handoff.tracks_to_observations(arrays), handoff.tracks_to_observations(d)):
        assert x == y if isinstance(x, list) else (x.dtype == y.dtype and np.array_equal(x, y))
    ma, md = handoff.traj_to_matches(arrays, 4), handoff.traj_to_matches(d, 4)
    for k in ("pair_images", "pair_ptr", "matches"):
        assert np.array_equal(getattr(ma, k), getattr(md, k))


@pytest.mark.skipif(_lib.lib().psfm_device_count() > 0, reason="needs a machine WITHOUT a GPU")
def test_resident_stage_has_no_cpu_fallback():
    h = C.c_void_p()
    assert _lib.lib().psfm_tracker_create(36, 52, 2, 7, None, C.byref(h)) == -2          # PSFM_ERR_NO_DEVICE
    assert not h
    g, fw, fb, f2, b2, occ, occ2 = _load()
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        tracker.track_optimize(fw, f2, occ, occ2, 2, device=True)
    with pytest.raises(_lib.PsfmError, match="no CUDA device"):
        tracker.main_connect_point_trajectories(fw, fb, f2, b2, 2, 1.0, 3, device=True)


def test_argument_errors_carry_a_message():
    """Bad arguments are refused before any device is needed, with the call named in psfm_last_error."""
    L = _lib.lib()
    assert L.psfm_tracker_create(36, 52, 2, 7, None, None) == -1
    assert b"psfm_tracker_create" in L.psfm_last_error()
    assert L.psfm_flow_check_device(None, None, 36, 52, 1.0, None, None, None) == -1
    assert b"psfm_flow_check_device" in L.psfm_last_error()
    assert L.psfm_tracker_advance(None, None, None, None, None, None, None) == -1
    assert b"psfm_tracker_advance" in L.psfm_last_error()


@pytest.mark.parametrize("ratio", [1, 2, 3])
def test_scipy_distance_transform_without_an_occupied_pixel(ratio):
    """The rule k_reseed_stage uses when no particle survives: scipy's distance_transform_edt of the
    [H, W, 1] occupancy map extend_all builds, with no occupied pixel, exceeds r exactly where
    (y + 1)^2 + x^2 > r^2 (its value there is sqrt((y + 1)^2 + x^2))."""
    ndimage = pytest.importorskip("scipy.ndimage")
    for h, w in [(36, 52), (101, 157)]:
        dist = ndimage.distance_transform_edt(1.0 - np.zeros((h, w, 1)))[..., 0]
        yy, xx = np.meshgrid(np.arange(h), np.arange(w), indexing="ij")
        assert np.array_equal(dist, np.sqrt((yy + 1.0) ** 2 + xx ** 2))
        assert np.array_equal((dist > ratio)[::ratio, ::ratio], (((yy + 1) ** 2 + xx ** 2) > ratio * ratio)[::ratio, ::ratio])


@pytest.mark.gpu
def test_c_abi_back_to_back_on_the_legacy_stream(gpu):
    """The C ABI with stream NULL (the legacy default stream), psfm_tracker_optimize called right after
    psfm_tracker_advance with nothing in between: HP1 is ordered after the kernels that build its inputs."""
    import torch
    g, fw, fb, f2, b2, occ, occ2 = _load()
    L = _lib.lib()
    dv = lambda a, dt: tracker._on_device(a, dt)
    flows = [dv(f, torch.float32) for f in fw]
    occs = [dv(o, torch.uint8) for o in occ]
    flows2 = [dv(f, torch.float32) for f in f2]
    occs2 = [dv(o, torch.uint8) for o in occ2]
    torch.cuda.synchronize()
    h, w = occ[0].shape
    handle = C.c_void_p()
    _lib.check(L.psfm_tracker_create(h, w, 2, len(fw) + 1, None, C.byref(handle)), "psfm_tracker_create")
    try:
        counts = (C.c_int32 * 3)()
        for t in range(len(fw)):
            prev = (flows[t - 1].data_ptr(), flows2[t - 1].data_ptr(), occs2[t - 1].data_ptr()) if t else (None, None, None)
            _lib.check(L.psfm_tracker_advance(handle, flows[t].data_ptr(), occs[t].data_ptr(), *prev, counts), "advance")
            if t:
                assert counts[2] > 0
                _lib.check(L.psfm_tracker_optimize(handle, None, None), "optimize")
        nt, m = C.c_int64(), C.c_int64()
        _lib.check(L.psfm_tracker_finish(handle, 0, C.byref(nt), C.byref(m)), "finish")
        ids, ptr = np.empty(nt.value, np.int64), np.empty(nt.value + 1, np.int64)
        frame_ids, xy = np.empty(m.value, np.int32), np.empty((m.value, 2))
        i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))
        _lib.check(L.psfm_tracker_result(handle, i64(ids), i64(ptr), frame_ids.ctypes.data_as(C.POINTER(C.c_int32)),
                                         _lib.dptr(xy)), "result")
    finally:
        L.psfm_tracker_destroy(handle)
    _compare(tracker.TrackArrays(ids, ptr, frame_ids, xy).to_dict(), g)
