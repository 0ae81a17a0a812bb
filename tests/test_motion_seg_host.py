"""The trajectory labeller's host side (particlesfm_b200.motion_seg): windows, the shuffle, the track-set export, the
weights loader, the command's refusals and the C ABI's argument checks, all without a device."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle.motion_seg_oracle as O
from particlesfm_b200 import _abi, _lib, device_count, launch_count, motion_seg


@pytest.mark.parametrize("length,window", [(1, 1), (5, 1), (12, 5), (10, 5), (10, 10), (9, 10), (80, 10), (81, 10),
                                           (7, 3), (3, 7), (13, 4)])
def test_windows_equal_load_cut_seq(length, window):
    starts, L = motion_seg.window_starts(length, window)
    assert [list(range(s, s + L)) for s in starts] == O.windows(length, window)


@pytest.mark.parametrize("K", [1, 2, 7, 1000])
def test_shuffle_is_the_track_sets_cut(K):
    from particlesfm_b200.point_trajectory import _particlesfm
    particlesfm = _particlesfm()
    s = particlesfm.TrajectorySet({i * 3 + 1: {"frame_ids": [0, 1, 2], "locations": [[0, 0]] * 3,
                                               "labels": [False] * 3} for i in range(K)})
    s.build_invert_indexes()
    cap = max(1, K // 2)
    got = s.sample_inside_window([0, 1, 2], 3, cap)["traj_ids"]
    ids = np.arange(K) * 3 + 1
    perm = motion_seg.shuffle_permutation(K)
    want = ids.tolist() if K <= cap else ids[perm[:cap]].tolist()
    assert list(got) == want


def test_csr_export_is_what_the_sampler_sees():
    from particlesfm_b200.point_trajectory import _particlesfm
    particlesfm = _particlesfm()
    s = particlesfm.TrajectorySet({9: {"frame_ids": [4, 2, 2, 3], "locations": [[1, 1], [2, 2], [3, 3], [4, 4]],
                                       "labels": [False] * 4},
                                   5: {"frame_ids": [0], "locations": [[7, 8]], "labels": [False]}})
    ids, ptr, frames, xy = s.csr()
    assert ids.tolist() == [5, 9] and ptr.tolist() == [0, 1, 4]
    assert frames.tolist() == [0, 2, 3, 4]
    assert xy.tolist() == [[7, 8], [2, 2], [4, 4], [1, 1]]


def _ckpt(tmp_path, sd, name="ckpt.pth", wrap=True):
    import torch
    p = str(tmp_path / name)
    torch.save({"model_state_dict": sd} if wrap else sd, p)
    return p


def test_loader_takes_the_seeded_weights(tmp_path):
    w = motion_seg.load_weights(_ckpt(tmp_path, O.seeded_state_dict(0)))
    assert motion_seg.pack_encoder(w).shape == (motion_seg.ENCODER_FLOATS,)


@pytest.mark.parametrize("bad", ["no_entry", "unexpected", "missing", "shape"])
def test_loader_refuses(tmp_path, bad):
    import torch
    sd = O.seeded_state_dict(0)
    if bad == "unexpected":
        sd["decoder.extra.weight"] = torch.zeros(1)
    elif bad == "missing":
        del sd["decoder.output.bias"]
    elif bad == "shape":
        sd["decoder.output.bias"] = torch.zeros(2)
    p = _ckpt(tmp_path, sd, wrap=bad != "no_entry")
    with pytest.raises(ValueError, match="ckpt.pth"):
        motion_seg.load_weights(p)


def _inputs(tmp_path, n=6, h=24, w=40):
    import cv2
    root = str(tmp_path)
    img, dep, trj = (os.path.join(root, d) for d in ("images", "depth", "traj"))
    for d in (img, dep, trj):
        os.makedirs(d)
    for i in range(n):
        cv2.imwrite(os.path.join(img, "%03d.png" % i), O.seeded_frames(1, h, w, i)[0])
        cv2.imwrite(os.path.join(dep, "%03d.png" % i), O.seeded_depth_pixels(1, h, w, i)[0])
    np.save(os.path.join(trj, "track.npy"), O.seeded_track_set(20, n, h, w, 1))
    return img, dep, trj, _ckpt(tmp_path, O.seeded_state_dict(0))


def _run(img, dep, trj, ckpt, *extra):
    return motion_seg.main(["--image_dir", img, "--depth_dir", dep, "--traj_dir", trj, "--model", ckpt] + list(extra))


@pytest.mark.parametrize("bad", ["image", "image_size", "depth_stem", "depth_bits", "depth_size", "track",
                                 "window", "cap", "weights"])
def test_refusals_exit_2_naming_the_file(tmp_path, capsys, bad):
    import cv2
    img, dep, trj, ckpt = _inputs(tmp_path)
    extra, name = [], None
    if bad == "image":
        name = os.path.join(img, "zzz.txt")
        open(name, "w").write("not an image")
    elif bad == "image_size":
        name = os.path.join(img, "003.png")
        cv2.imwrite(name, np.zeros((10, 10, 3), np.uint8))
    elif bad == "depth_stem":
        name = os.path.join(dep, "xyz.png")
        os.rename(os.path.join(dep, "005.png"), name)
    elif bad == "depth_bits":
        name = os.path.join(dep, "002.png")
        cv2.imwrite(name, np.zeros((24, 40), np.uint8))
    elif bad == "depth_size":
        name = os.path.join(dep, "004.png")
        cv2.imwrite(name, np.zeros((20, 40), np.uint16))
    elif bad == "track":
        name = os.path.join(trj, "track.npy")
        np.save(name, {1: {"frame_ids": [0]}})
    elif bad == "window":
        extra, name = ["--window_size", "0"], "window_size"
    elif bad == "cap":
        extra, name = ["--traj_max_num", "0"], "traj_max_num"
    else:
        name = ckpt
        _ckpt(tmp_path, {"x": 1}, wrap=False)
    n0 = launch_count()
    assert _run(img, dep, trj, ckpt, *extra) == 2
    assert name in capsys.readouterr().err
    assert launch_count() == n0
    assert not os.path.exists(trj + "_labeled/track.npy")


P = C.c_void_p(256)        # never dereferenced: every call below is refused before the device is touched
ENTRIES = ["psfm_seg_hits", "psfm_seg_windows", "psfm_seg_depth_resize", "psfm_seg_encode", "psfm_seg_merge",
           "psfm_seg_draw"]


def _calls(L, p=P, n=4, win=1, rows=8, h=24):
    return {
        "psfm_seg_hits": lambda: L.psfm_seg_hits(p, p, n, p, win, 5, p, None),
        "psfm_seg_windows": lambda: L.psfm_seg_windows(p, p, p, p, p, rows, p, 5, p, p, None),
        "psfm_seg_depth_resize": lambda: L.psfm_seg_depth_resize(p, n, h, 40, p, None),
        "psfm_seg_encode": lambda: L.psfm_seg_encode(p, p, p, p, win, rows, 5, p, n, h, 40, p, p, None),
        "psfm_seg_merge": lambda: L.psfm_seg_merge(p, p, n, p, win, 5, p, p, p, p, None),
        "psfm_seg_draw": lambda: L.psfm_seg_draw(p, p, p, p, rows, 5, h, 40, p, 3, p, 5, 5, 5, p, p, None),
    }


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("why", ["null", "count", "size"])
def test_bad_arguments_are_invalid_before_any_launch(entry, why):
    L = _lib.lib()
    if why == "null":
        call = _calls(L, p=None)[entry]
    elif why == "count":
        call = _calls(L, n=0, win=0, rows=-1)[entry]
    else:
        if entry in ("psfm_seg_hits", "psfm_seg_windows", "psfm_seg_merge"):
            pytest.skip("no frame size")
        call = _calls(L, h=0)[entry]
    n0 = launch_count()
    assert call() == _abi.PSFM_ERR_INVALID
    assert entry in L.psfm_last_error().decode()
    assert launch_count() == n0


def test_encoder_refuses_a_window_longer_than_shared_memory_holds():
    L = _lib.lib()
    longest = L.psfm_seg_max_window()
    assert longest >= 100
    assert L.psfm_seg_encode(P, P, P, P, 1, 8, longest + 1, P, 4, 24, 40, P, P, None) == _abi.PSFM_ERR_INVALID
    assert "exceeds" in L.psfm_last_error().decode()


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
@pytest.mark.parametrize("entry", ENTRIES)
def test_no_device_is_refused(entry):
    L = _lib.lib()
    assert _calls(L)[entry]() == _abi.PSFM_ERR_NO_DEVICE
    assert "%s: no CUDA device" % entry in L.psfm_last_error().decode()


def test_labels_reach_the_hand_off():
    from particlesfm_b200 import handoff
    from particlesfm_b200.tracker import TrackArrays
    t = TrackArrays(np.array([4, 7]), np.array([0, 2, 5]), np.array([0, 1, 0, 1, 2], np.int32),
                    np.arange(10, dtype=np.float64).reshape(5, 2))
    keys, traj, frames, _ = handoff._flatten(t, True)
    assert traj.tolist() == [0, 0, 1, 1, 1]
    t.labels = np.array([False, True, True, False, False])
    keys, traj, frames, xy = handoff._flatten(t, True)
    assert traj.tolist() == [0, 1, 1] and frames.tolist() == [0, 1, 2]
    assert handoff._flatten(t, False)[1].tolist() == [0, 0, 1, 1, 1]
    assert t.to_dict()[4]["labels"] == [False, True]


def test_a_window_longer_than_the_encoder_takes_is_refused():
    import torch
    from particlesfm_b200.tracker import TrackArrays
    longest = _lib.lib().psfm_seg_max_window()
    tracks = TrackArrays(np.array([1]), np.array([0, 1]), np.array([0], np.int32), np.zeros((1, 2)))
    with pytest.raises(ValueError, match="--window_size"):
        motion_seg.label_trajectories(tracks, torch.zeros((longest + 1, 2, 2), dtype=torch.uint16), (2, 2),
                                      {}, window_size=longest + 5)
    motion_seg.check_window_length(longest + 1, longest)       # windows of `longest` frames are taken
