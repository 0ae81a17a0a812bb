"""The point-trajectory command's host side (particlesfm_b200.point_trajectory, tracker.track): the .flo reader and
the checks that refuse malformed flow directories before anything is written, the skip-path-consistency tracker
against the reference's track.py (tests/golden/track_small.npz), and the track.npy state encoding of the numpy
oracle framed into a file that loads as the TrajectorySet of the same track set."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import track_npy_oracle as tno
from particlesfm_b200 import _lib, point_trajectory as pt, tracker

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden", "track_small.npz")
sys.path.insert(0, HERE)
from test_tracker import _compare, _load   # noqa: E402


def write_flo(path, flow, tag=pt.TAG_FLOAT, trailing=b""):
    h, w = flow.shape[:2]
    with open(path, "wb") as f:
        f.write(np.array([tag], "<f4").tobytes() + np.array([w, h], "<i4").tobytes())
        f.write(np.ascontiguousarray(flow, "<f4").tobytes() + trailing)


def write_flow_dir(root, fw, fb, f2=None, b2=None):
    for name, maps in (("flow_f", fw), ("flow_b", fb), ("flow_f2", f2), ("flow_b2", b2)):
        if maps is None:
            continue
        os.makedirs(os.path.join(root, name), exist_ok=True)
        for i, m in enumerate(maps):
            write_flo(os.path.join(root, name, "%05d.flo" % i), m)
    return root


def _flows(n=4, h=6, w=9, seed=0):
    rng = np.random.default_rng(seed)
    return [rng.normal(0, 1, (h, w, 2)).astype(np.float32) for _ in range(n)]


def test_read_flo_ignores_trailing_bytes(tmp_path):
    f = _flows(1, 5, 7)[0]
    p = str(tmp_path / "a.flo")
    write_flo(p, f, trailing=b"\x01\x02\x03")
    out = pt.read_flo(p)
    assert out.dtype == np.float32 and out.shape == (5, 7, 2) and np.array_equal(out, f)
    assert pt.flo_size(p) == (5, 7)


def _malformed_cases(root):
    """(name, flow_dir, path the message names, skip_path_consistency) for each refused input"""
    fw = _flows(4)
    cases = []
    d = write_flow_dir(os.path.join(root, "short"), fw, fw, fw[:3], fw[:3])
    bad = os.path.join(d, "flow_b", "00002.flo")
    with open(bad, "r+b") as f:
        f.truncate(12 + 8 * 6 * 9 - 4)
    cases.append(("short file", d, bad, False))
    d = write_flow_dir(os.path.join(root, "header"), fw, fw, fw[:3], fw[:3])
    bad = os.path.join(d, "flow_f", "00001.flo")
    with open(bad, "r+b") as f:
        f.truncate(7)
    cases.append(("file shorter than the header", d, bad, True))
    d = write_flow_dir(os.path.join(root, "tag"), fw, fw, fw[:3], fw[:3])
    bad = os.path.join(d, "flow_f2", "00001.flo")
    write_flo(bad, fw[0], tag=1.0)
    cases.append(("bad tag", d, bad, False))
    d = write_flow_dir(os.path.join(root, "sizes"), fw, fw, fw[:3], fw[:3])
    bad = os.path.join(d, "flow_f", "00003.flo")
    write_flo(bad, np.zeros((6, 10, 2), np.float32))
    cases.append(("maps of different sizes", d, bad, True))
    d = write_flow_dir(os.path.join(root, "empty"), [], fw)
    os.makedirs(os.path.join(d, "flow_f"), exist_ok=True)
    cases.append(("empty flow_f", d, os.path.join(d, "flow_f"), True))
    d = write_flow_dir(os.path.join(root, "count"), fw, fw[:3])
    cases.append(("flow_b count", d, os.path.join(d, "flow_b"), True))
    d = write_flow_dir(os.path.join(root, "f2"), fw, fw, fw[:2], fw[:3])
    cases.append(("too few flow_f2", d, os.path.join(d, "flow_f2"), False))
    d = write_flow_dir(os.path.join(root, "b2"), fw, fw, fw[:3])
    cases.append(("missing flow_b2", d, os.path.join(d, "flow_b2"), False))
    return cases


def test_malformed_flow_directories_are_refused_before_anything_is_written(tmp_path):
    for name, d, named, skip in _malformed_cases(str(tmp_path / "flows")):
        traj = str(tmp_path / "traj" / name.replace(" ", "_"))
        with pytest.raises(ValueError) as e:
            pt.main_connect_point_trajectories(d, traj, skip_path_consistency=skip)
        assert named in str(e.value), (name, str(e.value))
        assert not os.path.exists(os.path.join(traj, "track.npy")) and not os.path.exists(os.path.join(traj, "track.npy.tmp"))
        argv = ["--flow_dir", d, "--traj_dir", traj] + (["--skip_path_consistency"] if skip else [])
        assert pt.main(argv) != 0, name
        assert not os.path.exists(os.path.join(traj, "track.npy"))


def test_cli_exits_non_zero_with_the_message(tmp_path):
    name, d, named, skip = _malformed_cases(str(tmp_path / "flows"))[2]
    r = subprocess.run([sys.executable, "-m", "particlesfm_b200.point_trajectory", "--flow_dir", d, "--traj_dir",
                        str(tmp_path / "traj")], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode != 0 and named in r.stderr
    assert not os.path.exists(str(tmp_path / "traj" / "track.npy"))


def test_extra_maps_are_ignored_and_skip_mode_does_not_open_the_stride_two_maps(tmp_path):
    fw = _flows(4)
    d = write_flow_dir(str(tmp_path / "a"), fw, fw, fw + fw, fw)
    frames, h, w = pt.flow_frames(d)
    assert (h, w) == (6, 9) and [len(f) for f in frames] == [2, 4, 4, 4]
    assert frames[3][2].endswith(os.path.join("flow_f2", "00002.flo"))
    d = write_flow_dir(str(tmp_path / "b"), fw, fw)
    os.makedirs(os.path.join(d, "flow_f2"))
    write_flo(os.path.join(d, "flow_f2", "00000.flo"), fw[0], tag=3.0)
    frames, _, _ = pt.flow_frames(d, skip_path_consistency=True)
    assert [len(f) for f in frames] == [2, 2, 2, 2]
    with pytest.raises(ValueError, match="flow_f2"):
        pt.flow_frames(d)


def test_skip_exists_leaves_the_file_and_opens_no_flow(tmp_path):
    traj = tmp_path / "traj"
    traj.mkdir()
    (traj / "track.npy").write_bytes(b"keep me")
    name, d, _, _ = _malformed_cases(str(tmp_path / "flows"))[0]
    assert pt.main_connect_point_trajectories(d, str(traj), skip_exists=True) is None
    assert pt.main(["--flow_dir", str(tmp_path / "nowhere"), "--traj_dir", str(traj), "--skip_exists"]) == 0
    assert (traj / "track.npy").read_bytes() == b"keep me"
    new = tmp_path / "made" / "deeper"
    with pytest.raises(ValueError):
        pt.main_connect_point_trajectories(d, str(new), skip_exists=True)
    assert new.is_dir() and not (new / "track.npy").exists()        # created as the reference creates it


def test_host_track_reproduces_the_reference_track_py():
    g = np.load(GOLD)
    _, fw, fb, f2, b2, occ, occ2 = _load()
    res = tracker.track(fw, occ, 2)
    _compare(res, g)
    res3 = tracker.track(fw, occ, 2, traj_min_len=3)
    assert sorted(res3) == [int(i) for i, n in zip(g["ids"], g["lens"]) if n >= 3]
    assert np.diff(g["lens"]).any() and g["frames"].max() == len(fw)


def crafted_track_arrays():
    """TrackArrays whose opcode widths switch: ids below 256, from 256, from 65,536 and up to 2^31 - 1, frame ids
    from 256 and beyond 65,535, length-1 and length-0 trajectories, an id order that is not sorted."""
    rng = np.random.default_rng(5)
    ids = np.array([3, 0, 255, 256, 65535, 65536, 1 << 20, 2 ** 31 - 1], np.int64)
    lens = np.array([1, 2, 40, 0, 1, 33, 5, 1], np.int64)
    ptr = np.concatenate([[0], np.cumsum(lens)])
    frames = np.concatenate([np.sort(rng.choice(np.r_[0:300, 65530:65540, 2 ** 31 - 3:2 ** 31], n, replace=False))
                             for n in lens]).astype(np.int32)
    xy = rng.normal(0, 500.0, (ptr[-1], 2))
    xy[0] = [-0.0, np.inf]
    xy[1] = [5e-324, 1.0 / 3.0]
    return tracker.TrackArrays(ids, ptr, frames, xy)


def empty_track_arrays():
    return tracker.TrackArrays(np.zeros(0, np.int64), np.zeros(1, np.int64), np.zeros(0, np.int32), np.zeros((0, 2)))


def same_set(loaded, arrays):
    """loaded.as_dict() is identical to TrajectorySet(arrays.to_dict()).as_dict()"""
    ref = pt._particlesfm().TrajectorySet(arrays.to_dict()).as_dict()
    got = loaded.as_dict()
    assert type(loaded).__name__ == "TrajectorySet" and list(got) == list(ref) and all(type(k) is int for k in got)
    for k in ref:
        assert got[k]["frame_ids"] == ref[k]["frame_ids"] and all(type(f) is int for f in got[k]["frame_ids"])
        assert got[k]["labels"] == ref[k]["labels"] and not any(got[k]["labels"])
        assert len(got[k]["locations"]) == len(ref[k]["locations"])
        for a, b in zip(got[k]["locations"], ref[k]["locations"]):
            assert a.dtype == np.float64 and a.shape == (2,) and a.tobytes() == b.tobytes()


@pytest.mark.parametrize("arrays", [crafted_track_arrays(), empty_track_arrays()], ids=["crafted", "empty"])
def test_oracle_body_framed_into_track_npy_loads_as_the_track_set(tmp_path, arrays):
    body = tno.encode_body(arrays.ids, arrays.ptr, arrays.frame_ids, arrays.xy)
    path = str(tmp_path / "track.npy")
    pt.write_track_npy(path, body)
    same_set(np.load(path, allow_pickle=True).item(), arrays)
    assert not os.path.exists(path + ".tmp")
    if arrays.ids.shape[0]:
        m = arrays.frame_ids.shape[0]
        assert 20 * m < len(body) < 24 * m + 60 * arrays.ids.shape[0]


def test_oracle_body_uses_only_protocol_two_opcodes_without_memo():
    import pickletools
    a = crafted_track_arrays()
    body = tno.encode_body(a.ids, a.ptr, a.frame_ids, a.xy)
    codes = {op.code for op, _, _ in pickletools.genops(body + b".")} - {"."}
    assert codes == set("}(KMJX]eGu") | {"\x86", "\x89"}


def _bad_arrays():
    a = crafted_track_arrays()
    ids_hi, ids_neg, fr_neg, ptr_back = a.ids.copy(), a.ids.copy(), a.frame_ids.copy(), a.ptr.copy()
    ids_hi[2] = 2 ** 31
    ids_neg[0] = -1
    fr_neg[4] = -1
    ptr_back[2], ptr_back[3] = ptr_back[3], ptr_back[2]
    return [tracker.TrackArrays(ids_hi, a.ptr, a.frame_ids, a.xy), tracker.TrackArrays(ids_neg, a.ptr, a.frame_ids, a.xy),
            tracker.TrackArrays(a.ids, a.ptr, fr_neg, a.xy), tracker.TrackArrays(a.ids, ptr_back, a.frame_ids, a.xy)]


def test_bad_arrays_are_refused_by_both_encoders_before_the_device():
    for bad in _bad_arrays():
        with pytest.raises(ValueError):
            tno.encode_body(bad.ids, bad.ptr, bad.frame_ids, bad.xy)
        with pytest.raises(_lib.PsfmError) as e:
            tracker.track_npy_body_device(bad)
        assert e.value.code == -1 and "psfm_track_npy_create" in str(e.value)
