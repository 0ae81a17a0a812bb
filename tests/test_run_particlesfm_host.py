"""The whole-pipeline command without a device (particlesfm_b200.run_particlesfm, DESIGN.md §4.15): its refusals, its
file plan, the frame-readiness logic that feeds the tracker from the flow batches, and the --root_dir scheduler."""
import itertools
import os
import subprocess
import sys
import textwrap
import time

import numpy as np
import pytest
from PIL import Image

from oracle import raft_oracle as ro
from particlesfm_b200 import optical_flow as of, run_particlesfm as rp


# ------------------------------------------------------------------------------------------------ refusals

def _frames(d, n=3, h=123, w=125):
    os.makedirs(d, exist_ok=True)
    for i, f in enumerate(ro.seeded_frames(n, h, w, seed=1)):
        Image.fromarray(f).save(os.path.join(d, "%05d.png" % i))
    return d


@pytest.fixture(scope="module")
def weights(tmp_path_factory):
    import torch
    p = str(tmp_path_factory.mktemp("w") / "w.pth")
    torch.save(ro.seeded_state_dict(0), p)
    return p


def _run(argv, capsys):
    rc = rp.main(argv)
    return rc, capsys.readouterr().err


def test_refusals_write_nothing(tmp_path, weights, capsys):
    img = _frames(str(tmp_path / "img"))
    out = tmp_path / "out"
    out.mkdir()
    base = ["--model", weights, "-i", img, "-o", str(out), "--assume_static"]
    short = _frames(str(tmp_path / "short"), n=1)
    tiny = _frames(str(tmp_path / "tiny"), n=3, h=100, w=125)
    stray = _frames(str(tmp_path / "stray"))
    open(os.path.join(stray, "notes.txt"), "w").write("not a frame\n")
    jpeg = _frames(str(tmp_path / "jpeg"))
    Image.fromarray(ro.seeded_frames(1, 123, 125, seed=3)[0]).save(os.path.join(jpeg, "00009.jpeg"))
    bad_weights = str(tmp_path / "bad.pth")
    open(bad_weights, "wb").write(b"not a checkpoint")
    root = tmp_path / "root"
    (root / "a" / "images").mkdir(parents=True)
    (root / "b").mkdir()
    cases = [
        (["--model", weights, "-i", img, "-o", str(out)], "--assume_static"),
        (base + ["--sfm_type", "incremental_colmap"], "--sfm_type incremental_colmap"),
        (["--model", bad_weights, "-i", img, "-o", str(out), "--assume_static"], bad_weights),
        (["--model", str(tmp_path / "missing.pth"), "-i", img, "-o", str(out), "--assume_static"], "missing.pth"),
        (["--model", weights, "-i", short, "-o", str(out), "--assume_static"], short),
        (["--model", weights, "-i", tiny, "-o", str(out), "--assume_static"], "at least 121"),
        (["--model", weights, "-i", stray, "-o", str(out), "--assume_static"], "notes.txt"),
        (["--model", weights, "-i", jpeg, "-o", str(out), "--assume_static"], "00009.jpeg"),
        (["--model", weights, "-i", str(tmp_path / "nowhere"), "-o", str(out), "--assume_static"], "nowhere"),
        (["--model", weights, "--root_dir", str(root), "--assume_static"], os.path.join(str(root), "b")),
        (["--model", weights, "--assume_static"], "no input"),
    ]
    for argv, needle in cases:
        rc, err = _run(argv, capsys)
        assert rc == 2, (argv, err)
        assert needle in err, (needle, err)
        assert os.listdir(out) == [], argv
    assert sorted(os.listdir(root)) == ["a", "b"] and os.listdir(root / "a") == ["images"]
    # motion segmentation is named in the message, and --assume_static suggested
    _, err = _run(["--model", weights, "-i", img, "-o", str(out)], capsys)
    assert "motion segmentation" in err and "--assume_static" in err


def test_stray_file_is_no_refusal_without_sfm(tmp_path, weights):
    """The image-set check pairs frame ids with database ids; without the SfM step there is nothing to pair."""
    stray = _frames(str(tmp_path / "stray"))
    open(os.path.join(stray, "notes.txt"), "w").write("x")
    paths, h, w, _ = rp.check_inputs(stray, weights, None, with_sfm=False)
    assert len(paths) == 3 and (h, w) == (123, 125)


def test_help_names_the_forwarded_traj_min_len():
    text = rp.build_parser().format_help()
    assert "--traj_min_len" in text and "never passes it on" in " ".join(text.split())


# ------------------------------------------------------------------------------------------------ file plan

def _reference(keep, skip_sfm, skip_exists, has_track, has_flows):
    """What run_particlesfm.py:25-119 does with --assume_static: (stages run, intermediates it leaves written)."""
    stages = ["flows"]                                  # every pair, existing files skipped under skip_exists
    if not (skip_exists and has_track):
        stages.append("trajectories")
    if not skip_sfm:
        stages.append("sfm")
    left = set()
    if keep:
        left.add("optical_flows")
    if keep or skip_sfm:
        left.add("track.npy")
    return stages, left


@pytest.mark.parametrize("keep,skip_sfm,skip_exists,has_track,has_flows",
                         list(itertools.product((False, True), repeat=5)))
def test_file_plan(tmp_path, keep, skip_sfm, skip_exists, has_track, has_flows):
    out = str(tmp_path)
    flow_dir, traj_dir, npy = rp.workspace_paths(out)
    if has_track:
        os.makedirs(traj_dir)
        open(npy, "wb").close()
    if has_flows:
        os.makedirs(flow_dir)
    p = rp.plan(out, skip_sfm, skip_exists, keep)
    ref_stages, ref_left = _reference(keep, skip_sfm, skip_exists, has_track, has_flows)
    written = {n for n, w in (("optical_flows", p.write_flows), ("track.npy", p.write_track)) if w}
    stages = [s for st in p.stages() for s in (["flows", "trajectories"] if st == "flows_trajectories" else [st])]
    if skip_exists and has_track:
        # the existing track set is read: no flow is computed (the reference fills in missing flows it never reads),
        # nothing is written, and the existing files stay
        assert p.route == "track_npy" and written == set()
        assert stages == [s for s in ref_stages if s != "flows"]
        return
    assert stages == ref_stages
    if skip_exists and has_flows:
        # the existing flow directory is completed and tracked from, and is not deleted afterwards
        assert p.route == "flow_dir" and written == ref_left | {"optical_flows"}
    else:
        assert p.route == "fused" and written == ref_left


# ------------------------------------------------------------------------------------------------ frame readiness

def _tag(t, s, d):
    return float(1000 * t + 10 * s + d)


@pytest.mark.parametrize("pc", [True, False])
@pytest.mark.parametrize("per", [1, 2, 3, 4])
@pytest.mark.parametrize("n", [2, 3, 4, 7])
def test_frames_advance_once_in_order_with_bounded_maps(pc, per, n):
    calls, shared = [], []
    tag = lambda m: None if m is None else float(m[0])
    feed = rp.FrameFeed(n, pc, lambda t, f, b, prev, f2, b2: calls.append((t, tag(f), tag(b), tag(prev), tag(f2), tag(b2))),
                        keep=np.copy)
    pairs = of._pairs(n, pc)
    for b0 in range(0, len(pairs), per):
        batch = pairs[b0:b0 + per]
        flows = np.array([[_tag(t, s, 1)] for t, s in batch] + [[_tag(t, s, 2)] for t, s in batch])
        feed(batch, flows, None)
        assert feed.held() <= 3, (batch, feed.held())
        # nothing the sink keeps is a view of the batch, so the batch can be freed
        held = [m for fb in feed.maps.values() for m in fb] + ([feed.prev] if feed.prev is not None else [])
        assert not any(np.shares_memory(m, flows) for m in held)
        shared.append(feed.held())
    feed.done()
    assert [c[0] for c in calls] == list(range(n - 1))
    for t, f, b, prev, f2, b2 in calls:
        assert (f, b) == (_tag(t, 1, 1), _tag(t, 1, 2))
        if pc and t >= 1:
            assert (prev, f2, b2) == (_tag(t - 1, 1, 1), _tag(t - 1, 2, 1), _tag(t - 1, 2, 2))
        else:
            assert (prev, f2, b2) == (None, None, None)
    assert feed.held() == 0


def test_missing_pairs_are_reported():
    feed = rp.FrameFeed(4, True, lambda *a: None, keep=np.copy)
    feed([(0, 1), (0, 2)], np.zeros((4, 1)), None)
    with pytest.raises(RuntimeError, match="1 of 3 frames"):
        feed.done()


# ------------------------------------------------------------------------------------------------ --root_dir

STUB = textwrap.dedent("""
    import os, sys, time
    ws = sys.argv[sys.argv.index("--workspace_dir") + 1]
    t0 = time.time()
    time.sleep(0.4)
    with open(os.path.join(ws, "ran.txt"), "w") as f:
        f.write("%s %r %r\\n" % (os.environ.get("CUDA_VISIBLE_DEVICES"), t0, time.time()))
    sys.exit(3 if os.path.basename(ws).startswith("bad") else 0)
""")


def _root(tmp_path, names):
    root = tmp_path / "root"
    for n in names:
        (root / n / "images").mkdir(parents=True)
    return str(root)


def _records(root, names):
    out = {}
    for n in names:
        dev, t0, t1 = open(os.path.join(root, n, "ran.txt")).read().split()
        out[n] = (dev, float(t0), float(t1))
    return out


@pytest.mark.parametrize("devices", [["0"], ["3", "1"], ["2", "5", "7"]])
def test_root_dir_runs_one_child_per_device(tmp_path, devices):
    names = ["s%d" % i for i in range(5)]
    root = _root(tmp_path, names)
    args = rp.build_parser().parse_args(["--model", "w.pth", "--root_dir", root, "--assume_static"])
    lines = []
    rc = rp.run_root(args, devices=devices, command=[sys.executable, "-c", STUB], out=lines.append)
    assert rc == 0
    rec = _records(root, names)
    assert all(dev in devices for dev, _, _ in rec.values())
    for d in devices:
        spans = sorted((t0, t1) for dev, t0, t1 in rec.values() if dev == d)
        assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:])), (d, spans)
    if len(devices) > 1:
        assert len({dev for dev, _, _ in rec.values()}) > 1
    assert sum(1 for line in lines if ": done on device" in line) == len(names)


def test_a_failing_sequence_fails_the_run_and_the_others_still_run(tmp_path):
    names = ["a", "bad", "c", "d"]
    root = _root(tmp_path, names)
    args = rp.build_parser().parse_args(["--model", "w.pth", "--root_dir", root, "--assume_static"])
    lines = []
    rc = rp.run_root(args, devices=["0", "1"], command=[sys.executable, "-c", STUB], out=lines.append)
    assert rc == 1
    assert set(_records(root, names)) == set(names)
    assert any("bad: failed with status 3" in line for line in lines)


def test_child_gets_the_parent_flags(tmp_path):
    args = rp.build_parser().parse_args(["--model", "w.pth", "--root_dir", "R", "--assume_static", "--sample_ratio", "4",
                                         "--traj_min_len", "5", "--skip_sfm", "--keep_intermediate"])
    child = rp.build_parser().parse_args(rp.child_args(args, "R/x"))
    assert child.workspace_dir == "R/x" and child.root_dir == "none"
    for k in ("model", "sample_ratio", "traj_min_len", "flow_check_thres", "skip_sfm", "keep_intermediate",
              "assume_static", "skip_path_consistency", "skip_exists", "image_folder", "sfm_type"):
        assert getattr(child, k) == getattr(args, k), k


def test_an_exception_in_the_parent_leaves_no_child(tmp_path):
    procs = []

    def spawn(name, dev):
        p = subprocess.Popen([sys.executable, "-c", "import time, sys; time.sleep(0 if sys.argv[1] == 'quick' else 60)",
                              name])
        procs.append(p)
        return p

    def report(name, dev, rc, seconds):
        raise KeyboardInterrupt

    t0 = time.time()
    with pytest.raises(KeyboardInterrupt):
        rp.schedule(["slow1", "quick", "slow2", "slow3"], ["0", "1", "2"], spawn, report)
    assert len(procs) == 3 and time.time() - t0 < 30
    assert all(p.poll() is not None for p in procs)
