"""python tools/bench_point_trajectory.py [--shapes sintel,davis] [--modes pc,skip] [--repeats 3] [--out DIR]

Wall time of the point-trajectory stage from a flow directory to track.npy on disk, on seeded .flo directories
written from synthetic.make_flow_sequence at two user shapes:

    sintel   50 frames, 436 x 1024, sample_ratio 2
    davis    80 frames, 480 x 854,  sample_ratio 1

with path consistency (pc: flow_f, flow_b, flow_f2, flow_b2) and without it (skip: flow_f, flow_b).  Two arms,
alternated after a warm-up of each on a 5-frame directory:

    (a) today's route   every map read into host memory by a restatement of the reference's read_flo, then the
                        resident stage (pc: main_connect_point_trajectories_device; skip: flow_check_device and
                        track_device, the resident mode this tree adds), TrackArrays.to_dict(), and
                        np.save(track.npy, particlesfm.TrajectorySet(dict))
    (b) the command     point_trajectory.main_connect_point_trajectories: streamed maps, the state body written on
                        the device

Reports min / median / max of each arm, the two files' sizes, the time np.load(...).item() takes for each (what a
downstream reader pays) and whether the two files load to identical sets, at every shape run.  One JSON line, with
the card's name and power limit read in the same call.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SHAPES = {"sintel": (50, 436, 1024, 2), "davis": (80, 480, 854, 1)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def read_flo_reference(name):
    """utils.py:38-56 restated: tag, w, h, then np.fromfile and np.resize"""
    with open(name, "rb") as f:
        tag = np.fromfile(f, np.float32, count=1)[0]
        assert tag == 202021.25
        w = np.fromfile(f, np.int32, count=1)
        h = np.fromfile(f, np.int32, count=1)
        data = np.fromfile(f, np.float32, count=2 * w[0] * h[0])
    return np.resize(data, (int(h[0]), int(w[0]), 2))


def arm_a(flow_dir, traj_dir, ratio, skip):
    from particlesfm_b200 import point_trajectory as pt, tracker
    load = lambda name: [read_flo_reference(p) for p in pt.list_flows(os.path.join(flow_dir, name))]
    fw, fb = load("flow_f"), load("flow_b")
    if skip:
        _, occ = tracker.flow_check_device(fw, fb, 1.0)
        arrays = tracker.track_device(fw, occ, ratio, 3)
    else:
        arrays = tracker.main_connect_point_trajectories_device(fw, fb, load("flow_f2"), load("flow_b2"), ratio, 1.0, 3)
    os.makedirs(traj_dir, exist_ok=True)
    np.save(os.path.join(traj_dir, "track.npy"), pt._particlesfm().TrajectorySet(arrays.to_dict()))


def arm_b(flow_dir, traj_dir, ratio, skip):
    from particlesfm_b200 import point_trajectory as pt
    pt.main_connect_point_trajectories(flow_dir, traj_dir, ratio, 1.0, 3, skip_path_consistency=skip)


def timed(fn, *args):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def stats(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs)}


def write_dirs(root, n_frames, h, w, seed):
    from particlesfm_b200 import synthetic as syn
    from test_point_trajectory_host import write_flow_dir
    fw, fb, f2, b2 = syn.make_flow_sequence(n_frames, h, w, seed=seed)
    full = write_flow_dir(os.path.join(root, "full"), fw, fb, f2, b2)
    warm = write_flow_dir(os.path.join(root, "warm"), fw[:5], fb[:5], f2[:4], b2[:4])
    return full, warm


def same_loaded(p, q):
    a = np.load(p, allow_pickle=True).item().as_dict()
    b = np.load(q, allow_pickle=True).item().as_dict()
    if list(a) != list(b):
        return False
    for k in a:
        ta, tb = a[k], b[k]
        if ta["frame_ids"] != tb["frame_ids"] or ta["labels"] != tb["labels"]:
            return False
        if any(x.tobytes() != y.tobytes() for x, y in zip(ta["locations"], tb["locations"])):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="sintel,davis")
    ap.add_argument("--modes", default="pc,skip")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None, help="scratch directory for the .flo files (default: a temporary one)")
    a = ap.parse_args()
    import torch
    from particlesfm_b200 import device_count, point_trajectory as pt
    if device_count() <= 0:
        raise SystemExit("bench_point_trajectory: no CUDA device")
    torch.cuda.init()
    result = {"card": card(), "repeats": a.repeats, "shapes": {}}
    scratch = tempfile.mkdtemp(dir=a.out)
    try:
        for name in a.shapes.split(","):
            n_frames, h, w, ratio = SHAPES[name]
            root = os.path.join(scratch, name)
            full, warm = write_dirs(root, n_frames, h, w, seed=n_frames)
            res = {"frames": n_frames, "height": h, "width": w, "sample_ratio": ratio}
            for mode in a.modes.split(","):
                skip = mode == "skip"
                out_a, out_b = os.path.join(root, mode + "_a"), os.path.join(root, mode + "_b")
                arm_a(warm, os.path.join(root, "warm_a"), ratio, skip)
                arm_b(warm, os.path.join(root, "warm_b"), ratio, skip)
                ta, tb = [], []
                for _ in range(a.repeats):
                    ta.append(timed(arm_a, full, out_a, ratio, skip))
                    tb.append(timed(arm_b, full, out_b, ratio, skip))
                    print(json.dumps({name: {mode: {"a": ta[-1], "b": tb[-1]}}}), file=sys.stderr, flush=True)
                pa, pb = os.path.join(out_a, "track.npy"), os.path.join(out_b, "track.npy")
                la = [timed(lambda: np.load(pa, allow_pickle=True).item()) for _ in range(2)]
                lb = [timed(lambda: np.load(pb, allow_pickle=True).item()) for _ in range(2)]
                res[mode] = {"a_seconds": stats(ta), "b_seconds": stats(tb),
                             "a_bytes": os.path.getsize(pa), "b_bytes": os.path.getsize(pb),
                             "a_load_seconds": min(la), "b_load_seconds": min(lb),
                             "identical_sets": same_loaded(pa, pb)}
                arrays = pt.connect_point_trajectories(full, ratio, 1.0, 3, skip)
                res[mode]["observations"] = int(arrays.frame_ids.shape[0])
                res[mode]["trajectories"] = int(arrays.ids.shape[0])
                res[mode]["b_bytes_per_observation"] = res[mode]["b_bytes"] / max(1, res[mode]["observations"])
                print(json.dumps({name: {mode: res[mode]}}), file=sys.stderr, flush=True)
            result["shapes"][name] = res
            shutil.rmtree(root)
    finally:
        shutil.rmtree(scratch, ignore_errors=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
