"""python tools/bench_tracker.py [--shapes sintel,davis] [--repeats 3] [--arms host,device]

Wall time of the whole tracker stage, main_connect_point_trajectories (flow check, tracking, HP1, track set),
on deterministic synthetic sequences at two user shapes (synthetic.make_flow_sequence: smooth flows, composed
two-step flows, crude backward flows, a moving block the flow check marks occluded):

    sintel   50 frames, 436 x 1024, sample_ratio 2
    davis    80 frames, 480 x 854,  sample_ratio 1

Arms, alternated within one process after a warm-up of each on the first frames:
    host     device=False: torch-CPU sampling, scipy re-seeding, numpy bookkeeping, HP1 through the library
    device   the stage resident on the GPU; reported as the time to TrackArrays and the to_dict() time
On a tree without the resident stage the device arm times main_connect_point_trajectories(device=True) as a
whole.  With both arms, the track sets of the last repeat are checked to be bit-identical.  Prints one JSON
line with the device name and power limit beside the times.  Maps are numpy arrays in both arms, so the
device arm's times include their upload.
"""
import argparse
import gc
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"sintel": (50, 436, 1024, 2), "davis": (80, 480, 854, 1)}
WARMUP_FRAMES = 5


def _flat(d):
    """A track-set dict as (ids, ptr, frame_ids, xy) arrays, in dict order."""
    ids = np.fromiter(d.keys(), np.int64, len(d))
    lens = np.fromiter((len(v["frame_ids"]) for v in d.values()), np.int64, len(d))
    ptr = np.concatenate([[0], np.cumsum(lens)])
    frames = np.fromiter((f for v in d.values() for f in v["frame_ids"]), np.int64, int(ptr[-1]))
    xy = np.empty((int(ptr[-1]), 2))
    o = 0
    for v in d.values():
        n = len(v["locations"])
        if n:
            xy[o:o + n] = np.stack(v["locations"])
        o += n
    labels = any(l for v in d.values() for l in v["labels"])
    return ids, ptr, frames, xy, labels


def _stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": xs} if xs else None


def run_shape(name, repeats, arms):
    import torch
    from particlesfm_b200 import synthetic as syn, tracker
    n_frames, h, w, ratio = SHAPES[name]
    fw, fb, f2, b2 = syn.make_flow_sequence(n_frames, h, w, seed=n_frames)
    resident = hasattr(tracker, "main_connect_point_trajectories_device")

    def host(k=None):
        s = slice(None, k)
        return tracker.main_connect_point_trajectories(fw[s], fb[s], f2[s], b2[s], ratio, 1.0, 3, device=False)

    def device(k=None):
        s = slice(None, k)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if resident:
            arrays = tracker.main_connect_point_trajectories_device(fw[s], fb[s], f2[s], b2[s], ratio, 1.0, 3)
        else:
            arrays = None
            d = tracker.main_connect_point_trajectories(fw[s], fb[s], f2[s], b2[s], ratio, 1.0, 3, device=True)
        t1 = time.perf_counter()
        if resident:
            d = arrays.to_dict()
        t2 = time.perf_counter()
        return arrays, d, t1 - t0, t2 - t1

    for arm in arms:                                    # warm-up: modules, allocator, torch-CPU kernels
        host(WARMUP_FRAMES) if arm == "host" else device(WARMUP_FRAMES)
    times = {"host": [], "device": [], "device_to_arrays": [], "device_to_dict": []}
    last = {}
    for r in range(repeats):
        for arm in arms:
            last.pop(arm, None)
            gc.collect()
            if arm == "host":
                t0 = time.perf_counter()
                d = host()
                times["host"].append(time.perf_counter() - t0)
                if r == repeats - 1:
                    last["host"] = d
            else:
                arrays, d, ta, td = device()
                times["device"].append(ta + td)
                times["device_to_arrays"].append(ta if arrays is not None else None)
                times["device_to_dict"].append(td if arrays is not None else None)
                if r == repeats - 1:
                    last["device"] = (arrays, d)
            del d
    out = {"shape": name, "frames": n_frames, "h": h, "w": w, "sample_ratio": ratio, "traj_min_len": 3,
           "resident_stage": resident}
    for k, v in times.items():
        v = [x for x in v if x is not None]
        out[k + "_s"] = _stats(v)
    ref = last.get("host") if "host" in last else None
    if "device" in last:
        arrays, d = last["device"]
        ids, ptr, frames, xy, labels = _flat(d)
        out["trajectories"], out["observations"] = int(ids.shape[0]), int(ptr[-1])
        if ref is not None:
            hi, hp, hf, hx, hl = _flat(ref)
            same = (np.array_equal(ids, hi) and np.array_equal(ptr, hp) and np.array_equal(frames, hf)
                    and np.array_equal(xy, hx) and not labels and not hl)
            if arrays is not None:
                same = same and np.array_equal(arrays.ids, hi) and np.array_equal(arrays.ptr, hp) \
                    and np.array_equal(arrays.frame_ids, hf) and np.array_equal(arrays.xy, hx)
            out["bit_identical"] = bool(same)
    elif ref is not None:
        ids, ptr, _, _, _ = _flat(ref)
        out["trajectories"], out["observations"] = int(ids.shape[0]), int(ptr[-1])
    if "host" in times and times["host"] and times["device"]:
        out["speedup_median"] = statistics.median(times["host"]) / statistics.median(times["device"])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shapes", default="sintel,davis")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--arms", default="host,device")
    args = ap.parse_args()
    import torch
    import bench
    from particlesfm_b200 import device_count
    if device_count() <= 0 or not torch.cuda.is_available():
        raise SystemExit("bench_tracker: no CUDA device (the product has no CPU path)")
    arms = [a for a in args.arms.split(",") if a]
    results = []
    for name in [s for s in args.shapes.split(",") if s]:
        results.append(run_shape(name, args.repeats, arms))
        print("[bench_tracker]", json.dumps(results[-1]), file=sys.stderr, flush=True)
    print(json.dumps({"tool": "bench_tracker", "gpu": bench.gpu_info(bench.smi_device(0)), "repeats": args.repeats,
                      "arms": arms, "results": results}))


if __name__ == "__main__":
    main()
