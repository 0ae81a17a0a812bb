"""python tools/bench_two_view.py [--shapes check,sintel,davis] [--repeats 3] [--host-max-matches 3000000]

Wall time of the relative-pose step gcolmap runs when it loads a database (TwoViewGeometry::EstimateRelativePose
of every verified pair), on seeded geometric scenes: synthetic.make_two_view_scene (a camera moving 0.02 per frame,
static points 2 .. 40 away, locations = exact projections) with the tracker's counts, then traj_to_matches_device
and import_keypoints_matches_arrays, so that every image pair of the database rows is one pair here (config
CALIBRATED, E from the true poses):

    check     4 k trajectories,  30 k observations, 12 frames   (small enough for the numpy restatement)
    sintel  131 k trajectories, 5.52 M observations, 50 frames
    davis   489 k trajectories, 32.3 M observations, 80 frames

Arms, alternated within one process after a warm-up of each on the check shape:
    device   init_geometry.estimate_relative_poses (csrc/two_view.cu), host buffers in and out
    host     the numpy restatement oracle/two_view_oracle.py, NOT the reference (COLMAP is not built here); it is
             reported as not run above --host-max-matches inlier matches
Where both run, the device result is checked against the restatement pair by pair (quaternion and translation to
1e-12, num_points3D equal, tri_angle to 1e-12).  Prints one JSON line with the device name and power limit.
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

SHAPES = {"check": (4_000, 12, 30_000), "sintel": (131_000, 50, 5_520_000), "davis": (489_000, 80, 32_300_000)}


def _stats(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs), "all": xs} if xs else None


def _inputs(name):
    from particlesfm_b200 import handoff, synthetic as syn
    ntraj, nf, nobs = SHAPES[name]
    tracks, qvec, tvec, cam = syn.make_two_view_scene(ntraj, nf, nobs, seed=nf)
    names = ["%05d.png" % i for i in range(nf)]
    ids = [i + 1 for i in range(nf)]
    m = handoff.traj_to_matches_device(tracks, nf)
    del tracks
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), m, skip_geometric_verification=False)
    del m
    return syn.two_view_inputs(rows, ids, qvec, tvec, cam)


def _agreement(dev, ref):
    ok = {"pairs": len(ref), "pose": 0, "num_points3D": 0, "tri_angle": 0}
    for p, r in enumerate(ref):
        ok["pose"] += bool(np.abs(dev.qvec[p] - r["qvec"]).max() <= 1e-12 and np.abs(dev.tvec[p] - r["t"]).max() <= 1e-12)
        ok["num_points3D"] += int(dev.num_points3D[p]) == r["num_points3D"]
        ok["tri_angle"] += bool(np.isclose(dev.tri_angle[p], r["tri_angle"], rtol=0, atol=1e-12, equal_nan=True))
    return ok


def run_shape(name, repeats, host_max):
    from oracle import two_view_oracle as tv
    from particlesfm_b200 import init_geometry
    t0 = time.perf_counter()
    args = _inputs(name)
    ntraj, nf, nobs = SHAPES[name]
    n = int(args["inlier_ptr"][-1])
    out = {"shape": name, "frames": nf, "trajectories": ntraj, "observations": nobs, "pairs": int(args["config"].shape[0]),
           "inlier_matches": n, "setup_s": time.perf_counter() - t0}
    arms = ["device"] + (["host"] if n <= host_max else [])
    if n > host_max:
        out["host"] = "not run: %d inlier matches > --host-max-matches %d" % (n, host_max)
    run = {"device": lambda: init_geometry.estimate_relative_poses(**args), "host": lambda: tv.estimate_relative_poses(**args)}
    times = {a: [] for a in arms}
    last = {}
    for r in range(repeats):
        for arm in arms:
            last.pop(arm, None)
            gc.collect()
            t = time.perf_counter()
            res = run[arm]()
            times[arm].append(time.perf_counter() - t)
            last[arm] = res
    for arm in arms:
        out[arm + "_s"] = _stats(times[arm])
    dev = last["device"]
    out["num_points3D_total"] = int(dev.num_points3D.sum())
    out["tri_angle_deg_median"] = float(np.degrees(np.nanmedian(dev.tri_angle)))
    if "host" in last:
        out["host_arm"] = "numpy restatement (oracle/two_view_oracle.py), not the reference"
        out["agreement"] = _agreement(dev, last["host"])
        out["speedup_median"] = statistics.median(times["host"]) / statistics.median(times["device"])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shapes", default="check,sintel,davis")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-max-matches", type=int, default=3_000_000)
    args = ap.parse_args()
    import bench
    from particlesfm_b200 import device_count, init_geometry
    if device_count() <= 0:
        raise SystemExit("bench_two_view: no CUDA device (the product has no CPU path)")
    from oracle import two_view_oracle as tv
    warm = _inputs("check")                             # warm-up: modules, CUDA context, allocator
    init_geometry.estimate_relative_poses(**warm)
    tv.estimate_relative_poses(**warm)
    results = []
    for name in [s for s in args.shapes.split(",") if s]:
        results.append(run_shape(name, args.repeats, args.host_max_matches))
        print("[bench_two_view]", json.dumps(results[-1]), file=sys.stderr, flush=True)
    gpu = bench.gpu_info(bench.smi_device(0))
    print(json.dumps({"tool": "bench_two_view", "gpu": gpu, "repeats": args.repeats, "results": results}))


if __name__ == "__main__":
    main()
