"""python tools/bench_rotations.py [--shapes sintel,davis,target,config5,long] [--repeats 3] [--oracle-max-images 200]

Wall time of the global rotation averaging (EstimateGlobalRotations) on these view graphs:

    sintel   the two-view chain at 50 frames: make_two_view_scene -> traj_to_matches_device -> estimate_relative_poses,
             all 1,225 pairs (30 k trajectories: the view graph is the Sintel shape's, with fewer matches per pair,
             which this step does not read beyond their count)
    davis    the same at 80 frames, all 3,160 pairs (50 k trajectories)
    target   synthetic.make_view_graph, complete, F = 200 (19,900 pairs), 1 degree noise, 10 % outliers
    config5  the same at F = 500 (124,750 pairs)
    long     banded (pairs up to 10 frames apart), F = 1,000 (9,945 pairs), 0.5 degree noise

Arms, alternated within one process after a warm-up of each:
    device   init_geometry.estimate_global_rotations (csrc/rotation_averaging.cu), host buffers in and out
    oracle   the numpy / scipy restatement oracle/rotation_oracle.py, NOT the reference (gcolmap is not built here);
             it is reported as not run above --oracle-max-images images
Where both run, iteration counts, kept pairs and orientations (1e-9 rad) are compared.  Reports the device call's
split into host graph work and device loop, its launch count, and the device name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHAIN = {"sintel": (30_000, 50, 600_000), "davis": (50_000, 80, 1_600_000)}
SYNTH = {"target": dict(num_images=200, noise_deg=1.0, outlier_fraction=0.1, seed=5),
         "config5": dict(num_images=500, noise_deg=1.0, outlier_fraction=0.1, seed=6),
         "long": dict(num_images=1000, graph="banded", band=10, noise_deg=0.5, seed=7)}


def _inputs(name):
    from particlesfm_b200 import handoff, init_geometry, synthetic as syn
    if name in SYNTH:
        g = syn.make_view_graph(**SYNTH[name])
        return {k: g[k] for k in ("num_images", "pair_images", "qvec", "num_correspondences", "has_pose")}
    ntraj, nf, nobs = CHAIN[name]
    tracks, qvec, tvec, cam = syn.make_two_view_scene(ntraj, nf, nobs, seed=nf)
    names, ids = ["%05d.png" % i for i in range(nf)], list(range(1, nf + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, nf))
    args = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    poses = init_geometry.estimate_relative_poses(**args)
    return dict(num_images=nf, pair_images=args["pair_images"], qvec=poses.qvec,
                num_correspondences=np.diff(args["inlier_ptr"]), has_pose=poses.estimated)


def _stats(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs)} if xs else None


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="sintel,davis,target,config5,long")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-max-images", type=int, default=200)
    a = ap.parse_args()
    from oracle import rotation_oracle as ro
    from particlesfm_b200 import device_count, init_geometry
    if device_count() <= 0:
        raise SystemExit("no CUDA device: this benchmark measures the GPU path")
    results = {"device": _device_info(), "oracle": "numpy/scipy restatement (not the reference)", "shapes": {}}
    for name in a.shapes.split(","):
        args = _inputs(name)
        run_oracle = args["num_images"] <= a.oracle_max_images
        dev = init_geometry.estimate_global_rotations(**args)          # warm-up
        ref = ro.estimate_global_rotations(**args) if run_oracle else None
        times = {"device": [], "oracle": []}
        for _ in range(a.repeats):
            t = time.perf_counter()
            dev = init_geometry.estimate_global_rotations(**args)
            times["device"].append(time.perf_counter() - t)
            if run_oracle:
                t = time.perf_counter()
                ref = ro.estimate_global_rotations(**args)
                times["oracle"].append(time.perf_counter() - t)
        s = dev.summary
        r = {"images": int(args["num_images"]), "pairs": int(len(args["qvec"])), "device_s": _stats(times["device"]),
             "oracle_s": _stats(times["oracle"]) if run_oracle else "not run (above --oracle-max-images)",
             "l1_rounds": s["num_l1_rounds"], "admm_iterations": s["admm_iterations"],
             "irls_iterations": s["num_irls_iterations"], "launches": s["num_launches"], "host_ms": s["host_ms"],
             "device_ms": s["device_ms"], "pairs_kept": s["num_pairs_kept"]}
        if run_oracle:
            ang = max((np.linalg.norm(ro.quaternion_to_angle_axis(ro.concatenate_quaternions(
                dev.orientations[f], ro.invert_quaternion(ref["orientations"][f]))))
                for f in np.nonzero(ref["has_orientation"])[0]), default=0.0)
            r["agrees"] = bool(s["admm_iterations"] == ref["admm_iterations"] and
                               s["num_irls_iterations"] == ref["irls_iterations"] and
                               np.array_equal(dev.pair_kept, ref["pair_kept"]) and ang <= 1e-9)
            r["max_orientation_diff_rad"] = float(ang)
        results["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
