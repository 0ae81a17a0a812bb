"""python tools/bench_verification.py [--shapes check,sintel,davis,sintel_full] [--repeats 3]

Wall time of init_geometry.verify_two_view_geometries (the geometric verification of `colmap matches_importer` on the
device) with host buffers in and out:

    check        300 trajectories, 12 frames, 3,600 observations (the numpy restatement runs here only)
    sintel       30,000 trajectories, 50 frames, 600,000 observations (the Sintel chain of tools/bench_positions.py)
    davis        50,000 trajectories, 80 frames, 1,600,000 observations (the DAVIS chain)
    sintel_full  131,000 trajectories, 50 frames, 5,520,000 observations: about 54 M raw matches in 1,225 pairs

Each: make_two_view_scene (helix path) -> traj_to_matches_device -> MatchTables.from_rows, keypoints with 10 %
outliers (synthetic.corrupt_keypoints, 20 .. 60 px) and 0.5 px noise.  After one warm-up call, min - median - max of
`repeats` calls, the per-phase split of the last call's summary and its trial counts per kind (F, H, watermark).  The
device scores trials in their sequential order, so no scored trial is discarded.  `colmap matches_importer` itself is
not timed (COLMAP is not built here).  The device name and power limit are read in the same process.
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

SHAPES = {"check": (300, 12, 3_600), "sintel": (30_000, 50, 600_000), "davis": (50_000, 80, 1_600_000),
          "sintel_full": (131_000, 50, 5_520_000)}


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _tables(n_traj, n_frames, n_obs, seed=11):
    from particlesfm_b200 import handoff, synthetic as syn
    tracks, _, _, cam = syn.make_two_view_scene(n_traj, n_frames, n_obs, seed=seed, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, n_frames))
    mt = handoff.MatchTables.from_rows(rows, ids, names, cam, (1024, 436))
    mt.keypoints, _ = syn.corrupt_keypoints(mt.keypoints, 0.1, seed=seed, noise_px=0.5)
    return mt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="check,sintel,davis,sintel_full")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from particlesfm_b200 import device_count, init_geometry
    if device_count() <= 0:
        raise SystemExit("bench_verification: no CUDA device (there is no CPU path to time)")
    print(json.dumps({"device": _device_info()}), flush=True)
    for name in args.shapes.split(","):
        mt = _tables(*SHAPES[name])
        inputs = mt.verification_inputs()
        init_geometry.verify_two_view_geometries(**inputs)
        times, out = [], None
        for _ in range(args.repeats):
            t = time.perf_counter()
            out = init_geometry.verify_two_view_geometries(**inputs)
            times.append(time.perf_counter() - t)
        s = out.summary
        rec = {"shape": name, "pairs": int(len(out.config)), "raw_matches": int(mt.match_ptr[-1]),
               "inliers": int(out.inlier_ptr[-1]),
               "call_s": {"min": min(times), "median": statistics.median(times), "max": max(times)},
               "phases_ms": {k: round(s[k], 3) for k in ("host_ms", "gather_ms", "ransac_ms", "compact_ms")},
               "trials": s["num_trials"], "trials_scored": s["num_trials_scored"], "local_rounds": s["num_local_rounds"],
               "configs": s["num_config"], "launches": s["num_launches"]}
        if name == "check":
            from oracle import verification_oracle as vo
            t = time.perf_counter()
            ref = vo.verify_two_view_geometries(**inputs)
            rec["numpy_s"] = time.perf_counter() - t
            rec["numpy_agrees"] = bool(np.array_equal(ref["config"], out.config)
                                       and np.array_equal(ref["inlier_matches"], out.inlier_matches)
                                       and np.array_equal(ref["trials"], out.trials))
        print(json.dumps(rec), flush=True)
    print(json.dumps({"device": _device_info()}), flush=True)


if __name__ == "__main__":
    main()
