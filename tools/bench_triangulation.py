"""python tools/bench_triangulation.py [--shapes small,sintel,davis] [--repeats 3]

Wall time of init_geometry.triangulate_all_points (GlobalMapper::TriangulateAllPoints on the device) with host buffers
in and out, on the chain shapes of tools/bench_positions.py:

    small    300 trajectories, 25 frames, 4,000 observations (the numpy restatement runs here only)
    sintel   30,000 trajectories, 50 frames, 600,000 observations
    davis    50,000 trajectories, 80 frames, 1,600,000 observations

Each: make_two_view_scene (helix path, true poses, 0.5 px noise) -> traj_to_matches_device -> database arrays.  After
one warm-up call, min - median - max of `repeats` calls, and the per-phase split of the last call's summary (host
work, graph, components, replay, assembly).  The reference's own time is not measured (gcolmap is not built here).
The device name and power limit are read in the same process.
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

SHAPES = {"small": (300, 25, 4_000), "sintel": (30_000, 50, 600_000), "davis": (50_000, 80, 1_600_000)}
DB = ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr", "inlier_matches")


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _inputs(n_traj, n_frames, n_obs, seed=11):
    from particlesfm_b200 import handoff, synthetic as syn
    tracks, qvec, tvec, cam = syn.make_two_view_scene(n_traj, n_frames, n_obs, seed=seed, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, n_frames))
    a = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    db = {k: a[k] for k in DB}
    db["keypoints"], _ = syn.corrupt_keypoints(db["keypoints"], 0.0, seed=seed, noise_px=0.5)
    db.update(camera_size=np.array([[1024, 436]]), orientations=qvec, image_tvec=tvec,
              registered=np.ones(n_frames, bool))
    return db


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="small,sintel,davis")
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    from particlesfm_b200 import device_count, init_geometry
    if device_count() <= 0:
        raise SystemExit("bench_triangulation: no CUDA device (there is no CPU path to time)")
    print(json.dumps({"device": _device_info()}), flush=True)
    for name in args.shapes.split(","):
        db = _inputs(*SHAPES[name])
        init_geometry.triangulate_all_points(**db)
        times, out = [], None
        for _ in range(args.repeats):
            t = time.perf_counter()
            out = init_geometry.triangulate_all_points(**db)
            times.append(time.perf_counter() - t)
        s = out.summary
        rec = {"shape": name, "keypoints": int(db["keypoint_ptr"][-1]), "matches": int(db["inlier_ptr"][-1]),
               "call_s": {"min": min(times), "median": statistics.median(times), "max": max(times)},
               "phases_ms": {k: round(s[k], 3) for k in ("host_ms", "graph_ms", "components_ms", "replay_ms", "assembly_ms")},
               "counts": {k: s[k] for k in ("num_components", "largest_component", "num_points3D", "num_continued",
                                            "num_ransac_trials", "num_local_estimates", "num_launches")}}
        if name == "small":
            from oracle import triangulation_oracle as to
            t = time.perf_counter()
            ref = to.triangulate_all_points(**db)
            rec["numpy_s"] = time.perf_counter() - t
            rec["numpy_agrees"] = bool(np.array_equal(ref["point3D_of_keypoint"], out.point3D_of_keypoint)
                                       and np.array_equal(ref["track_ptr"], out.track_ptr))
        print(json.dumps(rec), flush=True)
    print(json.dumps({"device": _device_info()}), flush=True)


if __name__ == "__main__":
    main()
