"""python tools/bench_sfm.py [--shapes sintel,davis] [--repeats 3] [--step_route auto|on|off]

Per-stage wall time (min, median, max of `repeats` calls after one warm-up call) of sfm.main_global_sfm, from a
track set and PNG frames to SFM/model, on the trajectory counts of DESIGN.md §4.2:

    small    300 trajectories, 25 frames, 4,000 observations (a quick check of the tool itself)
    sintel   131,000 trajectories, 50 frames, 5,520,000 observations
    davis    489,000 trajectories, 80 frames, 32,300,000 observations

Each shape: make_two_view_scene (helix path, focal 1.2 x 1024, 0.5 px noise), handed over in memory as a
tracker.TrackArrays (reading a track.npy of tens of millions of samples is not part of what is timed), and plain
grey 1024 x 436 PNG frames written first.  Besides the stages, each call reports the database writer thread's own time
and how long the call waited for it at the end (stage `database`).

The step-by-step route runs once per shape in the same process: traj_to_matches_device,
import_keypoints_matches_arrays, MatchTables.from_rows, verify_two_view_geometries, a hand-written cameras/images
table plus write_colmap_database, global_mapper on that database, then convert.  With --step_route auto it runs only
when the host has room for its int64 copies (about 150 bytes per match); a shape where it did not run says so.
The device name and power limit are read in the same process.
"""
import argparse
import json
import os
import sqlite3
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"small": (300, 25, 4_000), "sintel": (131_000, 50, 5_520_000), "davis": (489_000, 80, 32_300_000)}
W, H = 1024, 436
STEP_ROUTE_BYTES_PER_MATCH = 150


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _host_bytes_free():
    with open("/proc/meminfo") as f:
        info = {line.split(":")[0]: int(line.split()[1]) * 1024 for line in f}
    return info.get("MemAvailable", 0)


def _inputs(root, n_traj, n_frames, n_obs, seed=11):
    from PIL import Image
    from particlesfm_b200 import synthetic as syn
    img = os.path.join(root, "images")
    os.makedirs(img)
    frame = Image.fromarray(np.full((H, W, 3), 128, np.uint8))
    for i in range(n_frames):
        frame.save(os.path.join(img, "%05d.png" % i))
    tracks = syn.make_two_view_scene(n_traj, n_frames, n_obs, seed=seed, path="helix", focal=1.2 * W)[0]
    tracks.xy = syn.corrupt_keypoints(tracks.xy, 0.0, seed=seed, noise_px=0.5)[0]
    return img, tracks


def _step_route(root, img, tracks):
    """The same work through the per-stage entries and SQLite: seconds per step."""
    from particlesfm_b200 import convert, global_mapper as gm, handoff, init_geometry, sfm
    t, names = {}, sorted(os.listdir(img))
    ids = list(range(1, len(names) + 1))
    images = sfm.read_image_set(img)
    t0 = time.perf_counter()
    tm = handoff.traj_to_matches_device(tracks, len(names))
    t["traj_to_matches_device"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), tm)
    t["import_keypoints_matches_arrays"] = time.perf_counter() - t0
    del tm
    t0 = time.perf_counter()
    mt = handoff.MatchTables.from_rows(rows, ids, names, images.camera, (images.width, images.height))
    t["from_rows"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    ver = init_geometry.verify_two_view_geometries(**mt.verification_inputs())
    t["verify_two_view_geometries"] = time.perf_counter() - t0
    path = os.path.join(root, "step", "database.db")
    os.makedirs(os.path.dirname(path))
    t0 = time.perf_counter()
    db = sqlite3.connect(path)
    sfm.write_schema(db, images)
    db.close()
    handoff.write_colmap_database(path, handoff.DatabaseRows(rows.keypoints, rows.matches, ver.two_view_rows(mt.pair_ids)))
    t["write_database"] = time.perf_counter() - t0
    del rows, mt, ver
    t0 = time.perf_counter()
    rep = gm.global_mapper(path, os.path.join(root, "step", "model"), sfm.mapper_options(), image_path=img)
    t["global_mapper"] = time.perf_counter() - t0
    if rep.success:
        t0 = time.perf_counter()
        convert.write_depth_pose_from_colmap_format(rep.output, os.path.join(root, "step", "converted"))
        t["convert"] = time.perf_counter() - t0
    t["total"] = sum(t.values())
    return t, rep.success


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="sintel,davis")
    ap.add_argument("--repeats", type=int, default=3, help="timed calls per shape, after one warm-up call")
    ap.add_argument("--step_route", default="auto", choices=("auto", "on", "off"))
    args = ap.parse_args()
    from particlesfm_b200 import device_count, sfm
    if device_count() <= 0:
        raise SystemExit("bench_sfm: no CUDA device (there is no CPU path to time)")
    print(json.dumps({"device": _device_info()}), flush=True)
    mmm = lambda v: [round(min(v), 3), round(statistics.median(v), 3), round(max(v), 3)]
    for name in args.shapes.split(","):
        with tempfile.TemporaryDirectory() as root:
            t0 = time.perf_counter()
            img, tracks = _inputs(root, *SHAPES[name])
            rec = {"shape": name, "trajectories": SHAPES[name][0], "frames": SHAPES[name][1],
                   "observations": SHAPES[name][2], "inputs_s": round(time.perf_counter() - t0, 2)}
            totals, stages, writer = [], {}, []
            for k in range(args.repeats + 1):
                t0 = time.perf_counter()
                rep = sfm.main_global_sfm(os.path.join(root, "sfm%d" % k), img, tracks)
                if k == 0:
                    continue
                totals.append(time.perf_counter() - t0)
                for n, s, summ in rep.stages:
                    stages.setdefault(n, []).append(s)
                    if n == "database":
                        writer.append(summ["writer_seconds"])
            rec.update({"success": rep.success, "calls": args.repeats, "call_s_min_median_max": mmm(totals),
                        "stages_s_min_median_max": {n: mmm(v) for n, v in stages.items()},
                        "writer_thread_s_min_median_max": mmm(writer), "stats": rep.stats})
            for n, _, summ in rep.stages:
                if n in ("table", "verification"):
                    rec[n] = summ
            need = STEP_ROUTE_BYTES_PER_MATCH * rec["table"]["matches"]
            run = args.step_route == "on" or (args.step_route == "auto" and _host_bytes_free() > need)
            if run:
                step, ok = _step_route(root, img, tracks)
                rec["step_route_s"] = {k: round(v, 3) for k, v in step.items()}
                rec["step_route_success"] = ok
            else:
                rec["step_route_s"] = "not run: the host has %.0f GB available, the route needs about %.0f GB" % (
                    _host_bytes_free() / 1e9, need / 1e9)
            print(json.dumps(rec), flush=True)
    print(json.dumps({"device": _device_info()}), flush=True)


if __name__ == "__main__":
    main()
