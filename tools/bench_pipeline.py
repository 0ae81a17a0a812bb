"""Times the whole-pipeline command (particlesfm_b200.run_particlesfm.particlesfm: flows straight into the resident
tracker, the track set straight into the match table) against the three staged commands (optical_flow's directory,
point_trajectory's track.npy, sfm from that file) on the same input, alternated in one process, at the Sintel shape
(50 frames of 1024 x 436).  Two legs:

    raft  seeded frames and seeded RAFT weights, through --skip_sfm, without path consistency: the fused flows +
          trajectories stage and its track.npy against write_optical_flows, then main_connect_point_trajectories.
          With path consistency the seeded weights' flows leave a frame without a particle of 3 observations at
          this shape, where the tracker stops as the reference does (optimize_buffer's np.stack([])).
    room  synthetic.make_room_sequence's exact flows, with path consistency, as the flow source (uploaded per batch
          as the RAFT stage hands its maps over), into the tracker and the SfM step: the fused route against the
          flows written as the flow directory, then main_connect_point_trajectories, then sfm_reconstruction from
          track.npy

Per stage: min / median / max of --reps calls after one warm-up call of each route.  Prints a table and one JSON
line with the card's name and power limit, read in the same call.

    python tools/bench_pipeline.py [--reps 3] [--legs raft,room] [--frames 50] [--out OUT_DIR]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W = 436, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def clock(stages, name, fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    stages[name] = time.perf_counter() - t0
    return out


def write_frames(d, frames):
    from PIL import Image
    os.makedirs(d, exist_ok=True)
    for i, f in enumerate(frames):
        Image.fromarray(f).save(os.path.join(d, "%05d.png" % i))
    return d


def fused(img, out, **kw):
    from particlesfm_b200 import run_particlesfm as rp
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    rep = rp.particlesfm(img, out, quiet=True, **kw)
    torch.cuda.synchronize()
    stages = dict(rep.stages)
    stages["total"] = time.perf_counter() - t0
    return stages, rep


def staged_raft(img, out, weights):
    from particlesfm_b200 import optical_flow as of, point_trajectory as pt
    s = {}
    flow_dir, traj = os.path.join(out, "optical_flows"), os.path.join(out, "trajectories")
    clock(s, "flows", lambda: of.write_optical_flows(img, flow_dir, weights, skip_path_consistency=True))
    clock(s, "trajectories", lambda: pt.main_connect_point_trajectories(flow_dir, traj, skip_path_consistency=True))
    s["total"] = s["flows"] + s["trajectories"]
    return s, None


def staged_room(img, out, source):
    from particlesfm_b200 import optical_flow as of, point_trajectory as pt, sfm
    s = {}
    flow_dir, traj = os.path.join(out, "optical_flows"), os.path.join(out, "trajectories")
    paths, h, w = of.frame_list(img)

    def flows():
        of.make_flow_dirs(flow_dir, True)
        writer = of.FlowWriter(of.flow_files(paths, flow_dir))
        try:
            source(paths, h, w, of._pairs(len(paths), True), writer)
        finally:
            writer.join()
        writer.close()
    clock(s, "flows", flows)
    clock(s, "trajectories", lambda: pt.main_connect_point_trajectories(flow_dir, traj))
    rep = clock(s, "sfm", lambda: sfm.sfm_reconstruction(img, out, traj, assume_static=True))
    s["total"] = s["flows"] + s["trajectories"] + s["sfm"]
    return s, rep


def summary(runs):
    names = list(runs[0])
    return {n: [round(float(v), 4) for v in (np.min([r[n] for r in runs]), np.median([r[n] for r in runs]),
                                             np.max([r[n] for r in runs]))] for n in names}


def leg(name, tmp, reps, routes):
    results = {}
    for rep in range(reps + 1):                         # call 0 of each route is the warm-up
        for route, fn in routes:
            out = os.path.join(tmp, "%s_%s_%d" % (name, route, rep))
            stages, _ = fn(out)
            if rep:
                results.setdefault(route, []).append(stages)
            shutil.rmtree(out, ignore_errors=True)
    return {route: summary(r) for route, r in results.items()}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--legs", default="raft,room")
    p.add_argument("--frames", type=int, default=50)
    p.add_argument("--out", default=None, help="also write the JSON result to OUT/bench_pipeline.json")
    a = p.parse_args()
    import torch
    from oracle import raft_oracle as ro
    from particlesfm_b200 import run_particlesfm as rp, synthetic as syn
    result = {"card": card(), "frames": a.frames, "shape": [H, W], "reps": a.reps,
              "tf32_convolutions": bool(torch.backends.cudnn.allow_tf32)}
    with tempfile.TemporaryDirectory() as tmp:
        if "raft" in a.legs:
            img = write_frames(os.path.join(tmp, "raft_img"), ro.seeded_frames(a.frames, H, W, seed=1))
            weights = os.path.join(tmp, "w.pth")
            torch.save(ro.seeded_state_dict(0), weights)
            result["raft"] = leg("raft", tmp, a.reps, [
                ("fused", lambda out: fused(img, out, model=weights, skip_sfm=True, skip_path_consistency=True)),
                ("staged", lambda out: staged_raft(img, out, weights))])
        if "room" in a.legs:
            t0 = time.perf_counter()
            frames, flows, qvec, tvec = syn.make_room_sequence(a.frames, H, W, seed=0)
            result["room_generation_s"] = round(time.perf_counter() - t0, 2)
            img = write_frames(os.path.join(tmp, "room_img"), frames)
            source = rp.array_flow_source(flows)
            # one checked pair of runs: the same database rows, and the registered images
            s1, rep1 = fused(img, os.path.join(tmp, "check_fused"), flow_source=source)
            s2, rep2 = staged_room(img, os.path.join(tmp, "check_staged"), source)
            import sqlite3
            rows = lambda d: [sqlite3.connect(os.path.join(d, "sfm", "database.db")).execute(
                "SELECT * FROM %s ORDER BY rowid" % t).fetchall() for t in ("keypoints", "matches", "two_view_geometries")]
            result["room_check"] = {"databases_equal": rows(os.path.join(tmp, "check_fused")) == rows(os.path.join(tmp, "check_staged")),
                                    "registered": [rep1.sfm.stats["num_reg_images"] if rep1.success else 0,
                                                   rep2.stats["num_reg_images"] if rep2.success else 0]}
            result["room"] = leg("room", tmp, a.reps, [
                ("fused", lambda out: fused(img, out, flow_source=source)),
                ("staged", lambda out: staged_room(img, out, source))])
    result["card_after"] = card()
    for lg in ("raft", "room"):
        if lg in result:
            for route, st in result[lg].items():
                for stage, (lo, med, hi) in st.items():
                    print("%-5s %-7s %-20s %8.3f %8.3f %8.3f s" % (lg, route, stage, lo, med, hi))
    line = json.dumps(result)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_pipeline.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
