"""python tools/bench_mapper.py [--shapes small,sintel,davis] [--repeats 3] [--out DIR]

Per-stage wall time (min, median, max of `repeats` calls) of global_mapper.global_mapper (gcolmap global_mapper on the
device) from a SQLite database to OUT/0, on the chain shapes of tools/bench_positions.py:

    small    300 trajectories, 25 frames, 4,000 observations (warms every stage up)
    sintel   30,000 trajectories, 50 frames, 600,000 observations
    davis    50,000 trajectories, 80 frames, 1,600,000 observations

Each: make_two_view_scene (helix path, 0.5 px noise) -> traj_to_matches_device -> a database whose pairs are
CALIBRATED with E from the true poses (synthetic.two_view_inputs) -> the mapper.  Beside the mapper's hand-off
(psfm_ba_create_from_triangulation) and write-back (psfm_ba_get_model + write_model_arrays), the same steps through the
Python containers the chain test uses are timed on the same triangulation and refined state:
Triangulation.to_reconstruction + ba.flatten + psfm_ba_create, and get_state + observation mask + scatter +
apply_observation_mask + write_model.  The device name and power limit are read in the same process.
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

SHAPES = {"small": (300, 25, 4_000), "sintel": (30_000, 50, 600_000), "davis": (50_000, 80, 1_600_000)}
W, H = 1024, 436


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _database(path, n_traj, n_frames, n_obs, seed=11):
    from particlesfm_b200 import handoff, synthetic as syn
    tracks, qvec, tvec, cam = syn.make_two_view_scene(n_traj, n_frames, n_obs, seed=seed, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, n_frames))
    a = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    kps, _ = syn.corrupt_keypoints(a["keypoints"], 0.0, seed=seed, noise_px=0.5)
    db = sqlite3.connect(path)
    db.execute("CREATE TABLE cameras (camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, "
               "width INTEGER NOT NULL, height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL)")
    db.execute("CREATE TABLE images (image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, "
               "camera_id INTEGER NOT NULL)")
    db.execute("INSERT INTO cameras VALUES (1, 0, ?, ?, ?, 0)", (W, H, np.asarray(cam, np.float64).tobytes()))
    for i, n in zip(ids, names):
        db.execute("INSERT INTO images (image_id, name, camera_id) VALUES (?, ?, 1)", (i, n))
    db.commit()
    db.close()
    kp = [(i, kps[a["keypoint_ptr"][k]:a["keypoint_ptr"][k + 1]]) for k, i in enumerate(ids)]
    tv = [(pid, m, 2, a["F"][p], a["E"][p], a["H"][p]) for p, (pid, m) in enumerate(rows.matches)]
    handoff.write_colmap_database(path, handoff.DatabaseRows(kp, [], tv))


def _python_route(path, o, out):
    """Hand-off and write-back through the Python containers, on the mapper's stages 1-7 (same triangulation)."""
    import ctypes as C
    from particlesfm_b200 import _abi, _lib, ba, colmap_io, global_mapper as gm, handoff, init_geometry
    g, used = handoff.load_database_cache(path, o.min_num_matches, o.ignore_watermarks)
    used, rot, pos, res = gm.poses_and_points(g, used, o, gm.MapperReport())
    res.close()
    db = {k: getattr(g, k) for k in ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr",
                                     "inlier_matches")}
    tri = init_geometry.triangulate_all_points(**db, camera_size=g.camera_size, orientations=rot.orientations,
                                               image_tvec=pos.image_tvec, registered=pos.has_position, pair_used=used)
    t = {}
    t0 = time.perf_counter()
    rec = tri.to_reconstruction(g.image_ids, g.image_names, g.camera_ids)
    t["to_reconstruction"] = time.perf_counter() - t0
    reg = rec.RegImageIds()
    cfg = ba.BundleAdjustmentConfig()
    for i in reg:
        cfg.AddImage(i)
    cfg.SetConstantPose(reg[0])
    cfg.SetConstantTvec(reg[1], [0])
    t0 = time.perf_counter()
    problem, maps = ba.flatten(rec, cfg)
    t["flatten"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    S = ba.ResidentSolver(problem)
    t["create"] = time.perf_counter() - t0
    ro = _abi.BARefineOptions()
    _lib.lib().psfm_ba_default_refine_options(C.byref(ro))
    for force in (False, True):
        S.iterative_refinement(gm._refine_options(o, force), ro)
    t0 = time.perf_counter()
    S.get_state()
    alive, err = S.observation_mask(), S.point_errors()
    S.close()
    ba.scatter(problem, maps, rec)
    t["get_state_and_mask"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    ba.apply_observation_mask(problem, maps, rec, alive, err)
    t["apply_observation_mask"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    colmap_io.write_model(rec, out)
    t["write_model"] = time.perf_counter() - t0
    return t, problem.num_observations


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="small,sintel,davis")
    ap.add_argument("--repeats", type=int, default=3, help="mapper calls per shape (the Python route runs once)")
    ap.add_argument("--out", default=None, help="where the models go (default: a temporary directory)")
    args = ap.parse_args()
    from particlesfm_b200 import device_count, global_mapper as gm
    if device_count() <= 0:
        raise SystemExit("bench_mapper: no CUDA device (there is no CPU path to time)")
    print(json.dumps({"device": _device_info()}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        base = args.out or tmp
        for name in args.shapes.split(","):
            path = os.path.join(tmp, name + ".db")
            t0 = time.perf_counter()
            _database(path, *SHAPES[name])
            build_s = time.perf_counter() - t0
            o = gm.GlobalMapperOptions(ba_refine_extra_params=False)
            totals, stages = [], {}
            for _ in range(args.repeats):
                t0 = time.perf_counter()
                rep = gm.global_mapper(path, os.path.join(base, name), o)
                totals.append(time.perf_counter() - t0)
                for n, s, _ in rep.stages:
                    stages.setdefault(n, []).append(1e3 * s)
            mmm = lambda v: [round(min(v), 2), round(statistics.median(v), 2), round(max(v), 2)]
            rec = {"shape": name, "database_build_s": round(build_s, 3), "calls": args.repeats,
                   "mapper_s_min_median_max": mmm(totals), "success": rep.success,
                   "stages_ms_min_median_max": {n: mmm(v) for n, v in stages.items()}}
            for n, _, summ in rep.stages:
                if n == "handoff":
                    rec["observations"] = summ["observations"]
                if n == "write":
                    rec["written"] = summ
            py, m = _python_route(path, o, os.path.join(base, name + "_python", "0"))
            rec["python_route_ms"] = {k: round(1e3 * v, 2) for k, v in py.items()}
            rec["python_route_observations"] = m
            print(json.dumps(rec), flush=True)
    print(json.dumps({"device": _device_info()}), flush=True)


if __name__ == "__main__":
    main()
