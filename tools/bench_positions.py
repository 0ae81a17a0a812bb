"""python tools/bench_positions.py [--shapes sintel,davis,target,config5,long] [--repeats 3] [--oracle-max-images 200]

Wall time of the two global-mapper steps after rotation averaging, on these shapes:

    sintel   the two-view chain at 50 frames (make_two_view_scene, helix path -> traj_to_matches_device ->
             estimate_relative_poses -> estimate_global_rotations), then all kept pairs through both calls
    davis    the same at 80 frames
    target   synthetic.make_view_graph, complete, F = 200 (19,900 pairs), 1 degree direction noise, 10 % outliers
    config5  the same at F = 500 (124,750 pairs)
    long     banded (pairs up to 10 frames apart), F = 1,000, 0.5 degree direction noise

Calls, after a warm-up of each:
    pairwise   init_geometry.optimize_pairwise_translations (chain shapes only), with the bytes its inputs take
    positions  init_geometry.estimate_global_positions, split into host graph work, building S, factoring S,
               inverting S and the ADMM loop (from its summary), with its ADMM iterations and launches
    oracle     oracle/position_oracle.py (NOT the reference: gcolmap is not built here), reported as not run above
               --oracle-max-images images; where it runs, iteration counts and positions are compared
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

CHAIN = {"sintel": (30_000, 50, 600_000), "davis": (50_000, 80, 1_600_000)}
SYNTH = {"target": dict(num_images=200, direction_noise_deg=1.0, direction_outlier_fraction=0.1, seed=5),
         "config5": dict(num_images=500, direction_noise_deg=1.0, direction_outlier_fraction=0.1, seed=6),
         "long": dict(num_images=1000, graph="banded", band=10, direction_noise_deg=0.5, seed=7)}
DB = ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr", "inlier_matches")


def _stats(xs):
    return {"min": min(xs), "median": statistics.median(xs), "max": max(xs)} if xs else None


def _device_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _timed(fn, repeats):
    fn()
    times, out = [], None
    for _ in range(repeats):
        t = time.perf_counter()
        out = fn()
        times.append(time.perf_counter() - t)
    return out, _stats(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="sintel,davis,target,config5,long")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--oracle-max-images", type=int, default=200)
    a = ap.parse_args()
    from oracle import position_oracle as po
    from particlesfm_b200 import device_count, handoff, init_geometry, synthetic as syn
    if device_count() <= 0:
        raise SystemExit("no CUDA device: this benchmark measures the GPU path")
    results = {"device": _device_info(), "oracle": "numpy/scipy restatement (not the reference)", "shapes": {}}
    for name in a.shapes.split(","):
        r = {}
        if name in CHAIN:
            ntraj, nf, nobs = CHAIN[name]
            tracks, qvec, tvec, cam = syn.make_two_view_scene(ntraj, nf, nobs, seed=nf, path="helix")
            ids = list(range(1, nf + 1))
            names = ["%05d.png" % i for i in range(nf)]
            rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(tracks, nf))
            args = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
            poses = init_geometry.estimate_relative_poses(**args)
            rot = init_geometry.estimate_global_rotations(nf, args["pair_images"], poses.qvec, np.diff(args["inlier_ptr"]),
                                                          poses.estimated)
            db = {k: args[k] for k in DB}
            kept = rot.pair_kept
            t, r["pairwise_s"] = _timed(lambda: init_geometry.optimize_pairwise_translations(
                **db, orientations=rot.orientations, pair_used=kept), a.repeats)
            n_used = int(np.diff(args["inlier_ptr"])[kept].sum())
            r["pairwise_pairs"], r["pairwise_matches"] = int(kept.sum()), n_used
            # bytes the call uploads: matches (8 per match of every pair), keypoints (8 each), offsets
            r["pairwise_input_bytes"] = int(8 * args["inlier_ptr"][-1] + 8 * args["keypoint_ptr"][-1] +
                                            8 * (len(args["inlier_ptr"]) + len(args["keypoint_ptr"])))
            pargs = dict(num_images=nf, pair_images=args["pair_images"], tvec=t, orientations=rot.orientations,
                         has_orientation=rot.has_orientation, pair_used=kept)
        else:
            g = syn.make_view_graph(**SYNTH[name])
            pargs = dict(num_images=g["num_images"], pair_images=g["pair_images"], tvec=g["tvec"], orientations=g["truth"])
        dev, r["positions_s"] = _timed(lambda: init_geometry.estimate_global_positions(**pargs), a.repeats)
        s = dev.summary
        r.update(images=int(pargs["num_images"]), pairs_used=s["num_pairs_used"], views=s["num_views"],
                 admm_iterations=s["admm_iterations"], admm_iterations_queued=s["admm_iterations_queued"],
                 converged=bool(s["converged"]), launches=s["num_launches"],
                 split_ms={k: s[k] for k in ("host_ms", "build_ms", "factor_ms", "inverse_ms", "admm_ms")},
                 admm_ms_per_iteration=s["admm_ms"] / max(1, s["admm_iterations_queued"]))
        if s["num_views"] <= a.oracle_max_images:
            ref, r["oracle_s"] = _timed(lambda: po.estimate_global_positions(**pargs), 1)
            c = ref["positions"][ref["has_position"]]
            extent = np.linalg.norm(c - c.mean(0), axis=1).max()
            diff = float(np.abs(dev.positions - ref["positions"]).max() / extent)
            r["max_position_diff_rel"] = diff
            r["agrees"] = bool(s["admm_iterations"] == ref["iterations"] and diff <= 1e-9)
        else:
            r["oracle_s"] = "not run (above --oracle-max-images)"
        results["shapes"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
    print(json.dumps(results))


if __name__ == "__main__":
    main()
