"""python tools/bench_handoff.py [--shapes sintel,davis] [--repeats 2] [--arms host,device]

Wall time of the hand-off from a track set to COLMAP database rows, on seeded synthetic track sets with the
tracker's counts at two user shapes (synthetic.make_track_arrays: contiguous frame windows, geometric lengths):

    sintel   131 k trajectories,  5.52 M observations, 50 frames
    davis    489 k trajectories, 32.3 M observations,  80 frames

Arms, alternated within one process after a warm-up of each on a small track set:
    host     traj_to_matches + as_reference + import_keypoints_matches (numpy and Python lists)
    device   traj_to_matches_device + import_keypoints_matches_arrays (csrc/handoff.cu, then one slice per pair)
Both end in the same DatabaseRows (skip_geometric_verification=True, database ids in reverse name order so that
the column flip is exercised).  With both arms, the TrajectoryMatches and the rows of the last repeat are checked
to be bit-identical.  The host arm holds about 0.13 GB per million matches; where that exceeds 80 % of the
available memory it is reported as not run.  Prints one JSON line with the device name and power limit.
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

SHAPES = {"sintel": (131_000, 50, 5_520_000), "davis": (489_000, 80, 32_300_000)}
HOST_GB_PER_MILLION_MATCHES = 0.13


def _mem_available_gb():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 2 ** 20
    return 0.0


def _num_matches(arrays, k=20):
    n = arrays.lengths()
    return int(np.where(n <= k, n * (n - 1), k * (n - 1)).sum())


def _stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "all": xs} if xs else None


def _same_matches(a, b):
    return (len(a.keypoints) == len(b.keypoints) and all(np.array_equal(x, y) for x, y in zip(a.keypoints, b.keypoints))
            and all(np.array_equal(getattr(a, k), getattr(b, k)) for k in ("pair_images", "pair_ptr", "matches")))


def _same_rows(a, b):
    return all(len(x) == len(y) and all(i == j and u.tobytes() == v.tobytes() for (i, u), (j, v) in zip(x, y))
               for x, y in ((a.keypoints, b.keypoints), (a.matches, b.matches), (a.two_view, b.two_view)))


def run_shape(name, repeats, arms):
    from particlesfm_b200 import handoff, synthetic as syn
    ntraj, nf, nobs = SHAPES[name]
    arrays = syn.make_track_arrays(ntraj, nf, nobs, seed=nf)
    names = ["%05d.png" % i for i in range(nf)]
    image_ids = {n: nf - i for i, n in enumerate(names)}
    nm = _num_matches(arrays)
    out = {"shape": name, "frames": nf, "trajectories": ntraj, "observations": nobs, "matches": nm}
    arms = list(arms)
    if "host" in arms:
        need, avail = HOST_GB_PER_MILLION_MATCHES * nm / 1e6, _mem_available_gb()
        if need > 0.8 * avail:
            arms.remove("host")
            out["host"] = "not run: about %.0f GB needed, %.0f GB available" % (need, avail)

    def host(a):
        t0 = time.perf_counter()
        m = handoff.traj_to_matches(a, nf)
        t1 = time.perf_counter()
        data = m.as_reference(names)
        rows = handoff.import_keypoints_matches(image_ids, data, skip_geometric_verification=True)
        del data
        return m, rows, t1 - t0, time.perf_counter() - t1

    def device(a):
        t0 = time.perf_counter()
        m = handoff.traj_to_matches_device(a, nf)
        t1 = time.perf_counter()
        rows = handoff.import_keypoints_matches_arrays(names, image_ids, m, skip_geometric_verification=True)
        return m, rows, t1 - t0, time.perf_counter() - t1

    small = syn.make_track_arrays(2000, nf, 2000 * (nobs // ntraj), seed=1)
    for arm in arms:                                    # warm-up: modules, CUDA context, allocator
        (host if arm == "host" else device)(small)
    times = {f"{arm}_{part}": [] for arm in arms for part in ("to_matches", "to_rows", "total")}
    last = {}
    for r in range(repeats):
        for arm in arms:
            last.pop(arm, None)
            gc.collect()
            m, rows, tm, tr = (host if arm == "host" else device)(arrays)
            times[arm + "_to_matches"].append(tm)
            times[arm + "_to_rows"].append(tr)
            times[arm + "_total"].append(tm + tr)
            if r == repeats - 1:
                last[arm] = (m, rows)
            del m, rows
    for k, v in times.items():
        out[k + "_s"] = _stats(v)
    if "device" in last:
        m, rows = last["device"]
        out["pairs"], out["database_rows"] = int(m.pair_images.shape[0]), len(rows.matches)
        assert int(m.matches.shape[0]) == nm
    if "host" in last and "device" in last:
        out["bit_identical"] = bool(_same_matches(last["host"][0], last["device"][0])
                                    and _same_rows(last["host"][1], last["device"][1]))
        out["speedup_median"] = statistics.median(times["host_total"]) / statistics.median(times["device_total"])
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--shapes", default="sintel,davis")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--arms", default="host,device")
    args = ap.parse_args()
    import bench
    from particlesfm_b200 import device_count
    arms = [a for a in args.arms.split(",") if a]
    if "device" in arms and device_count() <= 0:
        raise SystemExit("bench_handoff: no CUDA device (the product has no CPU path)")
    results = []
    for name in [s for s in args.shapes.split(",") if s]:
        results.append(run_shape(name, args.repeats, arms))
        print("[bench_handoff]", json.dumps(results[-1]), file=sys.stderr, flush=True)
    gpu = bench.gpu_info(bench.smi_device(0)) if device_count() > 0 else None
    print(json.dumps({"tool": "bench_handoff", "gpu": gpu, "repeats": args.repeats, "arms": arms, "results": results}))


if __name__ == "__main__":
    main()
