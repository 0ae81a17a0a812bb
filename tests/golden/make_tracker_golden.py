"""Generates tests/golden/tracker_small.npz by running the REFERENCE's own Python tracker
(the reference's point_trajectory/track_optimize.py, imported read-only) on a small synthetic
flow sequence.  The reference's native module is replaced by a stub whose `Trajectory` is
this repo's pybind11 class and whose `optimize_location` is the CPU oracle (the reference's
Ceres build is unavailable here — SURVEY.md §8c), so the fixture pins the TRACKER semantics
(sampling, survival test, re-seeding, id order), not the optimiser.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_tracker_golden.py
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "particle-sfm_b200"))
REF = os.environ["PSFM_REFERENCE"]            # a ParticleSfM checkout


def make_sequence(n_frames=7, h=36, w=52, seed=11):
    from particlesfm_b200 import synthetic as syn
    rng = np.random.default_rng(seed)
    fw = [syn.smooth_flow(h, w, rng, 3.0, 4).astype(np.float32) for _ in range(n_frames - 1)]
    yy, xx = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")

    def compose(a, b):   # a then b
        p = np.stack([xx + a[..., 0], yy + a[..., 1]], -1).reshape(-1, 2)
        return (a + syn.bilinear_zeros(b, p).reshape(h, w, 2)).astype(np.float32)

    def backward(a):     # crude inverse: -a sampled at x - a
        p = np.stack([xx - a[..., 0], yy - a[..., 1]], -1).reshape(-1, 2)
        return (-syn.bilinear_zeros(a, p).reshape(h, w, 2)).astype(np.float32)
    fb = [backward(f) for f in fw]
    f2 = [compose(fw[i], fw[i + 1]) + rng.normal(0, 0.05, (h, w, 2)).astype(np.float32) for i in range(n_frames - 2)]
    b2 = [backward(f) for f in f2]
    # a moving occluder so that particles die and new ones are seeded
    for i, f in enumerate(fw):
        f[10:18, 8 + 4 * i:16 + 4 * i] += 6.0
    return fw, fb, f2, b2


def main():
    import oracle
    import particlesfm as ours          # the pybind11 module of this repo (containers)
    stub = types.SimpleNamespace(Trajectory=ours.Trajectory, TrajectorySet=ours.TrajectorySet,
                                 optimize_location=lambda uv12, r1, r2, sc, fmap, n, w, h:
                                 oracle.traj_optimize(uv12, r1, r2, sc, fmap)[0])
    pkg = types.ModuleType("point_trajectory.optimize.build")
    pkg.particlesfm = stub
    sys.modules["point_trajectory.optimize"] = types.ModuleType("point_trajectory.optimize")
    sys.modules["point_trajectory.optimize.build"] = pkg
    sys.path.insert(0, REF)
    from point_trajectory.track_optimize import track_optimize as ref_track_optimize
    from point_trajectory.utils import flow_check as ref_flow_check

    fw, fb, f2, b2 = make_sequence()
    _, occ = ref_flow_check(fw, fb, thres=1.0)
    _, occ2 = ref_flow_check(f2, b2, thres=1.0)
    trajs = ref_track_optimize(fw, f2, occ, occ2, 2)
    ids, lens, frames, locs = [], [], [], []
    for idx, t in enumerate(trajs):
        ids.append(idx); lens.append(t.length())
        frames.extend(t.times); locs.extend([np.asarray(p) for p in t.xys])
    out = os.path.join(ROOT, "tests", "golden", "tracker_small.npz")
    np.savez_compressed(out, fw=np.stack(fw), fb=np.stack(fb), f2=np.stack(f2), b2=np.stack(b2),
                        occ=np.stack(occ), occ2=np.stack(occ2), ids=np.array(ids), lens=np.array(lens),
                        frames=np.array(frames), locs=np.array(locs))
    print("wrote", out, "trajectories", len(ids), "observations", len(frames), "mean len", np.mean(lens))


if __name__ == "__main__":
    main()
