"""Generates tests/golden/track_small.npz by running the REFERENCE's own Python tracker without path consistency
(the reference's point_trajectory/track.py, imported read-only) on the 7-frame 36 x 52 sequence of
tracker_small.npz, with that fixture's occlusion maps.  The reference's native module is replaced by the same stub
as in make_tracker_golden.py (this repo's pybind11 Trajectory; track.py never calls the optimiser), so the fixture
pins the tracker semantics of the skip-path-consistency mode: sampling, survival test, re-seeding, id order.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_track_golden.py
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "particle-sfm_b200"))
REF = os.environ["PSFM_REFERENCE"]            # a ParticleSfM checkout


def main():
    import particlesfm as ours          # the pybind11 module of this repo (containers)

    def no_optimiser(*args):
        raise AssertionError("track.py does not optimise")
    stub = types.SimpleNamespace(Trajectory=ours.Trajectory, TrajectorySet=ours.TrajectorySet, optimize_location=no_optimiser)
    pkg = types.ModuleType("point_trajectory.optimize.build")
    pkg.particlesfm = stub
    sys.modules["point_trajectory.optimize"] = types.ModuleType("point_trajectory.optimize")
    sys.modules["point_trajectory.optimize.build"] = pkg
    sys.path.insert(0, REF)
    from point_trajectory.track import track as ref_track

    g = np.load(os.path.join(HERE, "tracker_small.npz"))
    fw = [g["fw"][i] for i in range(g["fw"].shape[0])]
    occ = [g["occ"][i] for i in range(g["occ"].shape[0])]
    trajs = ref_track(fw, occ, 2)
    ids, lens, frames, locs = [], [], [], []
    for idx, t in enumerate(trajs):
        ids.append(idx); lens.append(t.length())
        frames.extend(t.times); locs.extend([np.asarray(p) for p in t.xys])
    out = os.path.join(HERE, "track_small.npz")
    np.savez_compressed(out, ids=np.array(ids), lens=np.array(lens), frames=np.array(frames), locs=np.array(locs))
    print("wrote", out, "trajectories", len(ids), "observations", len(frames), "mean len", np.mean(lens))


if __name__ == "__main__":
    main()
