"""Generates tests/golden/handoff_small.npz by running the REFERENCE's own
`traj_to_matches` (the reference's sfm/matches_from_flow.py:51-118, imported read-only) on
a small synthetic track file.  Pins keypoint order / indices, match lists and their order
and the pair-list order of particlesfm_b200.handoff.traj_to_matches.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_handoff_golden.py
"""
import os
import sys
import tempfile

import numpy as np

REF = os.environ["PSFM_REFERENCE"]            # a ParticleSfM checkout


def make_tracks(num_images=36, num_traj=160, seed=21):
    rng = np.random.default_rng(seed)
    tracks = {}
    tid = 0
    for _ in range(num_traj):
        n = int(rng.choice([1, 2, 3, 5, 9, 14, 20, 21, 25, 33, 36], p=[.05, .1, .15, .15, .15, .1, .05, .05, .1, .05, .05]))
        n = min(n, num_images)
        start = int(rng.integers(0, num_images - n + 1))
        labels = (rng.random(n) < 0.15).astype(int)
        if rng.random() < 0.1:
            labels[:] = 1                                   # fully dynamic trajectory
        tracks[tid] = {"locations": [list(map(float, rng.uniform(0, 100, 2))) for _ in range(n)],
                       "labels": labels.tolist(), "frame_ids": list(range(start, start + n))}
        tid += int(rng.integers(1, 4))                      # ids with holes, dict order = insertion order
    return tracks


def main():
    sys.path.insert(0, os.path.join(REF, "sfm"))
    import matches_from_flow as ref
    num_images = 36
    tracks = make_tracks(num_images)
    out = {}
    with tempfile.TemporaryDirectory() as d:
        img_dir, traj_dir = os.path.join(d, "images"), os.path.join(d, "traj")
        os.makedirs(img_dir); os.makedirs(traj_dir)
        names = [f"{i:05d}.png" for i in range(num_images)]
        for n in names:
            open(os.path.join(img_dir, n), "w").close()
        np.save(os.path.join(traj_dir, "track.npy"), tracks, allow_pickle=True)
        for tag, rd in (("static", True), ("all", False)):
            pair_file = os.path.join(d, f"pairs_{tag}.txt")
            datas = ref.traj_to_matches(img_dir, traj_dir, pair_file, remove_dynamic=rd)
            kp = [np.asarray(datas[n].keypoints, dtype=np.float64).reshape(-1, 2) for n in names]
            out[f"{tag}_kp_ptr"] = np.concatenate([[0], np.cumsum([k.shape[0] for k in kp])])
            out[f"{tag}_kp"] = np.concatenate(kp)
            pa, pb, ptr, mm = [], [], [0], []
            for line in open(pair_file).read().split("\n"):
                if not line:
                    continue
                n0, n1 = line.split(" ")
                m = np.asarray(datas[n0].match_pairs[n0 + "-" + n1], dtype=np.int64).reshape(-1, 2)
                pa.append(names.index(n0)); pb.append(names.index(n1)); mm.append(m); ptr.append(ptr[-1] + m.shape[0])
            out[f"{tag}_pairs"] = np.stack([pa, pb], 1).astype(np.int64)
            out[f"{tag}_pair_ptr"] = np.asarray(ptr, dtype=np.int64)
            out[f"{tag}_matches"] = np.concatenate(mm)
    keys = list(tracks.keys())
    out["track_keys"] = np.asarray(keys, dtype=np.int64)
    out["track_len"] = np.asarray([len(tracks[k]["frame_ids"]) for k in keys], dtype=np.int64)
    out["track_frames"] = np.concatenate([tracks[k]["frame_ids"] for k in keys]).astype(np.int64)
    out["track_labels"] = np.concatenate([tracks[k]["labels"] for k in keys]).astype(np.int64)
    out["track_locs"] = np.concatenate([np.asarray(tracks[k]["locations"]) for k in keys])
    out["num_images"] = np.int64(num_images)
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "handoff_small.npz"), **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
