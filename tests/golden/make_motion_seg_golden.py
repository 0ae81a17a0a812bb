"""Generates tests/golden/motion_seg_small.npz by running the REFERENCE's own main_motion_segmentation (motion_seg/
of a ParticleSfM checkout, imported read-only) on the CPU, so in float32, with the traj_oa_depth weights of
oracle.motion_seg_oracle.seeded_state_dict(4) saved as a checkpoint.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_motion_seg_golden.py

Patches that make the reference run here: .cuda() of tensors and modules is the identity; `cvbase` and `torchvision`
are stub modules (utils.py imports cvbase's flow2rgb, which the labeller never calls; only torchvision's ToTensor is
used, restated for the ndarrays it gets); a temporary config names the seeded checkpoint; cv2.VideoWriter is replaced
by a recorder that keeps the SHA-256 of every frame before encoding.  The track sets are this project's
particlesfm.TrajectorySet, and np.random.seed(0) precedes each run, so the video's random trajectories are those of
np.random.RandomState(0).

Cases (every input regenerated from seeds by the oracle's seeded_* helpers):
  0: 12 frames of 96 x 160 (up-scaled to 240 x 424), window 5 (the last window overlaps), no cut
  1: the same with traj_max_num 30, below the windows' sizes (the fixed-seed shuffle cuts them)
  2: 6 frames of 300 x 500 (down-scaled), window 10 >= length (one window, Python-int keys)

Stored per case c: feat_c_w and logit_c_w, each window's encoder features [K][16] and logits [K] (forward hooks on
joint_encoder and decoder); keys_c, key_int_c (whether the keys are Python ints), ptr_c, frames_c, labels_c,
locations_c, the saved dict flattened in its key order; sha_c, the frames' SHA-256.
"""
import hashlib
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["PSFM_REFERENCE"]

CASES = [dict(n=12, h=96, w=160, window=5, cap=100000, trajs=200, seed=17),
         dict(n=12, h=96, w=160, window=5, cap=30, trajs=200, seed=17),
         dict(n=6, h=300, w=500, window=10, cap=100000, trajs=150, seed=5)]


def _stubs():
    import torch
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    cvbase = types.ModuleType("cvbase")
    cvbase.optflow = types.ModuleType("cvbase.optflow")
    cvbase.optflow.visualize = types.ModuleType("cvbase.optflow.visualize")
    cvbase.optflow.visualize.flow2rgb = None
    for m in (cvbase, cvbase.optflow, cvbase.optflow.visualize):
        sys.modules[m.__name__] = m

    class ToTensor:
        def __call__(self, pic):
            pic = pic[:, :, None] if pic.ndim == 2 else pic
            t = torch.from_numpy(pic.transpose((2, 0, 1))).contiguous()
            return t.float().div(255) if t.dtype == torch.uint8 else t
    tv = types.ModuleType("torchvision")
    tv.transforms = types.SimpleNamespace(ToTensor=ToTensor)
    sys.modules["torchvision"] = tv


class Recorder:
    frames = []

    def __init__(self, *a, **k):
        pass

    def write(self, img):
        Recorder.frames.append(hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest())

    def release(self):
        pass


def main():
    _stubs()
    import cv2
    import torch
    import oracle.motion_seg_oracle as O
    from particlesfm_b200.point_trajectory import _particlesfm
    _particlesfm()                                   # track.npy unpickles to particlesfm.TrajectorySet
    sys.path.insert(0, REF)
    import motion_seg.main_motion_segmentation  # noqa: F401 (the package re-exports the function under this name)
    mms = sys.modules["motion_seg.main_motion_segmentation"]
    cv2.VideoWriter = Recorder
    out = {}
    for c, case in enumerate(CASES):
        with tempfile.TemporaryDirectory() as tmp:
            img, dep, trj, lab = (os.path.join(tmp, d) for d in ("images", "depth", "traj", "traj_labeled"))
            for d in (img, dep, trj):
                os.makedirs(d)
            frames = O.seeded_frames(case["n"], case["h"], case["w"], seed=9)
            px = O.seeded_depth_pixels(case["n"], case["h"], case["w"], seed=8)
            for i in range(case["n"]):
                cv2.imwrite(os.path.join(img, "%05d.png" % i), frames[i][:, :, ::-1])
                cv2.imwrite(os.path.join(dep, "%05d.png" % i), px[i])
            np.save(os.path.join(trj, "track.npy"),
                    O.seeded_track_set(case["trajs"], case["n"], case["h"], case["w"], case["seed"]))
            ckpt = os.path.join(tmp, "ckpt.pth")
            torch.save({"model_state_dict": O.seeded_state_dict(4)}, ckpt)
            cfg = os.path.join(tmp, "cfg.yaml")
            with open(cfg, "w") as f:
                f.write("model_name: traj_oa_depth\nresolution: [240, 424]\nresume_path: %s\n" % ckpt)
            feats, logits = [], []
            real = mms.traj_oa_depth

            def hooked(*a, **k):
                m = real(*a, **k)
                m.joint_encoder.register_forward_hook(lambda mod, i, o: feats.append(o[0].t().numpy().copy()))
                m.decoder.register_forward_hook(lambda mod, i, o: logits.append(o[0, 0].numpy().copy()))
                return m
            mms.traj_oa_depth = hooked
            Recorder.frames = []
            np.random.seed(0)
            with torch.no_grad():
                mms.main_motion_segmentation(img, dep, trj, lab, config_file=cfg, window_size=case["window"],
                                             traj_max_num=case["cap"])
            mms.traj_oa_depth = real
            d = np.load(os.path.join(lab, "track.npy"), allow_pickle=True).item()
        keys = list(d)
        out["keys_%d" % c] = np.array([int(k) for k in keys], np.int64)
        out["key_int_%d" % c] = np.array(all(type(k) is int for k in keys))
        lens = [len(d[k]["frame_ids"]) for k in keys]
        out["ptr_%d" % c] = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        out["frames_%d" % c] = np.concatenate([d[k]["frame_ids"] for k in keys]).astype(np.int64)
        out["labels_%d" % c] = np.concatenate([d[k]["labels"] for k in keys]).astype(bool)
        out["locations_%d" % c] = np.concatenate([d[k]["locations"] for k in keys]).astype(np.float64)
        out["sha_%d" % c] = np.array(Recorder.frames)
        for w, (f, l) in enumerate(zip(feats, logits)):
            out["feat_%d_%d" % (c, w)], out["logit_%d_%d" % (c, w)] = f, l
        near = sum(int(np.sum(np.abs(l) < 1e-3)) for l in logits)
        total = sum(l.size for l in logits)
        assert near <= 0.01 * total, (near, total)
        print("case %d: %d windows, %d trajectories, %d observations, %d of %d logits within 1e-3 of 0"
              % (c, len(logits), len(keys), out["frames_%d" % c].size, near, total))
    np.savez_compressed(os.path.join(HERE, "motion_seg_small.npz"), **out)


if __name__ == "__main__":
    main()
