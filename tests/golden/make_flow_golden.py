"""Generates tests/golden/flow_small.npz by running the REFERENCE's own RAFT (third_party/RAFT/core of a ParticleSfM
checkout, imported read-only) on the CPU, with the weights of oracle.raft_oracle.seeded_state_dict(0), on the three
123 x 125 frames of seeded_frames(3, 123, 125, seed=0), as compute_raft_custom_folder(_stride2).py call it:
InputPadder('sintel'), model(image1, image2, iters=32, test_mode=True) per direction, unpad.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_flow_golden.py

The shape pads both sides (123 -> 128 and 125 -> 128) and gives a 16 x 16 grid at 1/8, whose coarsest level is 2 x 2.
A smaller frame (under 121 pixels on a side) gives a 1-pixel coarsest level, where the reference's bilinear_sampler
divides by W - 1 = 0 and every flow it returns is NaN; the product refuses such frames.

Stored: f1, b1 [2][123][125][2] (stride 1), f2, b2 [1][123][125][2] (stride 2), the reference's
flow_viz.flow_to_image(f1[0], convert_to_bgr=True) pixels, the first 12 bytes and the SHA-256 of the reference's
flow_write(f1[0]) file, and the checks below.  The weights keep the flows away from both degenerate ends: the script
asserts that at least 75 % of the last iteration's lookup centres lie inside the 1/8 grid (87.5 % do), that the flows
are not all zero, and that none is NaN or beyond the frame.  The file is about 690 KB: six float32 maps of the
smallest frame size whose reference flows are not NaN do not compress.  With fan-in weights alone (flow_head_scale = 1) the centres leave the
grid; FLOW_HEAD_SCALE = 0.05 is the scale that keeps them in.
"""
import hashlib
import importlib.util
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = os.environ["PSFM_REFERENCE"]            # a ParticleSfM checkout
H, W = 123, 125


def main():
    import argparse
    import torch
    from oracle import raft_oracle as ro
    from particlesfm_b200 import optical_flow as of
    raft_dir = os.path.join(REF, "third_party", "RAFT")
    sys.path.insert(0, os.path.join(raft_dir, "core"))
    from raft import RAFT
    from utils import flow_viz
    from utils.utils import InputPadder
    spec = importlib.util.spec_from_file_location("raft_custom_utils", os.path.join(raft_dir, "custom_utils.py"))
    cu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cu)

    args = argparse.Namespace(small=False, alternate_corr=False, mixed_precision=False)
    model = RAFT(args)
    ref_sd = model.state_dict()
    ours = of.state_shapes()
    assert list(sorted(ref_sd)) == sorted(ours), set(ref_sd) ^ set(ours)
    assert all(tuple(ref_sd[k].shape) == ours[k] for k in ours)
    model.load_state_dict(ro.seeded_state_dict(0))
    model.eval()
    torch.set_grad_enabled(False)

    frames = ro.seeded_frames(3, H, W, seed=0)
    centres_inside = []

    def call(a, b):
        im1 = torch.from_numpy(a).permute(2, 0, 1).float()[None]
        im2 = torch.from_numpy(b).permute(2, 0, 1).float()[None]
        padder = InputPadder(im1.shape)
        im1, im2 = padder.pad(im1, im2)
        low, up = model(im1, im2, iters=32, test_mode=True)
        gh, gw = low.shape[2:]
        c = low + of.coords_grid(1, gh, gw, "cpu")
        centres_inside.append(float(((c[:, 0] >= 0) & (c[:, 0] <= gw - 1) & (c[:, 1] >= 0) & (c[:, 1] <= gh - 1)).float().mean()))
        return padder.unpad(up)[0].permute(1, 2, 0).numpy()

    f1 = np.stack([call(frames[t], frames[t + 1]) for t in range(2)])
    b1 = np.stack([call(frames[t + 1], frames[t]) for t in range(2)])
    f2 = np.stack([call(frames[0], frames[2])])
    b2 = np.stack([call(frames[2], frames[0])])
    maps = np.concatenate([f1, b1, f2, b2])
    inside = min(centres_inside)
    assert np.isfinite(maps).all(), "NaN flow"
    assert np.abs(maps).max() < max(H, W), "flow beyond the frame"
    assert (np.abs(maps) > 1e-3).mean() > 0.5, "flows mostly zero"
    assert inside >= 0.75, "lookup centres leave the grid: %.3f inside" % inside

    img = flow_viz.flow_to_image(f1[0], convert_to_bgr=True)
    with tempfile.TemporaryDirectory() as tmp:
        p = os.path.join(tmp, "a.flo")
        cu.flow_write(p, f1[0])
        flo = open(p, "rb").read()
    out = os.path.join(HERE, "flow_small.npz")
    np.savez_compressed(out, f1=f1, b1=b1, f2=f2, b2=b2, image=img, flo_head=np.frombuffer(flo[:12], np.uint8),
                        flo_sha256=np.array(hashlib.sha256(flo).hexdigest()), flo_size=np.array(len(flo)),
                        min_centres_inside=np.array(inside), max_abs_flow=np.array(np.abs(maps).max()),
                        mean_abs_flow=np.array(np.abs(maps).mean()))
    print("wrote", out, os.path.getsize(out), "bytes; lookup centres inside >= %.3f, |flow| mean %.3f max %.3f"
          % (inside, np.abs(maps).mean(), np.abs(maps).max()))


if __name__ == "__main__":
    main()
