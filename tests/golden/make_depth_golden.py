"""Generates tests/golden/depth_small.npz by running the REFERENCE's own run_midas (third_party/MiDaS of a ParticleSfM
checkout, imported read-only) on the CPU, so in float32, with model midas_v21, the weights of
oracle.midas_oracle.seeded_state_dict(0) saved as a .pt, on the three 192 x 40 frames of seeded_frames(3, 40, 192,
seed=0) written as PNGs.

    PSFM_REFERENCE=/path/to/particle-sfm python tests/golden/make_depth_golden.py

Two patches make the reference importable without a network or timm: torch.hub.load (the WSL ResNeXt entry) is
replaced by torchvision's resnext101_32x8d(weights=None), the architecture that entry builds (its weights are
overwritten by the load that follows), and `timm` is a stub module (midas/vit.py imports it at top level but uses it
only inside the DPT constructors).  The script asserts that the reference model's state-dict keys and shapes are
particlesfm_b200.midas.state_shapes().

The frame size gives a 384 x 64 network input: 40 * 384 / 192 / 32 = 2.5, which np.round takes to 2 (ties to even).

Stored: transform0, the reference transform's float32 network input of frame 0 [3][64][384]; maps, the three PFMs
read back with read_pfm [3][40][192]; pfm_sha256 and pfm_head, the SHA-256 and first 32 bytes of frame 0's PFM file;
pixels, the three PNGs read with cv2.imread(p, -1); max_activation, the largest |output| of any module of the
reference model over the three frames; sizes, a table of Resize.get_size (width, height -> width, height) over a few
hundred shapes, including exact ties of np.round and shapes that give a zero side.
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
REF = os.environ["PSFM_REFERENCE"]            # a ParticleSfM checkout
H, W = 40, 192


def size_table():
    rng = np.random.default_rng(0)
    shapes = {(int(w), int(h)) for w, h in rng.integers(1, 4000, (200, 2))}
    shapes |= {(int(w), int(h)) for w, h in rng.integers(16, 1200, (100, 2))}
    # exact ties: 12 h / w (or 12 w / h) is k + 1/2
    for w in (48, 96, 192, 240, 480, 960, 1920):
        for h in range(1, w + 1):
            if (24 * h) % w == 0 and (24 * h // w) % 2 == 1:
                shapes |= {(w, h), (h, w)}
    shapes |= {(1000, 40), (40, 1000), (1024, 436), (854, 480), (384, 384), (1, 1), (767, 16), (768, 16), (769, 16)}
    return sorted(shapes)


def main():
    import cv2
    import torch
    import torchvision
    from oracle import midas_oracle as mo
    from particlesfm_b200 import midas

    torch.hub.load = lambda *a, **k: torchvision.models.resnext101_32x8d(weights=None)
    sys.modules.setdefault("timm", types.ModuleType("timm"))
    mdir = os.path.join(REF, "third_party", "MiDaS")
    sys.path.insert(0, mdir)
    import midas_utils
    import run as midas_run
    from midas.midas_net import MidasNet
    from midas.transforms import NormalizeImage, PrepareForNet, Resize
    assert not torch.cuda.is_available(), "run on a CPU device: the reference then computes in float32"

    sd = mo.seeded_state_dict(0)
    frames = mo.seeded_frames(3, H, W, seed=0)
    with tempfile.TemporaryDirectory() as tmp:
        weights = os.path.join(tmp, "midas_v21.pt")
        torch.save(sd, weights)
        model = MidasNet(weights, non_negative=True)
        ref_sd = model.state_dict()
        ours = midas.state_shapes()
        assert sorted(ref_sd) == sorted(ours), set(ref_sd) ^ set(ours)
        assert all(tuple(ref_sd[k].shape) == ours[k] for k in ours)
        model.eval()
        largest = [0.0]

        def hook(mod, inp, out):
            if isinstance(out, torch.Tensor):
                largest[0] = max(largest[0], out.abs().max().item())
        for m in model.modules():
            m.register_forward_hook(hook)

        img_dir, out_dir = os.path.join(tmp, "images"), os.path.join(tmp, "midas_depth")
        os.makedirs(img_dir)
        names = ["%05d.png" % i for i in range(len(frames))]
        for n, f in zip(names, frames):
            cv2.imwrite(os.path.join(img_dir, n), f[:, :, ::-1])
        transform = lambda img: PrepareForNet()(NormalizeImage(mean=mo.MEAN, std=mo.STD)(Resize(
            384, 384, resize_target=None, keep_aspect_ratio=True, ensure_multiple_of=32, resize_method="upper_bound",
            image_interpolation_method=cv2.INTER_CUBIC)({"image": img})))["image"]
        inputs = [transform(midas_utils.read_image(os.path.join(img_dir, n))) for n in names]
        with torch.no_grad():
            for x in inputs:
                model(torch.from_numpy(x)[None])
        midas_run.run_midas(img_dir, out_dir, weights, "midas_v21", optimize=True)

        maps = np.stack([midas_utils.read_pfm(os.path.join(out_dir, n[:-4] + ".pfm"))[0] for n in names])
        pixels = np.stack([cv2.imread(os.path.join(out_dir, n[:-4] + ".png"), -1) for n in names])
        pfm = open(os.path.join(out_dir, names[0][:-4] + ".pfm"), "rb").read()

    assert maps.dtype == np.float32 and pixels.dtype == np.uint16
    assert (maps > 0).mean() > 0.9 and maps.max() > maps.min(), "maps constant or mostly clipped by the final ReLU"
    assert largest[0] < 60000, "activations leave fp16's range: %g" % largest[0]
    resize = Resize(384, 384, resize_target=None, keep_aspect_ratio=True, ensure_multiple_of=32,
                    resize_method="upper_bound")
    shapes = size_table()
    sizes = np.array([(w, h) + tuple(int(v) for v in resize.get_size(w, h)) for w, h in shapes], np.int64)
    out = os.path.join(HERE, "depth_small.npz")
    np.savez_compressed(out, transform0=inputs[0], maps=maps, pixels=pixels, pfm_head=np.frombuffer(pfm[:32], np.uint8),
                        pfm_sha256=np.array(hashlib.sha256(pfm).hexdigest()), pfm_size=np.array(len(pfm)),
                        max_activation=np.array(largest[0]), sizes=sizes)
    print("wrote", out, os.path.getsize(out), "bytes; largest activation %.1f, depth %.3f .. %.3f, %d sizes"
          % (largest[0], maps.min(), maps.max(), len(sizes)))


if __name__ == "__main__":
    main()
