"""MiDaS midas_v21 restated with the reference's call structure (TEST INFRASTRUCTURE, DESIGN.md §4.16).

third_party/MiDaS run.py:run_midas handles one frame per call: read_image (cv2.imread, RGB, / 255 in float64), the
Resize / NormalizeImage / PrepareForNet transform on the host (cv2.resize INTER_CUBIC of the float64 image), a batch-1
forward (fp16 channels_last with optimize on a CUDA device, else float32), F.interpolate(bicubic,
align_corners=False) to the frame size, .cpu().numpy(), then write_depth(bits=2).  This module keeps that structure,
so the product's batching and its kernels (csrc/midas.cu: the input transform, the upsampling with min / max, the
quantisation) are checked against it.  The network is particlesfm_b200.midas.forward (the same torch calls either
way); tests/golden/depth_small.npz pins it and this module to the reference's own run_midas.

The pixels are write_depth's float32 arithmetic on the float32 map that the PFM holds.  With a float16 prediction the
reference's own write_depth computes in float16, where 65535 overflows (reference_fp16_pixels shows it): DESIGN.md
§4.16.

seeded_state_dict(seed) draws reference-keyed weights, so tests and the golden share weights without a checkpoint.
"""
import os

import numpy as np

from particlesfm_b200 import midas

MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]

# Scales of the seeded weights.  With He fan-in weights and unit batch norm, every ResNeXt block adds its branch to
# the identity at full size, and on the golden frames the largest activation reaches 1.6e8, far past fp16's 65504;
# BN3_SCALE shrinks each block's last batch-norm weight so the branches stay small (the largest is then 236:
# make_depth_golden.py records it).  HEAD_SCALE and HEAD_BIAS set the
# last convolution so the depth varies across the frame and stays mostly above the final ReLU's 0.
BN3_SCALE = 0.2
HEAD_SCALE = 0.02
HEAD_BIAS = 2.0


def seeded_state_dict(seed=0):
    """Weights of every key of midas_v21, drawn from numpy.random.default_rng(seed) per sorted key: convolution weights
    N(0, 2 / fan_in), biases N(0, 0.01^2), batch-norm weight 1 + N(0, 0.1^2) (times BN3_SCALE for a block's bn3),
    bias and running mean N(0, 0.1^2), running variance U(0.5, 1.5); the last convolution's weight times HEAD_SCALE
    and its bias HEAD_BIAS."""
    import torch
    rng = np.random.default_rng(seed)
    out = {}
    for k, shape in sorted(midas.state_shapes().items()):
        if k.endswith("num_batches_tracked"):
            out[k] = torch.tensor(0, dtype=torch.int64)
            continue
        if len(shape) == 4:
            v = rng.standard_normal(shape) * np.sqrt(2.0 / np.prod(shape[1:]))
            if k == "scratch.output_conv.4.weight":
                v = v * HEAD_SCALE
        elif k.endswith(".running_var"):
            v = rng.uniform(0.5, 1.5, shape)
        elif k == "scratch.output_conv.4.bias":
            v = np.full(shape, HEAD_BIAS)
        elif k.startswith("scratch.") and k.endswith(".bias"):
            v = 0.01 * rng.standard_normal(shape)
        elif k.endswith(".weight"):
            v = 1.0 + 0.1 * rng.standard_normal(shape)
            if ".bn3." in k:
                v = v * BN3_SCALE
        else:
            v = 0.1 * rng.standard_normal(shape)
        out[k] = torch.tensor(v, dtype=torch.float32)
    return out


def seeded_frames(n, h, w, seed=0):
    """n seeded uint8 RGB frames [h][w][3]: a smooth random texture with a brighter disc moving across it, plus noise."""
    rng = np.random.default_rng(seed)
    base = rng.uniform(0, 255, (h // 8 + 3, w // 8 + 3, 3))
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    fy, fx = yy / 8.0, xx / 8.0
    y0, x0 = np.floor(fy).astype(int), np.floor(fx).astype(int)
    a, b = (fy - y0)[..., None], (fx - x0)[..., None]
    tex = ((1 - a) * (1 - b) * base[y0, x0] + (1 - a) * b * base[y0, x0 + 1] + a * (1 - b) * base[y0 + 1, x0]
           + a * b * base[y0 + 1, x0 + 1])
    frames = []
    for t in range(n):
        cy, cx = h * (0.3 + 0.1 * t), w * (0.3 + 0.15 * t)
        disc = (((yy - cy) ** 2 + (xx - cx) ** 2) < (0.2 * min(h, w)) ** 2)[..., None]
        v = np.where(disc, 0.5 * tex + 120, tex) + rng.normal(0, 4, tex.shape)
        frames.append(np.clip(v, 0, 255).astype(np.uint8))
    return frames


def get_size(width, height):
    """Resize(384, 384, resize_target=None, keep_aspect_ratio=True, ensure_multiple_of=32,
    resize_method="upper_bound").get_size(width, height), as midas/transforms.py computes it."""
    def constrain(x, max_val):
        y = (np.round(x / 32) * 32).astype(int)
        if max_val is not None and y > max_val:
            y = (np.floor(x / 32) * 32).astype(int)
        if y < 0:
            y = (np.ceil(x / 32) * 32).astype(int)
        return y
    scale_height, scale_width = 384 / height, 384 / width
    if scale_width < scale_height:
        scale_height = scale_width
    else:
        scale_width = scale_height
    return int(constrain(scale_width * width, 384)), int(constrain(scale_height * height, 384))


def transform(rgb):
    """read_image's / 255 and the Resize / NormalizeImage / PrepareForNet transform of a uint8 RGB frame [h][w][3], on
    the host in float64 -> the float32 network input [3][H][W]."""
    import cv2
    img = rgb / 255.0
    width, height = get_size(img.shape[1], img.shape[0])
    img = cv2.resize(img, (width, height), interpolation=cv2.INTER_CUBIC)
    img = (img - MEAN) / STD
    return np.ascontiguousarray(np.transpose(img, (2, 0, 1))).astype(np.float32)


def predict(weights, rgb, optimize):
    """One reference call: transform, the batch-1 forward (fp16 channels_last when optimize, with weights from
    midas.network_weights(..., optimize)), bicubic to the frame size -> the prediction [h][w] as numpy (float16 when
    optimize, as .cpu().numpy() gives it)."""
    import torch
    dev = next(iter(weights.values())).device
    with torch.no_grad():
        sample = torch.from_numpy(transform(rgb)).to(dev).unsqueeze(0)
        if optimize:
            sample = sample.to(memory_format=torch.channels_last).half()
        prediction = midas.forward(weights, sample)
        prediction = torch.nn.functional.interpolate(prediction.unsqueeze(1), size=rgb.shape[:2], mode="bicubic",
                                                     align_corners=False).squeeze().cpu().numpy()
    return prediction


def pixels(depth_map):
    """write_depth(bits=2)'s PNG pixels from the float32 map: float32 arithmetic, truncated to uint16; zeros when
    max - min is not above float64 eps."""
    depth = np.asarray(depth_map, np.float32)
    lo, hi = depth.min(), depth.max()
    if hi - lo > np.finfo("float").eps:
        return (65535 * (depth - lo) / (hi - lo)).astype("uint16")
    return np.zeros(depth.shape, np.uint16)


def reference_fp16_pixels(prediction):
    """What the reference's write_depth computes for a float16 prediction: 65535 * the float16 array stays float16
    under numpy's promotion and overflows, so the map becomes inf / NaN before the uint16 cast."""
    import warnings
    depth = np.asarray(prediction, np.float16)
    lo, hi = depth.min(), depth.max()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        return (65535 * (depth - lo) / (hi - lo)).astype("uint16")


def depth_maps(weights, frames, optimize):
    """run_midas on a list of uint8 RGB frames -> (maps [n][h][w] float32 (the PFM values), pixels [n][h][w] uint16)."""
    maps = np.stack([predict(weights, f, optimize).astype(np.float32) for f in frames])
    return maps, np.stack([pixels(m) for m in maps])


def run_directory(weights, image_dir, output_dir, optimize):
    """run_midas's loop over a directory, writing NAME.pfm and NAME.png per frame as it does (the pixels as pixels()
    computes them)."""
    import cv2
    os.makedirs(output_dir, exist_ok=True)
    for p in sorted(os.listdir(image_dir)):
        rgb = cv2.cvtColor(cv2.imread(os.path.join(image_dir, p)), cv2.COLOR_BGR2RGB)
        depth = predict(weights, rgb, optimize).astype(np.float32)
        base = midas.output_base(output_dir, p)
        with open(base + ".pfm", "wb") as f:
            f.write(midas.pfm_bytes(np.flipud(depth)))
        cv2.imwrite(base + ".png", pixels(depth))
