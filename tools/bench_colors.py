"""Time the colour extraction (particlesfm_b200.colors, csrc/colors.cu) at two sequence shapes (DESIGN.md §4.11).

    python tools/bench_colors.py [--repeat 3] [--json OUT]

  sintel  50 PNG frames of 1024 x 436, 12,000 keypoints per frame
  davis   80 JPEG frames of 854 x 480, 20,000 keypoints per frame
60 % of the keypoints have a point; a point is seen in 5 frames on average.  The frames are seeded noise over smooth
colour fields, written to a temporary directory.  Per shape, the median of the calls: decode (summed over the decoder
threads) and the wall time the batches waited for it, the pixels' copies into pinned memory, the uploads, the kernels
(CUDA events), the whole call, and the vectorised oracle on the host (decoding included), whose colours the device's
must equal.  The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"sintel": (50, 1024, 436, 12000, ".png"), "davis": (80, 854, 480, 20000, ".jpg")}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_shape(d, frames, w, h, per_frame, ext, seed=0):
    from PIL import Image
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    names = []
    for i in range(frames):
        f = np.stack([127 + 120 * np.sin(xx / (41.0 + i) + c) * np.cos(yy / 29.0 - c) for c in range(3)], -1)
        img = np.clip(f + rng.normal(0, 8, f.shape), 0, 255).astype(np.uint8)
        names.append("%05d%s" % (i, ext))
        Image.fromarray(img).save(os.path.join(d, names[-1]))
    K = frames * per_frame
    kp = np.stack([rng.uniform(0, w, K), rng.uniform(0, h, K)], 1)
    P = int(0.6 * K / 5)
    rows = np.where(rng.random(K) < 0.6, rng.integers(0, P, K), -1).astype(np.int32)
    ptr = np.arange(frames + 1, dtype=np.int64) * per_frame
    return names, ptr, kp, rows, P


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--json")
    args = ap.parse_args()
    from oracle import colors_oracle as co
    from particlesfm_b200 import colors, device_count
    if device_count() <= 0:
        raise SystemExit("bench_colors: no CUDA device")
    gpu = card()
    print("card:", gpu)
    results = []
    for shape, (frames, w, h, per_frame, ext) in SHAPES.items():
        with tempfile.TemporaryDirectory() as d:
            names, ptr, kp, rows, P = make_shape(d, frames, w, h, per_frame, ext)
            colors.extract_colors_for_all_images(d, names, ptr, kp, rows, P, verbose=False)      # warm-up
            runs = []
            for _ in range(args.repeat):
                t0 = time.perf_counter()
                rgb, rep = colors.extract_colors_for_all_images(d, names, ptr, kp, rows, P, verbose=False)
                runs.append((time.perf_counter() - t0, rep))
            t0 = time.perf_counter()
            ref = co.extract_colors([co.read_image(os.path.join(d, n)) for n in names], ptr, kp, rows, P)
            oracle_s = time.perf_counter() - t0
            assert np.array_equal(rgb, ref), "device colours differ from the oracle's"
            med = lambda f: float(np.median([f(r) for r in runs]))
            obs = int((rows >= 0).sum())
            row = dict(shape=shape, card=gpu, frames=frames, width=w, height=h, keypoints=int(ptr[-1]), observations=obs,
                       points=P, batches=runs[0][1].num_batches, call_ms=1e3 * med(lambda r: r[0]),
                       oracle_ms=1e3 * oracle_s,
                       **{k + "_ms": 1e3 * med(lambda r, k=k: r[1].seconds[k])
                          for k in ("open", "decode", "decode_wait", "setup", "stage", "upload", "sample", "mean")})
            # bytes the kernels must move: per observation 20 read (xy, image) + 16 written + 16 read back + 4 order,
            # 12 pixel bytes read; per pixel 3 uploaded
            row["kernel_bytes"] = obs * (20 + 16 + 16 + 4 + 12) + 7 * P
            print(json.dumps(row), flush=True)
            results.append(row)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
