"""Times the depth step (particlesfm_b200.midas.write_depth_maps: batched network, device transform, upsampling and
quantisation, files written on a writer thread) against the reference's per-frame structure writing the same files
(oracle/midas_oracle.py:run_directory: cv2.resize on the host, a batch-1 forward, torch's bicubic, the PNG arithmetic
on the host), alternated in one process, on 50 seeded frames of 1024 x 436 (network input 384 x 160) with seeded
weights, both with optimize (fp16 channels_last) and torch's defaults.  Prints min / median / max of the runs after a
warm-up, the network's share of the step (CUDA events around the forward calls), and the card's name and power limit.

    python tools/bench_depth.py [--reps 3] [--frames 50] [--fp32]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=3)
    p.add_argument("--frames", type=int, default=50)
    p.add_argument("--fp32", action="store_true", help="optimize=False on both routes")
    a = p.parse_args()
    import cv2
    import numpy as np
    import torch
    from oracle import midas_oracle as mo
    from particlesfm_b200 import midas
    optimize = not a.fp32
    h, w = 436, 1024
    with tempfile.TemporaryDirectory() as tmp:
        d = os.path.join(tmp, "img")
        os.makedirs(d)
        for i, f in enumerate(mo.seeded_frames(a.frames, h, w, seed=1)):
            cv2.imwrite(os.path.join(d, "%05d.png" % i), f[:, :, ::-1])
        sd = mo.seeded_state_dict(0)
        wpath = os.path.join(tmp, "midas_v21.pt")
        torch.save(sd, wpath)
        weights = midas.network_weights(midas.check_state_dict(sd, "seeded"), "cuda", optimize)
        paths, _, _ = midas.frame_list(d)

        def step(out):
            bases = [midas.output_base(out, q) for q in paths]
            os.makedirs(out, exist_ok=True)
            with midas.DepthWriter(bases) as writer:
                return midas._run(paths, h, w, midas.load_weights(wpath), optimize, writer)

        step(os.path.join(tmp, "warm_step"))                    # module load, cuDNN heuristics
        mo.run_directory(weights, d, os.path.join(tmp, "warm_oracle"), optimize)
        stage, oracle, net = [], [], []
        for r in range(a.reps):
            t, n = timed(lambda: step(os.path.join(tmp, "step%d" % r)))
            stage.append(t)
            net.append(n)
            t, _ = timed(lambda: mo.run_directory(weights, d, os.path.join(tmp, "oracle%d" % r), optimize))
            oracle.append(t)
        a0 = [cv2.imread(os.path.join(tmp, "step0", "%05d.png" % i), -1).astype(np.int64) for i in range(a.frames)]
        b0 = [cv2.imread(os.path.join(tmp, "oracle0", "%05d.png" % i), -1).astype(np.int64) for i in range(a.frames)]
        dpx = max(int(np.abs(x - y).max()) for x, y in zip(a0, b0))
        s, o = sorted(stage), sorted(oracle)
        share = [n / t for n, t in zip(net, stage)]
        print(json.dumps({"frames": a.frames, "h": h, "w": w, "net": list(midas.get_size(w, h)), "optimize": optimize,
                          "frames_per_batch": midas.frames_per_batch(*midas.get_size(w, h)[::-1], optimize),
                          "card": card(), "step_s": [s[0], s[len(s) // 2], s[-1]],
                          "oracle_s": [o[0], o[len(o) // 2], o[-1]],
                          "network_share": [min(share), sorted(share)[len(share) // 2], max(share)],
                          "max_png_difference": dpx}), flush=True)


if __name__ == "__main__":
    main()
