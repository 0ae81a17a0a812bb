"""Times the optical-flow stage (particlesfm_b200.optical_flow.compute_optical_flows, flows kept on the device) against
the reference's per-call structure (oracle/raft_oracle.py: batch-1 calls per pair and direction, the volume per call,
grid_sample lookups, upsampling every iteration), alternated in one process, on seeded frames with seeded weights and
path consistency, at the Sintel shape (50 frames of 1024 x 436) and the DAVIS shape (80 frames of 854 x 480).  Both
run with torch's defaults (cuDNN TF32 convolutions, fp32 matmul).  Prints min / median / max per shape with the
card's name and power limit, and the largest flow difference between the two.

    python tools/bench_optical_flow.py [--reps 3] [--shapes sintel,davis] [--profile OUT_DIR]

--profile instead takes the per-kernel split of one stage run of 6 frames per shape with torch.profiler and writes
the table under OUT_DIR.
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

SHAPES = {"sintel": (50, 436, 1024), "davis": (80, 480, 854)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def setup(tmp, n, h, w):
    import torch
    from PIL import Image
    from oracle import raft_oracle as ro
    frames = ro.seeded_frames(n, h, w, seed=1)
    d = os.path.join(tmp, "img_%d_%d_%d" % (n, h, w))
    os.makedirs(d, exist_ok=True)
    for i, f in enumerate(frames):
        Image.fromarray(f).save(os.path.join(d, "%05d.png" % i))
    sd = ro.seeded_state_dict(0)
    weights = os.path.join(tmp, "w.pth")
    torch.save(sd, weights)
    return frames, d, weights, {k: v.cuda() for k, v in sd.items()}


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
    p.add_argument("--shapes", default="sintel,davis")
    p.add_argument("--profile", default=None)
    a = p.parse_args()
    import torch
    from oracle import raft_oracle as ro
    from particlesfm_b200 import optical_flow as of
    dev_name = card()
    with tempfile.TemporaryDirectory() as tmp:
        for name in a.shapes.split(","):
            n, h, w = SHAPES[name]
            if a.profile:
                frames, d, weights, sd = setup(tmp, 6, h, w)
                of.compute_optical_flows(d, weights)
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    timed(lambda: of.compute_optical_flows(d, weights))
                table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)
                os.makedirs(a.profile, exist_ok=True)
                with open(os.path.join(a.profile, "optical_flow_%s_profile.txt" % name), "w") as f:
                    f.write("%s\n%s\n" % (dev_name, table))
                print(table)
                continue
            frames, d, weights, sd = setup(tmp, n, h, w)
            of.compute_optical_flows(d, weights)          # warm-up: module load, cuDNN heuristics
            with torch.no_grad():
                ro.flow_pair(sd, frames[0], frames[1])
            stage, oracle, err = [], [], 0.0
            for _ in range(a.reps):
                t, got = timed(lambda: of.compute_optical_flows(d, weights))
                stage.append(t)
                with torch.no_grad():
                    t, ref = timed(lambda: ro.optical_flows(sd, frames))
                oracle.append(t)
                err = max(err, max((x - y).abs().max().item() for gl, rl in zip(got, ref) for x, y in zip(gl, rl)))
                del got, ref
            s, o = sorted(stage), sorted(oracle)
            print(json.dumps({"shape": name, "frames": n, "h": h, "w": w, "card": dev_name,
                              "stage_s": [s[0], s[len(s) // 2], s[-1]], "oracle_s": [o[0], o[len(o) // 2], o[-1]],
                              "max_flow_difference_px": err}), flush=True)


if __name__ == "__main__":
    main()
