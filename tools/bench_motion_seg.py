"""Times the trajectory labeller (particlesfm_b200.motion_seg) phase by phase on a synthetic DAVIS-shaped clip: 80
frames of 854 x 480, a seeded track set whose every window holds more trajectories than the default cap of 100,000,
seeded depth pixels and frames, seeded weights.  Phases: sampling (psfm_seg_hits + psfm_seg_windows), depth
(psfm_seg_depth_resize), encoder (psfm_seg_encode, every window in one launch), OANet (torch, per window), merge
(psfm_seg_merge and the output arrays), drawing (psfm_seg_draw, every window), track.npy (the dict and np.save on the
host), video (mp4v encoding of every frame) and end to end (label_trajectories with the video sink, then track.npy).
In the same run, alternated with the fused encoder: the encoder as torch's nn.Transformer on the device over all
rows at once (the same weights), and the reference's structure (the oracle's per-window features and nn.Transformer
on the device, one window after another).  Prints min / median / max over the repetitions after a warm-up, with the
card's name and power limit.

    python tools/bench_motion_seg.py [--reps 5] [--trajs 120000] [--frames 80]
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


def track_arrays(num_trajs, num_frames, h, w, seed):
    """Seeded trajectories: each starts at a random frame and runs 3 .. 40 frames, every frame seen."""
    from particlesfm_b200.tracker import TrackArrays
    rng = np.random.default_rng(seed)
    start = rng.integers(0, num_frames - 3, num_trajs)
    lens = np.minimum(rng.integers(3, 41, num_trajs), num_frames - start)
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    owner = np.repeat(np.arange(num_trajs), lens)
    step = np.arange(ptr[-1]) - ptr[:-1][owner]
    frames = (start[owner] + step).astype(np.int32)
    p0 = rng.uniform([0, 0], [w - 1, h - 1], (num_trajs, 2))
    v = rng.normal(0, 2, (num_trajs, 2))
    xy = np.clip(p0[owner] + v[owner] * step[:, None], 0, [w - 1, h - 1]).astype(np.float64)
    return TrackArrays(np.arange(num_trajs, dtype=np.int64), ptr, frames, xy)


def stats(xs):
    xs = sorted(xs)
    return {"min_ms": 1e3 * xs[0], "median_ms": 1e3 * xs[len(xs) // 2], "max_ms": 1e3 * xs[-1]}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--trajs", type=int, default=600000)
    p.add_argument("--frames", type=int, default=80)
    a = p.parse_args()
    import torch
    import oracle.motion_seg_oracle as O
    from particlesfm_b200 import motion_seg as ms
    h, w, n, window, cap = 480, 854, a.frames, 10, 100000
    tracks = track_arrays(a.trajs, n, h, w, seed=1)
    weights = ms.check_state_dict({"model_state_dict": O.seeded_state_dict(4)}, "seeded")
    sd = {k: v.cuda() for k, v in weights.items()}
    packed = torch.from_numpy(ms.pack_encoder(weights)).cuda()
    pixels = torch.from_numpy(np.random.default_rng(2).integers(0, 65535, (n, h, w), dtype=np.uint16)).cuda()
    frames = torch.from_numpy(np.random.default_rng(3).integers(0, 256, (n, ms.H, ms.W, 3), dtype=np.uint8)).cuda()
    model = O.transformer(O.seeded_state_dict(4)).cuda()
    ids, ptr, fr, xy = ms._sorted_csr(tracks)
    d_ptr, d_fr, d_xy = (torch.from_numpy(x).cuda() for x in (ptr, fr, np.ascontiguousarray(xy)))
    times = {k: [] for k in ("sampling", "depth", "encoder", "encoder_nn_transformer", "encoder_reference_structure",
                             "oanet", "merge", "drawing", "track_npy", "video", "end_to_end")}
    tmp = tempfile.mkdtemp()

    def torch_encoder(win, maps):
        kinv = torch.from_numpy(ms.camera_inverse()).cuda()
        nor = win.loc.clone()
        nor[..., 0] = (nor[..., 0] / (w / 424.0) / 424).clamp(0, 1)
        nor[..., 1] = (nor[..., 1] / (h / 240.0) / 240).clamp(0, 1)
        t = nor.float()
        f0 = win.starts[win.row_window.long()].long()
        idx = ((t[..., 1] * 240).int() * 424 + (t[..., 0] * 424).int()).long().clamp(0, 240 * 424 - 1)
        frame = f0[:, None] + torch.arange(win.L, device="cuda")[None]
        d = maps.reshape(n, -1)[frame, idx]
        grid = torch.stack([(idx % 424).float(), (idx // 424).float(), torch.ones_like(d)], -1)
        xyz = d[..., None] * torch.einsum("ij,klj->kli", kinv, grid)
        m = win.valid.float()
        m2, m3 = torch.zeros_like(t), torch.zeros_like(xyz)
        m2[:, :-1] = (t[:, 1:] - t[:, :-1]) * m[:, 1:, None]
        m3[:, :-1] = (xyz[:, 1:] - xyz[:, :-1]) * m[:, 1:, None]
        f = torch.cat([t, m2, xyz, m3], -1)
        x = torch.relu(f @ sd["joint_encoder.input_fc1.weight"].reshape(16, 10).t() + sd["joint_encoder.input_fc1.bias"])
        x = torch.relu(x @ sd["joint_encoder.fc2.weight"].reshape(16, 16).t() + sd["joint_encoder.fc2.bias"])
        x = x.permute(1, 0, 2)
        pad = win.valid == 0
        with torch.no_grad():
            return model(x, x, src_key_padding_mask=pad, tgt_key_padding_mask=pad).max(0)[0]

    def reference_structure(win, maps):
        out = []
        for wi in range(win.starts.shape[0]):
            a_, b_ = int(win.bounds[wi]), int(win.bounds[wi + 1])
            sub = ms.Windows()
            sub.L, sub.starts, sub.bounds = win.L, win.starts[wi:wi + 1], None
            sub.row_window = torch.zeros(b_ - a_, dtype=torch.int32, device="cuda")
            sub.loc, sub.valid = win.loc[a_:b_], win.valid[a_:b_]
            out.append(torch_encoder(sub, maps))
        return out

    feat_err = None
    for rep in range(a.reps + 1):
        t, win = timed(lambda: ms.sample_windows(d_ptr, d_fr, d_xy, n, window, cap))
        times["sampling"].append(t)
        t, maps = timed(lambda: ms.depth_resize(pixels))
        times["depth"].append(t)
        t, feat = timed(lambda: ms.encode(win, maps, (h, w), packed))
        times["encoder"].append(t)
        t, ref = timed(lambda: torch_encoder(win, maps))
        times["encoder_nn_transformer"].append(t)
        feat_err = float((feat - ref).abs().max())
        t, _ = timed(lambda: reference_structure(win, maps))
        times["encoder_reference_structure"].append(t)

        def oanet():
            pred = torch.zeros(win.rows.shape[0], dtype=torch.bool, device="cuda")
            with torch.no_grad():
                for wi in range(win.starts.shape[0]):
                    a_, b_ = int(win.bounds[wi]), int(win.bounds[wi + 1])
                    pred[a_:b_] = torch.sigmoid(ms.oanet_logits(sd, feat[a_:b_])) > 0.5
            return pred
        t, pred = timed(oanet)
        times["oanet"].append(t)
        t, _ = timed(lambda: ms.merge(d_ptr, d_fr, win, pred))
        times["merge"].append(t)
        rs = np.random.RandomState(0)
        drawn = []

        def draw():
            for wi in range(win.starts.shape[0]):
                a_, b_ = int(win.bounds[wi]), int(win.bounds[wi + 1])
                s0 = int(win.starts[wi])
                draws = [rs.randint(b_ - a_) for _ in range(ms.RANDOM_DRAWS)]
                drawn.append(ms.draw_window(frames[s0:s0 + win.L], win.loc[a_:b_], win.valid[a_:b_], pred[a_:b_],
                                            (h, w), draws))
        t, _ = timed(draw)
        times["drawing"].append(t)
        t, out = timed(lambda: ms.label_trajectories(tracks, pixels, (h, w), weights, window, cap))
        t0 = time.perf_counter()
        np.save(os.path.join(tmp, "track.npy"), ms.labelled_dict(out))
        times["track_npy"].append(time.perf_counter() - t0)
        host = [d.cpu().numpy() for d in drawn]
        t0 = time.perf_counter()
        vw = ms.VideoWriter(os.path.join(tmp, "motion_seg.mp4"))
        for d in host:
            vw.write(None, torch.from_numpy(d))
        vw.join()
        times["video"].append(time.perf_counter() - t0)

        def end_to_end():
            with ms.VideoWriter(os.path.join(tmp, "e2e.mp4")) as video:
                o = ms.label_trajectories(tracks, pixels, (h, w), weights, window, cap, video, frames)
            np.save(os.path.join(tmp, "e2e.npy"), ms.labelled_dict(o))
            return o
        t, out = timed(end_to_end)
        times["end_to_end"].append(t)
        if rep == 0:                                            # warm-up
            for v in times.values():
                v.clear()
    rows = int(win.rows.shape[0])
    print(json.dumps({"card": card(), "frames": n, "size": [w, h], "trajectories": a.trajs, "window": window,
                      "cap": cap, "windows": int(win.starts.shape[0]), "rows": rows,
                      "observations_out": int(out.frame_ids.shape[0]),
                      "fused_vs_nn_transformer_max_abs": feat_err,
                      "phases": {k: stats(v) for k, v in times.items()}}, indent=1))


if __name__ == "__main__":
    main()
