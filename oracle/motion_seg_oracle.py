"""The trajectory labeller restated window by window on the host (numpy, cv2 and CPU torch), as load_cut_seq.py,
traj_oa_depth.py and main_motion_segmentation.py compute it, for the tests of particlesfm_b200.motion_seg.

The window sampler is the track set's own TrajectorySet.sample_inside_window; the encoder is torch's nn.Transformer
loaded with the checkpoint's weights; OANet is particlesfm_b200.motion_seg.oanet_logits on the CPU.
"""
import numpy as np

H, W = 240, 424


def seeded_state_dict(seed):
    """traj_oa_depth's state dict with seeded weights: kaiming-like scales, batch-norm statistics near 1."""
    import torch
    from particlesfm_b200 import motion_seg
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in motion_seg.state_shapes().items():
        if k.endswith("num_batches_tracked"):
            sd[k] = torch.tensor(0)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(shape, generator=g)
        elif k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:
            base = 1.0 if (".norm" in k or "conv." in k or "conv1.1" in k or "conv2.0" in k or "conv3.2" in k) \
                and k.endswith("weight") else 0.0
            sd[k] = base + 0.1 * torch.randn(shape, generator=g)
        else:
            fan_in = int(np.prod(shape[1:]))
            sd[k] = torch.randn(shape, generator=g) * (1.0 / np.sqrt(fan_in))
    return sd


def seeded_track_set(num_trajs, num_frames, h, w, seed):
    """A particlesfm.TrajectorySet of num_trajs trajectories over num_frames frames of h x w: each starts at a random
    frame, runs a random length and may skip a frame."""
    from particlesfm_b200.point_trajectory import _particlesfm
    particlesfm = _particlesfm()
    rng = np.random.default_rng(seed)
    d = {}
    for i in range(num_trajs):
        s = int(rng.integers(0, num_frames - 1))
        n = int(rng.integers(1, num_frames - s + 1))
        frames = [f for f in range(s, s + n) if rng.random() > 0.1] or [s]
        p0 = rng.uniform([0, 0], [w - 1, h - 1])
        v = rng.normal(0, 2, 2)
        locs = [[float(np.clip(p0[0] + v[0] * (f - s), 0, w - 1)), float(np.clip(p0[1] + v[1] * (f - s), 0, h - 1))]
                for f in frames]
        d[2 * i + 3] = {"frame_ids": frames, "locations": locs, "labels": [False] * len(frames)}
    return particlesfm.TrajectorySet(d)


def seeded_depth_pixels(num_frames, h, w, seed):
    """uint16 depth pixels [n][h][w]: smooth ramps with noise, the full 16-bit range."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    out = []
    for _ in range(num_frames):
        a, b = rng.uniform(-1, 1, 2)
        base = (a * xx / w + b * yy / h + 2) / 4
        out.append(np.clip((base + rng.normal(0, 0.05, (h, w))) * 65535, 0, 65535).astype(np.uint16))
    return np.stack(out)


def seeded_frames(num_frames, h, w, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 256, (num_frames, h, w, 3), dtype=np.uint8)


def windows(length, window):
    """load_cut_seq's window frame lists."""
    if window >= length:
        return [list(range(length))]
    num = int(np.ceil(1.0 * length / window))
    return [list(range(i * window, (i + 1) * window)) if i != num - 1 else list(range(length - window, length))
            for i in range(num)]


def depth_map(pixels):
    """cv2.imread(png, -1) / 65535.0 resized to 240 x 424 in float64, then float32."""
    import cv2
    return cv2.resize(pixels / 65535.0, (W, H)).astype(np.float32)


def transformer(sd):
    """nn.Transformer(d_model 16, 4 heads, 2 + 2 layers, FFN 64) loaded with the checkpoint's weights, in eval."""
    import torch
    m = torch.nn.Transformer(d_model=16, nhead=4, num_encoder_layers=2, num_decoder_layers=2, dim_feedforward=64,
                             dropout=0.1, activation="relu")
    pre = "joint_encoder.transformer_model."
    m.load_state_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
    return m.eval()


def features(sd, depth, traj, valid):
    """augment_traj and the two projections: depth [L][240][424] float32, traj [K][L][2] normalised float32, valid
    [K][L] -> (the 10 channels [K][L][10], the projected input [K][L][16])."""
    import torch
    import torch.nn.functional as F
    from particlesfm_b200 import motion_seg
    kinv = torch.from_numpy(motion_seg.camera_inverse())
    K, L = valid.shape
    t = torch.from_numpy(traj)
    idx = ((t[..., 1] * H).to(torch.int) * W + (t[..., 0] * W).to(torch.int)).to(torch.int64).clamp(0, H * W - 1)
    u, v = (idx % W).float(), (idx // W).float()
    grid = torch.stack([u, v, torch.ones_like(u)], -1)                      # [K][L][3]
    d = torch.from_numpy(depth).reshape(L, -1)
    dv = torch.stack([d[j][idx[:, j]] for j in range(L)], 1)                 # [K][L]
    xyz = dv[..., None] * torch.einsum("ij,klj->kli", kinv, grid)
    m = torch.from_numpy(valid.astype(np.float32))
    m2 = torch.zeros_like(t)
    m2[:, :-1] = (t[:, 1:] - t[:, :-1]) * m[:, 1:, None]
    m3 = torch.zeros_like(xyz)
    m3[:, :-1] = (xyz[:, 1:] - xyz[:, :-1]) * m[:, 1:, None]
    f = torch.cat([t, m2, xyz, m3], -1)
    x = F.relu(f @ sd["joint_encoder.input_fc1.weight"].reshape(16, 10).t() + sd["joint_encoder.input_fc1.bias"])
    x = F.relu(x @ sd["joint_encoder.fc2.weight"].reshape(16, 16).t() + sd["joint_encoder.fc2.bias"])
    return f, x, idx


def encode(model, proj, valid):
    """pt_transformer.extract_feature: [K][L][16] -> the max over time of the transformer's output [K][16]."""
    import torch
    x = proj.permute(1, 0, 2)                                                # [L][K][16]
    pad = torch.from_numpy(valid == 0)
    with torch.no_grad():
        out = model(x, x, src_key_padding_mask=pad, tgt_key_padding_mask=pad)
    return out.max(0)[0]


def label(image_size, pixels, tracks, sd, window_size, traj_max_num, frames=None):
    """The stage on the host: (the labelled dict as main_motion_segmentation saves it, per window (features [K][16],
    logits [K], the sampled trajectory ids [K]), the video frames [n][960][424][3] BGR when frames [n][h][w][3] RGB are given)."""
    import cv2
    import torch
    from particlesfm_b200 import motion_seg
    h, w = image_size
    sdf = {k: v.float() for k, v in sd.items() if not k.endswith("num_batches_tracked")}
    model = transformer(sd)
    tracks.build_invert_indexes()
    n = pixels.shape[0]
    depths = np.stack([depth_map(p) for p in pixels])
    rs = np.random.RandomState(0)
    out, win_out, video = {}, [], []
    single = window_size >= n
    for idx in windows(n, window_size):
        s = tracks.sample_inside_window(idx, 3, traj_max_num)
        raw = np.stack([s["locations"][0], s["locations"][1]], -1)
        valid = s["masks"].astype(np.uint8)
        nor = raw.copy()
        nor[..., 0] /= float(w) / float(W)
        nor[..., 1] /= float(h) / float(H)
        nor[..., 0] /= W
        nor[..., 1] /= H
        nor = np.clip(nor, 0.0, 1.0)
        K = nor.shape[0]
        if K:
            _, proj, _ = features(sdf, depths[idx], nor.astype(np.float32), valid)
            feat = encode(model, proj, valid)
            with torch.no_grad():
                logits = motion_seg.oanet_logits(sdf, feat)
            pred = (torch.sigmoid(logits) > 0.5).numpy()
            win_out.append((feat.numpy(), logits.numpy(), list(s["traj_ids"])))
        else:
            pred = np.zeros(0, bool)
            win_out.append((np.zeros((0, 16), np.float32), np.zeros(0, np.float32), []))
        if frames is not None:
            imgs = [cv2.resize(frames[f], (W, H))[:, :, ::-1].copy() for f in idx]
            rows = [[i.copy() for i in imgs] for _ in range(3)]
            for i in range(K):
                for j in range(len(idx)):
                    if valid[i, j]:
                        c = (int(nor[i, j, 0] * W), int(nor[i, j, 1] * H))
                        cv2.circle(rows[0][j], c, 1, motion_seg_colors()[int(pred[i])], 2)
                        cv2.circle(rows[1][j], c, 1, motion_seg_colors()[0], 1)
            for _ in range(100 if K else 0):
                i = rs.randint(K)
                for j in range(len(idx)):
                    if valid[i, j]:
                        c = (int(nor[i, j, 0] * W), int(nor[i, j, 1] * H))
                        cv2.circle(rows[2][j], c, 3, motion_seg_colors()[i % 6], 4)
            for j in range(len(idx)):
                video.append(np.concatenate([imgs[j], rows[0][j], rows[1][j], rows[2][j]], 0))
        keys = s["traj_ids"] if single else np.array(s["traj_ids"])
        time = np.array(idx)
        for i in range(K):
            m = valid[i] == 1
            key = keys[i]
            vt, vl, vtime = raw[i][m], np.full(int(m.sum()), pred[i]), time[m]
            if key not in out:
                out[key] = {"locations": vt.copy(), "labels": vl.copy(), "frame_ids": vtime}
            else:
                new = np.array([t not in out[key]["frame_ids"] for t in vtime], dtype=bool)
                o = out[key]
                o["locations"] = np.concatenate([o["locations"], vt[new]], 0)
                o["labels"] = np.concatenate([o["labels"], vl[new]], 0)
                o["frame_ids"] = np.concatenate([o["frame_ids"], vtime[new]], 0)
    return out, win_out, video


def motion_seg_colors():
    """draw_traj_cls's colour bank."""
    return [(255, 0, 0), (0, 255, 0), (0, 0, 255), (255, 255, 0), (255, 0, 255), (0, 255, 255)]


def deciding_logits(out, wins, window_size, num_frames):
    """For every observation of the labelled dict, in its order, the logit of the window row that decided its label
    (the first window that sampled the trajectory and holds the frame)."""
    seen = {}
    for (_, logits, ids), idx in zip(wins, windows(num_frames, window_size)):
        for k, l in zip(ids, logits):
            for f in idx:
                seen.setdefault((int(k), f), float(l))
    return np.concatenate([[seen[(int(k), int(f))] for f in out[k]["frame_ids"]] for k in out]) if out else np.zeros(0)
