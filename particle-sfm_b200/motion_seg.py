"""The trajectory labeller on the GPU: track.npy and the depth maps in, every observation marked static or dynamic
out (DESIGN.md §4.17).

    python -m particlesfm_b200.motion_seg --image_dir I --depth_dir D --traj_dir T [--output_traj_dir O]
        --model checkpoint.pth [--window_size 10] [--traj_max_num 100000] [--skip_exists]

Reference: motion_seg/main_motion_segmentation.py with load_cut_seq.py and the traj_oa_depth network (a transformer
over each trajectory's window, then OANet over the window's trajectories).  It writes O/track.npy, the sampled
observations with their labels, and O/motion_seg.mp4, draw_traj_cls's picture of every window; O defaults to T
followed by "_labeled".

The window sampler, the depth resize, the input channels with the whole transformer, the merge of the windows'
labels and the drawing are csrc/motion_seg.cu; OANet stays torch calls, one window at a time (its instance norms are
per window).
"""
import argparse
import ctypes
import glob
import os
import sys
from collections import OrderedDict

import numpy as np

from . import _lib
from ._stage import PinnedSink, Worker, check_keys, load_checkpoint, require_device, stream
from .tracker import TrackArrays

C_void = ctypes.c_void_p

H, W = 240, 424                 # example_test.yaml's resolution
MIN_HITS = 3                    # sample_inside_window's min_length
CLUSTERS = 100
CHANNELS = 128
RANDOM_DRAWS = 100              # draw_traj_cls's random trajectories per window
# draw_traj_cls's circles as (radius, thickness): labels, sampled points, random trajectories
CIRCLES = ((1, 2), (1, 1), (3, 4))
ENCODER_FLOATS = 15881          # the packed encoder (csrc/motion_seg.cu), camera included


# ----------------------------------------------------------------------------- weights

def state_shapes():
    """traj_oa_depth's state-dict keys and shapes: the projections and nn.Transformer under joint_encoder, OANBlock
    (net_channels 128, depth 8, 100 clusters) under decoder."""
    s = OrderedDict()

    def conv(p, o, i):
        s[p + ".weight"], s[p + ".bias"] = (o, i, 1, 1), (o,)

    def lin(p, o, i):
        s[p + ".weight"], s[p + ".bias"] = (o, i), (o,)

    def norm(p, c=16):
        s[p + ".weight"], s[p + ".bias"] = (c,), (c,)

    def bn(p, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            s["%s.%s" % (p, k)] = (c,)
        s[p + ".num_batches_tracked"] = ()

    def attn(p):
        s[p + ".in_proj_weight"], s[p + ".in_proj_bias"] = (48, 16), (48,)
        lin(p + ".out_proj", 16, 16)

    e = "joint_encoder."
    conv(e + "input_fc1", 16, 10)
    conv(e + "fc2", 16, 16)
    t = e + "transformer_model."
    for l in range(2):
        p = t + "encoder.layers.%d" % l
        attn(p + ".self_attn")
        lin(p + ".linear1", 64, 16)
        lin(p + ".linear2", 16, 64)
        norm(p + ".norm1")
        norm(p + ".norm2")
    norm(t + "encoder.norm")
    for l in range(2):
        p = t + "decoder.layers.%d" % l
        attn(p + ".self_attn")
        attn(p + ".multihead_attn")
        lin(p + ".linear1", 64, 16)
        lin(p + ".linear2", 16, 64)
        norm(p + ".norm1")
        norm(p + ".norm2")
        norm(p + ".norm3")
    norm(t + "decoder.norm")

    def pointcn(p, cin, cout):
        bn(p + ".conv.1", cin)
        conv(p + ".conv.3", cout, cin)
        bn(p + ".conv.5", cout)
        conv(p + ".conv.7", cout, cout)
        if cin != cout:
            conv(p + ".shot_cut", cout, cin)

    d = "decoder."
    conv(d + "conv1", CHANNELS, 16)
    for i in range(4):
        pointcn(d + "l1_1.%d" % i, CHANNELS, CHANNELS)
    bn(d + "down1.conv.1", CHANNELS)
    conv(d + "down1.conv.3", CLUSTERS, CHANNELS)
    for i in range(4):
        p = d + "l2.%d" % i
        bn(p + ".conv1.1", CHANNELS)
        conv(p + ".conv1.3", CHANNELS, CHANNELS)
        bn(p + ".conv2.0", CLUSTERS)
        conv(p + ".conv2.2", CLUSTERS, CLUSTERS)
        bn(p + ".conv3.2", CHANNELS)
        conv(p + ".conv3.4", CHANNELS, CHANNELS)
    bn(d + "up1.conv.1", CHANNELS)
    conv(d + "up1.conv.3", CLUSTERS, CHANNELS)
    pointcn(d + "l1_2.0", 2 * CHANNELS, CHANNELS)
    for i in range(1, 4):
        pointcn(d + "l1_2.%d" % i, CHANNELS, CHANNELS)
    conv(d + "output", 1, CHANNELS)
    return s


def check_state_dict(ckpt, what):
    """The network's float32 weights from a checkpoint's contents, its "model_state_dict" entry as the reference loads
    it.  ValueError naming the file: no such entry, an unexpected or missing key, or a wrong shape."""
    if not isinstance(ckpt, dict) or not isinstance(ckpt.get("model_state_dict"), dict):
        raise ValueError("%s: holds no \"model_state_dict\" entry" % what)
    sd = ckpt["model_state_dict"]
    shapes = state_shapes()
    check_keys(sd, shapes, what)
    return {k: sd[k].float() for k in shapes if not k.endswith("num_batches_tracked")}


def load_weights(path):
    return check_state_dict(load_checkpoint(path), path)


def camera_inverse():
    """traj_oa_depth.image_grid's K^-1 (fx = fy = (h + w) / 2, cx = w / 2, cy = h / 2) inverted in float64, then
    float32 [3][3]."""
    f = (H + W) / 2.0
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]])
    return np.linalg.inv(K).astype(np.float32)


def pack_encoder(sd):
    """The encoder's weights in csrc/motion_seg.cu's order, every matrix transposed to [in][out], then K^-1:
    float32 [ENCODER_FLOATS]."""
    parts = []

    def mat(k):
        v = sd[k].detach().cpu().float().numpy()
        parts.append(v.reshape(v.shape[0], -1).T.ravel())

    def vec(k):
        parts.append(sd[k].detach().cpu().float().numpy().ravel())

    def lin(p, w=".weight", b=".bias"):
        mat(p + w)
        vec(p + b)

    def attn(p):
        lin(p, ".in_proj_weight", ".in_proj_bias")
        lin(p + ".out_proj")

    def norm(p):
        vec(p + ".weight")
        vec(p + ".bias")

    lin("joint_encoder.input_fc1")
    lin("joint_encoder.fc2")
    t = "joint_encoder.transformer_model."
    for l in range(2):
        p = t + "encoder.layers.%d" % l
        attn(p + ".self_attn")
        lin(p + ".linear1")
        lin(p + ".linear2")
        norm(p + ".norm1")
        norm(p + ".norm2")
    norm(t + "encoder.norm")
    for l in range(2):
        p = t + "decoder.layers.%d" % l
        attn(p + ".self_attn")
        attn(p + ".multihead_attn")
        lin(p + ".linear1")
        lin(p + ".linear2")
        for n in (1, 2, 3):
            norm(p + ".norm%d" % n)
    norm(t + "decoder.norm")
    parts.append(camera_inverse().ravel())
    out = np.concatenate(parts).astype(np.float32)
    assert out.shape == (ENCODER_FLOATS,)
    return out


# ----------------------------------------------------------------------------- OANet

def _instance_norm(x):
    """InstanceNorm2d(eps=1e-3) over the window's trajectories; one trajectory normalises to 0."""
    import torch
    import torch.nn.functional as F
    return torch.zeros_like(x) if x.shape[2] == 1 else F.instance_norm(x, eps=1e-3)


def _bn(sd, p, x):
    import torch.nn.functional as F
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _conv(sd, p, x):
    import torch.nn.functional as F
    return F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"])


def _norm_relu(sd, p, x, instance=True):
    import torch
    return torch.relu(_bn(sd, p, _instance_norm(x) if instance else x))


def _pointcn(sd, p, x):
    y = _conv(sd, p + ".conv.3", _norm_relu(sd, p + ".conv.1", x))
    y = _conv(sd, p + ".conv.7", _norm_relu(sd, p + ".conv.5", y))
    return y + (_conv(sd, p + ".shot_cut", x) if p + ".shot_cut.weight" in sd else x)


def _oafilter(sd, p, x):
    out = _conv(sd, p + ".conv1.3", _norm_relu(sd, p + ".conv1.1", x)).transpose(1, 2)
    out = out + _conv(sd, p + ".conv2.2", _norm_relu(sd, p + ".conv2.0", out, instance=False))
    out = _conv(sd, p + ".conv3.4", _norm_relu(sd, p + ".conv3.2", out.transpose(1, 2)))
    return out + x


def oanet_logits(sd, feat):
    """OANBlock on one window's encoder features [K][16] (float32, on the network's device) -> the logits [K]."""
    import torch
    x = feat.t().reshape(1, 16, -1, 1)
    x1 = _conv(sd, "decoder.conv1", x)
    for i in range(4):
        x1 = _pointcn(sd, "decoder.l1_1.%d" % i, x1)
    embed = _conv(sd, "decoder.down1.conv.3", _norm_relu(sd, "decoder.down1.conv.1", x1))
    S = torch.softmax(embed, dim=2).squeeze(3)
    x2 = torch.matmul(x1.squeeze(3), S.transpose(1, 2)).unsqueeze(3)
    for i in range(4):
        x2 = _oafilter(sd, "decoder.l2.%d" % i, x2)
    embed = _conv(sd, "decoder.up1.conv.3", _norm_relu(sd, "decoder.up1.conv.1", x1))
    S = torch.softmax(embed, dim=1).squeeze(3)
    x_up = torch.matmul(x2.squeeze(3), S).unsqueeze(3)
    out = torch.cat([x1, x_up], dim=1)
    for i in range(4):
        out = _pointcn(sd, "decoder.l1_2.%d" % i, out)
    return _conv(sd, "decoder.output", out).reshape(-1)


# ----------------------------------------------------------------------------- windows and kernels

def window_starts(length, window):
    """load_cut_seq's windows -> (first frames, window length): [i w, (i + 1) w) for all but the last, which is
    [length - w, length); one window [0, length) when w >= length."""
    if window >= length:
        return [0], length
    num = -(-length // window)
    return [i * window for i in range(num - 1)] + [length - window], window


def shuffle_permutation(k):
    """psfm_seg_shuffle: the permutation of 0 .. k-1 of the track set's fixed-seed shuffle."""
    perm = np.empty(k, dtype=np.int32)
    _lib.check(_lib.lib().psfm_seg_shuffle(k, perm.ctypes.data_as(C_void)), "psfm_seg_shuffle")
    return perm


def _p(t):
    return C_void(t.data_ptr())


def depth_resize(pixels):
    """psfm_seg_depth_resize: uint16 pixels [n][h][w] on the device -> float32 [n][240][424]."""
    import torch
    pixels = pixels.contiguous()
    n, h, w = pixels.shape
    out = torch.empty((n, H, W), dtype=torch.float32, device=pixels.device)
    _lib.check(_lib.lib().psfm_seg_depth_resize(_p(pixels), n, h, w, _p(out), stream()), "psfm_seg_depth_resize")
    return out


class Windows:
    """The sampled windows on the device.  starts [W] int32 and L: the windows; rows [R] int32 (trajectory index) and
    row_window [R] int32 in window order, each window's rows in its sampler's order; bounds [W + 1]: each window's
    rows; loc [R][L][2] float64 and valid [R][L] uint8."""


def sample_windows(ptr, frames, xy, num_frames, window_size, traj_max_num):
    """The window sampler (psfm_seg_hits, psfm_seg_windows) on the device CSR track set (trajectories in ascending id
    order, frames ascending)."""
    import torch
    dev = ptr.device
    T = ptr.shape[0] - 1
    starts, L = window_starts(num_frames, window_size)
    out = Windows()
    out.L = L
    out.starts = torch.tensor(starts, dtype=torch.int32, device=dev)
    hits = torch.empty((len(starts), T), dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().psfm_seg_hits(_p(ptr), _p(frames), T, _p(out.starts), len(starts), L, _p(hits), stream()),
               "psfm_seg_hits")
    sampled = hits >= MIN_HITS
    counts = sampled.sum(1).tolist()
    rows = []
    for w, k in enumerate(counts):
        idx = torch.nonzero(sampled[w]).reshape(-1).to(torch.int32)
        if k > traj_max_num:
            idx = idx[torch.from_numpy(shuffle_permutation(k)[:traj_max_num]).to(dev, torch.int64)]
        rows.append(idx)
    counts = [int(r.shape[0]) for r in rows]
    out.bounds = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    out.rows = torch.cat(rows)
    out.row_window = torch.repeat_interleave(torch.arange(len(starts), dtype=torch.int32, device=dev),
                                             torch.tensor(counts, device=dev))
    R = out.rows.shape[0]
    out.loc = torch.zeros((R, L, 2), dtype=torch.float64, device=dev)
    out.valid = torch.zeros((R, L), dtype=torch.uint8, device=dev)
    if R:
        _lib.check(_lib.lib().psfm_seg_windows(_p(ptr), _p(frames), _p(xy), _p(out.rows), _p(out.row_window), R,
                                               _p(out.starts), L, _p(out.loc), _p(out.valid), stream()),
                   "psfm_seg_windows")
    return out


def encode(win, depth, raw_hw, packed):
    """psfm_seg_encode: the encoder features [R][16] of every window row."""
    import torch
    R = win.rows.shape[0]
    feat = torch.empty((R, 16), dtype=torch.float32, device=depth.device)
    if R:
        _lib.check(_lib.lib().psfm_seg_encode(_p(win.loc), _p(win.valid), _p(win.row_window), _p(win.starts),
                                              win.starts.shape[0], R, win.L, _p(depth), depth.shape[0],
                                              int(raw_hw[0]), int(raw_hw[1]), _p(packed), _p(feat), stream()),
                   "psfm_seg_encode")
    return feat


def merge(ptr, frames, win, pred):
    """psfm_seg_merge -> (labels [M] int8 on the device, -1 for a dropped observation; first_row [T] int32)."""
    import torch
    dev = ptr.device
    T = ptr.shape[0] - 1
    Wn = win.starts.shape[0]
    row_of = torch.full((Wn, T), -1, dtype=torch.int32, device=dev)
    R = win.rows.shape[0]
    if R:
        row_of[win.row_window.long(), win.rows.long()] = torch.arange(R, dtype=torch.int32, device=dev)
    labels = torch.empty(frames.shape[0], dtype=torch.int8, device=dev)
    first = torch.empty(T, dtype=torch.int32, device=dev)
    pred = pred.to(torch.uint8).contiguous()
    if R == 0:
        pred = torch.zeros(1, dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib().psfm_seg_merge(_p(ptr), _p(frames), T, _p(win.starts), Wn, win.L, _p(row_of), _p(pred),
                                         _p(labels), _p(first), stream()), "psfm_seg_merge")
    return labels, first


_STAMPS = None


def circle_stamps():
    """The pixel offsets (dx, dy) cv2.circle paints for each of CIRCLES, taken once from a blank canvas -> (int16
    [n][2] of the three stamps one after another, their counts)."""
    global _STAMPS
    if _STAMPS is None:
        import cv2
        parts = []
        for r, t in CIRCLES:
            c = np.zeros((32, 32), np.uint8)
            cv2.circle(c, center=(16, 16), radius=r, color=255, thickness=t)
            ys, xs = np.nonzero(c)
            parts.append(np.stack([xs - 16, ys - 16], 1).astype(np.int16))
        _STAMPS = (np.ascontiguousarray(np.concatenate(parts)), [len(p) for p in parts])
    return _STAMPS


def draw_window(frames, loc, valid, pred, raw_hw, draws):
    """psfm_seg_draw: draw_traj_cls's video frames [L][960][424][3] (BGR) of one window from its resized BGR frames
    [L][240][424][3], its rows' loc [K][L][2], valid [K][L] and labels pred [K] (device), and the random draws."""
    import torch
    dev = frames.device
    L = frames.shape[0]
    K = loc.shape[0]
    stamps, (na, nb, nc) = circle_stamps()
    st = torch.from_numpy(stamps).to(dev)
    d = torch.from_numpy(np.asarray(draws, dtype=np.int32)).to(dev)
    order = torch.empty((L, 3, H, W), dtype=torch.int32, device=dev)
    out = torch.empty((L, 4 * H, W, 3), dtype=torch.uint8, device=dev)
    pred = pred.to(torch.uint8).contiguous()
    none = C_void(0)
    _lib.check(_lib.lib().psfm_seg_draw(_p(frames.contiguous()), _p(loc) if K else none, _p(valid) if K else none,
                                        _p(pred) if K else none, K, L, int(raw_hw[0]), int(raw_hw[1]),
                                        _p(d) if len(draws) else none, len(draws), _p(st), na, nb, nc, _p(order),
                                        _p(out), stream()), "psfm_seg_draw")
    return out


# ----------------------------------------------------------------------------- the stage

def check_window_length(num_frames, window_size):
    """ValueError when the windows of num_frames frames (one window of all of them when window_size >= num_frames) are
    longer than the fused encoder's per-row state fits in shared memory (psfm_seg_max_window, 435 frames)."""
    L = window_starts(num_frames, window_size)[1]
    longest = _lib.lib().psfm_seg_max_window()
    if L > longest:
        raise ValueError("--window_size: a window of %d frames is longer than the fused encoder takes (%d); give a "
                         "--window_size of at most %d" % (L, longest, longest))


def _sorted_csr(tracks):
    """tracks' arrays with the trajectories in ascending id order; ValueError when a trajectory's frames are not
    strictly ascending."""
    ids, ptr = np.asarray(tracks.ids, np.int64), np.asarray(tracks.ptr, np.int64)
    frames, xy = np.asarray(tracks.frame_ids, np.int32), np.asarray(tracks.xy, np.float64).reshape(-1, 2)
    lens = np.diff(ptr)
    starts = np.zeros(frames.shape[0], dtype=bool)
    starts[ptr[:-1][lens > 0]] = True
    if frames.shape[0] and np.any((np.diff(frames) <= 0) & ~starts[1:]):
        raise ValueError("track set: a trajectory's frames are not strictly ascending")
    order = np.argsort(ids, kind="stable")
    if np.array_equal(order, np.arange(ids.shape[0])):
        return ids, ptr, frames, xy
    new_lens = lens[order]
    new_ptr = np.concatenate([[0], np.cumsum(new_lens)]).astype(np.int64)
    # observation j of new trajectory k comes from old position ptr[order[k]] + j
    sel = np.repeat(ptr[:-1][order] - new_ptr[:-1], new_lens) + np.arange(new_ptr[-1])
    return ids[order], new_ptr, frames[sel], xy[sel]


def label_trajectories(tracks, depth, raw_hw, weights, window_size=10, traj_max_num=100000, video=None,
                       frames=None):
    """The labeller on a tracker.TrackArrays and the depth pixels (uint16 CUDA tensor [n][h][w], n the number of
    frames; or the maps depth_resize made of them, float32 [n][240][424]) for frames of raw_hw = (height, width), with
    the checked weights (load_weights).  Returns a TrackArrays of
    the sampled observations with their labels: keys in first-appearance order over the windows, frames ascending.
    With video (a sink called as video(None, frames [L][960][424][3] uint8 BGR on the device) per window) frames
    must hold the resized BGR frames [n][240][424][3] uint8 on the device."""
    import torch
    if window_size < 1 or traj_max_num < 1:
        raise ValueError("window_size and traj_max_num must be at least 1")
    n = int(depth.shape[0])
    starts, L = window_starts(n, window_size)
    check_window_length(n, window_size)
    ids, ptr, fr, xy = _sorted_csr(tracks)
    require_device("motion_seg")
    empty = TrackArrays(np.zeros(0, np.int64), np.zeros(1, np.int64), np.zeros(0, np.int32),
                        np.zeros((0, 2), np.float64), np.zeros(0, bool))
    dev = "cuda"
    sd = {k: v.to(dev) for k, v in weights.items()}
    packed = torch.from_numpy(pack_encoder(weights)).to(dev)
    if ids.shape[0] == 0:
        return empty
    d_ptr, d_fr = torch.from_numpy(ptr).to(dev), torch.from_numpy(fr).to(dev)
    d_xy = torch.from_numpy(np.ascontiguousarray(xy)).to(dev)
    win = sample_windows(d_ptr, d_fr, d_xy, n, window_size, traj_max_num)
    maps = depth if depth.dtype == torch.float32 else depth_resize(depth)
    feat = encode(win, maps, raw_hw, packed)
    pred = torch.zeros(win.rows.shape[0], dtype=torch.bool, device=dev)
    rs = np.random.RandomState(0)
    with torch.no_grad():
        for w in range(len(starts)):
            a, b = int(win.bounds[w]), int(win.bounds[w + 1])
            if b > a:
                pred[a:b] = torch.sigmoid(oanet_logits(sd, feat[a:b])) > 0.5
            if video is not None:
                draws = [rs.randint(b - a) for _ in range(RANDOM_DRAWS)] if b > a else []
                video(None, draw_window(frames[starts[w]:starts[w] + L], win.loc[a:b], win.valid[a:b], pred[a:b],
                                        raw_hw, draws))
    labels, first = merge(d_ptr, d_fr, win, pred)
    labels, first = labels.cpu().numpy(), first.cpu().numpy()
    keep_t = np.nonzero(first >= 0)[0]
    keep_t = keep_t[np.argsort(first[keep_t], kind="stable")]
    if keep_t.shape[0] == 0:
        return empty
    kept = labels >= 0
    owner = np.repeat(np.arange(ids.shape[0]), np.diff(ptr))
    rank = np.full(ids.shape[0], -1, dtype=np.int64)
    rank[keep_t] = np.arange(keep_t.shape[0])
    obs = np.nonzero(kept & (rank[owner] >= 0))[0]
    sel = obs[np.argsort(rank[owner[obs]], kind="stable")]
    out_ptr = np.concatenate([[0], np.cumsum(np.bincount(rank[owner[sel]], minlength=keep_t.shape[0]))])
    return TrackArrays(ids[keep_t], out_ptr, fr[sel], xy[sel], labels[sel] == 1)


def labelled_dict(tracks, int_keys=False):
    """The dict main_motion_segmentation saves: {id: {"locations" [n][2] float64, "labels" [n] bool, "frame_ids" [n]
    int64}} in the tracks' order; keys are numpy int64 as the windowed reference makes them, Python ints for its
    single window (int_keys)."""
    out = {}
    ptr = tracks.ptr.tolist()
    for k, i in enumerate(tracks.ids.tolist()):
        s, e = ptr[k], ptr[k + 1]
        out[i if int_keys else np.int64(i)] = {"locations": tracks.xy[s:e].copy(),
                                                "labels": tracks.labels[s:e].copy(),
                                                "frame_ids": tracks.frame_ids[s:e].astype(np.int64)}
    return out


def read_tracks(traj_dir):
    """traj_dir/track.npy as the sampler sees it (TrajectorySet.csr) -> TrackArrays; ValueError naming the file when
    it does not unpickle to a TrajectorySet."""
    from .point_trajectory import _particlesfm
    particlesfm = _particlesfm()
    path = os.path.join(traj_dir, "track.npy")
    try:
        obj = np.load(path, allow_pickle=True).item()
    except Exception as e:
        raise ValueError("%s: not a readable track.npy (%s)" % (path, e)) from None
    if not isinstance(obj, particlesfm.TrajectorySet):
        raise ValueError("%s: holds a %s, not a TrajectorySet" % (path, type(obj).__name__))
    ids, ptr, frames, xy = obj.csr()
    return TrackArrays(ids, ptr, frames, xy)


def frame_list(image_dir):
    """load_cut_seq's frames, every entry of image_dir sorted, each decoded once -> (paths, (h, w), the frames as
    draw_traj_cls paints on them [n][240][424][3] uint8 BGR); ValueError naming the file for an entry cv2 cannot read
    or frames of mixed sizes."""
    import cv2
    if not os.path.isdir(image_dir):
        raise ValueError("%s: not a directory" % image_dir)
    paths = [os.path.join(image_dir, f) for f in sorted(os.listdir(image_dir))]
    size, resized = None, []
    for p in paths:
        img = cv2.imread(p) if os.path.isfile(p) else None
        if img is None:
            raise ValueError("%s: not an image cv2 can read" % p)
        if size is None:
            size = img.shape[:2]
        elif img.shape[:2] != size:
            raise ValueError("%s: %d x %d, the sequence's frames are %d x %d"
                             % (p, img.shape[1], img.shape[0], size[1], size[0]))
        resized.append(cv2.resize(img, (W, H)))
    if not paths:
        raise ValueError("%s: no frames" % image_dir)
    return paths, size, np.stack(resized)


def depth_list(depth_dir, paths):
    """The depth PNGs paired with the frames -> uint16 [n][h][w]; ValueError naming the file when the PNG stems are not
    exactly the frame stems, or a PNG is not 16-bit single-channel, or the sizes differ."""
    import cv2
    pngs = sorted(glob.glob(os.path.join(depth_dir, "*.png")))
    stems = [os.path.splitext(os.path.basename(p))[0] for p in paths]
    dstems = [os.path.splitext(os.path.basename(p))[0] for p in pngs]
    if dstems != stems:
        bad = next((p for p, s in zip(pngs, dstems) if s not in set(stems)), None)
        raise ValueError("%s: the depth PNGs' names are not the frames' names (%d PNGs, %d frames)"
                         % (bad or depth_dir, len(pngs), len(paths)))
    maps = []
    for p in pngs:
        d = cv2.imread(p, -1)
        if d is None or d.dtype != np.uint16 or d.ndim != 2:
            raise ValueError("%s: not a 16-bit single-channel PNG" % p)
        if maps and d.shape != maps[0].shape:
            raise ValueError("%s: %d x %d, the other depth maps are %d x %d"
                             % (p, d.shape[1], d.shape[0], maps[0].shape[1], maps[0].shape[0]))
        maps.append(d)
    return np.stack(maps)


def resized_frame(path):
    """load_cut_seq's frame as draw_traj_cls paints on it: cv2.imread resized to 424 x 240 (INTER_LINEAR), BGR."""
    import cv2
    return cv2.resize(cv2.imread(path), (W, H))


class VideoWriter(PinnedSink):
    """A sink for label_trajectories' video frames: mp4v at 5 fps, written on the writer thread."""

    def __init__(self, path):
        self.path, self.writer = path, None
        super().__init__("psfm-motion-seg-video")

    def write(self, meta, frames):
        import cv2
        if self.writer is None:
            self.writer = cv2.VideoWriter(self.path, cv2.VideoWriter_fourcc(*"mp4v"), 5.0, (W, 4 * H))
        for f in frames.numpy():
            self.writer.write(f)

    def join(self):
        error = super().join()
        if self.writer is not None:
            self.writer.release()
        return error


def main_motion_segmentation(image_dir, depth_dir, traj_dir, output_traj_dir=None, model=None, window_size=10,
                             traj_max_num=100000, skip_exists=False):
    """The command: output_traj_dir/track.npy and motion_seg.mp4.  Bad input raises ValueError naming the file before
    any device work.  Returns the labelled TrackArrays, or None when skipped."""
    import torch
    if output_traj_dir is None:
        output_traj_dir = traj_dir + "_labeled"
    video_name = os.path.join(output_traj_dir, "motion_seg.mp4")
    if skip_exists and os.path.exists(video_name) and os.path.exists(output_traj_dir):
        return None
    if window_size < 1 or traj_max_num < 1:
        raise ValueError("--window_size and --traj_max_num must be at least 1")
    paths, raw_hw, resized = frame_list(image_dir)
    check_window_length(len(paths), window_size)
    pixels = depth_list(depth_dir, paths)
    tracks = read_tracks(traj_dir)
    if model is None:
        raise ValueError("no --model checkpoint given")
    weights = load_weights(model)
    require_device("motion_seg")
    os.makedirs(output_traj_dir, exist_ok=True)
    frames = torch.from_numpy(resized).cuda()
    with VideoWriter(video_name) as video, Worker("psfm-motion-seg-npy") as saver:
        out = label_trajectories(tracks, torch.from_numpy(pixels).cuda(), raw_hw,
                                 weights, window_size, traj_max_num, video, frames)
        single = window_size >= len(paths)
        saver.submit(np.save, os.path.join(output_traj_dir, "track.npy"), labelled_dict(out, single))
    return out


def main(argv=None):
    p = argparse.ArgumentParser("Label point trajectories static or dynamic (traj_oa_depth) on the GPU")
    p.add_argument("--image_dir", required=True, help="path to the image folder")
    p.add_argument("--depth_dir", required=True, help="path to the depth folder (midas_depth)")
    p.add_argument("--traj_dir", required=True, help="path to the input trajectory folder (holding track.npy)")
    p.add_argument("--output_traj_dir", default=None, help="output folder; default: TRAJ_DIR + '_labeled'")
    p.add_argument("--model", required=True, help="the traj_oa_depth checkpoint (model_state_dict)")
    p.add_argument("--window_size", type=int, default=10, help="sliding window size to load the data")
    p.add_argument("--traj_max_num", type=int, default=100000, help="the maximum number of trajectories per window")
    p.add_argument("--skip_exists", action="store_true", help="skip when the output video and folder exist")
    a = p.parse_args(argv)
    try:
        main_motion_segmentation(a.image_dir, a.depth_dir, a.traj_dir, a.output_traj_dir, a.model, a.window_size,
                                 a.traj_max_num, a.skip_exists)
    except ValueError as e:
        print("motion_seg: %s" % e, file=sys.stderr)
        return 2
    except (_lib.PsfmError, RuntimeError, OSError) as e:
        print("motion_seg: %s" % e, file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
