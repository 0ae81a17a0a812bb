"""RAFT optical flow restated with the reference's call structure (TEST INFRASTRUCTURE, DESIGN.md §4.14).

third_party/RAFT/compute_raft_custom_folder.py (and _stride2) call the model once per pair and direction with batch 1:
each call encodes both frames, builds its own all-pairs volume (core/corr.py: torch.matmul / 16, avg_pool2d pyramid),
looks it up with grid_sample (bilinear_sampler, align_corners=True, zero padding) and upsamples the flow after every
one of the 32 iterations, returning the last.  This module keeps that structure on purpose, so the product's batched
schedule, its shared product of both directions, the lookup, the once-only upsampling and the flow image
(csrc/optical_flow.cu) are checked against it.  The convolution blocks are particlesfm_b200.optical_flow's (the same
torch calls in either structure); tests/golden/flow_small.npz pins them and this module to the reference's own RAFT.

seeded_state_dict(seed) draws reference-keyed weights, so tests and the golden share weights without a checkpoint.
"""
import numpy as np

from particlesfm_b200 import optical_flow as of

# scale of the flow head's last layer: with fan-in weights alone the update steps leave the 1/8 grid within a few
# iterations and the lookups read zeros; at 0.05 most (87 %) stay inside the volume (make_flow_golden.py)
FLOW_HEAD_SCALE = 0.05


def seeded_state_dict(seed=0, flow_head_scale=FLOW_HEAD_SCALE):
    """Weights of every key of the basic model (without `module.`), drawn from numpy.random.default_rng(seed) per
    sorted key: convolution weights N(0, 1 / fan_in), biases N(0, 0.01^2), batch-norm weight 1 + N(0, 0.1^2), bias and
    running mean N(0, 0.1^2), running variance U(0.5, 1.5)."""
    import torch
    rng = np.random.default_rng(seed)
    out = {}
    for k, shape in sorted(of.state_shapes().items()):
        if k.endswith("num_batches_tracked"):
            out[k] = torch.tensor(0, dtype=torch.int64)
            continue
        if len(shape) == 4:
            v = rng.standard_normal(shape) / np.sqrt(np.prod(shape[1:]))
            if k == "update_block.flow_head.conv2.weight":
                v = v * flow_head_scale
        elif k.endswith(".running_var"):
            v = rng.uniform(0.5, 1.5, shape)
        elif k.endswith(".bias") and ".norm" not in k and ".downsample.1" not in k:
            v = 0.01 * rng.standard_normal(shape)
        elif k.endswith(".weight"):
            v = 1.0 + 0.1 * rng.standard_normal(shape)
        else:
            v = 0.1 * rng.standard_normal(shape)
        out[k] = torch.tensor(v, dtype=torch.float32)
    # norm3 and downsample.1 are one module in the reference, listed under both names
    for k in list(out):
        if ".downsample.1." in k:
            out[k] = out[k.replace(".downsample.1.", ".norm3.")].clone()
    return out


def seeded_frames(n, h, w, seed=0):
    """n smooth seeded uint8 RGB frames [h][w][3] of a texture drifting by about a pixel per frame."""
    rng = np.random.default_rng(seed)
    base = rng.uniform(0, 255, (h // 4 + 8, w // 4 + 8, 3))
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    frames = []
    for t in range(n):
        fy, fx = (yy + 0.7 * t) / 4.0 + 2, (xx + 1.3 * t) / 4.0 + 2
        y0, x0 = np.floor(fy).astype(int), np.floor(fx).astype(int)
        a, b = (fy - y0)[..., None], (fx - x0)[..., None]
        y1, x1 = (y0 + 1) % base.shape[0], (x0 + 1) % base.shape[1]     # the texture wraps on long clips
        y0, x0 = y0 % base.shape[0], x0 % base.shape[1]
        v = ((1 - a) * (1 - b) * base[y0, x0] + (1 - a) * b * base[y0, x1] + a * (1 - b) * base[y1, x0]
             + a * b * base[y1, x1])
        frames.append(np.clip(v + rng.normal(0, 4, v.shape), 0, 255).astype(np.uint8))
    return frames


def corr_pyramid(fmap1, fmap2):
    """CorrBlock.__init__ for batch 1: [h w][1][h_l][w_l] per level."""
    import torch
    import torch.nn.functional as F
    _, dim, h, w = fmap1.shape
    corr = torch.matmul(fmap1.view(1, dim, h * w).transpose(1, 2), fmap2.view(1, dim, h * w))
    corr = (corr.view(1, h, w, 1, h, w) / torch.sqrt(torch.tensor(dim).float())).reshape(h * w, 1, h, w)
    pyr = [corr]
    for _ in range(3):
        corr = F.avg_pool2d(corr, 2, stride=2)
        pyr.append(corr)
    return pyr


def lookup(pyr, coords, radius=4):
    """CorrBlock.__call__: coords [B][2][h][w] -> [B][324][h][w] through grid_sample."""
    import torch
    import torch.nn.functional as F
    coords = coords.permute(0, 2, 3, 1)
    batch, h1, w1, _ = coords.shape
    out = []
    for i, corr in enumerate(pyr):
        d = torch.linspace(-radius, radius, 2 * radius + 1, device=coords.device)
        delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1)
        c = coords.reshape(batch * h1 * w1, 1, 1, 2) / 2 ** i + delta.view(1, 2 * radius + 1, 2 * radius + 1, 2)
        H, W = corr.shape[-2:]
        x, y = c.split([1, 1], dim=-1)
        grid = torch.cat([2 * x / (W - 1) - 1, 2 * y / (H - 1) - 1], dim=-1)
        out.append(F.grid_sample(corr, grid, align_corners=True).view(batch, h1, w1, -1))
    return torch.cat(out, dim=-1).permute(0, 3, 1, 2).contiguous().float()


def upsample_flow(flow, mask):
    """RAFT.upsample_flow: flow [N][2][h][w], mask [N][576][h][w] (already scaled by 0.25) -> [N][2][8h][8w]."""
    import torch
    import torch.nn.functional as F
    N, _, H, W = flow.shape
    mask = torch.softmax(mask.view(N, 1, 9, 8, 8, H, W), dim=2)
    up = F.unfold(8 * flow, [3, 3], padding=1).view(N, 2, 9, 1, 1, H, W)
    up = torch.sum(mask * up, dim=2).permute(0, 1, 4, 2, 5, 3)
    return up.reshape(N, 2, 8 * H, 8 * W)


def raft(sd, image1, image2, iters=32):
    """model(image1, image2, iters, test_mode=True)[1]: padded float images [1][3][H][W] in 0..255 -> [1][2][H][W]."""
    import torch
    image1, image2 = 2 * (image1 / 255.0) - 1.0, 2 * (image2 / 255.0) - 1.0
    f = of.encode(sd, "fnet", torch.cat([image1, image2]))
    pyr = corr_pyramid(f[:1], f[1:])
    net, inp = of.context(sd, image1)
    coords0 = of.coords_grid(1, image1.shape[2] // 8, image1.shape[3] // 8, image1.device)
    coords1 = coords0.clone()
    for _ in range(iters):
        corr = lookup(pyr, coords1)
        flow = coords1 - coords0
        net, mask, delta = of.update(sd, net, inp, corr, flow, True)
        coords1 = coords1 + delta
        flow_up = upsample_flow(coords1 - coords0, 0.25 * mask)
    return flow_up


def flow_pair(sd, frame1, frame2, iters=32):
    """One reference call pair: uint8 frames [h][w][3] -> (forward, backward) [h][w][2] float32 tensors."""
    import torch
    import torch.nn.functional as F
    dev = sd["fnet.conv1.weight"].device
    h, w = frame1.shape[:2]
    pad = of.padding(h, w)
    im1, im2 = (F.pad(torch.from_numpy(np.ascontiguousarray(f)).permute(2, 0, 1).float()[None].to(dev), pad,
                      mode="replicate") for f in (frame1, frame2))
    H, W = im1.shape[2:]
    crop = lambda f: f[0, :, pad[2]:H - pad[3], pad[0]:W - pad[1]].permute(1, 2, 0)
    return crop(raft(sd, im1, im2, iters)), crop(raft(sd, im2, im1, iters))


def optical_flows(sd, frames, path_consistency=True, iters=32):
    """compute_raft_custom_folder (+ _stride2) on a list of frames -> (flows_f, flows_b, flows_f2, flows_b2)."""
    out = ([], [], [], [])
    for t in range(len(frames) - 1):
        f, b = flow_pair(sd, frames[t], frames[t + 1], iters)
        out[0].append(f)
        out[1].append(b)
    if path_consistency:
        for t in range(len(frames) - 2):
            f, b = flow_pair(sd, frames[t], frames[t + 2], iters)
            out[2].append(f)
            out[3].append(b)
    return out


def _colorwheel():
    RY, YG, GC, CB, BM, MR = 15, 6, 4, 11, 13, 6
    cw = np.zeros((RY + YG + GC + CB + BM + MR, 3))
    c = 0
    cw[0:RY, 0], cw[0:RY, 1] = 255, np.floor(255 * np.arange(0, RY) / RY)
    c += RY
    cw[c:c + YG, 0], cw[c:c + YG, 1] = 255 - np.floor(255 * np.arange(0, YG) / YG), 255
    c += YG
    cw[c:c + GC, 1], cw[c:c + GC, 2] = 255, np.floor(255 * np.arange(0, GC) / GC)
    c += GC
    cw[c:c + CB, 1], cw[c:c + CB, 2] = 255 - np.floor(255 * np.arange(CB) / CB), 255
    c += CB
    cw[c:c + BM, 2], cw[c:c + BM, 0] = 255, np.floor(255 * np.arange(0, BM) / BM)
    c += BM
    cw[c:c + MR, 2], cw[c:c + MR, 0] = 255 - np.floor(255 * np.arange(MR) / MR), 255
    return cw


def flow_to_image(flow_uv):
    """flow_viz.flow_to_image(flow_uv, convert_to_bgr=True) of a float32 [h][w][2] map, with one change: the angle is
    the correctly rounded float32 arctan2 (arctan2 in float64, rounded once).  numpy's float32 arctan2 is not the same
    function on every CPU (SVML on AVX-512 machines, up to 3 units in the last place; libm elsewhere), so the
    reference's own pixels depend on the machine; the device kernel computes this definition."""
    u, v = flow_uv[:, :, 0], flow_uv[:, :, 1]
    rad_max = np.max(np.sqrt(np.square(u) + np.square(v)))
    u, v = u / (rad_max + 1e-5), v / (rad_max + 1e-5)
    img = np.zeros((u.shape[0], u.shape[1], 3), np.uint8)
    cw = _colorwheel()
    ncols = cw.shape[0]
    rad = np.sqrt(np.square(u) + np.square(v))
    a = np.arctan2(-v.astype(np.float64), -u.astype(np.float64)).astype(np.float32) / np.pi
    fk = (a + 1) / 2 * (ncols - 1)
    k0 = np.floor(fk).astype(np.int32)
    k1 = k0 + 1
    k1[k1 == ncols] = 0
    f = fk - k0
    for i in range(3):
        col0, col1 = cw[:, i][k0] / 255.0, cw[:, i][k1] / 255.0
        col = (1 - f) * col0 + f * col1
        idx = rad <= 1
        col[idx] = 1 - rad[idx] * (1 - col[idx])
        col[~idx] = col[~idx] * 0.75
        img[:, :, 2 - i] = np.floor(255 * col)
    return img
