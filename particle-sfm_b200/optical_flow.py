"""The optical-flow stage on the GPU: a frame directory in, the flow directory the point-trajectory stage reads out
(DESIGN.md §4.14).

    python -m particlesfm_b200.optical_flow --image_dir I --output_dir O/optical_flows --model raft-things.pth
        [--skip_path_consistency] [--skip_exists]

Reference: third_party/RAFT/compute_raft_custom_folder.py and compute_raft_custom_folder_stride2.py with their
defaults: the basic RAFT model (not small, no alternate correlation, no mixed precision), 32 iterations, weights from
the user's raft-things.pth.  It writes flow_f/NAME.flo, flow_b/NAME-bk.flo and flow_imgs/NAME for every pair of
consecutive frames, and with path consistency flow_f2, flow_b2 and flow_imgs2 for frames two apart.

The network is restated from the architecture.  Its convolutions are cuDNN calls through torch with torch's defaults
(the reference's precision class on the same card); the correlation pyramids, the lookup, the convex upsampling and
the flow image are csrc/optical_flow.cu.  Unlike the reference's four batch-1 calls per frame, every frame is
encoded once (instance norm in fnet and eval-mode batch norm in cnet act on each sample alone), one product gives
both directions' correlation pyramids, the mask head runs in the last iteration only, and the update loop runs
batched over the forward and backward problems of several pairs.
"""
import argparse
import ctypes
import glob
import os
import queue
import sys
import threading
from collections import OrderedDict
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _abi, _lib

C_void = ctypes.c_void_p

ITERS = 32
TAG_FLOAT = 202021.25
MIN_SIZE = 121          # smaller frames give a 1-pixel coarsest level, where the reference's lookup divides by 0
_BUDGET = 8 << 30       # device bytes of correlation pyramids and update activations per batch of problems
_LEVELS, _CORR = 4, 324
_SMALL_ONLY = ("update_block.gru.convz.weight", "fnet.layer1.0.conv3.weight", "cnet.layer1.0.conv3.weight")


# ----------------------------------------------------------------------------- weights

def state_shapes():
    """The basic RAFT model's state-dict keys (without DataParallel's `module.` prefix) and their shapes."""
    s = OrderedDict()

    def conv(p, o, i, kh, kw):
        s[p + ".weight"], s[p + ".bias"] = (o, i, kh, kw), (o,)

    def bn(p, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            s["%s.%s" % (p, k)] = (c,)
        s[p + ".num_batches_tracked"] = ()

    for net, out, batch in (("fnet", 256, False), ("cnet", 256, True)):
        conv(net + ".conv1", 64, 3, 7, 7)
        if batch:
            bn(net + ".norm1", 64)
        cin = 64
        for li, (dim, stride) in enumerate(((64, 1), (96, 2), (128, 2)), 1):
            for bi in (0, 1):
                p = "%s.layer%d.%d" % (net, li, bi)
                conv(p + ".conv1", dim, cin if bi == 0 else dim, 3, 3)
                conv(p + ".conv2", dim, dim, 3, 3)
                if batch:
                    bn(p + ".norm1", dim)
                    bn(p + ".norm2", dim)
                if bi == 0 and stride != 1:
                    if batch:
                        bn(p + ".norm3", dim)
                    conv(p + ".downsample.0", dim, cin, 1, 1)
                    if batch:
                        bn(p + ".downsample.1", dim)
            cin = dim
        conv(net + ".conv2", out, 128, 1, 1)
    u = "update_block."
    conv(u + "encoder.convc1", 256, _CORR, 1, 1)
    conv(u + "encoder.convc2", 192, 256, 3, 3)
    conv(u + "encoder.convf1", 128, 2, 7, 7)
    conv(u + "encoder.convf2", 64, 128, 3, 3)
    conv(u + "encoder.conv", 126, 256, 3, 3)
    for g in "zrq":
        conv(u + "gru.conv%s1" % g, 128, 384, 1, 5)
        conv(u + "gru.conv%s2" % g, 128, 384, 5, 1)
    conv(u + "flow_head.conv1", 256, 128, 3, 3)
    conv(u + "flow_head.conv2", 2, 256, 3, 3)
    conv(u + "mask.0", 256, 128, 3, 3)
    conv(u + "mask.2", 576, 256, 1, 1)
    return s


def check_state_dict(sd, what):
    """The basic model's weights from a state dict, DataParallel's `module.` prefix stripped.  ValueError naming the
    key for the small model's keys, an unexpected or missing key, or a wrong shape."""
    import torch
    if not isinstance(sd, dict):
        raise ValueError("%s: holds a %s, not a state dict" % (what, type(sd).__name__))
    sd = {(k[7:] if k.startswith("module.") else k): v for k, v in sd.items()}
    shapes = state_shapes()
    for k in _SMALL_ONLY:
        if k in sd:
            raise ValueError("%s: key %r is the small RAFT model's; only the basic model (raft-things) is supported" % (what, k))
    for k, v in sd.items():
        if k not in shapes:
            raise ValueError("%s: unexpected key %r" % (what, k))
        if not isinstance(v, torch.Tensor) or tuple(v.shape) != shapes[k]:
            raise ValueError("%s: key %r has shape %s, expected %s" % (what, k, tuple(getattr(v, "shape", ())), shapes[k]))
    for k in shapes:
        if k not in sd:
            raise ValueError("%s: missing key %r" % (what, k))
    return {k: (sd[k] if k.endswith("num_batches_tracked") else sd[k].float()) for k in shapes}


def load_weights(path):
    """check_state_dict of torch.load(path, weights_only=True) on the host; ValueError naming the file when it does
    not exist or cannot be read as a checkpoint."""
    import torch
    if not os.path.isfile(path):
        raise ValueError("%s: no such weights file" % path)
    try:
        sd = torch.load(path, map_location="cpu", weights_only=True)
    except Exception as e:
        raise ValueError("%s: not a readable checkpoint (%s)" % (path, e)) from None
    return check_state_dict(sd, path)


# ----------------------------------------------------------------------------- the network

def _conv(sd, p, x, stride=1, padding=0):
    import torch.nn.functional as F
    return F.conv2d(x, sd[p + ".weight"], sd[p + ".bias"], stride, padding)


def _norm(sd, p, x, batch):
    import torch.nn.functional as F
    if batch:
        return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                            False, 0.0, 1e-5)
    return F.instance_norm(x, eps=1e-5)


def encode(sd, net, x):
    """BasicEncoder `net` ("fnet": instance norm, "cnet": batch norm in eval mode) of images [N][3][H][W] already
    scaled to [-1, 1] -> [N][256][H/8][W/8]."""
    import torch
    batch = net == "cnet"
    x = torch.relu(_norm(sd, net + ".norm1", _conv(sd, net + ".conv1", x, 2, 3), batch))
    for li, stride in ((1, 1), (2, 2), (3, 2)):
        for bi in (0, 1):
            p, s = "%s.layer%d.%d" % (net, li, bi), stride if bi == 0 else 1
            y = torch.relu(_norm(sd, p + ".norm1", _conv(sd, p + ".conv1", x, s, 1), batch))
            y = torch.relu(_norm(sd, p + ".norm2", _conv(sd, p + ".conv2", y, 1, 1), batch))
            if s != 1:
                x = _norm(sd, p + ".norm3", _conv(sd, p + ".downsample.0", x, s, 0), batch)
            x = torch.relu(x + y)
    return _conv(sd, net + ".conv2", x)


def context(sd, x):
    """cnet split into the hidden state tanh(net) and the context relu(inp), 128 channels each."""
    import torch
    c = encode(sd, "cnet", x)
    return torch.tanh(c[:, :128]), torch.relu(c[:, 128:])


def update(sd, net, inp, corr, flow, with_mask):
    """BasicUpdateBlock: motion encoder, SepConvGRU, flow head; the mask head's output (before its 0.25 scale) only
    when with_mask.  -> (net, mask or None, delta_flow)."""
    import torch
    u = "update_block."
    relu = torch.relu
    cor = relu(_conv(sd, u + "encoder.convc1", corr))
    cor = relu(_conv(sd, u + "encoder.convc2", cor, 1, 1))
    flo = relu(_conv(sd, u + "encoder.convf1", flow, 1, 3))
    flo = relu(_conv(sd, u + "encoder.convf2", flo, 1, 1))
    out = relu(_conv(sd, u + "encoder.conv", torch.cat([cor, flo], 1), 1, 1))
    x = torch.cat([inp, out, flow], 1)
    for k, pad in (("1", (0, 2)), ("2", (2, 0))):
        hx = torch.cat([net, x], 1)
        z = torch.sigmoid(_conv(sd, u + "gru.convz" + k, hx, 1, pad))
        r = torch.sigmoid(_conv(sd, u + "gru.convr" + k, hx, 1, pad))
        q = torch.tanh(_conv(sd, u + "gru.convq" + k, torch.cat([r * net, x], 1), 1, pad))
        net = (1 - z) * net + z * q
    delta = _conv(sd, u + "flow_head.conv2", relu(_conv(sd, u + "flow_head.conv1", net, 1, 1)), 1, 1)
    mask = _conv(sd, u + "mask.2", relu(_conv(sd, u + "mask.0", net, 1, 1))) if with_mask else None
    return net, mask, delta


def padding(h, w):
    """InputPadder's 'sintel' padding of an h x w frame to multiples of 8: [left, right, top, bottom]."""
    ph, pw = (((h // 8) + 1) * 8 - h) % 8, (((w // 8) + 1) * 8 - w) % 8
    return [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2]


def coords_grid(n, h, w, device):
    """[n][2][h][w] pixel coordinates (x, y) of the 1/8 grid."""
    import torch
    y, x = torch.meshgrid(torch.arange(h, device=device), torch.arange(w, device=device), indexing="ij")
    return torch.stack([x, y]).float()[None].repeat(n, 1, 1, 1)


def _stream():
    import torch
    return C_void(torch.cuda.current_stream().cuda_stream)


def corr_pyramid_floats(h, w):
    return int(_lib.check(_lib.lib().psfm_corr_pyramid_floats(h, w), "psfm_corr_pyramid_floats"))


def corr_pyramids(fmap1, fmap2, fwd, bwd):
    """Both directions' pyramids of one pair: fmap1, fmap2 [256][h][w]; fwd, bwd: contiguous float32 CUDA tensors of
    corr_pyramid_floats(h, w) values, written in place."""
    import torch
    c, h, w = fmap1.shape
    torch.matmul(fmap1.reshape(c, h * w).t(), fmap2.reshape(c, h * w), out=fwd[:h * w * h * w].view(h * w, h * w))
    _lib.check(_lib.lib().psfm_corr_pyramids(C_void(fwd.data_ptr()), C_void(bwd.data_ptr()), h, w, _stream()),
               "psfm_corr_pyramids")


def corr_lookup(pyramids, coords, out):
    """psfm_corr_lookup: pyramids [P][corr_pyramid_floats], coords [P][2][h][w] -> out [P][324][h][w]."""
    P, _, h, w = coords.shape
    _lib.check(_lib.lib().psfm_corr_lookup(C_void(pyramids.data_ptr()), P, h, w, C_void(coords.data_ptr()),
                                           C_void(out.data_ptr()), _stream()), "psfm_corr_lookup")
    return out


def upsample(flow, mask, pad):
    """psfm_flow_upsample: flow [P][2][h][w], mask [P][576][h][w] (before the 0.25 scale), pad [left, right, top,
    bottom] -> [P][8h - top - bottom][8w - left - right][2]."""
    import torch
    P, _, h, w = flow.shape
    out = torch.empty((P, 8 * h - pad[2] - pad[3], 8 * w - pad[0] - pad[1], 2), dtype=torch.float32, device=flow.device)
    p = (ctypes.c_int32 * 4)(*pad)
    _lib.check(_lib.lib().psfm_flow_upsample(C_void(flow.data_ptr()), C_void(mask.data_ptr()), P, h, w, p,
                                             C_void(out.data_ptr()), _stream()), "psfm_flow_upsample")
    return out


def flow_to_image(flows):
    """psfm_flow_to_image: flows [M][H][W][2] float32 CUDA -> [M][H][W][3] uint8 BGR (flow_to_image(...,
    convert_to_bgr=True) per map)."""
    import torch
    M, H, W, _ = flows.shape
    out = torch.empty((M, H, W, 3), dtype=torch.uint8, device=flows.device)
    _lib.check(_lib.lib().psfm_flow_to_image(C_void(flows.data_ptr()), M, H, W, C_void(out.data_ptr()), _stream()),
               "psfm_flow_to_image")
    return out


def _per_problem_bytes(h, w, H, W):
    # the two pyramids' share, the lookup output and the update block's widest live set (about 3,000 channels at
    # 1/8), the mask and the output map
    return 4 * corr_pyramid_floats(h, w) + 4 * h * w * (_CORR + 3000 + 576) + 8 * H * W


def pairs_per_batch(H, W):
    """Pairs per batch of the update loop for H x W frames: as many forward + backward problems as the fixed budget
    holds, at least one pair."""
    Hp, Wp = H + sum(padding(H, W)[2:]), W + sum(padding(H, W)[:2])
    return max(1, _BUDGET // (2 * _per_problem_bytes(Hp // 8, Wp // 8, H, W)))


# ----------------------------------------------------------------------------- frames and names

def frame_list(image_dir):
    """The frames as the reference lists them, sorted(glob('*.png') + glob('*.jpg')), checked before any device work
    -> (paths, h, w).  ValueError naming the directory or file: fewer than 2 images, a file that is not an 8-bit
    3-channel (RGB) image, frames of different sizes, or frames under 121 x 121 (their coarsest correlation level is
    1 pixel wide, where the reference's lookup divides by zero and every flow is NaN)."""
    from PIL import Image, UnidentifiedImageError
    paths = sorted(glob.glob(os.path.join(image_dir, "*.png")) + glob.glob(os.path.join(image_dir, "*.jpg")))
    if len(paths) < 2:
        raise ValueError("%s: %d .png/.jpg image(s); optical flow needs at least 2" % (image_dir, len(paths)))
    size = None
    for p in paths:
        try:
            with Image.open(p) as im:
                mode, s = im.mode, im.size
        except (UnidentifiedImageError, OSError) as e:
            raise ValueError("%s: not a readable image (%s)" % (p, e)) from None
        if mode != "RGB":
            raise ValueError("%s: mode %s; the flow network takes 8-bit 3-channel (RGB) images" % (p, mode))
        if size is None:
            size = s
        elif s != size:
            raise ValueError("%s: %d x %d, the sequence's frames are %d x %d" % (p, s[0], s[1], size[0], size[1]))
    w, h = size
    if h < MIN_SIZE or w < MIN_SIZE:
        raise ValueError("%s: %d x %d; frames must be at least %d x %d" % (paths[0], w, h, MIN_SIZE, MIN_SIZE))
    return paths, h, w


def output_names(image_path):
    """(flow name, backward flow name, image name) of a pair's first frame, mapped as compute_raft_custom_folder.py
    maps them: .png and .jpg replaced by .flo, then .flo by -bk.flo (applied to the file name only), and the frame's
    own name for the image."""
    base = os.path.basename(image_path)
    flo = base.replace(".png", ".flo").replace(".jpg", ".flo")
    return flo, flo.replace(".flo", "-bk.flo"), base


def _subdirs(stride):
    s = "" if stride == 1 else "2"
    return "flow_f" + s, "flow_b" + s, "flow_imgs" + s


def _pairs(n, path_consistency):
    return [(t, s) for t in range(n - 1) for s in ((1, 2) if path_consistency else (1,)) if t + s < n]


def write_flo(path, flow):
    """flow_write: the tag, width and height, then the [H][W][2] float32 values."""
    h, w = flow.shape[:2]
    with open(path, "wb") as f:
        f.write(np.float32(TAG_FLOAT).tobytes() + np.int32(w).tobytes() + np.int32(h).tobytes())
        f.write(np.ascontiguousarray(flow, np.float32).tobytes())


# ----------------------------------------------------------------------------- the stage

class _FrameReader:
    """Decodes the frames a run needs, in order, on host threads into pinned [H][W][3] uint8 tensors, a few ahead of
    their use; upload(i) copies frame i on the copy stream and returns the device tensor, ordered before torch's
    current stream."""

    AHEAD = 6

    def __init__(self, paths, order):
        import torch
        self.paths, self.order, self.next = paths, list(order), 0
        self.pool = ThreadPoolExecutor(max_workers=4, thread_name_prefix="psfm-frame-reader")
        self.pending = OrderedDict()
        self.copy = torch.cuda.Stream()
        self._fill()

    def _decode(self, i):
        import torch
        from PIL import Image
        with Image.open(self.paths[i]) as im:
            a = np.asarray(im, dtype=np.uint8)
        t = torch.empty(a.shape, dtype=torch.uint8, pin_memory=True)
        t.numpy()[...] = a
        return t

    def _fill(self):
        while self.next < len(self.order) and len(self.pending) < self.AHEAD:
            i = self.order[self.next]
            self.pending[i] = self.pool.submit(self._decode, i)
            self.next += 1

    def upload(self, i):
        import torch
        host = self.pending.pop(i).result()
        self._fill()
        with torch.cuda.stream(self.copy):
            dev = host.to("cuda", non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy)
        torch.cuda.current_stream().wait_event(ev)
        dev.record_stream(torch.cuda.current_stream())
        ev.synchronize()            # the pinned buffer may be freed once the copy has left it
        return dev

    def close(self):
        for f in self.pending.values():
            f.cancel()
        self.pool.shutdown(wait=True)


def _run(paths, h, w, sd, pairs, sink):
    """The flows of `pairs` [(t, stride)] of the frames `paths` (h x w), in batches; sink(batch, flows, images) gets
    each batch's pairs, its maps [2 n][h][w][2] (forward maps first, then backward, in pair order) and the forward
    maps' BGR images [n][h][w][3], all on the device and ordered on torch's current stream."""
    import torch
    dev = torch.device("cuda")
    pad = padding(h, w)
    H, W = h + pad[2] + pad[3], w + pad[0] + pad[1]
    gh, gw = H // 8, W // 8
    S = corr_pyramid_floats(gh, gw)
    per = pairs_per_batch(h, w)
    needed = sorted({t for t, s in pairs} | {t + s for t, s in pairs})
    sd = {k: v.to(dev) for k, v in sd.items()}
    reader = _FrameReader(paths, needed)
    cache = {}          # frame -> (fmap, net, inp)
    try:
        with torch.no_grad():
            pyr = torch.empty((2 * min(per, len(pairs)), S), dtype=torch.float32, device=dev)
            for b0 in range(0, len(pairs), per):
                batch = pairs[b0:b0 + per]
                n = len(batch)
                first = min(t for t, _ in batch)
                for f in [f for f in cache if f < first]:
                    del cache[f]
                todo = sorted(({t for t, s in batch} | {t + s for t, s in batch}) - set(cache))
                for g in range(0, len(todo), 4):
                    ids = todo[g:g + 4]
                    x = torch.stack([reader.upload(i) for i in ids]).permute(0, 3, 1, 2).float()
                    x = torch.nn.functional.pad(x, pad, mode="replicate")
                    x = 2 * (x / 255.0) - 1.0
                    fmap = encode(sd, "fnet", x)
                    net, inp = context(sd, x)
                    for k, i in enumerate(ids):
                        cache[i] = (fmap[k], net[k], inp[k])
                src = [t for t, _ in batch] + [t + s for t, s in batch]
                dst = src[n:] + src[:n]
                for j in range(n):
                    corr_pyramids(cache[src[j]][0], cache[dst[j]][0], pyr[j], pyr[n + j])
                net = torch.stack([cache[i][1] for i in src])
                inp = torch.stack([cache[i][2] for i in src])
                coords0 = coords_grid(2 * n, gh, gw, dev)
                coords1 = coords0.clone()
                corr = torch.empty((2 * n, _CORR, gh, gw), dtype=torch.float32, device=dev)
                for it in range(ITERS):
                    corr_lookup(pyr, coords1, corr)
                    net, mask, delta = update(sd, net, inp, corr, coords1 - coords0, it == ITERS - 1)
                    coords1 = coords1 + delta
                flows = upsample(coords1 - coords0, mask, pad)
                sink(batch, flows, flow_to_image(flows[:n]))
    finally:
        reader.close()


def _require_device():
    from . import device_count
    if device_count() <= 0:
        raise _lib.PsfmError("optical flow: no CUDA device (the product has no CPU path)", _abi.PSFM_ERR_NO_DEVICE)


def compute_optical_flows(image_dir, model_path, path_consistency=True):
    """The stage's flows as CUDA tensors [H][W][2] float32, for tracker.main_connect_point_trajectories_device:
    (flows_f, flows_b, flows_f2, flows_b2), the stride-2 lists empty without path consistency.  Bad input raises
    ValueError naming the file before any device work."""
    paths, h, w = frame_list(image_dir)
    sd = load_weights(model_path)
    _require_device()
    n = len(paths)
    out = {1: ([None] * (n - 1), [None] * (n - 1)), 2: ([None] * max(0, n - 2), [None] * max(0, n - 2))}

    def keep(batch, flows, images):
        for j, (t, s) in enumerate(batch):
            out[s][0][t], out[s][1][t] = flows[j], flows[len(batch) + j]

    _run(paths, h, w, sd, _pairs(n, path_consistency), keep)
    return out[1][0], out[1][1], (out[2][0] if path_consistency else []), (out[2][1] if path_consistency else [])


class FlowWriter:
    """A sink for _run that writes each batch's files on a writer thread while the next batch runs: the maps and
    images go to pinned host buffers on torch's current stream, and the thread writes them once that copy is done.
    files(t, stride) -> (forward .flo, backward .flo, flow image) paths.  close() waits for the thread and raises
    the first failed write (join() only waits); a failed write also makes the next call raise."""

    def __init__(self, files):
        self.files = files
        self.work, self.failure = queue.Queue(maxsize=2), []
        self.thread = threading.Thread(target=self._write, name="psfm-flow-writer", daemon=True)
        self.thread.start()

    def _write(self):
        import cv2
        while True:
            item = self.work.get()
            if item is None:
                return
            if self.failure:
                continue
            try:
                batch, flows, images, ev = item
                ev.synchronize()
                for j, (t, s) in enumerate(batch):
                    ff, fb, fi = self.files(t, s)
                    if not cv2.imwrite(fi, images[j].numpy()):
                        raise OSError("%s: could not be written" % fi)
                    write_flo(ff, flows[j].numpy())
                    write_flo(fb, flows[len(batch) + j].numpy())
            except BaseException as e:
                self.failure.append(e)

    def __call__(self, batch, flows, images):
        import torch
        if self.failure:
            raise self.failure[0]
        hf = torch.empty(flows.shape, dtype=flows.dtype, pin_memory=True)
        hi = torch.empty(images.shape, dtype=images.dtype, pin_memory=True)
        hf.copy_(flows, non_blocking=True)
        hi.copy_(images, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        self.work.put((batch, hf, hi, ev))

    def join(self):
        """Ends the thread once the batches sent so far are written (or skipped after a failure)."""
        if self.thread is not None:
            self.work.put(None)
            self.thread.join()
            self.thread = None

    def close(self):
        self.join()
        if self.failure:
            raise self.failure[0]


def flow_files(paths, output_dir):
    """files(t, stride) of the flow directory output_dir for the frames `paths`: the forward .flo, backward .flo and
    flow image of pair (t, t + stride), named as compute_raft_custom_folder names them."""
    def files(t, s):
        f, b, i = output_names(paths[t])
        df, db, di = _subdirs(s)
        return os.path.join(output_dir, df, f), os.path.join(output_dir, db, b), os.path.join(output_dir, di, i)
    return files


def make_flow_dirs(output_dir, path_consistency):
    for s in ((1, 2) if path_consistency else (1,)):
        for d in _subdirs(s):
            os.makedirs(os.path.join(output_dir, d), exist_ok=True)


def missing_pairs(paths, output_dir, path_consistency):
    """The pairs of the frames `paths` whose three files are not all in output_dir (skip_exists)."""
    files = flow_files(paths, output_dir)
    return [p for p in _pairs(len(paths), path_consistency) if not all(os.path.exists(f) for f in files(*p))]


def write_optical_flows(image_dir, output_dir, model_path, skip_path_consistency=False, skip_exists=False):
    """compute_raft_custom_folder (and _stride2 unless skip_path_consistency) into output_dir.  With skip_exists, a
    pair whose three files exist is skipped, as the reference does.  Files are written on a writer thread while the
    next batch runs.  Returns the number of pairs computed."""
    paths, h, w = frame_list(image_dir)
    sd = load_weights(model_path)
    make_flow_dirs(output_dir, not skip_path_consistency)
    pairs = _pairs(len(paths), not skip_path_consistency)
    if skip_exists:
        pairs = missing_pairs(paths, output_dir, not skip_path_consistency)
    if not pairs:
        return 0
    _require_device()
    writer = FlowWriter(flow_files(paths, output_dir))
    try:
        _run(paths, h, w, sd, pairs, writer)
    finally:
        writer.join()
    writer.close()
    return len(pairs)


def main(argv=None):
    p = argparse.ArgumentParser("Pairwise optical flows (RAFT) of a frame directory on the GPU")
    p.add_argument("--image_dir", required=True, help="the folder containing input images")
    p.add_argument("--output_dir", required=True, help="the flow directory (WORKSPACE/optical_flows)")
    p.add_argument("--model", required=True, help="raft-things.pth")
    p.add_argument("--skip_path_consistency", action="store_true", help="only the stride-1 flows")
    p.add_argument("--skip_exists", action="store_true", help="skip a pair whose three files exist")
    a = p.parse_args(argv)
    try:
        write_optical_flows(a.image_dir, a.output_dir, a.model, a.skip_path_consistency, a.skip_exists)
    except ValueError as e:
        print("optical_flow: %s" % e, file=sys.stderr)
        return 2
    except (_lib.PsfmError, RuntimeError, OSError) as e:
        print("optical_flow: %s" % e, file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
