"""The monocular depth step on the GPU: a frame directory in, the depth directory the motion-segmentation stage reads
out (DESIGN.md §4.16).

    python -m particlesfm_b200.midas --image_dir I --output_dir O/midas_depth --model midas_v21-f6b98070.pt
        [--skip_exists]

Reference: third_party/MiDaS run.py:run_midas with the defaults run_particlesfm.py calls it with: model midas_v21
(MidasNet: a ResNeXt-101 32x8d encoder and a RefineNet decoder), optimize=True (on a CUDA device the network runs in
fp16 channels_last), one frame per call.  It writes NAME.pfm (the float prediction at frame size) and NAME.png (that
prediction quantised to 16 bits) for every entry of the image directory.

The network is restated from the architecture; its convolutions are cuDNN calls through torch.  The input transform
(cv2's bicubic resize of the float64 image and the ImageNet normalisation), the bicubic upsampling to frame size with
each map's minimum and maximum, and the 16-bit quantisation are csrc/midas.cu.  Unlike the reference's batch-1 calls,
frames go through the network in batches sized by a device byte budget (batch norm is in eval mode, so each sample is
computed alone).
"""
import argparse
import ctypes
import glob
import os
import sys
from collections import OrderedDict
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib
from ._stage import FrameReader, PinnedSink, check_keys, load_checkpoint, require_device, stream

C_void = ctypes.c_void_p

NET_SIZE = 384          # Resize(384, 384, keep_aspect_ratio=True, ensure_multiple_of=32, resize_method="upper_bound")
MULTIPLE = 32
FEATURES = 256
_BUDGET = 2 << 30       # device bytes of network activations per batch of frames
_BLOCKS = ((1, 3, 64), (2, 4, 128), (3, 23, 256), (4, 3, 512))    # ResNeXt-101 32x8d: (layer, blocks, planes)


# ----------------------------------------------------------------------------- weights

def state_shapes():
    """MidasNet's state-dict keys and shapes: the ResNeXt-101 32x8d encoder under `pretrained` (layer1 holds conv1,
    bn1 and resnet.layer1 as entries 0, 1 and 4), and the decoder under `scratch`."""
    s = OrderedDict()

    def bn(p, c):
        for k in ("weight", "bias", "running_mean", "running_var"):
            s["%s.%s" % (p, k)] = (c,)
        s[p + ".num_batches_tracked"] = ()

    s["pretrained.layer1.0.weight"] = (64, 3, 7, 7)
    bn("pretrained.layer1.1", 64)
    cin = 64
    for layer, blocks, planes in _BLOCKS:
        width, cout = planes * 4, planes * 4       # int(planes * 8 / 64) * 32 grouped channels, expansion 4
        for b in range(blocks):
            p = ("pretrained.layer1.4.%d" if layer == 1 else "pretrained.layer%d.%%d" % layer) % b
            s[p + ".conv1.weight"] = (width, cin if b == 0 else cout, 1, 1)
            bn(p + ".bn1", width)
            s[p + ".conv2.weight"] = (width, width // 32, 3, 3)
            bn(p + ".bn2", width)
            s[p + ".conv3.weight"] = (cout, width, 1, 1)
            bn(p + ".bn3", cout)
            if b == 0:
                s[p + ".downsample.0.weight"] = (cout, cin, 1, 1)
                bn(p + ".downsample.1", cout)
        cin = cout
    for i, c in enumerate((256, 512, 1024, 2048), 1):
        s["scratch.layer%d_rn.weight" % i] = (FEATURES, c, 3, 3)
    for i in (1, 2, 3, 4):
        for u in (1, 2):
            for c in (1, 2):
                p = "scratch.refinenet%d.resConfUnit%d.conv%d" % (i, u, c)
                s[p + ".weight"], s[p + ".bias"] = (FEATURES, FEATURES, 3, 3), (FEATURES,)
    for k, o, i, kk in ((0, 128, FEATURES, 3), (2, 32, 128, 3), (4, 1, 32, 1)):
        s["scratch.output_conv.%d.weight" % k], s["scratch.output_conv.%d.bias" % k] = (o, i, kk, kk), (o,)
    return s


def _other_model(k):
    return k.startswith(("pretrained.model.", "pretrained.act_postprocess")) or ".out_conv." in k


def check_state_dict(sd, what):
    """midas_v21's weights from a checkpoint's contents: a dict holding an "optimizer" key is unwrapped to its "model"
    entry, as BaseModel.load does.  ValueError naming the key for a DPT or midas_v21_small key, an unexpected or
    missing key, or a wrong shape (what the reference's strict load_state_dict refuses)."""
    if isinstance(sd, dict) and "optimizer" in sd:
        sd = sd.get("model")
    if not isinstance(sd, dict):
        raise ValueError("%s: holds a %s, not a state dict" % (what, type(sd).__name__))
    shapes = state_shapes()
    for k in sd:
        if isinstance(k, str) and _other_model(k):
            raise ValueError("%s: key %r is a DPT or midas_v21_small model's; only midas_v21 is built" % (what, k))
    check_keys(sd, shapes, what)
    return {k: sd[k].float() for k in shapes if not k.endswith("num_batches_tracked")}


def load_weights(path):
    """check_state_dict of load_checkpoint(path): ValueError naming the file when it does not exist or cannot be read
    as a checkpoint."""
    return check_state_dict(load_checkpoint(path), path)


def network_weights(sd, device, optimize):
    """The checked weights on `device` as the network runs them: fp16 with channels_last convolution weights when
    optimize (run_midas's model.to(memory_format=torch.channels_last).half() on a CUDA device), else fp32."""
    import torch
    out = {}
    for k, v in sd.items():
        v = v.to(device)
        if optimize:
            v = v.half()
            if v.dim() == 4:
                v = v.to(memory_format=torch.channels_last)
        out[k] = v
    return out


# ----------------------------------------------------------------------------- the network

def _bn(sd, p, x):
    import torch.nn.functional as F
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, 1e-5)


def _conv(sd, p, x, stride=1, padding=0, groups=1):
    import torch.nn.functional as F
    return F.conv2d(x, sd[p + ".weight"], sd.get(p + ".bias"), stride, padding, 1, groups)


def _bottleneck(sd, p, x, stride, downsample):
    """torchvision's Bottleneck with ResNeXt's 32 groups in conv2 (which carries the stride)."""
    import torch
    y = torch.relu(_bn(sd, p + ".bn1", _conv(sd, p + ".conv1", x)))
    y = torch.relu(_bn(sd, p + ".bn2", _conv(sd, p + ".conv2", y, stride, 1, 32)))
    y = _bn(sd, p + ".bn3", _conv(sd, p + ".conv3", y))
    if downsample:
        x = _bn(sd, p + ".downsample.1", _conv(sd, p + ".downsample.0", x, stride))
    return torch.relu(y + x)


def encode(sd, x):
    """pretrained.layer1 .. layer4 of the normalised input [N][3][H][W] -> the four feature maps (1/4 .. 1/32)."""
    import torch
    import torch.nn.functional as F
    x = torch.relu(_bn(sd, "pretrained.layer1.1", _conv(sd, "pretrained.layer1.0", x, 2, 3)))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    for layer, blocks, _ in _BLOCKS:
        for b in range(blocks):
            p = ("pretrained.layer1.4.%d" if layer == 1 else "pretrained.layer%d.%%d" % layer) % b
            x = _bottleneck(sd, p, x, 2 if (b == 0 and layer > 1) else 1, b == 0)
        feats.append(x)
    return feats


def _residual(sd, p, x):
    """ResidualConvUnit: its ReLU is in place, so the skip adds relu(x), not x."""
    import torch
    r = torch.relu(x)
    return _conv(sd, p + ".conv2", torch.relu(_conv(sd, p + ".conv1", r, 1, 1)), 1, 1) + r


def _fuse(sd, p, x, skip=None):
    """FeatureFusionBlock: x + resConfUnit1(skip), resConfUnit2, bilinear x 2 with align_corners=True."""
    import torch.nn.functional as F
    if skip is not None:
        x = x + _residual(sd, p + ".resConfUnit1", skip)
    x = _residual(sd, p + ".resConfUnit2", x)
    return F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)


def forward(sd, x):
    """MidasNet.forward(x) with non_negative=True: [N][3][H][W] -> [N][H][W] in x's dtype."""
    import torch
    import torch.nn.functional as F
    l1, l2, l3, l4 = encode(sd, x)
    rn = [_conv(sd, "scratch.layer%d_rn" % i, f, 1, 1) for i, f in enumerate((l1, l2, l3, l4), 1)]
    path = _fuse(sd, "scratch.refinenet4", rn[3])
    for i in (3, 2, 1):
        path = _fuse(sd, "scratch.refinenet%d" % i, path, rn[i - 1])
    out = _conv(sd, "scratch.output_conv.0", path, 1, 1)
    out = F.interpolate(out, scale_factor=2, mode="bilinear", align_corners=False)
    out = torch.relu(_conv(sd, "scratch.output_conv.2", out, 1, 1))
    out = torch.relu(_conv(sd, "scratch.output_conv.4", out))
    return torch.squeeze(out, dim=1)


# ----------------------------------------------------------------------------- sizes and kernels

def _constrain_to_multiple_of(x, max_val):
    y = (np.round(x / MULTIPLE) * MULTIPLE).astype(int)
    if y > max_val:
        y = (np.floor(x / MULTIPLE) * MULTIPLE).astype(int)
    return int(y)


def get_size(width, height):
    """Resize.get_size of run_midas's midas_v21 transform: keep the aspect ratio, fit the larger side's scale
    ("upper_bound"), round each side to a multiple of 32 with np.round (ties to even), floored when that exceeds
    384.  -> (network width, network height); a side can be 0 for a very elongated frame."""
    scale_height, scale_width = NET_SIZE / height, NET_SIZE / width
    if scale_width < scale_height:
        scale_height = scale_width
    else:
        scale_width = scale_height
    return (_constrain_to_multiple_of(scale_width * width, NET_SIZE),
            _constrain_to_multiple_of(scale_height * height, NET_SIZE))


def prepare(rgb, net_h, net_w, half):
    """psfm_depth_prepare: uint8 RGB frames [n][h][w][3] on the device -> the network input [n][3][net_h][net_w]
    (channels_last), fp16 when half else float32."""
    import torch
    n, h, w, _ = rgb.shape
    rgb = rgb.contiguous()
    out = torch.empty((n, 3, net_h, net_w), dtype=torch.float16 if half else torch.float32, device=rgb.device,
                      memory_format=torch.channels_last)
    _lib.check(_lib.lib().psfm_depth_prepare(C_void(rgb.data_ptr()), n, h, w, net_h, net_w, int(half),
                                             C_void(out.data_ptr()), stream()), "psfm_depth_prepare")
    return out


def upsample(pred, h, w):
    """psfm_depth_upsample: the prediction [n][H][W] (fp16 or float32) -> (the h x w maps as float32 with the rows
    flipped [n][h][w], each map's (min, max) [n][2])."""
    import torch
    pred = pred.contiguous()
    n, H, W = pred.shape
    flipped = torch.empty((n, h, w), dtype=torch.float32, device=pred.device)
    minmax = torch.empty((n, 2), dtype=torch.float32, device=pred.device)
    _lib.check(_lib.lib().psfm_depth_upsample(C_void(pred.data_ptr()), n, H, W, int(pred.dtype == torch.float16), h, w,
                                              C_void(flipped.data_ptr()), C_void(minmax.data_ptr()), stream()),
               "psfm_depth_upsample")
    return flipped, minmax


def quantize(flipped, minmax):
    """psfm_depth_quantize: the flipped maps [n][h][w] and their (min, max) -> write_depth's uint16 pixels [n][h][w]
    in frame orientation."""
    import torch
    n, h, w = flipped.shape
    out = torch.empty((n, h, w), dtype=torch.uint16, device=flipped.device)
    _lib.check(_lib.lib().psfm_depth_quantize(C_void(flipped.data_ptr()), n, h, w, C_void(minmax.data_ptr()),
                                              C_void(out.data_ptr()), stream()), "psfm_depth_quantize")
    return out


def frames_per_batch(net_h, net_w, optimize):
    """Frames per network batch for a net_h x net_w input: as many as the fixed budget holds at about 320 channels of
    the input's resolution per frame (the decoder's widest live set), at least one."""
    return max(1, _BUDGET // ((2 if optimize else 4) * 320 * net_h * net_w))


# ----------------------------------------------------------------------------- frames and names

def decode_rgb(path):
    """A frame as read_image reads it: cv2.imread (8-bit, 3 channels) converted to RGB; None when cv2 cannot read it."""
    import cv2
    img = cv2.imread(path)
    return None if img is None else np.ascontiguousarray(img[:, :, ::-1])


def frame_list(image_dir):
    """The frames as run_midas lists them, every entry of image_dir (glob '*'), sorted and checked before any device
    work -> (paths, h, w), h = w = 0 for an empty directory.  ValueError naming the file: an entry cv2 cannot read as
    an image, two entries with the same stem (a.png and a.jpg would write the same outputs), frames of different
    sizes, or a frame whose network input would have a zero side (get_size)."""
    import cv2
    if not os.path.isdir(image_dir):
        raise ValueError("%s: not a directory" % image_dir)
    paths = sorted(glob.glob(os.path.join(image_dir, "*")))
    stems = {}
    for p in paths:
        s = os.path.splitext(os.path.basename(p))[0]
        if s in stems:
            raise ValueError("%s: has the stem of %s, and both would write %s.pfm and %s.png" % (p, stems[s], s, s))
        stems[s] = p

    def shape(p):
        img = cv2.imread(p) if os.path.isfile(p) else None
        return None if img is None else img.shape[:2]

    with ThreadPoolExecutor(max_workers=4) as pool:
        shapes = list(pool.map(shape, paths))
    size = None
    for p, s in zip(paths, shapes):
        if s is None:
            raise ValueError("%s: not an image cv2 can read" % p)
        if size is None:
            size = s
            if 0 in get_size(s[1], s[0]):
                raise ValueError("%s: %d x %d gives a %d x %d network input; a side would be 0"
                                 % ((p, s[1], s[0]) + get_size(s[1], s[0])))
        elif s != size:
            raise ValueError("%s: %d x %d, the sequence's frames are %d x %d" % (p, s[1], s[0], size[1], size[0]))
    h, w = size if size is not None else (0, 0)
    return paths, h, w


def output_base(output_dir, image_path):
    """output_dir/NAME, NAME the frame's file name without its extension, as run_midas names the outputs."""
    return os.path.join(output_dir, os.path.splitext(os.path.basename(image_path))[0])


def pfm_bytes(flipped):
    """write_pfm's file of a float32 [h][w] map given with its rows already flipped: 'Pf', the width and height, the
    little-endian scale -1, then the values."""
    h, w = flipped.shape
    return b"Pf\n" + b"%d %d\n" % (w, h) + b"%f\n" % -1.0 + np.ascontiguousarray(flipped, "<f4").tobytes()


# ----------------------------------------------------------------------------- the step

def _require_device():
    require_device("midas")


def _run(paths, h, w, sd, optimize, sink):
    """The depth maps of the frames `paths` (h x w), in batches; sink(ids, flipped, pixels) gets each batch's frame
    indices, its flipped float32 maps [b][h][w] and the uint16 pixels [b][h][w], both on the device and ordered on
    torch's current stream.  Returns the seconds of device time spent in the network."""
    import torch
    net_w, net_h = get_size(w, h)
    per = frames_per_batch(net_h, net_w, optimize)
    weights = network_weights(sd, "cuda", optimize)
    reader = FrameReader(paths, range(len(paths)), decode_rgb)
    events = []
    try:
        with torch.no_grad():
            for b0 in range(0, len(paths), per):
                ids = list(range(b0, min(len(paths), b0 + per)))
                rgb = torch.stack([reader.upload(i) for i in ids])
                x = prepare(rgb, net_h, net_w, optimize)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                pred = forward(weights, x)
                e1.record()
                events.append((e0, e1))
                del x
                flipped, minmax = upsample(pred, h, w)
                del pred
                sink(ids, flipped, quantize(flipped, minmax))
    finally:
        reader.close()
    torch.cuda.current_stream().synchronize()
    return sum(a.elapsed_time(b) for a, b in events) / 1e3


def compute_depth_maps(image_dir, model_path, optimize=True):
    """The step's outputs as CUDA tensors: (paths, maps [n][h][w] float32 in frame orientation (the PFM values),
    pixels [n][h][w] uint16 (the PNG values)), the network in fp16 channels_last when optimize, else float32;
    ([], None, None) for an empty directory.  Bad input raises ValueError naming the file before any device work."""
    import torch
    paths, h, w = frame_list(image_dir)
    sd = load_weights(model_path)
    if not paths:
        return paths, None, None
    _require_device()
    maps, pixels = [], []

    def keep(ids, flipped, px):
        maps.append(torch.flip(flipped, [1]))
        pixels.append(px)

    _run(paths, h, w, sd, optimize, keep)
    return paths, torch.cat(maps), torch.cat(pixels)


class DepthWriter(PinnedSink):
    """A sink for _run that writes each batch's NAME.pfm and NAME.png files on a writer thread while the next batch
    runs, the batch's frames on 4 file threads; the first failed write is raised by the next call, by close() and on
    leaving a with block (PinnedSink).  bases[i] is frame i's output path without extension."""

    def __init__(self, bases):
        self.bases = bases
        self.pool = ThreadPoolExecutor(max_workers=4, thread_name_prefix="psfm-depth-files")
        super().__init__("psfm-depth-writer")

    def write(self, ids, flipped, pixels):
        import cv2

        def one(j):
            base = self.bases[ids[j]]
            with open(base + ".pfm", "wb") as f:
                f.write(pfm_bytes(flipped[j].numpy()))
            if not cv2.imwrite(base + ".png", pixels[j].numpy()):
                raise OSError("%s.png: could not be written" % base)
        list(self.pool.map(one, range(len(ids))))      # PNG encoding releases the GIL

    def join(self):
        error = super().join()
        self.pool.shutdown(wait=True)
        return error


def write_depth_maps(image_dir, output_dir, model_path, skip_exists=False, optimize=True):
    """run_midas(image_dir, output_dir) with midas_v21: NAME.pfm and NAME.png for every frame.  With skip_exists, a
    frame whose two files exist is skipped, as the reference does.  Returns the number of frames computed."""
    paths, h, w = frame_list(image_dir)
    sd = load_weights(model_path)
    os.makedirs(output_dir, exist_ok=True)
    bases = [output_base(output_dir, p) for p in paths]
    if skip_exists:
        keep = [i for i, b in enumerate(bases) if not (os.path.exists(b + ".pfm") and os.path.exists(b + ".png"))]
        paths, bases = [paths[i] for i in keep], [bases[i] for i in keep]
    if not paths:
        return 0
    _require_device()
    with DepthWriter(bases) as writer:
        _run(paths, h, w, sd, optimize, writer)
    return len(paths)


def main(argv=None):
    p = argparse.ArgumentParser("Monocular depth maps (MiDaS midas_v21) of a frame directory on the GPU")
    p.add_argument("--image_dir", required=True, help="the folder containing input images")
    p.add_argument("--output_dir", required=True, help="the depth directory (WORKSPACE/midas_depth)")
    p.add_argument("--model", required=True, help="midas_v21-f6b98070.pt")
    p.add_argument("--skip_exists", action="store_true", help="skip a frame whose .pfm and .png exist")
    a = p.parse_args(argv)
    try:
        write_depth_maps(a.image_dir, a.output_dir, a.model, a.skip_exists)
    except ValueError as e:
        print("midas: %s" % e, file=sys.stderr)
        return 2
    except (_lib.PsfmError, RuntimeError, OSError) as e:
        print("midas: %s" % e, file=sys.stderr)
        return 1
    return 0


if __name__ == "__main__":
    sys.exit(main())
