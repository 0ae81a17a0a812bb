"""The depth step on the GPU (csrc/midas.cu, particlesfm_b200.midas) against the oracle's reference call structure
(oracle/midas_oracle.py) and the reference's own float32 run (tests/golden/depth_small.npz): the kernels one by one,
then the whole step in float32 and in fp16, then the written files."""
import os
import re
import threading

import cv2
import numpy as np
import pytest
import torch

from oracle import midas_oracle as mo
from particlesfm_b200 import midas

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "depth_small.npz")


@pytest.fixture
def no_tf32():
    """The convolutions in full fp32 while a test runs, so the two call structures differ by reordering only."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _ulps(a, b, dtype):
    """|a - b| in units of the last place of dtype at |b| (a, b float64 arrays)."""
    spacing = np.spacing(np.abs(b).astype(dtype)).astype(np.float64)
    return np.abs(a - b) / spacing


def _write_frames(d, frames):
    os.makedirs(d, exist_ok=True)
    for i, f in enumerate(frames):
        assert cv2.imwrite(os.path.join(d, "%05d.png" % i), f[:, :, ::-1])
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w", [(3, 40, 192), (2, 436, 1024), (2, 480, 854), (1, 37, 23), (1, 500, 400)])
def test_prepare_equals_cv2_resize(gpu, n, h, w):
    frames = mo.seeded_frames(n, h, w, seed=0 if (n, h, w) == (3, 40, 192) else h)    # the golden's frames first
    W, H = midas.get_size(w, h)
    rgb = torch.from_numpy(np.stack(frames)).cuda()
    got = midas.prepare(rgb, H, W, False)
    assert got.shape == (n, 3, H, W) and got.is_contiguous(memory_format=torch.channels_last)
    ref = np.stack([mo.transform(f) for f in frames])
    u = _ulps(got.cpu().numpy().astype(np.float64), ref.astype(np.float64), np.float32)
    print("prepare %d x %d -> %d x %d: %d of %d values differ, at most %.0f ulp" % (w, h, W, H, (u > 0).sum(), u.size, u.max()))
    assert u.max() <= 4
    half = midas.prepare(rgb, H, W, True)
    assert half.dtype == torch.float16 and torch.equal(half, got.half())
    if (n, h, w) == (3, 40, 192):         # the reference's own transform of frame 0
        g = np.load(GOLDEN)["transform0"].astype(np.float64)
        assert _ulps(got[0].cpu().numpy().astype(np.float64), g, np.float32).max() <= 4


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("n,H,W,h,w", [(3, 64, 384, 40, 192), (2, 160, 384, 436, 1024), (1, 224, 384, 480, 854),
                                       (2, 64, 384, 64, 384), (1, 96, 64, 31, 17)])
def test_upsample_equals_interpolate(gpu, dtype, n, H, W, h, w):
    g = torch.Generator(device="cuda").manual_seed(H + w)
    pred = (torch.rand((n, H, W), device="cuda", generator=g) * 3 - 0.2).to(dtype)
    flipped, minmax = midas.upsample(pred, h, w)
    ref = torch.nn.functional.interpolate(pred.unsqueeze(1), size=(h, w), mode="bicubic", align_corners=False)[:, 0]
    got = torch.flip(flipped, [1]).cpu().numpy().astype(np.float64)
    r = ref.float().cpu().numpy().astype(np.float64)
    if dtype == torch.float16:
        u = _ulps(got, r, np.float16)
    else:
        # float32: torch's build fuses some products where this kernel's fused ones differ, an error of the inputs'
        # scale, so the unit is the last place at each map's largest magnitude (where a value nears 0 by
        # cancellation, the spacing at the value itself is no measure)
        scale = np.abs(r).reshape(n, -1).max(1)[:, None, None]
        u = np.abs(got - r) / np.spacing(scale.astype(np.float32)).astype(np.float64)
    print("upsample %s %d x %d -> %d x %d: %d of %d values differ, at most %.2f ulp"
          % (dtype, W, H, w, h, (u > 0).sum(), u.size, u.max()))
    # measured on an H100: fp16 at most 1 ulp (41 of 892,928 values at 1024 x 436), float32 at most 3 (DESIGN.md §4.16)
    assert u.max() <= (1 if dtype == torch.float16 else 4)
    mm = minmax.cpu().numpy()
    assert np.array_equal(mm[:, 0], got.reshape(n, -1).min(1).astype(np.float32))
    assert np.array_equal(mm[:, 1], got.reshape(n, -1).max(1).astype(np.float32))


@pytest.mark.gpu
def test_quantize_equals_the_golden_pixels(gpu):
    g = np.load(GOLDEN)
    maps = np.concatenate([g["maps"], np.full((1, 40, 192), 0.7, np.float32)])       # and a constant map
    flipped = torch.from_numpy(np.ascontiguousarray(maps[:, ::-1])).cuda()
    mm = torch.from_numpy(np.stack([maps.reshape(4, -1).min(1), maps.reshape(4, -1).max(1)], 1)).cuda()
    px = midas.quantize(flipped, mm).cpu().numpy()
    assert px.dtype == np.uint16
    assert np.array_equal(px[:3], g["pixels"]) and not px[3].any()
    _, got_mm = midas.upsample(torch.from_numpy(np.ascontiguousarray(g["maps"])).cuda(), 40, 192)   # same size: a copy
    assert np.array_equal(got_mm.cpu().numpy(), mm[:3].cpu().numpy())


@pytest.fixture(scope="module")
def golden_dir(tmp_path_factory):
    d = tmp_path_factory.mktemp("depth")
    w = str(d / "midas_v21.pt")
    torch.save(mo.seeded_state_dict(0), w)
    return _write_frames(str(d / "img"), mo.seeded_frames(3, 40, 192, seed=0)), w


@pytest.mark.gpu
def test_float32_step_equals_the_golden(gpu, no_tf32, golden_dir):
    d, w = golden_dir
    g = np.load(GOLDEN)
    paths, maps, pixels = midas.compute_depth_maps(d, w, optimize=False)
    assert [os.path.basename(p) for p in paths] == ["00000.png", "00001.png", "00002.png"]
    ref = g["maps"]
    rng = ref.max() - ref.min()
    err = np.abs(maps.cpu().numpy() - ref).max()
    dpx = np.abs(pixels.cpu().numpy().astype(np.int64) - g["pixels"]).max()
    print("float32 step against the reference's run: depth %.3g of the range, pixels within %d" % (err / rng, dpx))
    assert err <= 1e-4 * rng and dpx <= 8
    assert np.array_equal(pixels.cpu().numpy(), np.stack([mo.pixels(m) for m in maps.cpu().numpy()]))


@pytest.mark.gpu
def test_fp16_step_is_as_close_as_the_per_frame_fp16_route(gpu, no_tf32, golden_dir):
    d, w = golden_dir
    ref = np.load(GOLDEN)["maps"]
    frames = mo.seeded_frames(3, 40, 192, seed=0)
    _, maps, pixels = midas.compute_depth_maps(d, w)
    weights = midas.network_weights(midas.check_state_dict(mo.seeded_state_dict(0), "seeded"), "cuda", True)
    oracle = np.stack([mo.predict(weights, f, True).astype(np.float32) for f in frames])
    ours, theirs = np.abs(maps.cpu().numpy() - ref).max(), np.abs(oracle - ref).max()
    print("fp16 against the float32 golden: step %.3g, per-frame fp16 route %.3g (range %.3g)"
          % (ours, theirs, ref.max() - ref.min()))
    assert ours <= 1.5 * theirs
    assert np.array_equal(pixels.cpu().numpy(), np.stack([mo.pixels(m) for m in maps.cpu().numpy()]))


@pytest.mark.gpu
def test_written_files_equal_the_returned_tensors(gpu, tmp_path, monkeypatch):
    frames = mo.seeded_frames(5, 436, 1024, seed=3)
    d = _write_frames(str(tmp_path / "img"), frames)
    w = str(tmp_path / "w.pt")
    torch.save(mo.seeded_state_dict(2), w)
    # a batch per frame, so the writer overlaps several batches; both calls batch alike, since in fp16 another batch
    # size can pick other cuDNN algorithms
    monkeypatch.setattr(midas, "_BUDGET", 1)
    paths, maps, pixels = midas.compute_depth_maps(d, w)
    out = str(tmp_path / "midas_depth")
    assert midas.main(["--image_dir", d, "--output_dir", out, "--model", w]) == 0
    for i, p in enumerate(paths):
        base = midas.output_base(out, p)
        raw = open(base + ".pfm", "rb").read()
        assert raw.startswith(b"Pf\n1024 436\n-1.000000\n")
        pfm = np.flipud(np.frombuffer(raw[len(b"Pf\n1024 436\n-1.000000\n"):], "<f4").reshape(436, 1024))
        assert np.array_equal(pfm, maps[i].cpu().numpy())
        png = cv2.imread(base + ".png", -1)
        assert png.dtype == np.uint16 and np.array_equal(png, pixels[i].cpu().numpy())
        # what motion_seg/load_cut_seq.py reads: a non-zero map in [0, 1]
        depth = cv2.imread(base + ".png", -1) / 65535.0
        assert depth.max() == 1.0 and np.count_nonzero(depth) > 0.5 * depth.size
    assert midas.main(["--image_dir", d, "--output_dir", out, "--model", w, "--skip_exists"]) == 0


@pytest.mark.gpu
def test_a_failed_write_raises_and_writes_no_later_batch(gpu, tmp_path, monkeypatch):
    """A directory where one .pfm file goes: the step raises the OSError naming it, writes no later batch and leaves
    no thread behind, and the command exits 1."""
    d = _write_frames(str(tmp_path / "img"), mo.seeded_frames(4, 40, 192, seed=0))
    w = str(tmp_path / "w.pt")
    torch.save(mo.seeded_state_dict(0), w)
    monkeypatch.setattr(midas, "_BUDGET", 1)       # a batch per frame
    out = str(tmp_path / "midas_depth")
    bad = os.path.join(out, "00001.pfm")
    os.makedirs(bad)
    before = set(threading.enumerate())
    with pytest.raises(OSError, match=re.escape(bad)):
        midas.write_depth_maps(d, out, w)
    assert [t.name for t in threading.enumerate() if t not in before] == []
    assert os.path.isfile(os.path.join(out, "00000.pfm")) and os.path.isfile(os.path.join(out, "00000.png"))
    assert not any(os.path.exists(os.path.join(out, "%05d.%s" % (i, e))) for i in (2, 3) for e in ("pfm", "png"))
    assert midas.main(["--image_dir", d, "--output_dir", out, "--model", w]) == 1
    assert [t.name for t in threading.enumerate() if t not in before] == []
