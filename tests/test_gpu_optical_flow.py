"""The optical-flow stage on the GPU (csrc/optical_flow.cu, particlesfm_b200.optical_flow) against the oracle's
reference call structure (oracle/raft_oracle.py) run on the same GPU: the kernels one by one, then the whole stage,
then the point-trajectory stage fed from the written directory and from the returned tensors."""
import os
import re
import sys
import threading

import numpy as np
import pytest
import torch

from oracle import raft_oracle as ro
from particlesfm_b200 import optical_flow as of, point_trajectory as pt, tracker

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_gpu_tracker_stage import _same   # noqa: E402


@pytest.fixture
def no_tf32():
    """The convolutions in full fp32 while a test runs, so the two call structures differ by reordering only."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _fmaps(h, w, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return [torch.randn((256, h, w), device="cuda", generator=g) for _ in range(2)]


def _pyramids(f1, f2):
    S = of.corr_pyramid_floats(*f1.shape[1:])
    fwd, bwd = torch.empty(S, device="cuda"), torch.empty(S, device="cuda")
    of.corr_pyramids(f1, f2, fwd, bwd)
    return fwd, bwd


def _levels(pyr, h, w):
    out, off, hl, wl = [], 0, h, w
    for _ in range(4):
        n = h * w * hl * wl
        out.append(pyr[off:off + n].view(h * w, 1, hl, wl))
        off, hl, wl = off + n, hl // 2, wl // 2
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(16, 16), (55, 128), (60, 107)])
def test_pyramids_equal_two_separate_products(gpu, no_tf32, h, w):
    f1, f2 = _fmaps(h, w, h + w)
    fwd, bwd = _pyramids(f1, f2)
    for mine, ref in ((fwd, ro.corr_pyramid(f1[None], f2[None])), (bwd, ro.corr_pyramid(f2[None], f1[None]))):
        for a, b in zip(_levels(mine, h, w), ref):
            # values ~ 1; the backward product sums in another order: a few fp32 units
            assert (a - b).abs().max().item() <= 1e-4 * max(1.0, b.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("h,w", [(16, 16), (16, 17)])
def test_lookup_equals_grid_sample(gpu, no_tf32, h, w):
    f1, f2 = _fmaps(h, w, 7)
    fwd, bwd = _pyramids(f1, f2)
    g = torch.Generator(device="cuda").manual_seed(3)
    P = 2
    coords = ro.of.coords_grid(P, h, w, "cuda") + 6 * torch.randn((P, 2, h, w), device="cuda", generator=g)
    coords[0, :, 0, :3] = torch.tensor([[-30.0, -4.5, w + 3.25], [h + 9.0, -0.5, 2.0]], device="cuda")  # out of range
    pyr = torch.stack([fwd, bwd])
    got = of.corr_lookup(pyr, coords, torch.empty((P, 324, h, w), device="cuda"))
    for p, one in enumerate((fwd, bwd)):
        ref = ro.lookup(_levels(one, h, w), coords[p:p + 1])
        assert (got[p] - ref[0]).abs().max().item() <= 1e-5 * max(1.0, ref.abs().max().item())
    # the window order: channel a * 9 + b of level 0 moves x by a - 4 (and y by b - 4)
    c = torch.zeros((1, 2, h, w), device="cuda")
    c[0, 0], c[0, 1] = 8.0, 8.0
    out = of.corr_lookup(fwd[None], c, torch.empty((1, 324, h, w), device="cuda"))
    lvl0 = _levels(fwd, h, w)[0]
    assert out[0, 1 * 9 + 4, 0, 0].item() == lvl0[0, 0, 8, 5].item()      # a = 1: x = 8 - 3
    assert out[0, 4 * 9 + 1, 0, 0].item() == lvl0[0, 0, 5, 8].item()      # b = 1: y = 8 - 3


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,pad", [(16, 16, [1, 2, 2, 3]), (55, 128, [0, 0, 2, 2]), (60, 107, [1, 1, 0, 0])])
def test_upsampling_equals_the_references(gpu, h, w, pad):
    g = torch.Generator(device="cuda").manual_seed(h)
    flow = 3 * torch.randn((3, 2, h, w), device="cuda", generator=g)
    mask = 4 * torch.randn((3, 576, h, w), device="cuda", generator=g)
    got = of.upsample(flow, mask, pad)
    ref = ro.upsample_flow(flow, 0.25 * mask)
    H, W = ref.shape[2:]
    ref = ref[:, :, pad[2]:H - pad[3], pad[0]:W - pad[1]].permute(0, 2, 3, 1)
    assert got.shape == ref.shape
    assert (got - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()


@pytest.mark.gpu
def test_flow_images_equal_the_restatement(gpu):
    g = np.load(os.path.join(HERE, "golden", "flow_small.npz"))
    rng = np.random.default_rng(5)
    maps = [g["f1"][0], g["b1"][1], g["f2"][0], (rng.standard_normal((436, 1024, 2)) * 7).astype(np.float32),
            np.zeros((40, 30, 2), np.float32), (rng.standard_normal((480, 854, 2)) * 1e-3).astype(np.float32)]
    for m in maps:
        got = of.flow_to_image(torch.from_numpy(m)[None].cuda())[0].cpu().numpy()
        ref = ro.flow_to_image(m)
        assert np.array_equal(got, ref), (m.shape, int((got != ref).sum()))
    assert np.array_equal(ro.flow_to_image(g["f1"][0]), g["image"])


def _write_frames(d, frames):
    from PIL import Image
    os.makedirs(d, exist_ok=True)
    for i, f in enumerate(frames):
        Image.fromarray(f).save(os.path.join(d, "%05d.png" % i))
    return d


# measured on an H100 80GB HBM3 at 700 W with TF32 off: see DESIGN.md §4.14
FLOW_TOL = 2e-3


@pytest.mark.gpu
@pytest.mark.parametrize("n,h,w", [(3, 123, 125), (5, 436, 1024)])
def test_stage_equals_the_oracle(gpu, no_tf32, tmp_path, n, h, w):
    frames = ro.seeded_frames(n, h, w, seed=n)
    sd = ro.seeded_state_dict(0)
    weights = str(tmp_path / "w.pth")
    torch.save({"module." + k: v for k, v in sd.items()}, weights)
    d = _write_frames(str(tmp_path / "img"), frames)
    got = of.compute_optical_flows(d, weights)
    with torch.no_grad():
        ref = ro.optical_flows({k: v.cuda() for k, v in sd.items()}, frames)
    err = 0.0
    for a_list, b_list in zip(got, ref):
        assert len(a_list) == len(b_list)
        for a, b in zip(a_list, b_list):
            assert a.shape == (h, w, 2) and a.dtype == torch.float32 and a.is_cuda
            err = max(err, (a - b).abs().max().item())
    print("max flow difference against the oracle: %.3g px" % err)
    assert err <= FLOW_TOL
    # the written directory: .flo bytes of the returned maps, images of the forward ones
    out = str(tmp_path / "flows")
    assert of.main(["--image_dir", d, "--output_dir", out, "--model", weights]) == 0
    for s, (ff, fb) in ((1, got[:2]), (2, got[2:])):
        sub = "" if s == 1 else "2"
        for t in range(len(ff)):
            f = pt.read_flo(os.path.join(out, "flow_f" + sub, "%05d.flo" % t))
            b = pt.read_flo(os.path.join(out, "flow_b" + sub, "%05d-bk.flo" % t))
            assert np.array_equal(f, ff[t].cpu().numpy()) and np.array_equal(b, fb[t].cpu().numpy())
            import cv2
            img = cv2.imread(os.path.join(out, "flow_imgs" + sub, "%05d.png" % t))
            assert np.array_equal(img, ro.flow_to_image(f))


@pytest.mark.gpu
def test_one_pair_per_batch_gives_the_same_flows(gpu, no_tf32, tmp_path, monkeypatch):
    d = _write_frames(str(tmp_path / "img"), ro.seeded_frames(5, 123, 125, seed=2))
    weights = str(tmp_path / "w.pth")
    torch.save(ro.seeded_state_dict(3), weights)
    whole = of.compute_optical_flows(d, weights)
    monkeypatch.setattr(of, "_BUDGET", 1)          # every pair a batch of its own: frames kept across batches
    assert of.pairs_per_batch(123, 125) == 1
    split = of.compute_optical_flows(d, weights)
    for a_list, b_list in zip(whole, split):
        for a, b in zip(a_list, b_list):
            assert (a - b).abs().max().item() <= 1e-4


@pytest.mark.gpu
def test_point_trajectory_from_the_directory_equals_the_tensors(gpu, tmp_path):
    frames = ro.seeded_frames(5, 123, 125, seed=9)
    weights = str(tmp_path / "w.pth")
    torch.save(ro.seeded_state_dict(4), weights)
    d = _write_frames(str(tmp_path / "img"), frames)
    flows = of.compute_optical_flows(d, weights)
    dev = tracker.main_connect_point_trajectories_device(*flows)
    out = str(tmp_path / "flows")
    assert of.write_optical_flows(d, out, weights) == 4 + 3
    arrays = pt.main_connect_point_trajectories(out, str(tmp_path / "traj"))
    assert arrays.ids.shape[0] > 0
    _same(arrays.to_dict(), dev.to_dict())


@pytest.mark.gpu
def test_a_failed_write_raises_and_writes_no_later_batch(gpu, tmp_path, monkeypatch):
    """A directory where one .flo file goes: the step raises the OSError naming it, writes no later batch and leaves
    no thread behind, and the command exits 1."""
    d = _write_frames(str(tmp_path / "img"), ro.seeded_frames(5, 123, 125, seed=2))
    weights = str(tmp_path / "w.pth")
    torch.save(ro.seeded_state_dict(3), weights)
    monkeypatch.setattr(of, "_BUDGET", 1)          # a batch per pair
    out = str(tmp_path / "flows")
    bad = os.path.join(out, "flow_f", "00001.flo")
    os.makedirs(bad)
    pairs = of._pairs(5, True)
    files = of.flow_files(of.frame_list(d)[0], out)
    before = set(threading.enumerate())
    with pytest.raises(OSError, match=re.escape(bad)):
        of.write_optical_flows(d, out, weights)
    assert [t.name for t in threading.enumerate() if t not in before] == []
    k = pairs.index((1, 1))
    assert all(os.path.isfile(f) for p in pairs[:k] for f in files(*p))
    assert not any(os.path.exists(f) for p in pairs[k + 1:] for f in files(*p))
    assert of.main(["--image_dir", d, "--output_dir", out, "--model", weights]) == 1
    assert [t.name for t in threading.enumerate() if t not in before] == []
