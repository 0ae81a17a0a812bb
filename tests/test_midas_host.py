"""The depth step's host side (particlesfm_b200.midas): the weights' checks, the frame list and its refusals, the
output names, the command's exit statuses, skip_exists, the PFM bytes, and what the step does differently from the
reference (DESIGN.md §4.16), all without a device."""
import hashlib
import os

import cv2
import numpy as np
import pytest
import torch

from oracle import midas_oracle as mo
from particlesfm_b200 import _abi, device_count, launch_count, midas

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "depth_small.npz")


def _frames(d, names, size=(192, 40)):
    os.makedirs(d, exist_ok=True)
    for n in names:
        assert cv2.imwrite(os.path.join(d, n), np.full((size[1], size[0], 3), 90, np.uint8))
    return d


@pytest.fixture(scope="module")
def seeded():
    return mo.seeded_state_dict(1)


@pytest.fixture(scope="module")
def weights(tmp_path_factory, seeded):
    p = str(tmp_path_factory.mktemp("w") / "midas_v21-f6b98070.pt")
    torch.save(seeded, p)
    return p


def test_state_dict_checks(seeded, tmp_path):
    assert set(midas.check_state_dict(seeded, "w")) == {k for k in midas.state_shapes() if "num_batches" not in k}
    wrapped = {"optimizer": {}, "model": dict(seeded), "epoch": 3}
    p = str(tmp_path / "wrapped.pt")
    torch.save(wrapped, p)
    assert set(midas.load_weights(p)) == set(midas.check_state_dict(seeded, "w"))
    bad = dict(seeded)
    bad["scratch.output_conv.4.weight"] = torch.zeros(1, 32, 3, 3)
    with pytest.raises(ValueError, match="'scratch.output_conv.4.weight' has shape"):
        midas.check_state_dict(bad, "w")
    bad = dict(seeded)
    del bad["pretrained.layer3.22.bn3.running_var"]
    with pytest.raises(ValueError, match="missing key 'pretrained.layer3.22.bn3.running_var'"):
        midas.check_state_dict(bad, "w")
    bad = dict(seeded, extra=torch.zeros(1))
    with pytest.raises(ValueError, match="unexpected key 'extra'"):
        midas.check_state_dict(bad, "w")
    for key in ("pretrained.model.cls_token", "scratch.refinenet1.out_conv.weight"):
        with pytest.raises(ValueError, match="only midas_v21 is built"):
            midas.check_state_dict(dict(seeded, **{key: torch.zeros(1)}), "w")
    with pytest.raises(ValueError, match="no such weights file"):
        midas.load_weights(str(tmp_path / "none.pt"))


def test_frame_list_is_every_entry(tmp_path):
    d = _frames(str(tmp_path / "img"), ["b.png", "a.jpg", "c.bmp", "0.PNG"])
    paths, h, w = midas.frame_list(d)
    assert [os.path.basename(p) for p in paths] == ["0.PNG", "a.jpg", "b.png", "c.bmp"]
    assert (h, w) == (40, 192)
    os.makedirs(str(tmp_path / "empty"))
    assert midas.frame_list(str(tmp_path / "empty")) == ([], 0, 0)
    assert midas.output_base("/o", "/x/y/00012.png") == "/o/00012"
    assert midas.output_base("/o", "a.b.jpg") == "/o/a.b"


@pytest.mark.parametrize("why", ["text", "directory", "zero side", "sizes", "stem"])
def test_refusals_name_the_file_before_any_device_work(tmp_path, weights, why, monkeypatch):
    d = str(tmp_path / "img")
    _frames(d, ["0.png", "1.png"])
    if why == "text":
        open(os.path.join(d, "2.txt"), "w").write("not an image")
        bad = os.path.join(d, "2.txt")
    elif why == "directory":
        os.makedirs(os.path.join(d, "2"))
        bad = os.path.join(d, "2")
    elif why == "zero side":
        for n in ("0.png", "1.png"):
            _frames(d, [n], size=(1000, 40))      # get_size: 384 x 0
        bad = os.path.join(d, "0.png")
    elif why == "sizes":
        _frames(d, ["2.png"], size=(192, 41))
        bad = os.path.join(d, "2.png")
    else:
        _frames(d, ["1.jpg"])
        bad = os.path.join(d, "1.png")            # sorted after 1.jpg, whose outputs it would overwrite
    monkeypatch.setattr(midas, "_run", lambda *a: pytest.fail("device work after a refusal"))
    n0 = launch_count()
    with pytest.raises(ValueError, match="^" + bad.replace(".", r"\.") + ":"):
        midas.write_depth_maps(d, str(tmp_path / "out"), weights)
    with pytest.raises(ValueError, match="^" + bad.replace(".", r"\.") + ":"):
        midas.compute_depth_maps(d, weights)
    assert midas.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", weights]) == 2
    assert launch_count() == n0


def test_bad_weights_exit_2(tmp_path):
    d = _frames(str(tmp_path / "img"), ["0.png"])
    assert midas.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", str(tmp_path / "no.pt")]) == 2
    torch.save({"pretrained.model.cls_token": torch.zeros(1, 1, 1024)}, str(tmp_path / "dpt.pt"))
    assert midas.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", str(tmp_path / "dpt.pt")]) == 2


def test_skip_exists_skips_frames_whose_two_files_exist(tmp_path, weights, monkeypatch):
    d = _frames(str(tmp_path / "img"), ["0.png", "1.png", "2.jpg"])
    out = str(tmp_path / "depth")
    os.makedirs(out)
    for n in ("0.pfm", "0.png", "1.pfm", "1.png", "2.pfm", "2.png"):
        open(os.path.join(out, n), "wb").close()
    monkeypatch.setattr(midas, "_run", lambda *a: pytest.fail("nothing left to compute"))
    assert midas.write_depth_maps(d, out, weights, skip_exists=True) == 0
    os.remove(os.path.join(out, "1.png"))
    seen = []
    monkeypatch.setattr(midas, "_require_device", lambda: None)
    monkeypatch.setattr(midas, "_run", lambda paths, h, w, sd, optimize, sink: seen.extend(paths))
    assert midas.write_depth_maps(d, out, weights, skip_exists=True) == 1
    assert seen == [os.path.join(d, "1.png")]
    seen.clear()
    assert midas.write_depth_maps(d, out, weights) == 3 and len(seen) == 3


def test_pfm_bytes_are_the_references():
    g = np.load(GOLDEN)
    data = midas.pfm_bytes(np.flipud(g["maps"][0]))
    assert data[:32] == g["pfm_head"].tobytes() and len(data) == int(g["pfm_size"])
    assert hashlib.sha256(data).hexdigest() == str(g["pfm_sha256"])
    assert data.startswith(b"Pf\n192 40\n-1.000000\n")


def test_reference_fp16_pixels_are_zeros():
    """The reference's write_depth on a float16 prediction (its optimize route on a CUDA device): 65535 * float16 stays
    float16 under this numpy's promotion, overflows to inf, and the map casts to zeros.  The product quantises the
    float32 map instead, as the reference does for a float32 prediction."""
    g = np.load(GOLDEN)
    pred16 = g["maps"][0].astype(np.float16)
    with np.errstate(over="ignore", invalid="ignore"):
        assert (65535 * (pred16 - pred16.min())).dtype == np.float16
    assert not mo.reference_fp16_pixels(pred16).any()
    ours = mo.pixels(pred16.astype(np.float32))
    assert ours.max() == 65535 and ours.min() == 0 and np.count_nonzero(ours) > 0.9 * ours.size
    # the product's arithmetic on the float32 map is the reference's float32 write_depth
    m = g["maps"][1]
    assert np.array_equal(mo.pixels(m), (65535 * (m - m.min()) / (m.max() - m.min())).astype("uint16"))
    assert np.array_equal(mo.pixels(m), g["pixels"][1])


def test_constant_map_gives_zero_pixels():
    """The reference raises AttributeError here (depth.type); the product writes a zero PNG."""
    assert not mo.pixels(np.full((4, 5), 0.25, np.float32)).any()


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_no_device_is_a_library_error(tmp_path, weights):
    d = _frames(str(tmp_path / "img"), ["0.png"])
    assert midas.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", weights]) == 1
    with pytest.raises(midas._lib.PsfmError) as e:
        midas.compute_depth_maps(d, weights)
    assert e.value.code == _abi.PSFM_ERR_NO_DEVICE
