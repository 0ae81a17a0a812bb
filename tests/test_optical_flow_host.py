"""The optical-flow stage's host side (particlesfm_b200.optical_flow): the frame list and its refusals, the output
names, the command's exit statuses and skip_exists, all before any device work."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import raft_oracle as ro
from particlesfm_b200 import _abi, device_count, launch_count, optical_flow as of


def _frames(d, names, size=(125, 123), mode="RGB"):
    os.makedirs(d, exist_ok=True)
    for n in names:
        Image.fromarray(np.full((size[1], size[0], 3), 90, np.uint8)).convert(mode).save(os.path.join(d, n))
    return d


@pytest.fixture
def weights(tmp_path):
    p = str(tmp_path / "raft-things.pth")
    torch.save({"module." + k: v for k, v in ro.seeded_state_dict(2).items()}, p)
    return p


def test_frame_list_is_the_references(tmp_path):
    d = _frames(str(tmp_path / "img"), ["b.png", "a.jpg", "c.png", "0.jpg"])
    for n in ("d.jpeg", "e.PNG", "f.txt"):
        open(os.path.join(d, n), "wb").close()
    paths, h, w = of.frame_list(d)
    assert [os.path.basename(p) for p in paths] == ["0.jpg", "a.jpg", "b.png", "c.png"]
    assert (h, w) == (123, 125)


def test_output_names_map_as_the_reference():
    assert of.output_names("/x/y/00012.png") == ("00012.flo", "00012-bk.flo", "00012.png")
    assert of.output_names("frame.jpg") == ("frame.flo", "frame-bk.flo", "frame.jpg")
    assert of.output_names("a.png.jpg") == ("a.flo.flo", "a-bk.flo-bk.flo", "a.png.jpg")


def test_pairs_follow_the_two_scripts():
    assert of._pairs(4, True) == [(0, 1), (0, 2), (1, 1), (1, 2), (2, 1)]
    assert of._pairs(4, False) == [(0, 1), (1, 1), (2, 1)]
    assert of.padding(436, 1024) == [0, 0, 2, 2] and of.padding(123, 125) == [1, 2, 2, 3]


@pytest.mark.parametrize("why", ["one image", "rgba", "grey", "palette", "sizes", "small", "not an image"])
def test_refusals_name_the_file_before_any_device_work(tmp_path, weights, why, monkeypatch):
    d = str(tmp_path / "img")
    _frames(d, ["0.png", "1.png"])
    if why == "one image":
        os.remove(os.path.join(d, "1.png"))
        bad = d
    elif why in ("rgba", "grey", "palette"):
        _frames(d, ["2.png"], mode={"rgba": "RGBA", "grey": "L", "palette": "P"}[why])
        bad = os.path.join(d, "2.png")
    elif why == "sizes":
        _frames(d, ["2.png"], size=(126, 123))
        bad = os.path.join(d, "2.png")
    elif why == "small":
        for n in ("0.png", "1.png"):
            _frames(d, [n], size=(125, 120))
        bad = os.path.join(d, "0.png")
    else:
        open(os.path.join(d, "2.jpg"), "wb").write(b"not a jpeg")
        bad = os.path.join(d, "2.jpg")
    monkeypatch.setattr(of, "_run", lambda *a: pytest.fail("device work after a refusal"))
    n0 = launch_count()
    with pytest.raises(ValueError, match="^" + bad.replace(".", r"\.") + ":"):
        of.write_optical_flows(d, str(tmp_path / "out"), weights)
    with pytest.raises(ValueError, match="^" + bad.replace(".", r"\.") + ":"):
        of.compute_optical_flows(d, weights)
    assert of.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", weights]) == 2
    assert launch_count() == n0


def test_bad_weights_exit_2(tmp_path):
    d = _frames(str(tmp_path / "img"), ["0.png", "1.png"])
    assert of.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", str(tmp_path / "none.pth")]) == 2


def test_skip_exists_skips_pairs_whose_three_files_exist(tmp_path, weights, monkeypatch):
    d = _frames(str(tmp_path / "img"), ["0.png", "1.png", "2.jpg"])
    out = str(tmp_path / "flows")
    for sub, names in (("flow_f", ["0.flo", "1.flo"]), ("flow_b", ["0-bk.flo", "1-bk.flo"]), ("flow_imgs", ["0.png", "1.png"]),
                       ("flow_f2", ["0.flo"]), ("flow_b2", ["0-bk.flo"]), ("flow_imgs2", ["0.png"])):
        os.makedirs(os.path.join(out, sub))
        for n in names:
            open(os.path.join(out, sub, n), "wb").close()
    monkeypatch.setattr(of, "_run", lambda *a: pytest.fail("nothing left to compute"))
    assert of.write_optical_flows(d, out, weights, skip_exists=True) == 0
    os.remove(os.path.join(out, "flow_b", "1-bk.flo"))
    seen = []
    monkeypatch.setattr(of, "_require_device", lambda: None)
    monkeypatch.setattr(of, "_run", lambda paths, h, w, sd, pairs, sink: seen.extend(pairs))
    assert of.write_optical_flows(d, out, weights, skip_exists=True) == 1
    assert seen == [(1, 1)]


@pytest.mark.skipif(device_count() > 0, reason="checks the refusal without a device")
def test_no_device_is_a_library_error(tmp_path, weights):
    d = _frames(str(tmp_path / "img"), ["0.png", "1.png"])
    assert of.main(["--image_dir", d, "--output_dir", str(tmp_path / "o"), "--model", weights]) == 1
    with pytest.raises(of._lib.PsfmError) as e:
        of.compute_optical_flows(d, weights)
    assert e.value.code == _abi.PSFM_ERR_NO_DEVICE
