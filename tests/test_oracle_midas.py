"""The MiDaS oracle (oracle/midas_oracle.py) against tests/golden/depth_small.npz, the reference's own run_midas on the
CPU (tests/golden/make_depth_golden.py): the host transform, the float32 network and upsampling, the PNG arithmetic,
and Resize.get_size; the product's host restatement of get_size against the same table."""
import os

import numpy as np
import pytest

from oracle import midas_oracle as mo
from particlesfm_b200 import midas

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "depth_small.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_transform_equals_the_references(golden):
    frames = mo.seeded_frames(3, 40, 192, seed=0)
    assert np.array_equal(mo.transform(frames[0]), golden["transform0"])


def test_float32_route_equals_the_golden(golden):
    import torch
    frames = mo.seeded_frames(3, 40, 192, seed=0)
    weights = midas.network_weights(midas.check_state_dict(mo.seeded_state_dict(0), "seeded"), "cpu", False)
    maps, pixels = mo.depth_maps(weights, frames, optimize=False)
    ref = golden["maps"]
    # the same torch calls on the same CPU: equal up to the order oneDNN picks for the convolutions
    assert np.abs(maps - ref).max() <= 1e-5 * (ref.max() - ref.min())
    # a pixel may move by one where the map moved by an ulp
    assert np.abs(pixels.astype(np.int64) - golden["pixels"]).max() <= 1
    assert np.array_equal(np.stack([mo.pixels(m) for m in ref]), golden["pixels"])
    assert float(golden["max_activation"]) < 60000.0
    assert (ref > 0).mean() > 0.9 and torch.is_grad_enabled()


def test_get_size_equals_the_table(golden):
    for w, h, nw, nh in golden["sizes"]:
        assert mo.get_size(int(w), int(h)) == (nw, nh), (w, h)
        assert midas.get_size(int(w), int(h)) == (nw, nh), (w, h)
    sizes = {(int(w), int(h)): (int(a), int(b)) for w, h, a, b in golden["sizes"]}
    assert sizes[(192, 40)] == (384, 64)           # 2.5 goes to 2: np.round's ties to even
    assert sizes[(1000, 40)] == (384, 0) and sizes[(1024, 436)] == (384, 160)
