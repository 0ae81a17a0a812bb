"""The RAFT oracle (oracle/raft_oracle.py) against the reference's own RAFT (tests/golden/flow_small.npz, written by
tests/golden/make_flow_golden.py on the CPU), the flow image and .flo writer against the reference's bytes, and the
weight loader's refusals."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import raft_oracle as ro
from particlesfm_b200 import optical_flow as of

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flow_small.npz")


def test_oracle_equals_the_reference_raft():
    g = np.load(GOLD)
    frames = ro.seeded_frames(3, 123, 125, seed=0)
    with torch.no_grad():
        f1, b1, f2, b2 = ro.optical_flows(ro.seeded_state_dict(0), frames)
    for name, got in (("f1", f1), ("b1", b1), ("f2", f2), ("b2", b2)):
        ref = g[name]
        assert len(got) == len(ref)
        for a, b in zip(got, ref):
            # measured: 0 (the same torch CPU calls in the same order); the bound allows fp32 reordering
            assert np.abs(a.numpy() - b).max() <= 1e-4, (name, np.abs(a.numpy() - b).max())


def test_flow_image_equals_the_reference():
    g = np.load(GOLD)
    assert np.array_equal(ro.flow_to_image(g["f1"][0]), g["image"])


def test_flo_bytes_equal_the_reference(tmp_path):
    g = np.load(GOLD)
    p = str(tmp_path / "a.flo")
    of.write_flo(p, g["f1"][0])
    raw = open(p, "rb").read()
    assert len(raw) == int(g["flo_size"]) and raw[:12] == g["flo_head"].tobytes()
    assert hashlib.sha256(raw).hexdigest() == str(g["flo_sha256"])


def _save(tmp_path, sd):
    p = str(tmp_path / "w.pth")
    torch.save(sd, p)
    return p


def test_loader_accepts_the_dataparallel_prefix(tmp_path):
    sd = ro.seeded_state_dict(1)
    got = of.load_weights(_save(tmp_path, {"module." + k: v for k, v in sd.items()}))
    assert list(got) == list(of.state_shapes())
    assert all(torch.equal(got[k], sd[k]) for k in sd)


@pytest.mark.parametrize("why", ["small", "unexpected", "missing", "shape"])
def test_loader_refusals_name_the_key(tmp_path, why):
    sd = {"module." + k: v for k, v in ro.seeded_state_dict(1).items()}
    if why == "small":
        sd["module.update_block.gru.convz.weight"] = torch.zeros(96, 242, 3, 3)
        key = "update_block.gru.convz.weight"
    elif why == "unexpected":
        sd["module.extra.weight"] = torch.zeros(1)
        key = "extra.weight"
    elif why == "missing":
        del sd["module.cnet.layer2.0.norm3.running_var"]
        key = "cnet.layer2.0.norm3.running_var"
    else:
        sd["module.update_block.mask.2.weight"] = torch.zeros(576, 128, 1, 1)
        key = "update_block.mask.2.weight"
    with pytest.raises(ValueError, match=r"w\.pth: .*%s" % key.replace(".", r"\.")):
        of.load_weights(_save(tmp_path, sd))


def test_loader_refuses_a_missing_or_unreadable_file(tmp_path):
    with pytest.raises(ValueError, match="no such weights file"):
        of.load_weights(str(tmp_path / "none.pth"))
    (tmp_path / "bad.pth").write_bytes(b"not a checkpoint")
    with pytest.raises(ValueError, match="bad.pth: not a readable checkpoint"):
        of.load_weights(str(tmp_path / "bad.pth"))
