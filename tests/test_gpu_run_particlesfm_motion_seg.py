"""run_particlesfm without --assume_static on the GPU: flows -> track set -> depth maps -> labeller -> SfM without the
dynamic observations, on the seeded room clip with seeded MiDaS and labeller weights."""
import os
import sys

import pytest
import torch

from oracle import midas_oracle as mo, motion_seg_oracle as so
from particlesfm_b200 import run_particlesfm as rp, sfm, synthetic as syn

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_run_particlesfm import ROOM, _write_room   # noqa: E402
from test_gpu_sfm import _tables_of   # noqa: E402

pytestmark = pytest.mark.gpu


def test_default_route_equals_sfm_on_the_kept_labelled_track_set(gpu, tmp_path):
    frames, flows, _, _ = syn.make_room_sequence(**ROOM)
    img = _write_room(str(tmp_path), frames)
    midas_w, seg_w = str(tmp_path / "midas.pt"), str(tmp_path / "seg.pth")
    torch.save(mo.seeded_state_dict(0), midas_w)
    torch.save({"model_state_dict": so.seeded_state_dict(4)}, seg_w)
    out = str(tmp_path / "out")
    rep = rp.particlesfm(img, out, flow_source=rp.array_flow_source(flows), keep_intermediate=True, quiet=True,
                         assume_static=False, midas_model=midas_w, motion_seg_model=seg_w, window_size=5)
    assert [n for n, _ in rep.stages] == ["flows_trajectories", "track_npy", "depth", "motion_seg", "sfm"]
    assert rep.success, (rep.sfm.failed_stage, rep.sfm.reason)
    assert os.path.getsize(os.path.join(out, "motion_seg.mp4")) > 0
    assert len([f for f in os.listdir(os.path.join(out, "midas_depth")) if f.endswith(".png")]) == ROOM["n_frames"]
    assert os.path.isdir(os.path.join(out, "sfm", "model"))
    labelled = os.path.join(out, "trajectories_labeled")
    staged = str(tmp_path / "staged")
    srep = sfm.main_global_sfm(os.path.join(staged, "sfm"), img, labelled, remove_dynamic=True)
    assert srep.success
    got, ref = _tables_of(os.path.join(out, "sfm", "database.db")), _tables_of(os.path.join(staged, "sfm", "database.db"))
    assert sorted(got) == sorted(ref)
    for t in ref:
        assert got[t] == ref[t], t
    # --skip_exists takes the kept labelled track set straight to the SfM step
    again = rp.particlesfm(img, out, flow_source=rp.array_flow_source(flows), skip_exists=True, quiet=True,
                           assume_static=False, midas_model=midas_w, motion_seg_model=seg_w, window_size=5)
    assert again.plan.route == "labeled_npy" and [n for n, _ in again.stages] == ["sfm"]
