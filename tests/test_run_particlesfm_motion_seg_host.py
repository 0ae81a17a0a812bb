"""run_particlesfm's labelling route on the host: its file plan, the flags a --root_dir child gets, and the refusals
before anything is written."""
import os

import numpy as np
import pytest

from particlesfm_b200 import run_particlesfm as rp


@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("skip_sfm", [False, True])
def test_plan_of_the_labelling_route(tmp_path, keep, skip_sfm):
    p = rp.plan(str(tmp_path), skip_sfm, False, keep, motion_segmentation=True)
    assert p.route == "fused" and p.motion_seg
    assert p.stages() == ["flows_trajectories", "depth", "motion_seg"] + ([] if skip_sfm else ["sfm"])
    assert p.write_depth == keep and p.write_labeled == (keep or skip_sfm)
    assert not rp.plan(str(tmp_path), skip_sfm, False, keep).motion_seg       # the default keeps today's plan


def test_skip_exists_takes_the_labelled_track_set_to_sfm(tmp_path):
    os.makedirs(tmp_path / "trajectories_labeled")
    np.save(str(tmp_path / "trajectories_labeled" / "track.npy"), {})
    p = rp.plan(str(tmp_path), False, True, False, motion_segmentation=True)
    assert p.route == "labeled_npy" and p.stages() == ["sfm"]
    assert rp.plan(str(tmp_path), False, True, False).route == "fused"       # --assume_static ignores it


def test_child_args_forward_the_weights():
    args = rp.build_parser().parse_args(["--model", "w.pth", "--root_dir", "R", "--midas_model", "m.pt",
                                         "--motion_seg_model", "s.pth", "--window_size", "7", "--traj_max_num", "50"])
    child = rp.build_parser().parse_args(rp.child_args(args, "R/x"))
    assert (child.midas_model, child.motion_seg_model, child.window_size, child.traj_max_num) == ("m.pt", "s.pth", 7, 50)
    assert not child.assume_static


@pytest.mark.parametrize("missing", ["--midas_model", "--motion_seg_model"])
def test_one_weights_flag_alone_is_refused(tmp_path, capsys, missing):
    argv = ["--model", "w.pth", "-i", str(tmp_path), "-o", str(tmp_path / "out"), "--midas_model", "m.pt",
            "--motion_seg_model", "s.pth"]
    i = argv.index(missing)
    del argv[i:i + 2]
    assert rp.main(argv) == 2
    err = capsys.readouterr().err
    assert "motion segmentation" in err and "--assume_static" in err
    assert not os.path.exists(tmp_path / "out")
