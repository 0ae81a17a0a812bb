"""oracle/motion_seg_oracle.py against tests/golden/motion_seg_small.npz, which the reference's own
main_motion_segmentation wrote on the CPU (tests/golden/make_motion_seg_golden.py): the labelled dict exactly, the
windows' encoder features and logits within float32 tolerance, and the video frames' SHA-256 exactly."""
import hashlib
import os

import numpy as np
import pytest

import oracle.motion_seg_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "motion_seg_small.npz")
CASES = [dict(n=12, h=96, w=160, window=5, cap=100000, trajs=200, seed=17),
         dict(n=12, h=96, w=160, window=5, cap=30, trajs=200, seed=17),
         dict(n=6, h=300, w=500, window=10, cap=100000, trajs=150, seed=5)]


@pytest.mark.parametrize("c", range(len(CASES)))
def test_oracle_equals_the_reference(c):
    g = np.load(GOLDEN)
    case = CASES[c]
    frames = O.seeded_frames(case["n"], case["h"], case["w"], seed=9)
    px = O.seeded_depth_pixels(case["n"], case["h"], case["w"], seed=8)
    tracks = O.seeded_track_set(case["trajs"], case["n"], case["h"], case["w"], case["seed"])
    got, wins, video = O.label((case["h"], case["w"]), px, tracks, O.seeded_state_dict(4), case["window"],
                               case["cap"], frames)
    keys = list(got)
    assert [int(k) for k in keys] == g["keys_%d" % c].tolist()
    assert all(type(k) is int for k in keys) == bool(g["key_int_%d" % c])
    ptr = g["ptr_%d" % c]
    for i, k in enumerate(keys):
        s, e = ptr[i], ptr[i + 1]
        assert np.array_equal(got[k]["frame_ids"], g["frames_%d" % c][s:e])
        assert np.array_equal(got[k]["labels"], g["labels_%d" % c][s:e])
        assert np.array_equal(got[k]["locations"], g["locations_%d" % c][s:e])
    assert len(wins) == len([f for f in g.files if f.startswith("logit_%d_" % c)])
    for w, (feat, logit, _) in enumerate(wins):
        np.testing.assert_allclose(feat, g["feat_%d_%d" % (c, w)], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(logit, g["logit_%d_%d" % (c, w)], rtol=1e-5, atol=1e-5)
    assert [hashlib.sha256(np.ascontiguousarray(f).tobytes()).hexdigest() for f in video] == g["sha_%d" % c].tolist()
