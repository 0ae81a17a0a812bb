"""Global rotation averaging on the GPU (init_geometry.estimate_global_rotations, csrc/rotation_averaging.cu) against
the numpy restatement (oracle/rotation_oracle.py, pinned by tests/test_oracle_rotations.py)."""
import numpy as np
import pytest

from oracle import init_oracle as io, rotation_oracle as ro
from particlesfm_b200 import handoff, init_geometry, synthetic as syn

pytestmark = pytest.mark.gpu

FIXTURES = {
    "exact": dict(num_images=25, seed=11),
    "outliers": dict(num_images=30, noise_deg=1.0, outlier_fraction=0.2, seed=1),
    "banded": dict(num_images=120, graph="banded", band=10, noise_deg=0.5, seed=2),
    "two_components": dict(num_images=40, graph="two_components", num_isolated=3, unposed_fraction=0.2, noise_deg=0.5,
                           seed=4),
    "two_images": dict(num_images=2, noise_deg=0.3, seed=3),
    "complete_200": dict(num_images=200, noise_deg=1.0, outlier_fraction=0.1, seed=5),
}


def _angle(q1, q2):
    return np.linalg.norm(ro.quaternion_to_angle_axis(ro.concatenate_quaternions(q1, ro.invert_quaternion(q2))))


def _compare(g, dev, ref):
    assert dev.success and ref["success"]
    s = dev.summary
    assert s["num_l1_rounds"] == ref["l1_rounds"]
    assert s["admm_iterations"] == ref["admm_iterations"]
    assert s["num_irls_iterations"] == ref["irls_iterations"]
    assert s["gauge_image"] == ref["gauge_image"]
    assert np.array_equal(dev.pair_kept, ref["pair_kept"])
    assert np.array_equal(dev.has_orientation, ref["has_orientation"])
    for f in np.nonzero(ref["has_orientation"])[0]:
        assert _angle(dev.orientations[f], ref["orientations"][f]) <= 1e-9, f


@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_matches_the_restatement(gpu, name):
    g = syn.make_view_graph(**FIXTURES[name])
    args = dict(num_images=g["num_images"], pair_images=g["pair_images"], qvec=g["qvec"],
                num_correspondences=g["num_correspondences"], has_pose=g["has_pose"])
    ref = ro.estimate_global_rotations(**args)
    # no pair within 1e-6 of the 5 degree filter threshold: the kept set is decided with margin
    ang = ref["residual_angles"][ref["residual_angles"] >= 0]
    assert np.abs(ang - np.deg2rad(5.0)).min() > 1e-6
    dev = init_geometry.estimate_global_rotations(**args)
    _compare(g, dev, ref)
    if name == "outliers":
        assert not (dev.pair_kept & g["outlier"]).any()
    again = init_geometry.estimate_global_rotations(**args)
    assert np.array_equal(again.orientations, dev.orientations) and np.array_equal(again.pair_kept, dev.pair_kept)


def test_exact_rotations_are_recovered(gpu):
    g = syn.make_view_graph(**FIXTURES["exact"])
    dev = init_geometry.estimate_global_rotations(g["num_images"], g["pair_images"], g["qvec"], g["num_correspondences"])
    gauge = dev.summary["gauge_image"]
    for f in range(g["num_images"]):
        truth = ro.concatenate_quaternions(ro.invert_quaternion(g["truth"][gauge]), g["truth"][f])
        assert _angle(dev.orientations[f], truth) <= 1e-12
    assert dev.pair_kept.all()


def test_chain_from_two_view_scene_to_known_rotation_translations(gpu):
    scene, qvec, tvec, cam = syn.make_two_view_scene(800, 8, 4000, seed=7)
    names, ids = ["%05d.png" % i for i in range(8)], list(range(1, 9))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(scene, 8))
    args = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    poses = init_geometry.estimate_relative_poses(**args)
    rot_args = dict(num_images=8, pair_images=args["pair_images"], qvec=poses.qvec,
                    num_correspondences=np.diff(args["inlier_ptr"]), has_pose=poses.estimated)
    dev = init_geometry.estimate_global_rotations(**rot_args)
    ref = ro.estimate_global_rotations(**rot_args)
    _compare(None, dev, ref)
    # error against the truth within what the restatement itself reaches on the same inputs (plus 1e-9 rad)
    gauge = dev.summary["gauge_image"]
    truth = [ro.concatenate_quaternions(ro.invert_quaternion(qvec[gauge]), qvec[f]) for f in range(8)]
    for f in range(8):
        assert _angle(dev.orientations[f], truth[f]) <= _angle(ref["orientations"][f], truth[f]) + 1e-9
    # the orientations feed the known-rotation pairwise translations
    pts = []
    kp_ptr, kps = args["keypoint_ptr"], args["keypoints"].astype(np.float64)
    f0, cx, cy = cam
    # the widest baselines: every point lies well inside max_depth, so the translation's sign is decided with margin
    pairs = []
    kept = np.nonzero(dev.pair_kept)[0]
    gap = np.abs(np.diff(args["pair_images"][kept], axis=1)[:, 0])
    for p in kept[np.argsort(-gap, kind="stable")][:5]:
        a, b = args["pair_images"][p]
        pairs.append((a, b))
        m = args["inlier_matches"][args["inlier_ptr"][p]:args["inlier_ptr"][p + 1]]
        x1 = (kps[kp_ptr[a] + m[:, 0]] - [cx, cy]) / f0
        x2 = (kps[kp_ptr[b] + m[:, 1]] - [cx, cy]) / f0
        pts.append((x1, x2, dev.orientations[a], dev.orientations[b]))
    t = init_geometry.batch_optimize_relative_position_with_known_rotation(pts)
    for k, (x1, x2, q1, q2) in enumerate(pts):
        ref_t = io.optimize_relative_position_with_known_rotation(x1, x2, ref["orientations"][pairs[k][0]],
                                                                  ref["orientations"][pairs[k][1]])
        assert np.abs(t[k] - ref_t).max() <= 1e-6, k
