"""Global position estimation and pairwise translations on the GPU (init_geometry.estimate_global_positions /
optimize_pairwise_translations, csrc/position_estimation.cu and csrc/init_geometry.cu) against the numpy restatement
(oracle/position_oracle.py, pinned by tests/test_oracle_positions.py)."""
import numpy as np
import pytest

from oracle import position_oracle as po, rotation_oracle as ro
from particlesfm_b200 import handoff, init_geometry, launch_count, synthetic as syn

pytestmark = pytest.mark.gpu

FIXTURES = {
    "exact": dict(num_images=25, seed=11),
    "outliers": dict(num_images=30, direction_noise_deg=1.0, direction_outlier_fraction=0.2, seed=1),
    "banded": dict(num_images=120, graph="banded", band=10, direction_noise_deg=0.5, seed=2),
    "two_images": dict(num_images=2, direction_noise_deg=0.3, seed=3),
    "complete_200": dict(num_images=200, direction_noise_deg=1.0, direction_outlier_fraction=0.1, seed=5),
    "unused_pairs": dict(num_images=40, graph="banded", band=6, direction_noise_deg=0.5, seed=4),
    "outliers_stops_mid_chunk": dict(num_images=30, direction_noise_deg=1.0, direction_outlier_fraction=0.2, seed=1),
    # long videos: S of 2,997 unknowns, and of 8,190 at the accepted bound of 2,731 views.  Seed 2 keeps every stopping
    # test at least 1e-2 relative away from its bound at both sizes.
    "banded_1000": dict(num_images=1000, graph="banded", band=10, direction_noise_deg=0.5, seed=2),
    "banded_2731": dict(num_images=2731, graph="banded", band=10, direction_noise_deg=0.5, seed=2),
}
# With the default options only two_images passes the stopping test (at its first iteration); these options make it
# fire at iteration 702, 30 iterations into a chunk of 32, so the test decides the count and the done flag must stop
# the two iterations queued after it in that chunk.
OPTIONS = {"outliers_stops_mid_chunk": dict(absolute_tolerance=1e-3, relative_tolerance=0.05)}


def _args(name):
    g = syn.make_view_graph(**FIXTURES[name])
    args = dict(num_images=g["num_images"], pair_images=g["pair_images"], tvec=g["tvec"], orientations=g["truth"])
    if name == "unused_pairs":
        used = np.random.default_rng(9).random(len(g["pair_images"])) >= 0.3
        used[np.abs(np.diff(g["pair_images"], axis=1)[:, 0]) == 1] = True     # the chain keeps the graph connected
        args["pair_used"] = used
    return g, args


def _options(name):
    return OPTIONS.get(name, {})


def _assert_margin(ref):
    """Every stopping test is decided with margin: no norm within 1e-6 relative of its bound."""
    h = np.array(ref["history"])
    assert (np.abs(h[:, 0] / h[:, 1] - 1) > 1e-6).all() and (np.abs(h[:, 2] / h[:, 3] - 1) > 1e-6).all()


def _compare(dev, ref):
    s = dev.summary
    assert s["admm_iterations"] == ref["iterations"] and bool(s["converged"]) == ref["converged"]
    # the last stopping test's four norms, each to 1e-9 of the larger of itself and its bound (a residual near zero
    # is a difference of O(bound) terms)
    r, pe, sn, de = ref["history"][-1]
    for key, val, bound in (("primal_residual", r, pe), ("primal_tolerance", pe, pe), ("dual_residual", sn, de),
                            ("dual_tolerance", de, de)):
        assert abs(s[key] - val) <= 1e-9 * max(abs(val), bound), (key, s[key], val)
    assert s["gauge_image"] == ref["gauge_image"]
    assert np.array_equal(dev.has_position, ref["has_position"])
    c = ref["positions"][ref["has_position"]]
    extent = np.linalg.norm(c - c.mean(0), axis=1).max()
    assert np.abs(dev.positions - ref["positions"]).max() <= 1e-9 * extent
    assert np.abs(dev.image_tvec - ref["image_tvec"]).max() <= 1e-9 * extent
    assert np.abs(dev.scales - ref["scales"]).max() <= 1e-9 * np.abs(ref["scales"]).max()


@pytest.mark.parametrize("name", list(FIXTURES))
def test_device_matches_the_restatement(gpu, name):
    g, args = _args(name)
    ref = po.estimate_global_positions(**args, options=_options(name))
    _assert_margin(ref)
    if name in OPTIONS:
        assert ref["converged"] and ref["iterations"] % 32 != 0
    opts = init_geometry.ConstrainedL1SolverOptions(**_options(name))
    args["options"] = opts
    n0 = launch_count()
    dev = init_geometry.estimate_global_positions(**args)
    s = dev.summary
    # 4 launches to build, factor and invert S, 4 per queued ADMM iteration (chunks of 32)
    queued = min(1000, -(-s["admm_iterations"] // 32) * 32)
    assert s["admm_iterations_queued"] == queued
    assert s["num_launches"] == 4 + 4 * queued == launch_count() - n0
    _compare(dev, ref)
    again = init_geometry.estimate_global_positions(**args)
    for k in ("positions", "image_tvec", "scales"):
        assert np.array_equal(getattr(again, k), getattr(dev, k)), k
    if name == "exact":
        pos = dev.positions
        assert syn.umeyama_ate(pos, g["centres"]) <= 1e-8 * np.linalg.norm(g["centres"] - g["centres"].mean(0), axis=1).max()


def test_tight_options_reach_the_linear_program_optimum(gpu):
    from test_oracle_positions import TIGHT, _lp_optimum
    g = syn.make_view_graph(8, direction_noise_deg=2.0, direction_outlier_fraction=0.2, seed=3)
    dev = init_geometry.estimate_global_positions(g["num_images"], g["pair_images"], g["tvec"], g["truth"],
                                                  options=init_geometry.ConstrainedL1SolverOptions(**TIGHT))
    ref = po.estimate_global_positions(g["num_images"], g["pair_images"], g["tvec"], g["truth"], options=TIGHT)
    _assert_margin(ref)
    assert ref["converged"] and dev.summary["converged"] and dev.summary["admm_iterations"] == ref["iterations"]
    obj = 0.0
    for k, (a, b) in enumerate(g["pair_images"]):
        d = po.rotated_translation(g["truth"][b], g["tvec"][k])
        obj += np.abs(dev.positions[a] - dev.positions[b] - dev.scales[k] * d).sum()
    lp = _lp_optimum(g)
    assert abs(obj - lp) <= 1e-6 * lp and (dev.scales >= 1 - 1e-8).all()


def _helix_chain(n_traj=800, n_frames=8, n_obs=4000, seed=7):
    scene, qvec, tvec, cam = syn.make_two_view_scene(n_traj, n_frames, n_obs, seed=seed, path="helix")
    names, ids = ["%05d.png" % i for i in range(n_frames)], list(range(1, n_frames + 1))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches_device(scene, n_frames))
    return syn.two_view_inputs(rows, ids, qvec, tvec, cam), qvec, tvec


DB = ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr", "inlier_matches")


def test_pairwise_translations_from_database_arrays(gpu):
    args, qvec, _ = _helix_chain(seed=3)
    db = {k: args[k] for k in DB}
    R = len(args["pair_images"])
    used = np.arange(R) % 4 != 2
    t, its = init_geometry.optimize_pairwise_translations(**db, orientations=qvec, pair_used=used, return_iterations=True)
    assert (t[~used] == 0).all() and (its[~used] == 0).all()
    # bit-identical to the normalised-points call on points normalised on the host with the same expression
    pts = []
    for p in np.nonzero(used)[0]:
        a, b = args["pair_images"][p]
        x1, x2 = po.normalized_points(**db, p=p)
        pts.append((x1, x2, qvec[a], qvec[b]))
    t2, its2 = init_geometry.batch_optimize_relative_position_with_known_rotation(pts, return_iterations=True)
    assert np.array_equal(t[used], t2) and np.array_equal(its[used], its2)
    # and agrees with the restatement on the widest baselines.  The other pairs are left out: their sign comes from the
    # cheirality majority, and where points lie close to max_depth = 1000 |R't| (short baselines) a count one point
    # away from the majority can flip with the rounding of the two triangulations (Jacobi on the device, LAPACK SVD in
    # numpy); the bit-identity above covers those pairs.
    ref, _ = po.optimize_pairwise_translations(**db, orientations=qvec, pair_used=used)
    gap = np.abs(np.diff(args["pair_images"], axis=1)[:, 0])
    for p in np.nonzero(used & (gap >= gap.max() - 1))[0]:
        assert np.abs(t[p] - ref[p]).max() <= 1e-6, p


def test_chain_from_database_rows_to_image_poses(gpu):
    args, qvec, tvec = _helix_chain()
    F = 8
    poses = init_geometry.estimate_relative_poses(**args)
    rot_args = dict(num_images=F, pair_images=args["pair_images"], qvec=poses.qvec,
                    num_correspondences=np.diff(args["inlier_ptr"]), has_pose=poses.estimated)
    rot = init_geometry.estimate_global_rotations(**rot_args)
    rot_ref = ro.estimate_global_rotations(**rot_args)
    db = {k: args[k] for k in DB}
    t = init_geometry.optimize_pairwise_translations(**db, orientations=rot.orientations, pair_used=rot.pair_kept)
    t_ref, _ = po.optimize_pairwise_translations(**db, orientations=rot_ref["orientations"], pair_used=rot_ref["pair_kept"])
    pos_args = dict(num_images=F, pair_images=args["pair_images"], orientations=rot.orientations,
                    has_orientation=rot.has_orientation, pair_used=rot.pair_kept)
    dev = init_geometry.estimate_global_positions(tvec=t, **pos_args)
    _compare(dev, po.estimate_global_positions(tvec=t, **pos_args))
    ref = po.estimate_global_positions(num_images=F, pair_images=args["pair_images"], tvec=t_ref,
                                       orientations=rot_ref["orientations"], has_orientation=rot_ref["has_orientation"],
                                       pair_used=rot_ref["pair_kept"])
    truth = syn.camera_centres(qvec, tvec)
    have = dev.has_position
    assert np.array_equal(have, ref["has_position"]) and have.sum() >= 3
    ate_dev = syn.umeyama_ate(dev.positions[have], truth[have])
    ate_ref = syn.umeyama_ate(ref["positions"][have], truth[have])
    assert ate_dev <= ate_ref + 1e-9
    assert ate_dev <= 0.05 * np.linalg.norm(truth - truth.mean(0), axis=1).max()
