"""Known answers of the numpy restatement of the global position estimation (oracle/position_oracle.py): exact
directions, a linear program, the Schur-reduced x update, the gauge, outliers, RegisterAllImages, the argument rules,
and the pairwise-translation step from database arrays."""
import numpy as np
import pytest
import scipy.optimize

from oracle import init_oracle as io, position_oracle as po
from particlesfm_b200 import handoff, synthetic as syn

TIGHT = dict(max_num_iterations=60000, absolute_tolerance=1e-11, relative_tolerance=1e-11)


def _run(g, **kw):
    return po.estimate_global_positions(g["num_images"], g["pair_images"], g["tvec"], g["truth"], **kw)


def _rel_ate(pos, truth):
    return syn.umeyama_ate(pos, truth) / np.linalg.norm(truth - truth.mean(0), axis=1).max()


def test_exact_directions_recover_the_truth_up_to_similarity():
    g = syn.make_view_graph(12, seed=11)
    r = _run(g, options=TIGHT)
    assert _rel_ate(r["positions"], g["centres"]) <= 1e-8
    assert r["min_scale"] >= 1 - 1e-8


def _lp_optimum(g):
    """min sum |c1 - c2 - s d|_1 subject to s >= 1 by HiGHS, the gauge (image 0) at the origin."""
    pairs, F = g["pair_images"], g["num_images"]
    R, n = len(pairs), 3 * (F - 1)
    d = np.array([po.rotated_translation(g["truth"][b], t) for (a, b), t in zip(pairs, g["tvec"])])
    A = np.zeros((3 * R, n + R))
    for k, (a, b) in enumerate(pairs):
        for img, sg in ((a, 1.0), (b, -1.0)):
            if img > 0:
                A[3 * k:3 * k + 3, 3 * (img - 1):3 * img] = sg * np.eye(3)
        A[3 * k:3 * k + 3, n + k] = -d[k]
    nv = n + R + 3 * R
    c = np.concatenate([np.zeros(n + R), np.ones(3 * R)])
    I = np.eye(3 * R)
    A_ub = np.block([[A, -I], [-A, -I]])
    bounds = [(None, None)] * n + [(1, None)] * R + [(0, None)] * (3 * R)
    res = scipy.optimize.linprog(c, A_ub=A_ub, b_ub=np.zeros(6 * R), bounds=bounds, method="highs")
    assert res.status == 0 and nv == len(res.x)
    return res.fun


def test_admm_reaches_the_linear_program_optimum():
    g = syn.make_view_graph(8, direction_noise_deg=2.0, direction_outlier_fraction=0.2, seed=3)
    r = _run(g, options=TIGHT)
    lp = _lp_optimum(g)
    assert abs(r["objective"] - lp) <= 1e-6 * lp
    used = r["scales"] != 0
    assert (r["scales"][used] >= 1 - 1e-8).all()


def test_schur_reduced_x_update_equals_the_full_solve():
    g = syn.make_view_graph(10, graph="banded", band=3, direction_noise_deg=1.0, seed=4)
    pairs, F = g["pair_images"], g["num_images"]
    index = {f: f - 1 for f in range(F)}
    d = np.array([po.rotated_translation(g["truth"][b], t) for (a, b), t in zip(pairs, g["tvec"])])
    A, _ = po.stacked_system(index, pairs, d, list(range(len(pairs))))
    rhs = np.random.default_rng(0).normal(size=A.shape[1])
    full = np.linalg.solve((A.T @ A).toarray(), rhs)
    red = po.schur_x_update([(index[a], index[b]) for a, b in pairs], d, F - 1, rhs)
    assert np.abs(red - full).max() <= 1e-12 * np.abs(full).max()


def test_gauge_moves_every_position_by_one_vector():
    g = syn.make_view_graph(15, direction_noise_deg=1.0, direction_outlier_fraction=0.1, seed=6)
    r0, r1 = _run(g), _run(g, gauge=7)
    assert r0["gauge_image"] == 0 and r1["gauge_image"] == 7
    shift = r1["positions"] - r0["positions"]
    assert np.abs(shift - shift[0]).max() <= 1e-9 * np.abs(r0["positions"]).max()
    assert np.abs(r1["scales"] - r0["scales"]).max() <= 1e-9 * np.abs(r0["scales"]).max()


def test_outliers_leave_the_centres_close_to_the_truth():
    g = syn.make_view_graph(40, direction_noise_deg=0.5, direction_outlier_fraction=0.15, seed=8)
    r = _run(g)
    assert _rel_ate(r["positions"], g["centres"]) <= 0.05


def test_image_tvec_is_minus_r_c():
    g = syn.make_view_graph(10, direction_noise_deg=1.0, seed=9)
    r = _run(g)
    R = syn.qvec_to_rotmat(g["truth"])
    assert np.abs(r["image_tvec"] + np.einsum("fij,fj->fi", R, r["positions"])).max() <= 1e-12
    assert np.abs(syn.camera_centres(g["truth"], r["image_tvec"]) - r["positions"]).max() <= 1e-12


BASE = dict(num_images=4, pair_images=np.array([[0, 1], [1, 2], [2, 3]]), tvec=np.tile([1.0, 0.0, 0.0], (3, 1)),
            orientations=np.tile([1.0, 0.0, 0.0, 0.0], (4, 1)))


@pytest.mark.parametrize("change, why", [
    (dict(pair_used=np.zeros(3)), "no used image pair"),
    (dict(pair_images=np.array([[0, 1], [1, 2], [2, 4]])), "outside"),
    (dict(pair_images=np.array([[0, 1], [1, 1], [2, 3]])), "with itself"),
    (dict(pair_images=np.array([[0, 1], [1, 0], [2, 3]])), "listed twice"),
    (dict(has_orientation=np.array([1, 1, 0, 1])), "no orientation"),
    (dict(orientations=np.array([[1.0, 0, 0, 0]] * 3 + [[np.nan, 0, 0, 0]])), "non-finite orientation"),
    (dict(tvec=np.array([[1.0, 0, 0], [np.inf, 0, 0], [1.0, 0, 0]])), "non-finite pair tvec"),
    (dict(pair_images=np.array([[0, 1], [2, 3], [0, 2]]), pair_used=np.array([1, 1, 0])), "connected"),
    (dict(options=dict(alpha=2.0)), "Check()"),
    (dict(options=dict(rho=0.0)), "Check()"),
    (dict(options=dict(max_num_iterations=0)), "Check()"),
])
def test_argument_rules(change, why):
    with pytest.raises(po.InvalidError, match=why.replace("(", r"\(").replace(")", r"\)")):
        po.estimate_global_positions(**{**BASE, **change})


def test_too_many_views_are_unsupported():
    F = 2733
    pairs = np.stack([np.arange(F - 1), np.arange(1, F)], 1)
    with pytest.raises(po.UnsupportedError):
        po.estimate_global_positions(F, pairs, np.tile([1.0, 0, 0], (F - 1, 1)), np.tile([1.0, 0, 0, 0], (F, 1)))


def test_unused_pairs_keep_zero_scales_and_their_images_have_no_position():
    g = syn.make_view_graph(6, direction_noise_deg=1.0, seed=2)
    used = np.ones(len(g["pair_images"]), bool)
    used[[p for p, (a, b) in enumerate(g["pair_images"]) if 5 in (a, b)]] = False
    r = _run(g, pair_used=used)
    assert not r["has_position"][5] and r["has_position"][:5].all()
    assert (r["scales"][~used] == 0).all() and (r["scales"][used] >= 1 - 1e-3).all()


def test_database_array_pairwise_step_equals_the_per_pair_oracle():
    scene, qvec, tvec, cam = syn.make_two_view_scene(300, 5, 1200, seed=3, path="helix")
    names, ids = ["%05d.png" % i for i in range(5)], list(range(1, 6))
    rows = handoff.import_keypoints_matches_arrays(names, dict(zip(names, ids)), handoff.traj_to_matches(scene, 5))
    args = syn.two_view_inputs(rows, ids, qvec, tvec, cam)
    db = {k: args[k] for k in ("keypoint_ptr", "keypoints", "image_camera", "cameras", "pair_images", "inlier_ptr",
                               "inlier_matches")}
    used = np.arange(len(args["pair_images"])) % 3 != 1
    t, its = po.optimize_pairwise_translations(**db, orientations=qvec, pair_used=used)
    for p, (a, b) in enumerate(args["pair_images"]):
        if not used[p]:
            assert (t[p] == 0).all() and its[p] == 0
            continue
        x1, x2 = po.normalized_points(**db, p=p)
        assert np.array_equal(t[p], io.optimize_relative_position_with_known_rotation(x1, x2, qvec[a], qvec[b]))


def test_view_graph_keeps_every_existing_key():
    old = syn.make_view_graph(20, noise_deg=1.0, outlier_fraction=0.2, seed=5)
    new = syn.make_view_graph(20, noise_deg=1.0, outlier_fraction=0.2, seed=5, direction_noise_deg=1.0,
                              direction_outlier_fraction=0.3)
    for k in ("pair_images", "qvec", "num_correspondences", "has_pose", "truth", "outlier"):
        assert np.array_equal(old[k], new[k]), k
    assert np.array_equal(old["centres"], new["centres"])


def test_helix_scene_is_opt_in():
    a = syn.make_two_view_scene(200, 6, 800, seed=2)
    b = syn.make_two_view_scene(200, 6, 800, seed=2, path="line")
    assert np.array_equal(a[0].xy, b[0].xy) and np.array_equal(a[2], b[2])
    h = syn.make_two_view_scene(200, 6, 800, seed=2, path="helix")
    c = syn.camera_centres(h[1], h[2])
    # not near-collinear: the second singular value of the centred centres is a sizeable share of the first
    sv = np.linalg.svd(c - c.mean(0), compute_uv=False)
    assert sv[1] > 0.2 * sv[0]
