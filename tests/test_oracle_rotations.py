"""Known answers for the numpy restatement of the global rotation averaging (oracle/rotation_oracle.py), which the
GPU tests compare the device against."""
import numpy as np
import pytest
import scipy.linalg
import scipy.optimize
import scipy.sparse
from scipy.spatial.transform import Rotation

from oracle import rotation_oracle as ro
from particlesfm_b200 import synthetic as syn


def _scipy_quat(q):                    # (w, x, y, z) -> scipy's (x, y, z, w)
    return Rotation.from_quat([q[1], q[2], q[3], q[0]])


def _angle(q1, q2):
    return np.linalg.norm(ro.quaternion_to_angle_axis(ro.concatenate_quaternions(q1, ro.invert_quaternion(q2))))


def _run(g, **kw):
    return ro.estimate_global_rotations(g["num_images"], g["pair_images"], g["qvec"], g["num_correspondences"],
                                        g.get("has_pose"), **kw)


def _max_error_to_truth(g, out):
    gauge = out["gauge_image"]
    return max(_angle(out["orientations"][f], ro.concatenate_quaternions(ro.invert_quaternion(g["truth"][gauge]),
                                                                         g["truth"][f]))
               for f in np.nonzero(out["has_orientation"])[0])


@pytest.mark.parametrize("graph", ["tree", "cyclic"])
def test_exact_relative_rotations_give_the_truth(graph):
    g = syn.make_view_graph(12, graph="banded", band=1 if graph == "tree" else 4, seed=3)
    out = _run(g)
    assert out["success"] and out["pair_kept"].all()
    assert _max_error_to_truth(g, out) <= 1e-12


@pytest.mark.parametrize("angle", [0.0, 1e-12, 1e-6, 0.3, 2.0, np.pi - 1e-9, np.pi])
def test_quaternion_helpers_agree_with_scipy(angle):
    rng = np.random.default_rng(int(angle * 1000) + 1)
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    aa = axis * angle
    q = ro.angle_axis_to_quaternion(aa)
    ref = Rotation.from_rotvec(aa)
    assert np.allclose(_scipy_quat(q).as_matrix(), ref.as_matrix(), atol=1e-14)
    back = ro.quaternion_to_angle_axis(q)
    assert np.allclose(Rotation.from_rotvec(back).as_matrix(), ref.as_matrix(), atol=1e-12)
    assert np.linalg.norm(back) <= np.pi + 1e-12
    if angle < 3.0:                    # the cos < 0 branch gives -q the same (shortest) angle-axis as q
        assert np.allclose(ro.quaternion_to_angle_axis(-q), back, atol=1e-12)
    assert np.allclose(ro.quaternion_to_rotation_matrix(q), ref.as_matrix(), atol=1e-14)
    q2 = ro.angle_axis_to_quaternion(rng.normal(size=3))
    cat = ro.concatenate_quaternions(q, q2)                      # q2 after q
    assert np.allclose(_scipy_quat(cat).as_matrix(), (_scipy_quat(q2) * ref).as_matrix(), atol=1e-13)
    assert np.allclose(_scipy_quat(ro.invert_quaternion(q)).as_matrix(), ref.inv().as_matrix(), atol=1e-14)


def test_weighted_normal_matrix_is_the_kronecker_laplacian():
    g = syn.make_view_graph(9, graph="banded", band=3, seed=2)
    index = {f: f - 1 for f in range(9)}
    pairs = list(range(len(g["qvec"])))
    A = ro.incidence_matrix(index, g["pair_images"], pairs)
    B = ro.incidence_matrix(index, g["pair_images"], pairs, scalar=True)
    w = np.random.default_rng(0).random(len(pairs))
    lhs = (A.T @ scipy.sparse.diags(np.repeat(w, 3)) @ A).toarray()
    rhs = np.kron((B.T @ scipy.sparse.diags(w) @ B).toarray(), np.eye(3))
    assert np.array_equal(lhs, rhs)


def test_admm_agrees_with_a_linear_program():
    rng = np.random.default_rng(4)
    g = syn.make_view_graph(6, seed=4)
    index = {f: f - 1 for f in range(6)}
    A = ro.incidence_matrix(index, g["pair_images"], list(range(len(g["qvec"]))))
    b = rng.normal(scale=0.1, size=A.shape[0])
    b[::7] += 1.0                                                 # a few gross errors
    factor = scipy.linalg.cho_factor((A.T @ A).toarray(), lower=True)
    x, its = ro.l1_solve(A, factor, b, 5000)
    assert its < 5000
    m, n = A.shape
    Ad = A.toarray()
    lp = scipy.optimize.linprog(np.r_[np.zeros(n), np.ones(m)], A_ub=np.block([[Ad, -np.eye(m)], [-Ad, -np.eye(m)]]),
                                b_ub=np.r_[b, -b], bounds=[(None, None)] * n + [(0, None)] * m, method="highs")
    best = lp.fun
    got = np.abs(A @ x - b).sum()
    assert got <= best * (1 + 1e-2) + np.sqrt(m) * 1e-4 * 10


def test_outliers_are_filtered():
    g = syn.make_view_graph(30, noise_deg=1.0, outlier_fraction=0.2, seed=1)
    out = _run(g)
    assert g["outlier"].sum() > 50
    assert not (out["pair_kept"] & g["outlier"]).any()
    assert out["pair_kept"][~g["outlier"]].mean() > 0.95
    assert _max_error_to_truth(g, out) <= np.deg2rad(1.0)       # 1 degree pair noise, 29 pairs per image


def test_components_gauge_and_spanning_tree_ties():
    # two components of 3 images: {1, 2, 4} and {0, 3, 5}; the one holding image 0 is kept, image 0 is the gauge
    pairs = np.array([[2, 1], [4, 2], [3, 0], [5, 3]])
    q5 = np.tile([1.0, 0.0, 0.0, 0.0], (4, 1))
    out = ro.estimate_global_rotations(6, pairs, q5, [10, 10, 10, 10])
    assert out["gauge_image"] == 0
    assert list(np.nonzero(out["has_orientation"])[0]) == [0, 3, 5]
    assert list(np.nonzero(out["pair_kept"])[0]) == [2, 3]
    # the larger component wins over the one holding image 0
    pairs = np.array([[0, 1], [2, 3], [3, 4], [4, 2]])
    out = ro.estimate_global_rotations(5, pairs, np.tile([1.0, 0, 0, 0], (4, 1)), [1, 1, 1, 1])
    assert out["gauge_image"] == 2 and list(np.nonzero(out["pair_kept"])[0]) == [1, 2, 3]
    # spanning tree: a triangle with inconsistent rotations; equal weights pick (0, 1) and (0, 2) by image order
    rot = lambda deg: ro.angle_axis_to_quaternion(np.array([0.0, 0.0, np.deg2rad(deg)]))
    pairs = np.array([[1, 2], [0, 2], [0, 1]])
    qv = np.array([rot(30), rot(20), rot(10)])
    o = ro.spanning_tree_orientations([0, 1, 2], pairs, qv, [5, 5, 5], [0, 1, 2])
    assert _angle(o[1], rot(10)) < 1e-15 and _angle(o[2], rot(20)) < 1e-15
    # a heavier edge wins over image order
    o = ro.spanning_tree_orientations([0, 1, 2], pairs, qv, [9, 5, 5], [0, 1, 2])
    assert _angle(o[1], rot(10)) < 1e-15 and _angle(o[2], rot(40)) < 1e-15


def test_no_posed_pair_fails():
    pairs = np.array([[0, 1]])
    assert not ro.estimate_global_rotations(2, pairs, [[1.0, 0, 0, 0]], [3], has_pose=[0])["success"]
    assert not ro.estimate_global_rotations(2, pairs, [[np.nan, 0, 0, 0]], [3])["success"]
    assert not ro.estimate_global_rotations(2, np.zeros((0, 2)), np.zeros((0, 4)), [])["success"]


@pytest.mark.parametrize("name", list(ro.DEFAULTS))
def test_each_check_violation(name):
    with pytest.raises(ro.OptionsError):
        ro.estimate_global_rotations(2, [[0, 1]], [[1.0, 0, 0, 0]], [3], options={name: 0})
