"""HP1 parity on the GPU: the CUDA kernel (through the C ABI and through the pybind11
`particlesfm` module) against the CPU oracle — BIT-EXACT (integer track connectivity is
thresholded from these doubles)."""
import os
import sys

import numpy as np
import pytest

import oracle
from particlesfm_b200 import synthetic as syn, traj

pytestmark = pytest.mark.gpu


def _case(n, h, w, seed):
    return syn.make_traj_inputs(n, h, w, seed=seed)


@pytest.mark.parametrize("n,h,w,seed", [(1, 32, 48, 0), (31, 32, 48, 1), (256, 64, 96, 2), (257, 64, 96, 3),
                                        (5000, 128, 256, 4), (70001, 218, 512, 5)])
def test_bit_exact_vs_oracle(gpu, n, h, w, seed):
    uv12, r1, r2, sc, f12 = _case(n, h, w, seed)
    ref, sref = oracle.traj_optimize(uv12, r1, r2, sc, f12)
    out, s = traj.optimize_location(uv12, r1, r2, sc, f12, n, w, h, return_summary=True)
    assert s.num_iterations == sref.num_iterations
    assert s.termination == sref.termination
    assert s.num_successful_steps == sref.num_successful_steps
    assert s.initial_cost == sref.initial_cost
    assert s.final_cost == sref.final_cost
    assert np.array_equal(out, ref), f"max abs diff {np.abs(out - ref).max()}"


@pytest.mark.parametrize("n,h,w,seed", [(1, 32, 48, 0), (31, 32, 48, 1), (256, 64, 96, 2), (257, 64, 96, 3),
                                        (5000, 128, 256, 4), (70001, 218, 512, 5)])
def test_against_reference_dump_when_present(gpu, n, h, w, seed):
    """Outputs of the REAL reference module (Ceres 2.0.0), dumped by oracle/ref_recipe/dump_ref_vectors.py
    on a machine that can build it.  Skipped until the files exist."""
    import hashlib
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", f"ref_traj_{n}_{h}_{w}_{seed}.npz")
    if not os.path.exists(path):
        pytest.skip("no reference dump (oracle/ref_recipe/RECIPE.md): parity is pinned to the oracle only")
    uv12, r1, r2, sc, f12 = _case(n, h, w, seed)
    g = np.load(path)
    hsh = hashlib.sha256()
    for a in (uv12, r1, r2, sc, f12):
        hsh.update(np.ascontiguousarray(a).tobytes())
    assert str(g["inputs_sha256"]) == hsh.hexdigest(), "the dump was made for other inputs"
    out = traj.optimize_location(uv12, r1, r2, sc, f12, n, w, h)
    assert np.abs(out - g["out"]).max() < 1e-9


def test_edge_inputs(gpu):
    # trajectories at / beyond the image border (Grid2D clamps), zero weights, a flat map
    h, w = 24, 40
    uv12, r1, r2, sc, f12 = _case(300, h, w, 7)
    uv12[:50, 0] = -3.7
    uv12[50:100, 1] = h + 5.2
    uv12[100:150, 0] = w - 1.0
    uv12[150:200, 1] = 0.0
    sc[:] = 0.0
    ref, _ = oracle.traj_optimize(uv12, r1, r2, sc, f12)
    out = traj.optimize_location(uv12, r1, r2, sc, f12, 300, w, h)
    assert np.array_equal(out, ref)
    flat = np.full((h, w, 2), 1.25, np.float32)
    ref, _ = oracle.traj_optimize(uv12, r1, r2, sc + 1.0, flat)
    out = traj.optimize_location(uv12, r1, r2, sc + 1.0, flat, 300, w, h)
    assert np.array_equal(out, ref)


def test_inputs_not_mutated_and_empty(gpu):
    uv12, r1, r2, sc, f12 = _case(100, 32, 32, 9)
    keep = [a.copy() for a in (uv12, r1, r2, sc, f12)]
    traj.optimize_location(uv12, r1, r2, sc, f12, 100, 32, 32)
    for a, b in zip(keep, (uv12, r1, r2, sc, f12)):
        assert np.array_equal(a, b)
    out = traj.optimize_location(np.zeros((0, 4)), np.zeros((0, 2)), np.zeros((0, 2)), np.zeros((0, 1)), f12, 0, 32, 32)
    assert out.shape == (0, 4)


def test_pybind_module_matches(gpu):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "particle-sfm_b200"))
    import particlesfm
    uv12, r1, r2, sc, f12 = _case(3000, 96, 128, 11)
    ref, _ = oracle.traj_optimize(uv12, r1, r2, sc, f12)
    out = particlesfm.optimize_location(uv12, r1, r2, sc, f12, 3000, 128, 96)
    assert out.shape == (3000, 4) and np.array_equal(out, ref)
    # float64 maps that are float32-representable are accepted, like the reference's force-cast
    out = particlesfm.optimize_location(uv12, r1, r2, sc, f12.astype(np.float64), 3000, 128, 96)
    assert np.array_equal(out, ref)


def test_constant_flow_closed_form(gpu):
    # constant flow c: minimiser of (x1-a)^2 + s^2 (x2-b)^2 + (x2-x1-c)^2 per axis
    h, w, n = 40, 60, 500
    rng = np.random.default_rng(0)
    c = np.array([1.5, -0.75])
    flow = np.tile(c.astype(np.float32), (h, w, 1))
    x1 = rng.uniform(5, 30, (n, 2)); x2 = x1 + c + rng.normal(0, 0.3, (n, 2))
    a = x1 + rng.normal(0, 0.2, (n, 2)); b = x2 + rng.normal(0, 0.2, (n, 2))
    out = traj.optimize_location(np.concatenate([x1, x2], 1), a, b, np.ones((n, 1)), flow, n, w, h)
    # normal equations: [[2,-1],[-1,2]] [x1;x2] = [a - c; b + c]
    x1s = (2 * (a - c) + (b + c)) / 3.0
    x2s = ((a - c) + 2 * (b + c)) / 3.0
    assert np.abs(out[:, :2] - x1s).max() < 1e-6 and np.abs(out[:, 2:] - x2s).max() < 1e-6
