"""When every tile of a problem takes the dense pair phase, the fused exact step runs k_schur_dense_p, the
Schur tile kernel compiled without its pair loop.  It must give the pair loop's LM trajectory and
parameters (PSFM_SCHUR_PAIRS=loop runs k_schur_tile_p on every tile) to the drift bound of
test_run_to_run_drift_is_bounded, with and without rotations and focal length refined."""
import numpy as np
import pytest

import oracle
from particlesfm_b200 import _abi, ba, synthetic as syn

pytestmark = pytest.mark.gpu

NUM_POINTS, TRACK_LEN = 6000, 12


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


@pytest.mark.parametrize("rot,focal", [(False, False), (True, True)])
def test_all_dense_kernel_agrees_with_the_pair_loop(gpu, monkeypatch, rot, focal):
    # 12-frame windows, the headline's shape at a small size: 21 whole tracks per 256-observation tile
    prob = syn.make_ba_problem(40, NUM_POINTS, TRACK_LEN, seed=45)[0]
    o = oracle.ba_global_options(refine_rotation=rot, refine_focal_length=focal)
    o.linear_solver = _abi.SOLVER_EXACT_SCHUR
    out = {}
    for arm in ("dense", "loop"):
        monkeypatch.setenv("PSFM_SCHUR_PAIRS", arm)
        p = prob.copy()
        out[arm] = (ba.solve_problem(p, o), p)
        monkeypatch.delenv("PSFM_SCHUR_PAIRS")
    (sd, pd), (sl, pl) = out["dense"], out["loop"]
    tiles = -(-NUM_POINTS // (256 // TRACK_LEN))
    assert sd.explicit_fused == 1 and sd.explicit_dense_tiles == tiles and sl.explicit_dense_tiles == 0
    assert sd.num_explicit_solves > 0
    assert sd.num_iterations == sl.num_iterations and sd.termination == sl.termination
    assert abs(sd.final_cost - sl.final_cost) <= 1e-11 * sl.final_cost
    for a, b in ((pd.qvec, pl.qvec), (pd.tvec, pl.tvec), (pd.xyz, pl.xyz), (pd.cam_params, pl.cam_params)):
        assert _rel(a, b) < 1e-9
