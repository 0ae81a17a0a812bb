"""The two pair phases of the fused Schur tile kernel: the per-entry loop and the dense Z Z'
product on fp64 tensor cores (PSFM_SCHUR_PAIRS=loop | dense), and the unfused fallback
(PSFM_SCHUR_UNFUSED=1: k_schur_w + k_schur_pairs over the same pair tasks) are the same Schur
complement summed in a different order.  They must give the same LM trajectory and the same
parameters to the drift bound of test_run_to_run_drift_is_bounded."""
import numpy as np
import pytest

import oracle
from particlesfm_b200 import _abi, ba, synthetic as syn

pytestmark = pytest.mark.gpu


def _opts(rot, focal):
    o = oracle.ba_global_options(refine_rotation=rot, refine_focal_length=focal)
    o.linear_solver = _abi.SOLVER_EXACT_SCHUR
    return o


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _with_duplicates(prob, fraction, seed):
    """Every `fraction` of the observations observed a second time in the same image (a point
    tracked twice into one frame), 0.3 px away from the first."""
    rng = np.random.default_rng(seed)
    dup = rng.choice(prob.obs_image.size, int(fraction * prob.obs_image.size), replace=False)
    xy = prob.obs_xy[dup] + rng.normal(0.0, 0.3, (dup.size, 2))
    return _abi.BAProblem(prob.qvec, prob.tvec, prob.xyz, prob.cam_params,
                          np.concatenate([prob.obs_image, prob.obs_image[dup]]),
                          np.concatenate([prob.obs_point, prob.obs_point[dup]]),
                          np.concatenate([prob.obs_xy, xy]), prob.image_camera,
                          prob.pose_constant, prob.tvec_constant_mask, prob.camera_constant)


def _problem(kind):
    if kind == "windows":
        return syn.make_ba_problem(40, 6000, 9, seed=31)[0]
    if kind == "dynamic":
        return syn.make_ba_problem(40, 6000, 12, seed=32, dynamic_fraction=0.3)[0]
    return _with_duplicates(syn.make_ba_problem(30, 4000, 8, seed=33)[0], 0.05, seed=34)


@pytest.mark.parametrize("rot,focal", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("kind", ["windows", "dynamic", "duplicates"])
def test_dense_and_loop_pair_phases_agree(gpu, monkeypatch, kind, rot, focal):
    prob = _problem(kind)
    o = _opts(rot, focal)
    out = {}
    for arm in ("loop", "dense", "unfused"):
        env = ("PSFM_SCHUR_UNFUSED", "1") if arm == "unfused" else ("PSFM_SCHUR_PAIRS", arm)
        monkeypatch.setenv(*env)
        p = prob.copy()
        out[arm] = (ba.solve_problem(p, o), p)
        monkeypatch.delenv(env[0])
    (sl, pl), (sd, pd), (su, pu) = out["loop"], out["dense"], out["unfused"]
    assert sl.explicit_fused == 1 and sd.explicit_fused == 1 and su.explicit_fused == 0
    assert sl.explicit_dense_tiles == 0 and sd.explicit_dense_tiles > 0 and su.explicit_dense_tiles == 0
    assert sl.num_pair_tasks > 0 and sd.num_pair_tasks == sl.num_pair_tasks and su.num_pair_tasks == sl.num_pair_tasks
    for s, q in ((sd, pd), (su, pu)):
        assert s.num_iterations == sl.num_iterations and s.termination == sl.termination
        assert abs(s.final_cost - sl.final_cost) <= 1e-11 * sl.final_cost
        for a, b in ((q.qvec, pl.qvec), (q.tvec, pl.tvec), (q.xyz, pl.xyz), (q.cam_params, pl.cam_params)):
            assert _rel(a, b) < 1e-9
