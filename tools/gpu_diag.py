"""Step-by-step diagnostic for GPU runs (prints, never swallows)."""
import ctypes as C
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np


def main():
    from particlesfm_b200 import _lib, _abi
    print("lib path", _lib.LIB_PATH, os.path.exists(_lib.LIB_PATH))
    L = _lib.lib()
    n = L.psfm_device_count()
    print("device_count", n, "last_error", L.psfm_last_error())
    if n <= 0:
        try:
            cudart = C.CDLL("libcudart.so")
            cnt = C.c_int()
            rc = cudart.cudaGetDeviceCount(C.byref(cnt))
            cudart.cudaGetErrorString.restype = C.c_char_p
            print("system cudart: rc", rc, cudart.cudaGetErrorString(rc), "count", cnt.value)
        except Exception:
            traceback.print_exc()
        try:
            cu = C.CDLL("libcuda.so.1")
            rc = cu.cuInit(0)
            v = C.c_int()
            cu.cuDriverGetVersion(C.byref(v))
            print("cuInit rc", rc, "driver version", v.value)
        except Exception:
            traceback.print_exc()
        return 1
    import oracle
    from particlesfm_b200 import synthetic as syn, traj, ba
    # HP1
    for n_, h, w, seed in [(1, 32, 48, 0), (257, 64, 96, 3), (5000, 128, 256, 4)]:
        uv12, r1, r2, sc, f12 = syn.make_traj_inputs(n_, h, w, seed=seed)
        ref, sref = oracle.traj_optimize(uv12, r1, r2, sc, f12)
        try:
            out, s = traj.optimize_location(uv12, r1, r2, sc, f12, n_, w, h, return_summary=True)
            print("HP1 n=%d: iters gpu %d oracle %d term %d/%d cost %.17g/%.17g equal=%s maxdiff=%g solve_ms=%.3f" % (
                n_, s.num_iterations, sref.num_iterations, s.termination, sref.termination, s.final_cost, sref.final_cost,
                np.array_equal(out, ref), np.abs(out - ref).max(), s.solve_ms))
        except Exception:
            traceback.print_exc()
    # HP2 evaluate / linear step / solve
    rel = lambda a, b: np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)
    for rot, focal in [(False, False), (True, True)]:
        prob, truth = syn.make_ba_problem(10, 600, 6, seed=5)
        o = oracle.ba_global_options(refine_rotation=rot, refine_focal_length=focal)
        o.linear_solver = _abi.SOLVER_EXACT_SCHUR
        try:
            c0, r0, gc0, gp0 = oracle.ba_evaluate(prob, o)
            S = ba.ResidentSolver(prob)
            c1, r1_, gc1, gp1 = S.evaluate(o)
            print("HP2 eval rot=%s: cost %.15g/%.15g r %.2e gc %.2e gp %.2e" % (rot, c1, c0, rel(r1_, r0), rel(gc1, gc0), rel(gp1, gp0)))
            for solver in (_abi.SOLVER_EXACT_SCHUR, _abi.SOLVER_ITERATIVE_SCHUR):
                o.linear_solver = solver
                sc0, sp0, it0 = oracle.ba_linear_step(prob, o, 1e4, solver)
                sc1, sp1, it1 = S.linear_step(o, 1e4)
                print("  linear step solver=%d: iters %d/%d cam %.2e pts %.2e" % (solver, it1, it0, rel(sc1, sc0), rel(sp1, sp0)))
                p0, p1 = prob.copy(), prob.copy()
                s0 = oracle.ba_solve(p0, o)
                s1 = ba.solve_problem(p1, o)
                print("  solve solver=%d: iters %d/%d lin %d/%d term %d/%d cost %.12g/%.12g q %.2e t %.2e X %.2e K %.2e dev_ms %.2f" % (
                    solver, s1.num_iterations, s0.num_iterations, s1.num_linear_iterations, s0.num_linear_iterations,
                    s1.termination, s0.termination, s1.final_cost, s0.final_cost, rel(p1.qvec, p0.qvec), rel(p1.tvec, p0.tvec),
                    rel(p1.xyz, p0.xyz), rel(p1.cam_params, p0.cam_params), s1.device_ms))
        except Exception:
            traceback.print_exc()
    return 0


if __name__ == "__main__":
    sys.exit(main())
