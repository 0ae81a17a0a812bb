"""In-tree build of the sm_90a (H100) library and the pybind11 `particlesfm` module.

    python -m particlesfm_b200.build            # build what is stale
    python -m particlesfm_b200.build --force

nvcc cross-compiles for sm_90a without a GPU.  Outputs (git-ignored):  particle-sfm_b200/libpsfm_b200.so  and
particle-sfm_b200/particlesfm.cpython-*.so
"""
import os
import subprocess
import sys
import sysconfig

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
LIB = os.path.join(HERE, "libpsfm_b200.so")
BUILD = os.path.join(HERE, "build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC", "-ccbin", CXX]

# (source, extra flags).  traj_solver.cu: -fmad=false so that its iterates are
# bit-identical to the oracle compiled with -ffp-contract=off (DESIGN.md §4).  convert.cu: the same, so that its
# depths and percentiles equal the numpy restatement's (DESIGN.md §4.10).  colors.cu: the same, so that its
# interpolated samples equal the oracle's (DESIGN.md §4.11).  midas.cu: the same, so that its input transform
# restates cv2's unfused float64 arithmetic (DESIGN.md §4.16).
UNITS = [
    ("common.cu", []),
    ("pair_inputs.cu", []),
    ("microbench.cu", []),
    ("tracker.cu", []),
    ("track_npy.cu", []),
    ("handoff.cu", []),
    ("init_geometry.cu", []),
    ("two_view.cu", []),
    ("rotation_averaging.cu", []),
    ("position_estimation.cu", []),
    ("triangulation.cu", []),
    ("verification.cu", []),
    ("dlt.cu", []),
    ("convert.cu", ["-fmad=false"]),
    ("colors.cu", ["-fmad=false"]),
    ("optical_flow.cu", ["-fmad=false"]),
    ("midas.cu", ["-fmad=false"]),
    ("motion_seg.cu", []),
    ("dist.cu", []),
    ("ba_solver.cu", []),
    ("traj_solver.cu", ["-fmad=false"]),
]
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h")))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def pybind_target():
    return os.path.join(HERE, "particlesfm" + sysconfig.get_config_var("EXT_SUFFIX"))


def build_library(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.join(INCLUDE, "psfm_b200.h")]
    objs = []
    for src, extra in UNITS:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            cmd = [NVCC] + ARCH + COMMON + extra + ["-c", s, "-o", o]
            if verbose:
                cmd += ["-Xptxas", "-v"]
            print("[build]", " ".join(cmd), flush=True)
            subprocess.check_call(cmd)
    if force or _stale(LIB, objs):
        # link beside the target and rename: a process loading it meanwhile never sees a half-written library
        cmd = [NVCC] + ARCH + ["-shared", "-ccbin", CXX, "-o", LIB + ".tmp"] + objs + ["-ldl"]
        print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        os.replace(LIB + ".tmp", LIB)
    return LIB


def build_pybind(force=False):
    import pybind11
    src = os.path.join(CSRC, "bindings.cc")
    tgt = pybind_target()
    deps = [src, os.path.join(CSRC, "trajectory_base.h"), os.path.join(INCLUDE, "psfm_b200.h")]
    if force or _stale(tgt, deps):
        cmd = [CXX, "-O2", "-std=c++17", "-shared", "-fPIC", "-fvisibility=hidden",
               "-I", pybind11.get_include(), "-I", sysconfig.get_paths()["include"], "-I", INCLUDE,
               src, "-o", tgt + ".tmp", "-ldl"]
        print("[build]", " ".join(cmd), flush=True)
        subprocess.check_call(cmd)
        os.replace(tgt + ".tmp", tgt)
    return tgt


def build_all(force=False, verbose=False):
    return build_library(force, verbose), build_pybind(force)


if __name__ == "__main__":
    build_all(force="--force" in sys.argv, verbose="-v" in sys.argv)
