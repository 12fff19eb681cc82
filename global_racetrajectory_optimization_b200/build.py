"""In-tree build of libmincurv_b200.so (H100, sm_90a only).  Used by __graft_entry__.build() and by the
loader when the shared library is missing or older than its sources."""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(_HERE, "libmincurv_b200.so")
SOURCES = ["capi.cu", "mincurv_setup.cu", "mincurv_ipm.cu", "mincurv_finalize.cu", "splines.cu", "shortest_path.cu",
           "vel_profile.cu", "traj_check.cu", "synth.cu", "prep_track.cu"]
HEADERS = ["common.cuh", "mincurv_ws.cuh", "mincurv_ops.cuh", "vel_profile_core.cuh", "traj_check_core.cuh", os.path.join("..", "..", "include", "mincurv_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _nvcc() -> str:
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found: the CUDA extension of global_racetrajectory_optimization_b200 cannot be built")
    return cand


def needs_build() -> bool:
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps)


PROFILE_LIB_PATH = os.path.join(_HERE, "libmincurv_b200_prof.so")


def build_profile(verbose: bool = False, extra=(), out=None) -> str:
    """Instrumented build (-DMC_PROFILE: cycle counters inside the interior-point kernel, read with mc_debug_read_profile);
    a separate file, loaded only when MC_B200_LIB points at it (tools/prof_run.py).  Never the product library."""
    out = out or PROFILE_LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-DMC_PROFILE", *extra, "-o", out, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB_PATH, *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
