"""In-tree build of libmincurv_b200.so (H100, sm_90a only).  Used by __graft_entry__.build() and by the
loader when the shared library is missing or older than its sources."""
from __future__ import annotations

import glob
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
HEADER = os.path.join(INCLUDE, "mincurv_b200.h")      # the C-ABI; _lib derives its ctypes signatures from it
SP_SENS_HEADER = os.path.join(CSRC, "shortest_path_sens.h")     # the shortest path's sensitivity entries, bound the same way
LAP_SENS_HEADER = os.path.join(CSRC, "lap_time_sens.h")         # the lap time's sensitivity entries, bound the same way
LIB_PATH = os.path.join(_HERE, "libmincurv_b200.so")
SOURCES = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
HEADERS = sorted(glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) +
                 glob.glob(os.path.join(INCLUDE, "*.h")))
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
    return any(os.path.getmtime(d) > t for d in SOURCES + HEADERS)


PROFILE_LIB_PATH = os.path.join(_HERE, "libmincurv_b200_prof.so")


def build_profile(verbose: bool = False, extra=(), out=None) -> str:
    """Instrumented build (-DMC_PROFILE: cycle counters inside the interior-point kernel, read with mc_debug_read_profile);
    a separate file, loaded only when MC_B200_LIB points at it (tools/prof_run.py).  Never the product library."""
    out = out or PROFILE_LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-DMC_PROFILE", *extra, "-o", out, *SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB_PATH
    cmd = [_nvcc(), *NVCC_FLAGS, "-o", LIB_PATH, *SOURCES]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force=True, verbose=True))
