"""ctypes binding of the C-ABI in include/mincurv_b200.h.  There is no CPU fallback: importing the
compute entry points without the shared library (or calling them without a CUDA device) raises."""
from __future__ import annotations

import ctypes
import os
import re

from . import build as _build

_LIB = None


class MinCurvLibError(RuntimeError):
    pass


def _c_source(path: str) -> str:
    """The C source in path without its comments and preprocessor lines."""
    with open(path) as f:
        txt = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    return re.sub(r"^[ \t]*#[^\n]*", "", txt, flags=re.M)


_SCALARS = {"int": ctypes.c_int, "double": ctypes.c_double, "size_t": ctypes.c_size_t}


def _ctype(c: str, decl: str, ret: bool = False):
    c = " ".join(c.replace("*", " * ").split())
    if ret and c == "const char *":
        return ctypes.c_char_p
    if c.endswith("*"):
        return ctypes.c_void_p
    if c not in _SCALARS:
        raise MinCurvLibError(f"{decl}: no ctypes type for the C type '{c}'")
    return _SCALARS[c]


def header_signatures(path: str) -> dict:
    """name -> (restype, argtypes) of every declaration `ret mc_name(type name, ...);` in the C header at path."""
    sigs = {}
    for ret, name, args in re.findall(r"([\w\s*]+?)\b(mc_\w+)\s*\(([^)]*)\)\s*;", _c_source(path)):
        params = [] if args.strip() in ("", "void") else [re.sub(r"\w+\s*$", "", p) for p in args.split(",")]
        sigs[name] = (_ctype(ret, name, ret=True), [_ctype(p, name) for p in params])
    return sigs


_SIGS = header_signatures(_build.HEADER)
EXPORTED_SYMBOLS = tuple(_SIGS)
# the shortest path's sensitivity entries (batch.opt_shortest_path_diff): exported by the same library, declared in a header
# of their own; load() binds them with the rest
_SP_SENS_SIGS = header_signatures(_build.SP_SENS_HEADER)
SP_SENS_SYMBOLS = tuple(_SP_SENS_SIGS)
_SIGS.update(_SP_SENS_SIGS)
# the lap time's sensitivity entries (batch.vel_profile_diff): the same library, a header of their own; load() binds them
# too, but they stay out of _SIGS (the table of the public header and the shortest path's entries)
LAP_SENS_SIGS = header_signatures(_build.LAP_SENS_HEADER)
LAP_SENS_SYMBOLS = tuple(LAP_SENS_SIGS)


def slab_mirror():
    """The names of enum Vec in csrc/mincurv_ws.cuh without V_ (the O(N) vectors at the head of a minimum-curvature
    workspace slab, in slab order) and the constexpr ints of csrc/common.cuh, so that the host reads the layout the
    kernels were compiled with."""
    enum = re.search(r"enum\s+Vec\b[^{]*\{([^}]*)\}", _c_source(os.path.join(_build.CSRC, "mincurv_ws.cuh"))).group(1)
    names = []
    for i, (name, value) in enumerate(re.findall(r"(\w+)\s*(?:=\s*(\d+))?", enum)):
        if name == "NUM_VEC":
            break
        if not name.startswith("V_") or (value and int(value) != i):
            raise MinCurvLibError(f"enum Vec: cannot mirror entry {i} '{name}'")
        names.append(name[2:])
    consts = re.findall(r"constexpr\s+int\s+(\w+)\s*=\s*(\d+)\s*;", _c_source(os.path.join(_build.CSRC, "common.cuh")))
    return names, {k: int(v) for k, v in consts}


def lib_path() -> str:
    return _build.LIB_PATH


def load(build_if_missing: bool = True):
    """Load libmincurv_b200.so (building it with nvcc first if needed)."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = os.environ.get("MC_B200_LIB") or _build.LIB_PATH      # (override: the instrumented build of tools/prof_run.py)
    if path == _build.LIB_PATH and build_if_missing and _build.needs_build():
        _build.build()
    if not os.path.exists(path):
        raise MinCurvLibError(f"{path} is missing: build it with `python -m global_racetrajectory_optimization_b200.build` "
                              "(there is no CPU fallback for this path)")
    lib = ctypes.CDLL(path)
    for name, (res, args) in {**_SIGS, **LAP_SENS_SIGS}.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _LIB = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().mc_last_error()
        raise MinCurvLibError(f"{what} failed with code {rc}: {msg.decode() if msg else ''}")
