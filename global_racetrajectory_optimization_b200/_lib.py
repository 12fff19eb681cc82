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


def _declarations(path: str):
    """(restype, name, [parameter types]) of every declaration `ret mc_name(type name, ...);` in the C header at path."""
    for ret, name, args in re.findall(r"([\w\s*]+?)\b(mc_\w+)\s*\(([^)]*)\)\s*;", _c_source(path)):
        yield ret, name, [] if args.strip() in ("", "void") else [re.sub(r"\w+\s*$", "", p) for p in args.split(",")]


def header_signatures(path: str) -> dict:
    """name -> (restype, argtypes) of every declaration `ret mc_name(type name, ...);` in the C header at path."""
    return {name: (_ctype(ret, name, ret=True), [_ctype(re.sub(r"\bMC_OPTIONAL[2-6]?\b", " ", p), name) for p in params])
            for ret, name, params in _declarations(path)}


def optional_parameters(path: str, marker: str = "MC_OPTIONAL") -> dict:
    """name -> (first, count) of the MC_OPTIONAL parameters (or those of another marker, such as MC_OPTIONAL2,
    MC_OPTIONAL3, MC_OPTIONAL4, MC_OPTIONAL5 or MC_OPTIONAL6) of each declaration in the C header at path that has them
    (one run of consecutive parameters)."""
    out = {}
    for _, name, params in _declarations(path):
        k = [i for i, p in enumerate(params) if re.search(rf"\b{marker}\b", p)]
        if k:
            if k != list(range(k[0], k[-1] + 1)):
                raise MinCurvLibError(f"{name}: the {marker} parameters must be consecutive")
            out[name] = (k[0], len(k))
    return out


def header_struct(path: str, name: str):
    """A ctypes.Structure with the fields of `typedef struct { ... } name;` in the C header at path (the scalar and
    pointer types of header_signatures)."""
    m = re.search(rf"typedef\s+struct\s*\{{([^}}]*)\}}\s*{name}\s*;", _c_source(path))
    if m is None:
        raise MinCurvLibError(f"{path}: no typedef struct {name}")
    fields = []
    for decl in filter(str.strip, m.group(1).split(";")):
        base, *rest = decl.split(",")
        first = re.match(r"\s*(.*?)([\s*]+)(\w+)\s*$", base)
        if first is None:
            raise MinCurvLibError(f"{name}: cannot read the field declaration '{decl.strip()}'")
        typ = first.group(1).strip()
        for stars, field in [(first.group(2), first.group(3))] + [re.match(r"\s*([\s*]*)(\w+)\s*$", r).groups()
                                                                  for r in rest]:
            stars = stars.strip()        # (a const scalar is passed as the scalar)
            fields.append((field, _ctype(typ + " " + stars if stars else re.sub(r"\bconst\b", "", typ), name)))
    return type(name, (ctypes.Structure,), {"_fields_": fields})


def header_define(path: str, name: str) -> int:
    """The integer value of `#define name value` (or `(value)`) in the C header at path."""
    with open(path) as f:
        m = re.search(rf"^[ \t]*#[ \t]*define[ \t]+{name}[ \t]+\(?(-?\d+)\)?", f.read(), flags=re.M)
    if m is None:
        raise MinCurvLibError(f"{path}: no #define {name}")
    return int(m.group(1))


_SIGS = header_signatures(_build.HEADER)
_OPTIONAL = optional_parameters(_build.HEADER)
_OPTIONAL2 = optional_parameters(_build.HEADER, "MC_OPTIONAL2")
_OPTIONAL3 = optional_parameters(_build.HEADER, "MC_OPTIONAL3")
_OPTIONAL4 = optional_parameters(_build.HEADER, "MC_OPTIONAL4")
_OPTIONAL5 = optional_parameters(_build.HEADER, "MC_OPTIONAL5")
_OPTIONAL6 = optional_parameters(_build.HEADER, "MC_OPTIONAL6")
EXPORTED_SYMBOLS = tuple(_SIGS)


def _with_optional(fn, *groups):
    """fn, which may also be called without its parameters [first, first + count) of the last of groups ((first, count)
    each, in release order), or without those of the last two, and so on: they are then NULL (0 for an int or a
    double), as the header documents for the MC_OPTIONAL .. MC_OPTIONAL6 parameters, so that a call written for the
    entry before they were added still binds its arguments to the right parameters."""
    forms = {}
    left_out = []
    for first, count in sorted(groups, reverse=True):       # (the later groups come after the earlier ones)
        left_out.append((first, tuple(0 if t is ctypes.c_int else 0.0 if t is ctypes.c_double else None
                                      for t in fn.argtypes[first:first + count])))
        forms[len(fn.argtypes) - sum(len(f) for _, f in left_out)] = list(reversed(left_out))

    def call(*args):
        for first, fill in forms.get(len(args), ()):
            args = args[:first] + fill + args[first:]
        return fn(*args)
    call.__name__, call.argtypes, call.restype = fn.__name__, fn.argtypes, fn.restype
    return call


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
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
        groups = [g[name] for g in (_OPTIONAL, _OPTIONAL2, _OPTIONAL3, _OPTIONAL4, _OPTIONAL5, _OPTIONAL6)
                  if name in g]
        if groups:
            setattr(lib, name, _with_optional(fn, *groups))
    _LIB = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().mc_last_error()
        raise MinCurvLibError(f"{what} failed with code {rc}: {msg.decode() if msg else ''}")
