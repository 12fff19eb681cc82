"""ctypes binding of the C-ABI in include/mincurv_b200.h.  There is no CPU fallback: importing the
compute entry points without the shared library (or calling them without a CUDA device) raises."""
from __future__ import annotations

import ctypes
import os

from . import build as _build

_c_int = ctypes.c_int
_c_dbl = ctypes.c_double
_vp = ctypes.c_void_p
_sz = ctypes.c_size_t

_LIB = None

_SIGS = {
    "mc_version": (_c_int, []),
    "mc_last_error": (ctypes.c_char_p, []),
    "mc_calc_splines_workspace_bytes": (_sz, [_c_int, _c_int]),
    "mc_calc_splines_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _vp, _c_int, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_workspace_bytes": (_sz, [_c_int, _c_int]),
    "mc_mincurv_solve_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _c_dbl, _vp, _vp, _vp, _vp, _vp, _vp,
                                        _vp, _sz, _vp]),
    "mc_mincurv_solve_batch_ex": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _c_dbl, _vp, _c_dbl, _vp, _vp, _vp, _vp,
                                           _vp, _vp, _sz, _vp]),
    "mc_mincurv_solve_batch_shared": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _c_dbl, _vp, _c_dbl, _vp, _vp, _vp,
                                               _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_setup_batch_shared": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _vp, _c_dbl, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_solve_batch_sens": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _c_dbl, _vp, _c_dbl, _vp, _vp, _vp, _vp,
                                             _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_adjoint_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _vp, _c_dbl, _vp, _vp, _vp, _vp, _vp, _vp,
                                          _vp, _vp, _sz, _vp]),
    "mc_mincurv_setup_batch_ex": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _vp, _c_dbl, _vp, _vp, _sz, _vp]),
    "mc_mincurv_setup_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_dbl, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_pdip_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_finalize_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_dbl, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_mincurv_kappa_batch": (_c_int, [_c_int, _c_int, _vp, _c_dbl, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_shortest_path_workspace_bytes": (_sz, [_c_int, _c_int]),
    "mc_shortest_path_solve_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _c_dbl, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_create_raceline_workspace_bytes": (_sz, [_c_int, _c_int]),
    "mc_create_raceline_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _vp, _vp, _c_dbl, _c_int, _vp, _vp, _vp, _vp,
                                          _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_calc_head_curv_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "mc_iqp_relinearise_workspace_bytes": (_sz, [_c_int, _c_int, _c_int]),
    "mc_iqp_relinearise_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _c_dbl, _c_int, _vp, _vp, _vp, _vp,
                                          _sz, _vp]),
    "mc_scale_alpha_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_dbl, _vp]),
    "mc_iqp_finish_batch": (_c_int, [_c_int, _c_int, _c_int, _c_int, _c_int, _c_dbl, _c_int, _c_int] + [_vp] * 16),
    "mc_vel_profile_workspace_bytes": (_sz, [_c_int, _c_int, _c_int]),
    "mc_vel_profile_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_int, _vp, _vp, _c_dbl, _c_int, _vp, _c_int, _vp,
                                      _c_dbl, _c_dbl, _c_dbl, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_vel_profile_batch_ex": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _c_int, _vp, _vp, _c_dbl, _c_int, _vp, _c_int, _vp,
                                         _c_dbl, _c_dbl, _c_dbl, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "mc_calc_ax_t_profile_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _vp, _vp, _c_dbl, _vp, _vp, _vp]),
    "mc_interp_track_workspace_bytes": (_sz, [_c_int, _c_int]),
    "mc_interp_track_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _vp, _c_dbl, _c_int, _c_dbl, _c_int, _vp, _vp, _vp,
                                       _sz, _vp]),
    "mc_min_bound_dists_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _c_int, _vp, _vp, _c_int, _vp, _vp, _c_int, _c_dbl,
                                          _c_dbl, _vp, _vp]),
    "mc_traj_extrema_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _c_dbl, _c_dbl, _vp, _vp]),
    "mc_assemble_trajectory_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _vp, _vp, _vp, _vp]),
    "mc_check_normals_crossing_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _c_int, _vp, _vp]),
    "mc_prep_track_workspace_bytes": (_sz, [_c_int, _c_int, _c_int]),
    "mc_prep_track_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _c_dbl, _c_dbl, _c_dbl, _c_dbl, _c_int, _c_int, _vp, _vp, _vp,
                                     _vp, _sz, _vp]),
    "mc_polygon_length_batch": (_c_int, [_c_int, _c_int, _vp, _vp, _c_int, _vp, _vp, _c_int, _c_dbl, _vp, _vp]),
    "mc_jitter_widths_batch": (_c_int, [_c_int, _c_int, _vp, _c_int, _vp, _vp, _vp, _c_dbl, _vp, _vp, _vp]),
    "mc_debug_read_profile": (_c_int, [_vp, _c_int]),
    "mc_debug_factor_solve": (_c_int, [_c_int, _c_int, _vp, _vp, _vp, _sz, _vp]),
}

EXPORTED_SYMBOLS = tuple(_SIGS)


class MinCurvLibError(RuntimeError):
    pass


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
    _LIB = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != 0:
        msg = load().mc_last_error()
        raise MinCurvLibError(f"{what} failed with code {rc}: {msg.decode() if msg else ''}")
