"""Batched device API of the H100 minimum-curvature path.

Thin host logic above the C-ABI (include/mincurv_b200.h): torch tensors are used only as device
buffer holders (allocation, streams); every computation happens in the CUDA kernels of
``libmincurv_b200.so``.  There is no CPU fallback -- without a CUDA device these functions raise.

The batched entry points have no counterpart in the reference (which solves one track per call);
the single-track modules next to this file (``opt_min_curv.py`` ...) mirror the tph call surface
used by main_globaltraj.py:264-290,371-387 on top of them.
"""
from __future__ import annotations

import ctypes
import functools
import math
from types import SimpleNamespace
from typing import Optional, Union

import torch

from . import _lib

# the workspace layout of the minimum-curvature path as the kernels were compiled with it (csrc/mincurv_ws.cuh,
# csrc/common.cuh): debugging and tests read intermediate results out of the workspace
SLAB_VECTORS, _CONSTS = _lib.slab_mirror()
HB_PITCH, ZB_PITCH = _CONSTS["HB_PITCH"], _CONSTS["ZB_PITCH"]
N_MIN = _CONSTS["N_MIN"]     # smallest closed track the banded solver supports
STATUS_TEXT = {
    0: "ok",
    1: "Problem not solvable, track might be too small to run with current safety distance!",
    2: "interior-point iteration cap reached",
    3: "numerical breakdown (non-positive pivot)",
    4: "curvature rows still violated after the curvature-row phase (constraints inconsistent)",
    -1: "unsupported track size",
}

# The two constants of trajectory_planning_helpers that cannot be confirmed offline (include/mincurv_b200.h,
# DESIGN.md section 2).  Run-time parameters of the C-ABI (*_ex entry points); tools/pin_against_tph.py determines them
# from the real package when it is importable and tests/test_real_tph.py then runs with what it found.
F_SCALE = 2.0               # tph.opt_min_curv: f = F_SCALE * E^T k_ref
VP_DECEL_SLICE_UPPER = 1    # tph.calc_vel_profile (closed): half of the doubled lap kept after the backward pass

_WS = {}


def mincurv_slab_layout(n_max: int) -> dict:
    """make_layout of csrc/mincurv_ws.cuh: offsets of one instance's slab, in doubles."""
    np_ = ((n_max + 31) // 32) * 32 + 64
    o = len(SLAB_VECTORS) * np_
    o_zb = o
    o += n_max * ZB_PITCH
    o_hb = o
    o += np_ * HB_PITCH
    o_tiles = o
    o += np_ * 67
    return dict(np=np_, o_zb=o_zb, o_hb=o_hb, o_tiles=o_tiles, stride=(o + 15) & ~15)


def _require_cuda() -> None:
    if not torch.cuda.is_available():
        raise _lib.MinCurvLibError("global_racetrajectory_optimization_b200 needs a CUDA device (H100, sm_90a); "
                                   "there is no CPU fallback")


def _ptr(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _device_guard(fn):
    """Run fn with the device of its first CUDA tensor argument current: the library launches on the calling thread's
    current device and on that device's current stream."""
    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        dev = next((a.device for a in list(args) + list(kwargs.values()) if isinstance(a, torch.Tensor) and a.is_cuda), None)
        if dev is None:
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    return wrapper


def _workspace(kind: str, nbytes: int, device) -> torch.Tensor:
    """Scratch buffer of the library for one (kind, device, stream): calls on different streams never share slabs or the
    work counter of the persistent solver kernels.  A buffer is allocated while its stream is current, so when a larger
    one replaces it the caching allocator re-uses the old block in that stream's order only."""
    dev = torch.device(device)
    key = (kind, str(dev), int(torch.cuda.current_stream(dev).cuda_stream) if dev.type == "cuda" else 0)
    ws = _WS.get(key)
    if ws is None or ws.numel() < nbytes:
        _WS[key] = None
        ws = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
        _WS[key] = ws
    return ws


def release_workspaces() -> None:
    _WS.clear()


def _f64(t: torch.Tensor, name: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise TypeError(f"{name} must be a CUDA tensor")
    if t.dtype != torch.float64:
        raise TypeError(f"{name} must be float64")
    return t.contiguous()


def _npts(n_pts, B, device):
    if n_pts is None:
        return None
    n_pts = n_pts.to(device=device, dtype=torch.int32).contiguous()
    if n_pts.numel() != B:
        raise ValueError("n_pts must have one entry per track")
    return n_pts


# ------------------------------------------------------------------------------------------------
@_device_guard
def calc_splines_batch(xy: torch.Tensor, n_pts: Optional[torch.Tensor] = None,
                       el_lengths: Optional[torch.Tensor] = None, use_dist_scaling: bool = True,
                       want_coeffs: bool = True):
    """Closed cubic splines through the points of every track.

    xy: [B, n_max, 2] (or a reftrack [B, n_max, 4]); returns (coeffs_x, coeffs_y, normvec, h)."""
    _require_cuda()
    xy = _f64(xy, "xy")
    B, n_max, stride = xy.shape
    dev = xy.device
    n_pts = _npts(n_pts, B, dev)
    cx = torch.zeros((B, n_max, 4), dtype=torch.float64, device=dev) if want_coeffs else None
    cy = torch.zeros((B, n_max, 4), dtype=torch.float64, device=dev) if want_coeffs else None
    nv = torch.zeros((B, n_max, 2), dtype=torch.float64, device=dev)
    h = torch.ones((B, n_max), dtype=torch.float64, device=dev)
    if el_lengths is not None:
        el_lengths = _f64(el_lengths, "el_lengths")
    ws = _workspace("splines", _lib.load().mc_calc_splines_workspace_bytes(B, n_max), dev)
    _call("mc_calc_splines_batch", B, n_max, n_pts, xy, stride, el_lengths, int(bool(use_dist_scaling)), cx, cy, nv, h,
          ws=ws)
    return cx, cy, nv, h


def _wveh(w_veh, B, dev):
    """(scalar, None) for a number, (0.0, [B] float64 tensor) for a tensor: the w_veh / w_veh_batch pair of the C-ABI."""
    if isinstance(w_veh, torch.Tensor):
        if w_veh.numel() != B:
            raise ValueError("w_veh tensor must have one entry per track")
        return 0.0, w_veh.to(device=dev, dtype=torch.float64).reshape(B).contiguous()
    return float(w_veh), None


def _chunk(B: int, per_item_bytes: int, device) -> int:
    free, _ = torch.cuda.mem_get_info(device)
    budget = max(int(free * 0.6), per_item_bytes)
    return max(1, min(B, budget // max(per_item_bytes, 1)))


def _rows(t: Optional[torch.Tensor]):
    """A per-instance argument of _launch_chunks: rows s:e of t for the chunk of instances s:e (anything but a tensor,
    None for NULL among it, stays as it is)."""
    return lambda s, e: t[s:e] if isinstance(t, torch.Tensor) else t


def _call(entry: str, *args, ws: Optional[torch.Tensor] = None) -> None:
    """Runs the C-ABI entry with args, a tensor passed as its pointer, None as NULL and anything else as it is, followed
    by the workspace and its size (with ws) and the current stream.  A nonzero return raises MinCurvLibError naming the
    entry."""
    c_args = [_ptr(a) if isinstance(a, torch.Tensor) else a for a in args]      # (args holds the tensors until the call)
    if ws is not None:
        c_args += [_ptr(ws), ws.numel()]
    _lib.check(getattr(_lib.load(), entry)(*c_args, _stream()), entry)


def _launch_chunks(entry: str, B: int, chunk: int, ws: torch.Tensor, *args) -> None:
    """_call of the entry on chunks of at most chunk of the B instances, with the chunk's size as B.  args are the entry's
    arguments between B and the workspace: a callable of (s, e) such as _rows gives the argument of the chunk of instances
    s:e, anything else is passed as _call passes it."""
    for s in range(0, B, chunk):
        e = min(B, s + chunk)
        _call(entry, e - s, *(a(s, e) if callable(a) else a for a in args), ws=ws)


def _mincurv_inputs(tracks: dict, shape_error: str, n_pts, w_veh, centre_id, max_chunk, f_scale) -> SimpleNamespace:
    """The checked and normalised inputs of opt_min_curv_batch and opt_min_curv_diff.  tracks: name -> (tensor, cols), every
    tensor [B, n_max, cols] ([B, n_max] for cols None; the first fixes B and n_max).  Returns a namespace of the tracks as
    contiguous float64 CUDA tensors, B, n_max, dev, n_pts, w_scalar and w_batch (see _wveh), centre_id (int32 or None),
    f_scale (None: F_SCALE) and chunk, the instances per launch."""
    t = {name: _f64(x, name) for name, (x, _) in tracks.items()}
    first = next(iter(t.values()))
    B, n_max = first.shape[:2]
    if any(t[name].shape != (B, n_max) + ((cols,) if cols else ()) for name, (_, cols) in tracks.items()):
        raise RuntimeError(shape_error)
    if n_max < N_MIN:
        raise NotImplementedError(f"closed tracks with fewer than {N_MIN} points are not supported by the banded solver")
    dev = first.device
    n_pts = _npts(n_pts, B, dev)
    w_scalar, w_batch = _wveh(w_veh, B, dev)
    if centre_id is not None:
        if centre_id.shape != (B,):
            raise ValueError("centre_id must be [B]")
        centre_id = centre_id.to(device=dev, dtype=torch.int32).contiguous()
    per_item = _lib.load().mc_mincurv_workspace_bytes(1, n_max)
    return SimpleNamespace(**t, B=B, n_max=n_max, dev=dev, n_pts=n_pts, w_scalar=w_scalar, w_batch=w_batch,
                           centre_id=centre_id, f_scale=float(F_SCALE if f_scale is None else f_scale),
                           chunk=_chunk(B, per_item, dev) if max_chunk is None else min(B, max_chunk))


def _mincurv_results(B: int, n_max: int, dev) -> dict:
    """Buffers for the per-instance results of a solve, in the order of the C-ABI."""
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    return dict(alpha=torch.empty((B, n_max), **f64), curv_error_max=torch.empty((B,), **f64),
                kappa_lin_max=torch.empty((B,), **f64), status=torch.empty((B,), **i32), iters=torch.empty((B,), **i32))


@_device_guard
def opt_min_curv_batch(reftrack: torch.Tensor, normvec: torch.Tensor, h: torch.Tensor, kappa_bound: float,
                       w_veh: Union[float, torch.Tensor], n_pts: Optional[torch.Tensor] = None,
                       max_chunk: Optional[int] = None, f_scale: Optional[float] = None,
                       centre_id: Optional[torch.Tensor] = None, lin_alpha: Optional[torch.Tensor] = None) -> dict:
    """Batched tph.opt_min_curv (closed tracks).  Returns a dict of device tensors:
    alpha [B, n_max], curv_error_max [B], kappa_lin_max [B], status [B] (int32), iters [B] (int32).
    f_scale: None = the module default F_SCALE (see there).
    centre_id [B] (optional): for batches in which several instances share a centreline (x, y, normvec, h, n_pts identical;
    only the widths differ -- a width sweep of one track): centre_id[b] = index of the instance that owns b's centreline
    (owners: centre_id[b] == b).  H, f and k_ref are then assembled once per centreline (same results, less work);
    shared_centre_ids() builds the tensor from group labels.
    lin_alpha [B, n_max] (optional): the QP linearised about the line reftrack + lin_alpha * normvec on the same grid
    instead of the centre line (the step of tph's iterative QP without re-sampling; DESIGN.md section 3.2): the curvature
    rows, H and f use that line's first derivatives, and curv_error_max and kappa_lin_max refer to that linearisation.
    alpha is still the shift from the centre line.  With centre_id a follower is linearised about its owner's row."""
    _require_cuda()
    if lin_alpha is not None and (lin_alpha.shape != h.shape):
        raise ValueError(f"opt_min_curv_batch: lin_alpha must be [B, n_max] like h, got {tuple(lin_alpha.shape)}")
    a = _mincurv_inputs(dict(reftrack=(reftrack, 4), normvec=(normvec, 2), h=(h, None)),
                        "Array size of reftrack should be the same as normvectors!", n_pts, w_veh, centre_id, max_chunk, f_scale)
    out = _mincurv_results(a.B, a.n_max, a.dev)
    if lin_alpha is not None:
        lin = _f64(lin_alpha, "lin_alpha")
        invalid = None
        if a.centre_id is not None:
            # a follower is linearised about its owner's row, as the shared assembly does; the instances are solved one by
            # one (bitwise what the shared solve gives), a follower without a valid owner gets status -1 as there
            o = a.centre_id.long()
            oc = o.clamp(0, a.B - 1)
            invalid = (o < 0) | (o >= a.B) | (a.centre_id[oc] != oc.to(torch.int32))
            if a.n_pts is not None:
                invalid |= a.n_pts[oc] != a.n_pts
            lin = lin[oc].contiguous()
        ws = _workspace("mincurv", _lib.load().mc_mincurv_workspace_bytes(a.chunk, a.n_max), a.dev)
        _launch_chunks("mc_mincurv_solve_batch_ex", a.B, a.chunk, ws, a.n_max, *map(_rows, (a.n_pts, a.reftrack, a.normvec,
                       a.h)), float(kappa_bound), a.w_scalar, _rows(a.w_batch), a.f_scale, *map(_rows, out.values()), 0.0,
                       None, None, _rows(lin))
        if invalid is not None:
            out["status"] = torch.where(invalid, -1, out["status"]).to(torch.int32)
        return out
    _mincurv_launch("mc_mincurv_solve_batch_shared", a.chunk, a.n_pts, a.reftrack, a.normvec, a.h, float(kappa_bound),
                    a.w_scalar, a.w_batch, a.f_scale, a.centre_id, *out.values())
    return out


def shared_centre_ids(group: torch.Tensor) -> torch.Tensor:
    """centre_id for opt_min_curv_batch from group labels [B] (any integers: instances with equal labels share a
    centreline): the first instance of every group becomes its owner.  Returns int32 [B] on the labels' device."""
    vals, inv = torch.unique(group, return_inverse=True)
    idx = torch.arange(group.shape[0], device=group.device, dtype=torch.int64)
    first = torch.full((vals.shape[0],), group.shape[0], device=group.device, dtype=torch.int64)
    first = first.scatter_reduce(0, inv, idx, reduce="amin")
    return first[inv].to(torch.int32)


def _chunk_centre_ids(centre_id, B):
    """centre_id as a per-instance argument of _launch_chunks: owners are addressed inside the chunk, the first instance of
    the chunk with the same owner takes the role."""
    return lambda s, e: centre_id if centre_id is None or (s == 0 and e == B) else shared_centre_ids(centre_id[s:e])


def _mincurv_launch(entry: str, chunk: int, n_pts, reftrack, normvec, h, kappa_bound, w_scalar, w_batch, f_scale, centre_id,
                    *outputs) -> None:
    """Runs the C-ABI entry mc_mincurv_solve_batch_shared, mc_mincurv_solve_batch_sens or mc_mincurv_adjoint_batch on
    chunks of at most chunk instances.  The arguments are the entry's own in its order, outputs the arguments after
    centre_id: a tensor is split by instances, a callable of (s, e) gives the argument of the chunk s:e, anything else
    is passed as it is; kappa_bound is None for the adjoint, which takes none."""
    B, n_max = h.shape
    ws = _workspace("mincurv", _lib.load().mc_mincurv_workspace_bytes(chunk, n_max), h.device)
    kb = () if kappa_bound is None else (kappa_bound,)
    _launch_chunks(entry, B, chunk, ws, n_max, *map(_rows, (n_pts, reftrack, normvec, h)), *kb, w_scalar, _rows(w_batch),
                   f_scale, _chunk_centre_ids(centre_id, B), *(o if callable(o) else _rows(o) for o in outputs))


def _wanted(B: int, *grads, device=None) -> torch.Tensor:
    """bool [B]: the instances with a nonzero upstream gradient in any of grads (each [B, ...] or None, which counts as
    zero).  device: where the mask lives when every gradient is None (autograd passes None for an output it has no
    gradient for when the function does not materialise them)."""
    wanted = torch.zeros((B,), dtype=torch.bool, device=next((g.device for g in grads if g is not None), device))
    for g in grads:
        if g is not None:
            wanted |= (g != 0).flatten(1).any(dim=1) if g.ndim > 1 else g != 0
    return wanted


def _refuse(strict: bool, wanted: torch.Tensor, gs: torch.Tensor, who: str, what: str) -> None:
    """strict: raise if an instance with a nonzero upstream gradient (wanted [B]) has grad_status gs != 0."""
    bad = wanted & (gs != 0)
    if strict and bool(bad.any()):
        idx = bad.nonzero().flatten()
        raise _lib.MinCurvLibError(f"{who} for {idx.numel()} instance(s) {what} (first: {idx[:8].tolist()}, "
                                   f"grad_status {gs[idx[:8]].tolist()}); strict=False gives them zero gradients")


class _MinCurvDiff(torch.autograd.Function):
    """alpha of the min-curvature QP as a function of the widths; see opt_min_curv_diff."""

    @staticmethod
    def forward(ctx, widths, w_veh_t, centre, normvec, h, kappa_bound, w_scalar, n_pts, centre_id, chunk, f_scale, strict,
                curvature_rows):
        B, n_max, _ = centre.shape
        dev = centre.device
        reftrack = torch.cat((centre, widths), dim=2).contiguous()
        alpha, cerr, kmax, status, iters = _mincurv_results(B, n_max, dev).values()
        sens = torch.empty((B, 2, n_max), dtype=torch.float64, device=dev)
        grad_status = torch.empty((B,), dtype=torch.int32, device=dev)
        sens_rows = torch.empty((B, n_max), dtype=torch.float64, device=dev) if curvature_rows else None
        n_rows = torch.empty((B,), dtype=torch.int32, device=dev) if curvature_rows else None
        _mincurv_launch("mc_mincurv_solve_batch_sens", chunk, n_pts, reftrack, normvec, h, kappa_bound, w_scalar, w_veh_t,
                        f_scale, centre_id, alpha, cerr, kmax, status, iters, sens, grad_status, sens_rows, n_rows)
        ctx.save_for_backward(widths, centre, normvec, h, w_veh_t, n_pts, centre_id, sens, grad_status, sens_rows, n_rows)
        ctx.w_scalar, ctx.chunk, ctx.f_scale, ctx.strict = w_scalar, chunk, f_scale, strict
        ctx.mark_non_differentiable(cerr, kmax, status, iters, grad_status)
        return alpha, cerr, kmax, status, iters, grad_status

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_alpha, *_unused):
        widths, centre, normvec, h, w_veh_t, n_pts, centre_id, sens, grad_status, sens_rows, n_rows = ctx.saved_tensors
        B, n_max, _ = centre.shape
        dev = centre.device
        grad_alpha = grad_alpha.to(dtype=torch.float64).contiguous()
        wanted = _wanted(B, grad_alpha)
        who = "opt_min_curv_diff: no width gradient"
        _refuse(ctx.strict, wanted, grad_status, who, "with a nonzero upstream gradient")
        gs = grad_status.clone()            # (the adjoint sets 3 where its factorisation breaks down)
        reftrack = torch.cat((centre, widths), dim=2).contiguous()
        gwr = torch.empty((B, n_max), dtype=torch.float64, device=dev)
        gwl = torch.empty((B, n_max), dtype=torch.float64, device=dev)
        gwv = torch.empty((B,), dtype=torch.float64, device=dev)
        chunk, rows = ctx.chunk, (None, None, None, 0)
        if sens_rows is not None:
            # the Schur complement of the strong rows: cap^2 doubles per instance of a chunk, next to its slab
            cap = int(n_rows.max())
            per_item = _lib.load().mc_mincurv_workspace_bytes(1, n_max) + 8 * cap * cap
            chunk = min(chunk, _chunk(B, per_item, dev))
            schur = torch.empty((chunk, max(cap * cap, 1)), dtype=torch.float64, device=dev)
            rows = (sens_rows, n_rows, lambda s, e: schur, cap)
        _mincurv_launch("mc_mincurv_adjoint_batch", chunk, n_pts, reftrack, normvec, h, None, ctx.w_scalar, w_veh_t,
                        ctx.f_scale, centre_id, sens, gs, grad_alpha, gwr, gwl, gwv, *rows, None)
        _refuse(ctx.strict, wanted, gs, who, "whose adjoint factorisation broke down")
        return (torch.stack((gwr, gwl), dim=2), gwv if w_veh_t is not None else None) + (None,) * 11


@_device_guard
def opt_min_curv_diff(centre: torch.Tensor, widths: torch.Tensor, normvec: torch.Tensor, h: torch.Tensor, kappa_bound: float,
                      w_veh: Union[float, torch.Tensor], n_pts: Optional[torch.Tensor] = None,
                      centre_id: Optional[torch.Tensor] = None, max_chunk: Optional[int] = None,
                      f_scale: Optional[float] = None, strict: bool = True, curvature_rows: bool = False) -> dict:
    """opt_min_curv_batch with alpha differentiable with respect to the track widths and the vehicle width (autograd).

    centre [B, n_max, 2] (x, y) and widths [B, n_max, 2] (w_tr_right, w_tr_left) make up the reftrack of
    opt_min_curv_batch; w_veh is a float or a [B] tensor.  Returns the dict of opt_min_curv_batch (alpha, curv_error_max,
    kappa_lin_max, status, iters: the same values) plus grad_status [B] (int32).  alpha carries a grad_fn: backward() /
    torch.autograd.grad give dL/dwidths [B, n_max, 2] and, for a tensor w_veh, dL/dw_veh, at the cost of one assembly, one
    factorisation and one solve per instance (implicit differentiation of the KKT conditions, DESIGN.md section 3.10).
    centre, normvec and h are constants: they must not require grad.
    grad_status: 0 = the gradient is computed; 4 = the curvature rows were active (solved by the curvature-row phase),
    not supported; otherwise the solve's status (1, 2, 3, -1).  strict=True: backward raises if an instance with a
    nonzero upstream gradient has grad_status != 0 (or its adjoint factorisation breaks down); strict=False: such
    instances get zero gradients.
    curvature_rows=True: the instances the curvature-row phase solved are differentiated too, at that phase's final
    iterate (DESIGN.md section 3.10, curvature rows): the forward exports 8 more bytes per point, grad_status is the final
    solve status (4 only where the rows stay violated), and the backward reads the largest count of strongly active rows
    once from the device to size their Schur complements.  The forward's values are those of curvature_rows=False bit
    for bit, and so are the gradients of the instances the box phase solved."""
    _require_cuda()
    for t, name in ((centre, "centre"), (normvec, "normvec"), (h, "h")):
        if isinstance(t, torch.Tensor) and t.requires_grad:
            raise ValueError(f"opt_min_curv_diff: {name} is a constant (no gradient with respect to it); detach it")
    a = _mincurv_inputs(dict(centre=(centre, 2), widths=(widths, 2), normvec=(normvec, 2), h=(h, None)),
                        "opt_min_curv_diff: centre and widths must be [B, n_max, 2], normvec [B, n_max, 2], h [B, n_max]",
                        n_pts, w_veh, centre_id, max_chunk, f_scale)
    alpha, cerr, kmax, status, iters, grad_status = _MinCurvDiff.apply(
        a.widths, a.w_batch, a.centre, a.normvec, a.h, float(kappa_bound), a.w_scalar, a.n_pts, a.centre_id, a.chunk,
        a.f_scale, bool(strict), bool(curvature_rows))
    return dict(alpha=alpha, curv_error_max=cerr, kappa_lin_max=kmax, status=status, iters=iters, grad_status=grad_status)


@_device_guard
def opt_shortest_path_batch(reftrack: torch.Tensor, normvec: torch.Tensor, w_veh: Union[float, torch.Tensor],
                            n_pts: Optional[torch.Tensor] = None) -> dict:
    """Batched tph.opt_shortest_path.  Returns dict(alpha, status, iters)."""
    _require_cuda()
    reftrack, normvec, n_pts, w_scalar, w_batch = _shortest_path_inputs(reftrack, normvec, w_veh, n_pts)
    B, n_max, _ = reftrack.shape
    dev = reftrack.device
    alpha = torch.empty((B, n_max), dtype=torch.float64, device=dev)
    status = torch.empty((B,), dtype=torch.int32, device=dev)
    iters = torch.empty((B,), dtype=torch.int32, device=dev)
    ws = _workspace("shortest", _lib.load().mc_shortest_path_workspace_bytes(B, n_max), dev)
    _call("mc_shortest_path_solve_batch", B, n_max, n_pts, reftrack, normvec, w_scalar, w_batch, alpha, status, iters, ws=ws)
    return dict(alpha=alpha, status=status, iters=iters)


def _shortest_path_inputs(reftrack, normvec, w_veh, n_pts):
    """The checked inputs of opt_shortest_path_batch and opt_shortest_path_diff: reftrack [B, n_max, 4] and normvec
    [B, n_max, 2] as contiguous float64 CUDA tensors, n_pts (int32 or None) and the w_veh pair of _wveh."""
    reftrack = _f64(reftrack, "reftrack")
    normvec = _f64(normvec, "normvec")
    B, n_max, four = reftrack.shape
    if four != 4 or normvec.shape != (B, n_max, 2):
        raise RuntimeError("Array size of reftrack should be the same as normvectors!")
    return (reftrack, normvec, _npts(n_pts, B, reftrack.device)) + _wveh(w_veh, B, reftrack.device)


class _ShortestPathDiff(torch.autograd.Function):
    """alpha of the shortest-path QP as a function of the reftrack, the normals and w_veh; see opt_shortest_path_diff."""

    @staticmethod
    def forward(ctx, reftrack, normvec, w_veh_t, w_scalar, n_pts, strict):
        B, n_max, _ = reftrack.shape
        f64, i32 = dict(dtype=torch.float64, device=reftrack.device), dict(dtype=torch.int32, device=reftrack.device)
        alpha, status, iters = torch.empty((B, n_max), **f64), torch.empty((B,), **i32), torch.empty((B,), **i32)
        sens, grad_status = torch.empty((B, 2, n_max), **f64), torch.empty((B,), **i32)
        ws = _workspace("shortest", _lib.load().mc_shortest_path_workspace_bytes(B, n_max), reftrack.device)
        _call("mc_shortest_path_solve_batch_sens", B, n_max, n_pts, reftrack, normvec, w_scalar, w_veh_t, alpha, status, iters,
              sens, grad_status, ws=ws)
        ctx.save_for_backward(reftrack, normvec, w_veh_t, n_pts, alpha, sens, grad_status)
        ctx.w_scalar, ctx.strict = w_scalar, strict
        ctx.mark_non_differentiable(status, iters, grad_status)
        return alpha, status, iters, grad_status

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_alpha, *_unused):
        reftrack, normvec, w_veh_t, n_pts, alpha, sens, grad_status = ctx.saved_tensors
        B, n_max, _ = reftrack.shape
        f64 = dict(dtype=torch.float64, device=reftrack.device)
        grad_alpha = grad_alpha.to(dtype=torch.float64).contiguous()
        wanted = _wanted(B, grad_alpha)
        who = "opt_shortest_path_diff: no gradient"
        _refuse(ctx.strict, wanted, grad_status, who, "with a nonzero upstream gradient")
        gs = grad_status.clone()            # (the adjoint sets 3 where its solution is not finite)
        need_rt, need_nv, need_wv = ctx.needs_input_grad[:3]
        grt = torch.empty((B, n_max, 4), **f64)
        gnv = torch.empty((B, n_max, 2), **f64) if need_nv else None
        gwv = torch.empty((B,), **f64) if need_wv else None
        ws = _workspace("shortest", _lib.load().mc_shortest_path_workspace_bytes(B, n_max), reftrack.device)
        _call("mc_shortest_path_adjoint_batch", B, n_max, n_pts, reftrack, normvec, ctx.w_scalar, w_veh_t, alpha, sens, gs,
              grad_alpha, grt, gnv, gwv, ws=ws)
        _refuse(ctx.strict, wanted, gs, who, "whose adjoint solution is not finite")
        return grt if need_rt else None, gnv, gwv, None, None, None


@_device_guard
def opt_shortest_path_diff(reftrack: torch.Tensor, normvec: torch.Tensor, w_veh: Union[float, torch.Tensor],
                           n_pts: Optional[torch.Tensor] = None, strict: bool = True) -> dict:
    """opt_shortest_path_batch with alpha differentiable with respect to the reftrack, the normals and the vehicle width
    (autograd).

    Returns the dict of opt_shortest_path_batch (alpha, status, iters: the same values) plus grad_status [B] (int32).
    alpha carries a grad_fn: backward() / torch.autograd.grad give dL/dreftrack [B, n_max, 4] (x, y at fixed normals,
    w_tr_right, w_tr_left), dL/dnormvec [B, n_max, 2] and, for a tensor w_veh, dL/dw_veh, at the cost of one cyclic
    tridiagonal solve per instance (implicit differentiation of the KKT conditions, DESIGN.md section 3.11).  Any of the
    three may be a constant.  Widths whose bound tph clamps to 0.001 m get zero gradients.
    grad_status: 0 = the gradient is computed; otherwise the solve's status (2, 3, -1).  strict=True: backward raises if
    an instance with a nonzero upstream gradient has grad_status != 0 (or a non-finite adjoint solution); strict=False:
    such instances get zero gradients."""
    _require_cuda()
    reftrack, normvec, n_pts, w_scalar, w_batch = _shortest_path_inputs(reftrack, normvec, w_veh, n_pts)
    alpha, status, iters, grad_status = _ShortestPathDiff.apply(reftrack, normvec, w_batch, w_scalar, n_pts, bool(strict))
    return dict(alpha=alpha, status=status, iters=iters, grad_status=grad_status)


def _closed_polygon_length(pts: torch.Tensor, n_pts: Optional[torch.Tensor], normvec: Optional[torch.Tensor] = None,
                           shift: Optional[torch.Tensor] = None, shift_stride: int = 1, sign: float = 1.0) -> torch.Tensor:
    """Length [B] of the closed polygon through the first n_pts[b] points p_i (+ sign * shift_i * n_i) of every row
    (mc_polygon_length_batch: a block reduction per track on the device)."""
    B, n_max, stride = pts.shape
    out = torch.zeros((B,), dtype=torch.float64, device=pts.device)
    _call("mc_polygon_length_batch", B, n_max, n_pts, pts, stride, normvec, shift, int(shift_stride), float(sign), out)
    return out


@_device_guard
def create_raceline_batch(refline: torch.Tensor, normvec: torch.Tensor, alpha: torch.Tensor, stepsize_interp: float,
                          n_pts: Optional[torch.Tensor] = None, n_out_max: Optional[int] = None,
                          with_head_curv: bool = True) -> dict:
    """Batched tph.create_raceline (+ tph.calc_head_curv_an at the resampled points).

    refline: [B, n_max, 2] or a reftrack [B, n_max, 4].  If n_out_max is None an upper bound is derived from
    the polygon length of the shifted line (one small device->host read) and the call is repeated with a larger one if
    a track still does not fit; with an explicit n_out_max an overflow is reported as n_out[b] = -(points needed)."""
    _require_cuda()
    refline = _f64(refline, "refline")
    normvec = _f64(normvec, "normvec")
    alpha = _f64(alpha, "alpha")
    B, n_max, stride = refline.shape
    dev = refline.device
    f64, i32 = dict(dtype=torch.float64, device=dev), dict(dtype=torch.int32, device=dev)
    n_pts = _npts(n_pts, B, dev)
    derived = n_out_max is None
    if derived:
        poly = _closed_polygon_length(refline, n_pts, normvec=normvec, shift=alpha)
        n_out_max = int(math.ceil(float(poly.max().item()) * 1.1 / float(stepsize_interp))) + 16
    n_out_max = int(n_out_max)
    while True:
        out = dict(       # (in the order of the C-ABI)
            coeffs_x=torch.zeros((B, n_max, 4), **f64), coeffs_y=torch.zeros((B, n_max, 4), **f64),
            spline_lengths=torch.zeros((B, n_max), **f64), n_out=torch.zeros((B,), **i32),
            raceline_interp=torch.zeros((B, n_out_max, 2), **f64), spline_inds=torch.zeros((B, n_out_max), **i32),
            t_values=torch.zeros((B, n_out_max), **f64), s_interp=torch.zeros((B, n_out_max), **f64),
            el_lengths_interp=torch.zeros((B, n_out_max), **f64),
            psi=torch.zeros((B, n_out_max), **f64) if with_head_curv else None,
            kappa=torch.zeros((B, n_out_max), **f64) if with_head_curv else None,
        )
        ws = _workspace("splines", _lib.load().mc_create_raceline_workspace_bytes(B, n_max), dev)
        _call("mc_create_raceline_batch", B, n_max, n_pts, refline, stride, normvec, alpha, float(stepsize_interp), n_out_max,
              *out.values(), ws=ws)
        if not derived:           # the caller fixed the capacity: an overflow is reported as n_out[b] = -(points needed)
            return out
        need = int((-out["n_out"]).max().item())
        if need <= 0:
            return out
        n_out_max = need + 16     # (the spline is longer than 1.1 x its polygon: re-run with what the kernel asked for)


_RL_KEYS = ("raceline_interp", "kappa", "el_lengths_interp", "coeffs_x", "coeffs_y", "spline_lengths", "n_out",
            "spline_inds", "t_values", "s_interp", "psi")


class _CreateRacelineDiff(torch.autograd.Function):
    """raceline_interp, kappa and el_lengths_interp of create_raceline as functions of alpha, the reference line and the
    normals; see create_raceline_diff."""

    @staticmethod
    def forward(ctx, refline, normvec, alpha, stepsize_interp, n_pts, n_out_max, strict):
        out = create_raceline_batch(refline, normvec, alpha, stepsize_interp, n_pts=n_pts, n_out_max=n_out_max)
        res = tuple(out[k] for k in _RL_KEYS)
        ctx.save_for_backward(normvec, alpha, n_pts, out["coeffs_x"], out["coeffs_y"], out["spline_lengths"], out["n_out"],
                              out["spline_inds"], out["t_values"])
        ctx.ref_cols, ctx.strict = refline.shape[2], strict
        ctx.mark_non_differentiable(*res[3:])
        ctx.set_materialize_grads(False)
        return res

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_ri, g_kappa, g_el, *_unused):
        normvec, alpha, n_pts, cx, cy, sl, n_out, si, tv = ctx.saved_tensors
        lib = _lib.load()
        B, n_max = alpha.shape
        f64 = dict(dtype=torch.float64, device=alpha.device)
        g_ri, g_kappa, g_el = (None if g is None else g.to(**f64).contiguous() for g in (g_ri, g_kappa, g_el))
        wanted = _wanted(B, g_ri, g_kappa, g_el, device=alpha.device)
        # n_out <= 0: an overflow of an explicit n_out_max (-points needed) or an inactive track: nothing to differentiate
        _refuse(ctx.strict, wanted, (n_out <= 0).to(torch.int32), "create_raceline_diff: no gradient",
                "with n_out <= 0 (overflow of n_out_max or an inactive track)")
        need_ref, need_nv, _ = ctx.needs_input_grad[:3]
        g_alpha = torch.empty((B, n_max), **f64)
        g_ref = torch.empty((B, n_max, 2), **f64) if need_ref else None
        g_nv = torch.empty((B, n_max, 2), **f64) if need_nv else None
        chunk = _chunk(B, lib.mc_create_raceline_adjoint_workspace_bytes(1, n_max), alpha.device)
        ws = _workspace("raceline_adjoint", lib.mc_create_raceline_adjoint_workspace_bytes(chunk, n_max), alpha.device)
        _launch_chunks("mc_create_raceline_adjoint_batch", B, chunk, ws, n_max, *map(_rows, (n_pts, normvec, alpha)),
                       si.shape[1], *map(_rows, (cx, cy, sl, n_out, si, tv, g_ri, g_kappa, g_el, g_alpha, g_ref, g_nv)))
        if g_ref is not None and ctx.ref_cols != 2:               # the width columns of a reftrack: no influence
            g_ref = torch.cat((g_ref, torch.zeros((B, n_max, ctx.ref_cols - 2), **f64)), dim=2)
        return g_ref, g_nv, g_alpha if ctx.needs_input_grad[2] else None, None, None, None, None


@_device_guard
def create_raceline_diff(refline: torch.Tensor, normvec: torch.Tensor, alpha: torch.Tensor, stepsize_interp: float,
                         n_pts: Optional[torch.Tensor] = None, n_out_max: Optional[int] = None, strict: bool = True) -> dict:
    """create_raceline_batch with raceline_interp, kappa and el_lengths_interp differentiable with respect to alpha, the
    reference line (x, y; the width columns of a [B, n, 4] reftrack get zeros) and the normals (autograd).

    Returns the dict of create_raceline_batch (the same values).  Every other entry, psi included, is not differentiable.
    The derivative holds n_out and every station's spline segment at the forward's; one CTA per track walks the
    stations, the lengths and the moment system backwards (DESIGN.md section 3.12).  Any input may be a constant.
    strict=True: backward raises for a track with n_out <= 0 (an overflow of an explicit n_out_max, or an inactive track)
    that received a nonzero upstream gradient; strict=False: such tracks get zero gradients."""
    _require_cuda()
    refline, normvec, alpha = _f64(refline, "refline"), _f64(normvec, "normvec"), _f64(alpha, "alpha")
    B, n_max, cols = refline.shape
    if cols not in (2, 4) or normvec.shape != (B, n_max, 2) or alpha.shape != (B, n_max):
        raise RuntimeError("create_raceline_diff: refline must be [B, n_max, 2 or 4], normvec [B, n_max, 2], alpha [B, n_max]")
    res = _CreateRacelineDiff.apply(refline, normvec, alpha, float(stepsize_interp), _npts(n_pts, B, refline.device),
                                    n_out_max, bool(strict))
    return dict(zip(_RL_KEYS, res))


@_device_guard
def calc_head_curv_batch(coeffs_x: torch.Tensor, coeffs_y: torch.Tensor, ind_spls: torch.Tensor, t_spls: torch.Tensor,
                         n_eval: Optional[torch.Tensor] = None, calc_curv: bool = True, calc_dcurv: bool = False):
    _require_cuda()
    if not calc_curv and calc_dcurv:
        raise ValueError("dkappa cannot be calculated without kappa!")
    coeffs_x = _f64(coeffs_x, "coeffs_x")
    coeffs_y = _f64(coeffs_y, "coeffs_y")
    t_spls = _f64(t_spls, "t_spls")
    B, n_max, _ = coeffs_x.shape
    dev = coeffs_x.device
    ind = ind_spls.to(device=dev, dtype=torch.int32).contiguous()
    n_eval_max = t_spls.shape[1]
    psi = torch.empty((B, n_eval_max), dtype=torch.float64, device=dev)
    kappa = torch.empty_like(psi) if calc_curv else None
    dkappa = torch.empty_like(psi) if calc_dcurv else None
    _call("mc_calc_head_curv_batch", B, n_max, coeffs_x, coeffs_y, n_eval_max, _npts(n_eval, B, dev), ind, t_spls, psi, kappa,
          dkappa)
    return psi, kappa, dkappa


@_device_guard
def iqp_relinearise_batch(reftrack, normvec, alpha, stepsize_interp, n_pts=None, active=None, n_max_new=None):
    """One re-linearisation step of tph.iqp_handler for every (active) track: returns
    (reftrack_new [B, n_max_new, 4], normvec_new [B, n_max_new, 2], n_pts_new [B])."""
    _require_cuda()
    reftrack = _f64(reftrack, "reftrack")
    normvec = _f64(normvec, "normvec")
    alpha = _f64(alpha, "alpha")
    B, n_max, _ = reftrack.shape
    dev = reftrack.device
    n_pts = _npts(n_pts, B, dev)
    if n_max_new is None:
        n_max_new = n_max + 64
    if active is not None:
        active = active.to(device=dev, dtype=torch.int32).contiguous()
    rnew = torch.zeros((B, n_max_new, 4), dtype=torch.float64, device=dev)
    nnew = torch.zeros((B, n_max_new, 2), dtype=torch.float64, device=dev)
    npn = torch.zeros((B,), dtype=torch.int32, device=dev)
    ws = _workspace("iqp", _lib.load().mc_iqp_relinearise_workspace_bytes(B, n_max, n_max_new), dev)
    _call("mc_iqp_relinearise_batch", B, n_max, n_pts, active, reftrack, normvec, alpha, float(stepsize_interp), int(n_max_new),
          rnew, nnew, npn, ws=ws)
    return rnew, nnew, npn


@_device_guard
def scale_alpha_batch(alpha: torch.Tensor, scale: Union[float, torch.Tensor]) -> None:
    B, n_max = alpha.shape
    sb = scale.to(device=alpha.device, dtype=torch.float64).contiguous() if isinstance(scale, torch.Tensor) else None
    _call("mc_scale_alpha_batch", B, n_max, alpha, sb, 1.0 if sb is not None else float(scale))


@_device_guard
def iqp_batch(reftrack: torch.Tensor, normvec: torch.Tensor, h: torch.Tensor, kappa_bound: float,
              w_veh: Union[float, torch.Tensor], stepsize_interp: float, iters_min: int = 3,
              curv_error_allowed: float = 0.01, n_pts: Optional[torch.Tensor] = None, max_iters: int = 50,
              fixed_iters: Optional[int] = None, _n_cap_min: int = 0) -> dict:
    """Batched tph.iqp_handler (SURVEY.md A.5): per-instance outer iterations with damping and
    re-linearisation; an instance leaves the loop once iter >= iters_min and its curv_error_max <=
    curv_error_allowed.  Returns dict(alpha [B, n_cap], reftrack [B, n_cap, 4], normvec [B, n_cap, 2],
    n_pts [B], outer_iters [B], status [B], qp_solves) -- every array refers to the instance's LAST iteration.
    status: the QP status of that iteration, or 2 if max_iters outer iterations did not reach curv_error_allowed (tph
    would keep iterating).  One small device->host read per outer iteration.

    fixed_iters: run exactly that many outer iterations for every instance (bench config C3).  Nothing has to be decided
    on the host between the iterations then, so they are queued back to back and the one thing the host would have
    looked at -- a re-sampled track that does not fit the capacity -- is checked once at the end (and the call repeated
    with the larger capacity, which the 5 % + 50 m of slack makes a rare event)."""
    _require_cuda()
    reftrack0, normvec0, h0 = reftrack, normvec, h           # (the caller's arrays: never written)
    reftrack = _f64(reftrack, "reftrack").clone()
    normvec = _f64(normvec, "normvec").clone()
    h = _f64(h, "h").clone()
    B, n_max, _ = reftrack.shape
    dev = reftrack.device
    cur_n = (n_pts.to(device=dev, dtype=torch.int32).clone() if n_pts is not None
             else torch.full((B,), n_max, dtype=torch.int32, device=dev))
    # capacity of the re-sampled tracks: the raceline is re-sampled every stepsize_interp metres, so its point count
    # follows from its length, not from n_max (a track given at a coarser spacing grows); 5 % + 50 m of slack on the
    # reference polygon, and the relinearisation step below grows the buffers if a track still does not fit
    poly = float(_closed_polygon_length(reftrack, cur_n).max().item())
    n_cap = max(n_max + 64, int(math.ceil((1.05 * poly + 50.0) / float(stepsize_interp))) + 16, int(_n_cap_min))

    def _alloc(cap):
        return dict(alpha=torch.zeros((B, cap), dtype=torch.float64, device=dev),
                    reftrack=torch.zeros((B, cap, 4), dtype=torch.float64, device=dev),
                    normvec=torch.zeros((B, cap, 2), dtype=torch.float64, device=dev))

    fin = _alloc(n_cap)
    fin.update(n_pts=torch.zeros((B,), dtype=torch.int32, device=dev),
               outer_iters=torch.zeros((B,), dtype=torch.int32, device=dev),
               status=torch.zeros((B,), dtype=torch.int32, device=dev),
               curv_error_max=torch.zeros((B,), dtype=torch.float64, device=dev))
    active = torch.ones((B,), dtype=torch.int32, device=dev)
    counters = torch.zeros((2,), dtype=torch.int32, device=dev)
    n_active = B
    qp_solves = 0
    it = 0
    limit = fixed_iters if fixed_iters is not None else max_iters
    worst = None              # fixed_iters: smallest new point count seen so far (device scalar; negative = overflow)
    while True:
        it += 1
        n_cur_max = reftrack.shape[1]
        res = opt_min_curv_batch(reftrack, normvec, h, kappa_bound, w_veh, n_pts=cur_n)     # (finished tracks: n_pts = 0, skipped)
        qp_solves += n_active
        alpha = res["alpha"]
        if it < iters_min:
            scale_alpha_batch(alpha, it * 1.0 / iters_min)
        # per-track termination and the copy of finished tracks into the result buffers: on the device
        _call("mc_iqp_finish_batch", B, n_cur_max, n_cap, it, int(iters_min), float(curv_error_allowed),
              int(fixed_iters) if fixed_iters is not None else 0, int(limit), active, res["status"], res["curv_error_max"],
              cur_n, alpha, reftrack, normvec,
              *(fin[k] for k in ("alpha", "reftrack", "normvec", "n_pts", "outer_iters", "status", "curv_error_max")), counters)
        if it >= limit:                       # every track was finished by this call (fixed count or cap): nothing to read back
            break
        if fixed_iters is not None:
            rt_new, nv_new, n_new = iqp_relinearise_batch(reftrack, normvec, alpha, stepsize_interp, n_pts=cur_n,
                                                          active=active, n_max_new=n_cap)
            worst = n_new.min() if worst is None else torch.minimum(worst, n_new.min())
            reftrack, normvec, cur_n = rt_new, nv_new, n_new
            h = torch.ones((B, n_cap), dtype=torch.float64, device=dev)
            continue
        while True:
            rt_new, nv_new, n_new = iqp_relinearise_batch(reftrack, normvec, alpha, stepsize_interp, n_pts=cur_n,
                                                          active=active, n_max_new=n_cap)
            # the ONE host read of the iteration: tracks still active, and the smallest new point count (negative = -(points
            # needed) for a track that does not fit the capacity)
            n_active, n_min = (int(v) for v in torch.stack((counters[0], n_new.min())).tolist())
            if n_active == 0 or n_min >= 0:
                break
            n_cap = -n_min + 64
            grown = _alloc(n_cap)
            for k in ("alpha", "reftrack", "normvec"):
                grown[k][:, :fin[k].shape[1]] = fin[k]
                fin[k] = grown[k]
        if n_active == 0:
            break
        reftrack, normvec, cur_n = rt_new, nv_new, n_new
        h = torch.ones((B, n_cap), dtype=torch.float64, device=dev)   # use_dist_scaling=False from iteration 2 on
    if worst is not None:
        n_min = int(worst.item())
        if n_min < 0:         # a re-sampled track did not fit: its later iterations ran on nothing -- repeat with room for it
            return iqp_batch(reftrack0, normvec0, h0, kappa_bound, w_veh, stepsize_interp, iters_min=iters_min,
                             curv_error_allowed=curv_error_allowed, n_pts=n_pts, max_iters=max_iters,
                             fixed_iters=fixed_iters, _n_cap_min=-n_min + 64)
    fin["qp_solves"] = qp_solves
    return fin


# ------------------------------------------------------------------------------------------------
# velocity-profile stage (SURVEY.md 8f-1): tph.calc_vel_profile + calc_ax_profile + calc_t_profile
# ------------------------------------------------------------------------------------------------
def _table(t, cols: int, name: str) -> torch.Tensor:
    """The checked table t as a float64 tensor where t lives (a host table stays on the host, so that the range checks
    of _vp_inputs read no device memory)."""
    t = torch.as_tensor(t, dtype=torch.float64)
    if t.ndim != 2 or t.shape[1] != cols:
        raise RuntimeError({3: "ggv diagram must consist of the three columns [vx, ax_max, ay_max]!",
                            2: "ax_max_machines must consist of the two columns [vx, ax_max_machines]!"}[cols])
    if t.shape[0] > 256:
        raise ValueError(f"{name}: at most 256 rows are supported")
    return t


def _to_device(t: torch.Tensor, dev) -> torch.Tensor:
    """t on dev.  A host table goes through pinned memory with a non-blocking copy: a copy from pageable memory would
    synchronise the stream on every call."""
    if t.device.type == "cpu" and torch.device(dev).type == "cuda":
        return t.contiguous().pin_memory().to(dev, non_blocking=True)
    return t.to(dev).contiguous()


class Vehicles:
    """K vehicles for the vehicles= argument of the velocity-profile entry points (vel_profile_batch, vel_profile_diff,
    lap_time_matrix_batch, lap_time_matrix_diff, raceline_refine.refine_raceline_batch), each with its own tables and
    scalars; veh_id [B] then picks the vehicle of each track.

    ggv, ax_max_machines: sequences of K tables ([rows, 3] and [rows, 2], 1 to 256 rows each; e.g. the pairs
    import_veh_dyn_info returns); v_max, drag_coeff, m_veh: K-sequences (a number stands for all K).  The checks of tph
    run here, once, per vehicle (each table must cover that vehicle's v_max; a call with per-variant top speeds checks
    those against every vehicle's tables on the host).  The tables are packed back to back and copied to device once,
    through pinned memory: a reused object costs no copy and no stream synchronisation per call.  device: where the
    tracks will be (default: the current CUDA device)."""

    def __init__(self, ggv, ax_max_machines, v_max, drag_coeff, m_veh, device=None):
        if isinstance(ggv, torch.Tensor) or isinstance(ax_max_machines, torch.Tensor):
            raise TypeError("Vehicles: ggv and ax_max_machines are sequences of one table per vehicle")
        ggv, mach = list(ggv), list(ax_max_machines)
        K = len(ggv)
        if K < 1 or len(mach) != K:
            raise ValueError("Vehicles: ggv and ax_max_machines need one table per vehicle (at least one vehicle)")
        vm, drag, mass = (self._per_vehicle(x, K, name) for x, name in ((v_max, "v_max"), (drag_coeff, "drag_coeff"),
                                                                         (m_veh, "m_veh")))
        ggv = [_table(g, 3, f"ggv[{k}]") for k, g in enumerate(ggv)]
        mach = [_table(m, 2, f"ax_max_machines[{k}]") for k, m in enumerate(mach)]
        for k in range(K):
            if ggv[k].shape[0] < 1 or mach[k].shape[0] < 1:
                raise ValueError(f"Vehicles: vehicle {k} has an empty table")
            if not (math.isfinite(vm[k]) and vm[k] > 0.0):
                raise ValueError(f"Vehicles: v_max[{k}] must be a finite speed > 0")
            if not (math.isfinite(mass[k]) and mass[k] > 0.0):
                raise ValueError(f"Vehicles: m_veh[{k}] must be > 0")
        self.n_veh = K
        self.v_max, self.drag_coeff, self.m_veh = vm, drag, mass
        self._ggv_top = [float(g[-1, 0]) for g in ggv]
        self._mach_top = [float(m[-1, 0]) for m in mach]
        for k in range(K):
            self.check_covers(vm[k], k)
        rows = torch.zeros((K + 1, 2), dtype=torch.int32)
        rows[1:, 0] = torch.cumsum(torch.tensor([g.shape[0] for g in ggv]), 0)
        rows[1:, 1] = torch.cumsum(torch.tensor([m.shape[0] for m in mach]), 0)
        par = torch.tensor([vm, drag, mass], dtype=torch.float64).T.contiguous()
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.ggv, self.ax_max_machines = _to_device(torch.cat(ggv), dev), _to_device(torch.cat(mach), dev)
        self.rows, self.par = _to_device(rows, dev), _to_device(par, dev)
        self.device = self.ggv.device

    @staticmethod
    def _per_vehicle(x, K, name):
        if isinstance(x, torch.Tensor):
            x = x.detach().cpu().reshape(-1).tolist()
        elif not hasattr(x, "__len__"):
            x = [x] * K
        x = [float(v) for v in x]
        if len(x) != K:
            raise ValueError(f"Vehicles: {name} needs one value per vehicle ({K})")
        return x

    def check_covers(self, v_top: float, k: Optional[int] = None) -> None:
        """tph's range checks: the tables of vehicle k (None: of every vehicle) cover the speed v_top."""
        for j in range(self.n_veh) if k is None else (k,):
            if self._mach_top[j] < v_top:
                raise RuntimeError("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!")
            if self._ggv_top[j] < v_top:
                raise RuntimeError("ggv has to cover the entire velocity range of the car (i.e. >= v_max)!")

    def veh_id(self, veh_id, B: int, dev) -> torch.Tensor:
        """veh_id as the [B] int32 device tensor the C-ABI takes.  None: one vehicle per track (K == B).  A host veh_id
        is range-checked here and copied through pinned memory; a device veh_id is not read (the kernels refuse a track
        whose id is out of range)."""
        if veh_id is None:
            if self.n_veh != B:
                raise ValueError(f"veh_id is required unless there is one vehicle per track ({self.n_veh} vehicles, "
                                 f"{B} tracks)")
            veh_id = torch.arange(B, dtype=torch.int32)
        if isinstance(veh_id, torch.Tensor) and veh_id.device.type != "cpu":
            if veh_id.numel() != B or veh_id.dtype.is_floating_point or veh_id.dtype == torch.bool:
                raise ValueError("veh_id must hold one integer per track")
            return veh_id.to(device=dev, dtype=torch.int32).reshape(B).contiguous()
        ids = torch.as_tensor(veh_id).reshape(-1)
        if ids.numel() != B or ids.dtype.is_floating_point or ids.dtype == torch.bool:
            raise ValueError("veh_id must hold one integer per track")
        if bool(((ids < 0) | (ids >= self.n_veh)).any()):
            raise ValueError(f"veh_id must be in 0 .. {self.n_veh - 1}")
        return _to_device(ids.to(torch.int32), dev)


# vehicle mode of the velocity-profile entries: n_ggv = MC_VP_VEHICLES, ggv = the address of an mc_vp_vehicles
VP_VEHICLES = _lib.header_define(_lib._build.HEADER, "MC_VP_VEHICLES")
_VpVehiclesDesc = _lib.header_struct(_lib._build.HEADER, "mc_vp_vehicles")


def _vp_vehicles(vehicles: Vehicles, veh_id, ggv, ax_max_machines, v_max, ggv_scales, drag_coeff, m_veh, B, dev):
    """The vehicle-mode part of _vp_inputs: (V, vmax_t, scale_t, the table arguments of the C-ABI (n_ggv, ggv, n_mach,
    ax_max_machines)).  ggv is a callable of the chunk (s, e) as _launch_chunks takes it: a reference to the
    mc_vp_vehicles of tracks s:e (held by the reference until the call has read it)."""
    if not isinstance(vehicles, Vehicles):
        raise TypeError("vehicles must be a batch.Vehicles")
    if (any(x is not None for x in (ggv, ax_max_machines, drag_coeff, m_veh))
            or (v_max is not None and ggv_scales is None)):
        raise ValueError("with vehicles= the ggv, ax_max_machines, v_max, drag_coeff and m_veh arguments must be None "
                         "(each vehicle has its own; v_max may give per-variant top speeds with ggv_scales)")
    if vehicles.device != torch.device(dev):
        raise ValueError(f"vehicles are on {vehicles.device}, the tracks on {dev}")
    ids = vehicles.veh_id(veh_id, B, dev)
    V, vmax_t, scale_t = 1, None, None
    if ggv_scales is not None:
        sc = torch.as_tensor(ggv_scales, dtype=torch.float64).reshape(-1)
        V, scale_t = int(sc.numel()), sc.to(dev).contiguous()
        if v_max is not None:
            vm = torch.as_tensor(v_max, dtype=torch.float64).reshape(-1)
            if vm.numel() == 1 and V > 1:
                vm = vm.expand(V).clone()
            if vm.numel() != V:
                raise ValueError("v_max and ggv_scales must have one entry per variant")
            vehicles.check_covers(float(vm.max().item()))
            vmax_t = vm.to(dev).contiguous()
    def desc(s, e):
        d = _VpVehiclesDesc(n_veh=vehicles.n_veh, n_ggv=int(vehicles.ggv.shape[0]),
                            n_mach=int(vehicles.ax_max_machines.shape[0]), ggv=vehicles.ggv.data_ptr(),
                            ax_max_machines=vehicles.ax_max_machines.data_ptr(), veh_rows=vehicles.rows.data_ptr(),
                            veh_par=vehicles.par.data_ptr(), veh_id=ids[s:e].data_ptr())
        d.tensors = (vehicles, ids)                       # (the buffers outlive the descriptor)
        return ctypes.byref(d)
    return V, vmax_t, scale_t, (VP_VEHICLES, desc, 0, None)


def _vp_inputs(kappa, el_lengths, ggv, ax_max_machines, v_max, ggv_scales, drag_coeff, m_veh, dyn_model_exp, filt_window,
               n_pts, decel_slice_upper, mu=None, max_chunk=None, vehicles=None, veh_id=None):
    """The checked and normalised inputs of vel_profile_batch, vel_profile_diff and lap_time_matrix_diff: kappa and
    el_lengths as contiguous float64 CUDA tensors [B, n_max], and a namespace of the rest as the C-ABI takes it: B, n_max,
    dev, mu, n_pts, V variants per track with their top speeds vmax_t and ggv scales scale_t ([V] on the device; both None
    for one profile per track at top speed v_scalar), common: the arguments from n_ggv to decel_slice_upper, which
    mc_vel_profile_batch_ex and mc_vel_profile_adjoint_batch take alike (with vehicles: n_ggv = MC_VP_VEHICLES and the
    chunk's mc_vp_vehicles in place of ggv), and max_chunk (see _vp_chunk)."""
    kappa = _f64(kappa, "kappa")
    el_lengths = _f64(el_lengths, "el_lengths")
    B, n_max = kappa.shape
    if el_lengths.shape != (B, n_max):
        raise RuntimeError("kappa and el_lengths must have the same length if closed!")
    dev = kappa.device
    if mu is not None:
        mu = _f64(mu, "mu")
        if mu.shape != (B, n_max):
            raise RuntimeError("kappa and mu must have the same length!")
    n_pts = _npts(n_pts, B, dev)
    if filt_window is not None and int(filt_window) % 2 != 1:
        raise RuntimeError("Window width of moving average filter must be odd!")
    upper = int(VP_DECEL_SLICE_UPPER if decel_slice_upper is None else decel_slice_upper)
    filt = 0 if filt_window is None else int(filt_window)
    if vehicles is not None or veh_id is not None:
        if vehicles is None:
            raise ValueError("veh_id needs vehicles=")
        V, vmax_t, scale_t, tables = _vp_vehicles(vehicles, veh_id, ggv, ax_max_machines, v_max, ggv_scales, drag_coeff,
                                                  m_veh, B, dev)
        return kappa, el_lengths, SimpleNamespace(B=B, n_max=n_max, dev=dev, mu=mu, n_pts=n_pts, V=V, vmax_t=vmax_t,
                                                  scale_t=scale_t, v_scalar=0.0, max_chunk=max_chunk,
                                                  common=(*tables, float(dyn_model_exp), 0.0, 0.0, filt, upper))
    if any(x is None for x in (ggv, ax_max_machines, v_max, drag_coeff, m_veh)):
        raise TypeError("the velocity profile needs ggv, ax_max_machines, v_max, drag_coeff and m_veh (or vehicles=)")
    ggv_h = _table(ggv, 3, "ggv")
    mach_h = _table(ax_max_machines, 2, "ax_max_machines")
    vmax_t = scale_t = None
    if ggv_scales is not None or isinstance(v_max, torch.Tensor) or hasattr(v_max, "__len__"):
        vm = torch.as_tensor(v_max, dtype=torch.float64).reshape(-1)
        sc = torch.ones_like(vm) if ggv_scales is None else torch.as_tensor(ggv_scales, dtype=torch.float64).reshape(-1)
        if vm.numel() == 1 and sc.numel() > 1:
            vm = vm.expand(sc.numel()).clone()
        if sc.numel() != vm.numel():
            raise ValueError("v_max and ggv_scales must have one entry per variant")
        V = int(vm.numel())
        vmax_t, scale_t = vm.to(dev).contiguous(), sc.to(dev).contiguous()
        v_hi, v_scalar = float(vm.max().item()), 0.0
    else:
        V, v_hi, v_scalar = 1, float(v_max), float(v_max)
    # tph's range checks (the tables must cover the whole velocity range of the car)
    if float(mach_h[-1, 0].item()) < v_hi:
        raise RuntimeError("ax_max_machines has to cover the entire velocity range of the car (i.e. >= v_max)!")
    if float(ggv_h[-1, 0].item()) < v_hi:
        raise RuntimeError("ggv has to cover the entire velocity range of the car (i.e. >= v_max)!")
    ggv_t, mach_t = _to_device(ggv_h, dev), _to_device(mach_h, dev)
    common = (int(ggv_t.shape[0]), ggv_t, int(mach_t.shape[0]), mach_t, float(dyn_model_exp), float(drag_coeff), float(m_veh),
              filt, upper)
    return kappa, el_lengths, SimpleNamespace(B=B, n_max=n_max, dev=dev, mu=mu, n_pts=n_pts, V=V, vmax_t=vmax_t,
                                              scale_t=scale_t, v_scalar=v_scalar, common=common, max_chunk=max_chunk)


def _vp_chunk(p: SimpleNamespace, per_track: int) -> int:
    """Tracks per launch of a velocity-profile entry whose workspace takes per_track bytes per track: as many as free
    device memory holds (or p.max_chunk), and at most (2 ** 31 - 1024) // V, so that one launch's B * V profiles stay
    within what the entry accepts."""
    chunk = _chunk(p.B, per_track, p.dev) if p.max_chunk is None else min(p.B, int(p.max_chunk))
    return max(1, min(chunk, (2 ** 31 - 1024) // p.V))


def _vel_profile_launch(kappa: torch.Tensor, el_lengths: torch.Tensor, p: SimpleNamespace, want_profiles: bool) -> dict:
    """The velocity profiles of the inputs of _vp_inputs: dict(laptime [B, V], status [B, V] and, if want_profiles,
    vx [B, V, n_max], ax [B, V, n_max], t [B, V, n_max + 1])."""
    lib = _lib.load()
    B, V, n_max = p.B, p.V, p.n_max
    f64 = dict(dtype=torch.float64, device=p.dev)
    laptime = torch.zeros((B, V), **f64)
    status = torch.zeros((B, V), dtype=torch.int32, device=p.dev)
    vx = torch.zeros((B, V, n_max), **f64) if want_profiles else None
    ax = torch.zeros((B, V, n_max), **f64) if want_profiles else None
    t = torch.zeros((B, V, n_max + 1), **f64) if want_profiles else None
    chunk = _vp_chunk(p, lib.mc_vel_profile_workspace_bytes(1, V, n_max))
    ws = _workspace("velprofile", lib.mc_vel_profile_workspace_bytes(chunk, V, n_max), p.dev)
    _launch_chunks("mc_vel_profile_batch_ex", B, chunk, ws, n_max, *map(_rows, (p.n_pts, kappa, el_lengths, p.mu)), V,
                   p.scale_t, p.vmax_t, p.v_scalar, *p.common, *map(_rows, (vx, ax, t, laptime, status)), None, None, None,
                   None)
    out = dict(laptime=laptime, status=status)
    if want_profiles:
        out.update(vx=vx, ax=ax, t=t)
    return out


@_device_guard
def vel_profile_batch(kappa: torch.Tensor, el_lengths: torch.Tensor, ggv=None, ax_max_machines=None, v_max=None,
                      drag_coeff: Optional[float] = None, m_veh: Optional[float] = None, dyn_model_exp: float = 1.0,
                      filt_window: Optional[int] = None, mu: Optional[torch.Tensor] = None,
                      n_pts: Optional[torch.Tensor] = None, ggv_scales=None, want_profiles: bool = True,
                      max_chunk: Optional[int] = None, decel_slice_upper: Optional[int] = None,
                      vehicles: Optional[Vehicles] = None, veh_id=None) -> dict:
    """Batched tph.calc_vel_profile (closed, ggv branch) + calc_ax_profile + calc_t_profile.

    kappa, el_lengths: [B, n_max] device tensors (n_pts[b] valid entries), e.g. the ``kappa`` /
    ``el_lengths_interp`` / ``n_out`` results of create_raceline_batch.  ``v_max`` is a float, or -- together with
    ``ggv_scales`` -- a sequence of V per-variant values: variant v of every track runs with
    ggv[:, 1:] * ggv_scales[v] and top speed v_max[v] (one cell of the reference's lap-time matrix,
    main_globaltraj.py:442-496).  Returns dict(laptime [B, V], status [B, V] and, if want_profiles,
    vx [B, V, n_max], ax [B, V, n_max], t [B, V, n_max + 1]).

    vehicles: a Vehicles of K vehicles, one per track picked by veh_id [B] (host or device integers; None: K == B, track
    b drives vehicle b).  ggv, ax_max_machines, drag_coeff and m_veh are then None, and so is v_max unless ggv_scales is
    given (v_max then gives per-variant top speeds; None: each track's variants run at its vehicle's v_max).  A track's
    results are bit for bit those of a call with its vehicle alone.  A track whose device veh_id is out of range gets
    lap time 0 and status 5 (VP_STATUS_BAD_VEHICLE), its neighbours are untouched."""
    _require_cuda()
    kappa, el_lengths, p = _vp_inputs(kappa, el_lengths, ggv, ax_max_machines, v_max, ggv_scales, drag_coeff, m_veh,
                                      dyn_model_exp, filt_window, n_pts, decel_slice_upper, mu=mu, max_chunk=max_chunk,
                                      vehicles=vehicles, veh_id=veh_id)
    return _vel_profile_launch(kappa, el_lengths, p, want_profiles)


class _VelProfileDiff(torch.autograd.Function):
    """laptime and vx of the velocity profile as functions of kappa and el_lengths; see vel_profile_diff.  p: the
    namespace of _vp_inputs (V = 1) and strict."""

    @staticmethod
    def forward(ctx, kappa, el_lengths, p):
        res = _vel_profile_launch(kappa, el_lengths, p, want_profiles=True)
        laptime, status = res["laptime"][:, 0], res["status"][:, 0]
        vx, ax, t = res["vx"][:, 0], res["ax"][:, 0], res["t"][:, 0]
        grad_status = status.clone()
        ctx.save_for_backward(kappa, el_lengths, grad_status)
        ctx.p = p
        ctx.mark_non_differentiable(ax, t, status, grad_status)
        ctx.set_materialize_grads(False)
        return laptime, vx, ax, t, status, grad_status

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_laptime, grad_vx, *_unused):
        kappa, el_lengths, grad_status = ctx.saved_tensors
        p = ctx.p
        lib = _lib.load()
        B, n_max = kappa.shape
        f64 = dict(dtype=torch.float64, device=kappa.device)
        grad_laptime = None if grad_laptime is None else grad_laptime.to(**f64).contiguous()
        grad_vx = None if grad_vx is None else grad_vx.to(**f64).contiguous()
        wanted = _wanted(B, grad_laptime, grad_vx, device=kappa.device)
        who = "vel_profile_diff: no gradient"
        _refuse(p.strict, wanted, grad_status, who, "with a nonzero upstream gradient")
        need_k, need_e = ctx.needs_input_grad[:2]
        gk = torch.empty((B, n_max), **f64) if need_k else None
        ge = torch.empty((B, n_max), **f64) if need_e else None
        gs = torch.empty((B,), dtype=torch.int32, device=kappa.device)
        chunk = _vp_chunk(p, lib.mc_vel_profile_adjoint_workspace_bytes(1, n_max))
        ws = _workspace("velprofile_adjoint", lib.mc_vel_profile_adjoint_workspace_bytes(chunk, n_max), kappa.device)
        _launch_chunks("mc_vel_profile_adjoint_batch", B, chunk, ws, n_max, *map(_rows, (p.n_pts, kappa, el_lengths)),
                       p.v_scalar, *p.common, *map(_rows, (grad_laptime, grad_vx, gk, ge, gs)))
        _refuse(p.strict, wanted, gs, who, "whose gradient is not finite")
        return gk, ge, None


@_device_guard
def vel_profile_diff(kappa: torch.Tensor, el_lengths: torch.Tensor, ggv=None, ax_max_machines=None,
                     v_max: Optional[float] = None, drag_coeff: Optional[float] = None, m_veh: Optional[float] = None,
                     dyn_model_exp: float = 1.0, filt_window: Optional[int] = None,
                     n_pts: Optional[torch.Tensor] = None, decel_slice_upper: Optional[int] = None,
                     strict: bool = True, vehicles: Optional[Vehicles] = None, veh_id=None,
                     max_chunk: Optional[int] = None) -> dict:
    """vel_profile_batch for one profile per track (no ggv scales, one top speed, no mu) with the lap time and the speed
    profile differentiable with respect to kappa and el_lengths (autograd).

    Returns dict(laptime [B], vx [B, n_max], ax [B, n_max], t [B, n_max + 1], status [B], grad_status [B]): the values of
    vel_profile_batch with V = 1.  laptime and vx carry a grad_fn; backward() / torch.autograd.grad give dL/dkappa and
    dL/del_lengths [B, n_max] (zero beyond n_pts) at the cost of running the profile again with a tape and walking it
    backwards, one thread per track (DESIGN.md section 3.12).  The derivative is that of the function the forward
    evaluates, with its discrete decisions (phase starts, which limit wins each min, table segments, the v_max clip)
    frozen.  Chain it to create_raceline_batch's kappa / el_lengths_interp with n_pts=rl["n_out"].
    grad_status: 0 = the gradient is computed; 3 = a non-finite lap time or gradient; for an inactive slot (n_pts < 2)
    the forward's status.  strict=True: backward raises if an instance with a nonzero upstream gradient has
    grad_status != 0; strict=False: such instances get zero gradients.  vehicles, veh_id: a vehicle per track, as for
    vel_profile_batch (each track at its vehicle's v_max; grad_status 5 for a refused veh_id).  max_chunk: at most that
    many tracks per launch (the results do not depend on it)."""
    _require_cuda()
    if isinstance(v_max, torch.Tensor) or hasattr(v_max, "__len__"):
        raise ValueError("vel_profile_diff: v_max must be one number (no per-variant top speeds)")
    kappa, el_lengths, p = _vp_inputs(kappa, el_lengths, ggv, ax_max_machines, v_max, None, drag_coeff, m_veh, dyn_model_exp,
                                      filt_window, n_pts, decel_slice_upper, max_chunk=max_chunk, vehicles=vehicles,
                                      veh_id=veh_id)
    p.strict = bool(strict)
    laptime, vx, ax, t, status, grad_status = _VelProfileDiff.apply(kappa, el_lengths, p)
    return dict(laptime=laptime, vx=vx, ax=ax, t=t, status=status, grad_status=grad_status)


def _lap_time_variants(ggv_scales, top_speeds, vehicles=None):
    """(top speed [V], ggv scale [V], T, S): the V = T * S variants of the lap-time matrix in its order, variant
    v = (top-speed index) * S + (scale index).  With vehicles, top_speeds None stands for each vehicle's v_max (T = 1,
    top speed None)."""
    if ggv_scales is None or (top_speeds is None and vehicles is None):
        raise TypeError("the lap-time matrix needs ggv_scales and top_speeds (top_speeds may be None with vehicles=)")
    gs = torch.as_tensor(ggv_scales, dtype=torch.float64).reshape(-1)
    if top_speeds is None:
        return None, gs, 1, gs.numel()
    ts = torch.as_tensor(top_speeds, dtype=torch.float64).reshape(-1)
    return ts.repeat_interleave(gs.numel()), gs.repeat(ts.numel()), ts.numel(), gs.numel()


def lap_time_matrix_batch(kappa: torch.Tensor, el_lengths: torch.Tensor, ggv=None, ax_max_machines=None,
                          ggv_scales=None, top_speeds=None, drag_coeff: Optional[float] = None, m_veh: Optional[float] = None,
                          dyn_model_exp: float = 1.0, filt_window: Optional[int] = None,
                          n_pts: Optional[torch.Tensor] = None, vehicles: Optional[Vehicles] = None,
                          veh_id=None) -> torch.Tensor:
    """The lap-time matrix of main_globaltraj.py:442-496 for every track of the batch in one launch:
    returns [B, len(top_speeds), len(ggv_scales)] lap times (top speeds in m/s).  vehicles, veh_id: a vehicle per track
    as for vel_profile_batch; cell v then scales the ggv of the track's vehicle, and top_speeds None runs every cell at
    the vehicle's v_max ([B, 1, len(ggv_scales)])."""
    vm, sc, T, S = _lap_time_variants(ggv_scales, top_speeds, vehicles)
    res = vel_profile_batch(kappa, el_lengths, ggv, ax_max_machines, vm, drag_coeff, m_veh, dyn_model_exp, filt_window,
                            n_pts=n_pts, ggv_scales=sc, want_profiles=False, vehicles=vehicles, veh_id=veh_id)
    bad_ = res["status"] != 0
    if bool(bad_.any().item()):
        raise RuntimeError("lap_time_matrix_batch: non-finite lap time or refused vehicle for %i profile(s)"
                           % int(bad_.sum().item()))
    return res["laptime"].reshape(kappa.shape[0], T, S)


class _LapTimeMatrixDiff(torch.autograd.Function):
    """The lap times [B, V] of V (ggv scale, top speed) variants per track as functions of kappa and el_lengths; see
    lap_time_matrix_diff.  p: the namespace of _vp_inputs and strict."""

    @staticmethod
    def forward(ctx, kappa, el_lengths, p):
        res = _vel_profile_launch(kappa, el_lengths, p, want_profiles=False)
        laptime, status = res["laptime"], res["status"]
        grad_status = status.clone()
        ctx.save_for_backward(kappa, el_lengths, grad_status)
        ctx.p = p
        ctx.mark_non_differentiable(status, grad_status)
        ctx.set_materialize_grads(False)
        return laptime, status, grad_status

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_laptime, *_unused):
        kappa, el_lengths, grad_status = ctx.saved_tensors
        if grad_laptime is None:
            return None, None, None
        p = ctx.p
        lib = _lib.load()
        B, n_max, V = p.B, p.n_max, p.V
        f64 = dict(dtype=torch.float64, device=kappa.device)
        grad_laptime = grad_laptime.to(**f64).contiguous()
        wanted = (grad_laptime != 0).flatten()                  # per profile b * V + v
        who, cells = "lap_time_matrix_diff: no gradient", " (instance: the cell b * V + v)"
        _refuse(p.strict, wanted, grad_status.flatten(), who, "with a nonzero upstream gradient" + cells)
        need_k, need_e = ctx.needs_input_grad[:2]
        gk = torch.empty((B, n_max), **f64) if need_k else None
        ge = torch.empty((B, n_max), **f64) if need_e else None
        gs = torch.empty((B, V), dtype=torch.int32, device=kappa.device)
        chunk = _vp_chunk(p, lib.mc_vel_profile_adjoint_workspace_bytes(V, n_max))
        ws = _workspace("velprofile_adjoint", lib.mc_vel_profile_adjoint_workspace_bytes(chunk * V, n_max), kappa.device)
        _launch_chunks("mc_vel_profile_batch_ex", B, chunk, ws, n_max, *map(_rows, (p.n_pts, kappa, el_lengths)), None, V,
                       p.scale_t, p.vmax_t, p.v_scalar, *p.common, None, None, None, None, None,
                       *map(_rows, (grad_laptime, gk, ge, gs)))
        _refuse(p.strict, wanted, gs.flatten(), who, "whose gradient is not finite" + cells)
        return gk, ge, None


@_device_guard
def lap_time_matrix_diff(kappa: torch.Tensor, el_lengths: torch.Tensor, ggv=None, ax_max_machines=None,
                         ggv_scales=None, top_speeds=None, drag_coeff: Optional[float] = None,
                         m_veh: Optional[float] = None, dyn_model_exp: float = 1.0, filt_window: Optional[int] = None,
                         n_pts: Optional[torch.Tensor] = None, decel_slice_upper: Optional[int] = None,
                         strict: bool = True, vehicles: Optional[Vehicles] = None, veh_id=None,
                         max_chunk: Optional[int] = None) -> dict:
    """lap_time_matrix_batch with the lap-time matrix differentiable with respect to kappa and el_lengths (autograd).

    Returns dict(laptime, status, grad_status), each [B, len(top_speeds), len(ggv_scales)]: laptime holds the values of
    lap_time_matrix_batch bit for bit (a non-finite cell is reported in status, not raised) and carries a grad_fn;
    backward() / torch.autograd.grad give dL/dkappa and dL/del_lengths [B, n_max] (zero beyond n_pts): for each track the
    sum over its cells, in cell order, of what vel_profile_diff gives for one cell with the ggv scaled by that cell's
    scale and that cell's top speed (DESIGN.md section 3.12).  The backward runs every profile of the matrix again with a
    tape (17 n_max + 1 doubles per profile; tracks are chunked by free device memory).
    grad_status per cell: 0 = the gradient is computed; 3 = a non-finite lap time or gradient; for an inactive slot
    (n_pts < 2) the forward's status.  strict=True: backward raises if a cell with a nonzero upstream gradient has
    grad_status != 0; strict=False: such cells add nothing to their track's gradient.  vehicles, veh_id: a vehicle per
    track, as for lap_time_matrix_batch.  max_chunk: at most that many tracks per launch (the results do not depend on
    it)."""
    _require_cuda()
    vm, sc, T, S = _lap_time_variants(ggv_scales, top_speeds, vehicles)
    kappa, el_lengths, p = _vp_inputs(kappa, el_lengths, ggv, ax_max_machines, vm, sc, drag_coeff, m_veh, dyn_model_exp,
                                      filt_window, n_pts, decel_slice_upper, max_chunk=max_chunk, vehicles=vehicles,
                                      veh_id=veh_id)
    p.strict = bool(strict)
    laptime, status, grad_status = _LapTimeMatrixDiff.apply(kappa, el_lengths, p)
    B = p.B
    return dict(laptime=laptime.reshape(B, T, S), status=status.reshape(B, T, S), grad_status=grad_status.reshape(B, T, S))


@_device_guard
def calc_ax_t_profile_batch(vx: torch.Tensor, el_lengths: torch.Tensor, ax_in: Optional[torch.Tensor] = None,
                            t_start: float = 0.0, n_pts: Optional[torch.Tensor] = None, want_t: bool = True):
    """Stand-alone tph.calc_ax_profile (ax_in None: vx holds n + 1 values per row) / tph.calc_t_profile.
    Returns (ax [P, n_max], t [P, n_max + 1] or None)."""
    _require_cuda()
    vx = _f64(vx, "vx")
    el_lengths = _f64(el_lengths, "el_lengths")
    P, n_max = el_lengths.shape
    dev = vx.device
    if ax_in is not None:
        ax_in = _f64(ax_in, "ax_in")
    ax_out = torch.zeros((P, n_max), dtype=torch.float64, device=dev)
    t_out = torch.zeros((P, n_max + 1), dtype=torch.float64, device=dev) if want_t else None
    _call("mc_calc_ax_t_profile_batch", P, n_max, _npts(n_pts, P, dev), vx, int(vx.shape[1]), el_lengths, ax_in, float(t_start),
          ax_out, t_out)
    return ax_out, t_out


# ------------------------------------------------------------------------------------------------
# trajectory back end (SURVEY.md 8f-3/8f-4): the reference's in-tree helpers interp_track, calc_min_bound_dists,
# check_traj and the trajectory assembly of main_globaltraj.py:501-512, batched
# ------------------------------------------------------------------------------------------------
@_device_guard
def interp_track_batch(pts: torch.Tensor, stepsize_approx: float = 1.0, n_pts: Optional[torch.Tensor] = None,
                       normvec: Optional[torch.Tensor] = None, normal_sign: float = 1.0, width_col: int = 2,
                       n_out_max: Optional[int] = None):
    """Batched helper_funcs_glob.src.interp_track.interp_track (helper_funcs_glob/src/interp_track.py).

    pts: [B, n_max, 2 or 4].  With ``normvec`` the re-sampled polyline is pts.xy + normal_sign * normvec * pts[..., width_col]
    (the track boundaries of check_traj.py:50-61).  Returns (out [B, n_out_max, 4], n_out [B])."""
    _require_cuda()
    pts = _f64(pts, "pts")
    B, n_max, stride = pts.shape
    dev = pts.device
    n_pts = _npts(n_pts, B, dev)
    if normvec is not None:
        normvec = _f64(normvec, "normvec")
        if normvec.shape != (B, n_max, 2) or stride != 4:
            raise ValueError("normvec needs a [B, n_max, 4] track and must be [B, n_max, 2]")
    if n_out_max is None:
        if normvec is None:
            poly = _closed_polygon_length(pts, n_pts)
        else:       # the boundary polyline p + sign * w n: the width column of the track is the per-point shift (stride 4)
            poly = _closed_polygon_length(pts, n_pts, normvec=normvec, shift=pts.reshape(-1)[int(width_col):].view(-1),
                                          shift_stride=4, sign=float(normal_sign))
        n_out_max = int(math.ceil(float(poly.max().item()) / float(stepsize_approx))) + 8
    ws = _workspace("interp_track", _lib.load().mc_interp_track_workspace_bytes(B, n_max), dev)
    while True:
        out = torch.zeros((B, int(n_out_max), 4), dtype=torch.float64, device=dev)
        n_out = torch.zeros((B,), dtype=torch.int32, device=dev)
        _call("mc_interp_track_batch", B, n_max, n_pts, pts, stride, normvec, float(normal_sign), int(width_col),
              float(stepsize_approx), int(n_out_max), out, n_out, ws=ws)
        need = int((-n_out).max().item())
        if need <= 0:
            return out, n_out
        n_out_max = need + 8


@_device_guard
def min_bound_dists_batch(xy: torch.Tensor, psi: torch.Tensor, bound1: torch.Tensor, bound2: torch.Tensor,
                          length_veh: float, width_veh: float, n_traj: Optional[torch.Tensor] = None,
                          nb1: Optional[torch.Tensor] = None, nb2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Batched helper_funcs_glob.src.calc_min_bound_dists.calc_min_bound_dists: [B, n_traj_max] minimum distances of
    the vehicle corners to the boundary points (bound1/bound2: [B, nb_max, >= 2], x and y first)."""
    _require_cuda()
    xy, psi, bound1, bound2 = _f64(xy, "xy"), _f64(psi, "psi"), _f64(bound1, "bound1"), _f64(bound2, "bound2")
    B, n_traj_max, _ = xy.shape
    if bound1.shape[2] != bound2.shape[2]:
        raise ValueError("bound1 and bound2 must have the same row layout")
    dev = xy.device
    out = torch.zeros((B, n_traj_max), dtype=torch.float64, device=dev)
    n_traj, nb1, nb2 = _npts(n_traj, B, dev), _npts(nb1, B, dev), _npts(nb2, B, dev)
    _call("mc_min_bound_dists_batch", B, n_traj_max, n_traj, xy, psi, int(bound1.shape[1]), nb1, bound1, int(bound2.shape[1]),
          nb2, bound2, int(bound1.shape[2]), float(length_veh), float(width_veh), out)
    return out


EXTREMA = ("min_dist", "kappa_abs_max", "ay_max", "ax_wo_drag_max", "ax_wo_drag_min", "a_tot_max", "vx_max", "n_points")


@_device_guard
def traj_extrema_batch(kappa: torch.Tensor, vx: torch.Tensor, ax: torch.Tensor, dragcoeff: float, mass_veh: float,
                       min_dists: Optional[torch.Tensor] = None, n_traj: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[B, 8] extrema per trajectory, columns as in EXTREMA (min_dist = inf without min_dists)."""
    _require_cuda()
    kappa, vx, ax = _f64(kappa, "kappa"), _f64(vx, "vx"), _f64(ax, "ax")
    B, n_max = kappa.shape
    dev = kappa.device
    if min_dists is not None:
        min_dists = _f64(min_dists, "min_dists")
    ext = torch.zeros((B, 8), dtype=torch.float64, device=dev)
    _call("mc_traj_extrema_batch", B, n_max, _npts(n_traj, B, dev), kappa, vx, ax, min_dists, float(dragcoeff), float(mass_veh),
          ext)
    return ext


@_device_guard
def check_traj_batch(reftrack: torch.Tensor, normvec: torch.Tensor, xy: torch.Tensor, psi: torch.Tensor,
                     kappa: torch.Tensor, vx: torch.Tensor, ax: torch.Tensor, length_veh: float, width_veh: float,
                     dragcoeff: float, mass_veh: float, n_pts: Optional[torch.Tensor] = None,
                     n_traj: Optional[torch.Tensor] = None, bound_stepsize: float = 1.0) -> dict:
    """The quantities helper_funcs_glob.src.check_traj.check_traj tests, for a batch of trajectories: boundaries
    re-sampled every ``bound_stepsize`` metres, minimum distance of the vehicle corners to them for every trajectory
    point (against ALL boundary points -- the reference passes only the first point of each boundary, check_traj.py:58-61,
    which the single-track mirror reproduces), and the extrema of curvature, accelerations and speed.
    Returns dict(min_dists [B, n_traj_max], bound_r/bound_l [B, nb, 4] with nb_r/nb_l [B], and one [B] tensor per name
    in EXTREMA)."""
    _require_cuda()
    kappa = _f64(kappa, "kappa")
    B = kappa.shape[0]
    n_traj = _npts(n_traj, B, kappa.device)
    br, nbr = interp_track_batch(reftrack, bound_stepsize, n_pts=n_pts, normvec=normvec, normal_sign=1.0, width_col=2)
    bl, nbl = interp_track_batch(reftrack, bound_stepsize, n_pts=n_pts, normvec=normvec, normal_sign=-1.0, width_col=3)
    md = min_bound_dists_batch(xy, psi, br, bl, length_veh, width_veh, n_traj=n_traj, nb1=nbr, nb2=nbl)
    ext = traj_extrema_batch(kappa, vx, ax, dragcoeff, mass_veh, min_dists=md, n_traj=n_traj)
    out = dict(min_dists=md, bound_r=br, bound_l=bl, nb_r=nbr, nb_l=nbl)
    out.update({name: ext[:, i] for i, name in enumerate(EXTREMA)})
    return out


def check_traj_flags(chk: dict, ggv, ax_max_machines, v_max: float, curvlim: float, min_dist_warn: float = 1.0) -> dict:
    """The comparisons of check_traj.py:74-139 as boolean [B] tensors (True = the reference would print the warning)."""
    import numpy as _np
    f = dict(min_dist=chk["min_dist"] < min_dist_warn, curvature=chk["kappa_abs_max"] > curvlim,
             v_max=chk["vx_max"] > v_max + 0.1)
    if ggv is not None:
        g = _np.asarray(ggv, dtype=float)
        f.update(ay=chk["ay_max"] > float(g[:, 2].max()) + 0.1, ax_pos=chk["ax_wo_drag_max"] > float(g[:, 1].max()) + 0.1,
                 ax_neg=chk["ax_wo_drag_min"] < float((-g[:, 1]).min()) - 0.1, a_tot=chk["a_tot_max"] > float(g[:, 1:].max()) + 0.1)
    if ax_max_machines is not None:
        m = _np.asarray(ax_max_machines, dtype=float)
        f["ax_machines"] = chk["ax_wo_drag_max"] > float(m[:, 1].max()) + 0.1
    return f


@_device_guard
def assemble_trajectory_batch(s: torch.Tensor, xy: torch.Tensor, psi: torch.Tensor, kappa: torch.Tensor, vx: torch.Tensor,
                              ax: torch.Tensor, spline_lengths: torch.Tensor, n_traj: Optional[torch.Tensor] = None,
                              n_spl: Optional[torch.Tensor] = None) -> torch.Tensor:
    """trajectory_opt / traj_race_cl of main_globaltraj.py:501-512 for a batch: [B, n_max + 1, 7] rows
    [s, x, y, psi, kappa, vx, ax]; row n_traj[b] closes the lap with s = sum(spline_lengths[b])."""
    _require_cuda()
    s, xy, psi, kappa, vx, ax = (_f64(t, nm) for t, nm in ((s, "s"), (xy, "xy"), (psi, "psi"), (kappa, "kappa"), (vx, "vx"),
                                                          (ax, "ax")))
    spline_lengths = _f64(spline_lengths, "spline_lengths")
    B, n_max = s.shape
    dev = s.device
    traj = torch.zeros((B, n_max + 1, 7), dtype=torch.float64, device=dev)
    _call("mc_assemble_trajectory_batch", B, n_max, _npts(n_traj, B, dev), s, xy, psi, kappa, vx, ax, int(spline_lengths.shape[1]),
          _npts(n_spl, B, dev), spline_lengths, traj)
    return traj


@_device_guard
def check_normals_crossing_batch(track: torch.Tensor, normvec: torch.Tensor, horizon: int = 10,
                                 n_pts: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Batched tph.check_normals_crossing (helper_funcs_glob/src/prep_track.py:57-59): bool [B], True where
    two normals at most ``horizon`` points apart cross inside the track."""
    _require_cuda()
    track, normvec = _f64(track, "track"), _f64(normvec, "normvec")
    B, n_max, four = track.shape
    if four != 4 or normvec.shape != (B, n_max, 2):
        raise ValueError("track must be [B, n_max, 4] and normvec [B, n_max, 2]")
    dev = track.device
    n_pts = _npts(n_pts, B, dev)
    smallest = n_max if n_pts is None else int(n_pts.min().item())
    if horizon >= smallest:
        raise RuntimeError("Horizon of %i points is too large for a track with %i points, reduce horizon!" % (horizon, smallest))
    crossing = torch.zeros((B,), dtype=torch.int32, device=dev)
    _call("mc_check_normals_crossing_batch", B, n_max, n_pts, track, normvec, int(horizon), crossing)
    return crossing != 0


# ------------------------------------------------------------------------------------------------
# sweep inputs generated on the device (SURVEY.md section 8d): width-jitter variants from seeds
# ------------------------------------------------------------------------------------------------
@_device_guard
def jitter_widths_batch(base: torch.Tensor, seeds: torch.Tensor, rel: float = 0.1, centre_id: Optional[torch.Tensor] = None,
                        n_pts_base: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None):
    """V = len(seeds) width-jitter variants of the prepared tracks ``base`` [n_base, n_max, 4] (variant v uses track
    centre_id[v], default v % n_base): w <- w (1 + rel g(s)), g smooth with |g| <= 1 drawn from seeds[v] (int64) by the
    stateless hash that synth.jitter_widths_hash mirrors on the host.  Returns (tracks [V, n_max, 4], n_pts [V])."""
    _require_cuda()
    base = _f64(base, "base")
    n_base, n_max, four = base.shape
    if four != 4:
        raise ValueError("base must be [n_base, n_max, 4]")
    dev = base.device
    seeds = seeds.to(device=dev, dtype=torch.int64).contiguous()
    V = int(seeds.numel())
    if centre_id is not None:
        centre_id = centre_id.to(device=dev, dtype=torch.int32).contiguous()
        if centre_id.numel() != V:
            raise ValueError("centre_id must have one entry per variant")
    if out is None:
        out = torch.empty((V, n_max, 4), dtype=torch.float64, device=dev)
    n_out = torch.empty((V,), dtype=torch.int32, device=dev)
    _call("mc_jitter_widths_batch", V, n_max, _npts(n_pts_base, n_base, dev), n_base, base, centre_id, seeds, float(rel), out,
          n_out)
    return out, n_out


# ------------------------------------------------------------------------------------------------
# prep_track front end (SURVEY.md section 8f-2): tph.spline_approximation + min-width inflation + splines + normals check
# ------------------------------------------------------------------------------------------------
# n_out[b] of mc_prep_track_batch (include/mincurv_b200.h): >= 0 points; -(points needed) above -PREP_REFUSED for a
# capacity; -PREP_REFUSED - reason for a refused track
PREP_REFUSED = 1 << 30
PREP_REASONS = {
    1: "n_raw is outside [0, n_raw_max]",
    2: "fewer than 5 points (raw, or after the pre-interpolation)",
    3: "a non-finite coordinate, width or length",
    4: "a point count (length / step) too large to hold",
    5: "the residual budget s_reg is not reached (s_reg >= the residual of the best constant fit, or the root search ran out)",
    6: "fewer than 3 re-sampled points",
}


def _prep_refuse(b: int, why: str):
    return ValueError(f"spline_approximation_batch: track {b} is refused: {why}")


@_device_guard
def spline_approximation_batch(track: torch.Tensor, k_reg: int = 3, s_reg: float = 10.0, stepsize_prep: float = 1.0,
                               stepsize_reg: float = 3.0, n_raw: Optional[torch.Tensor] = None,
                               min_width: Optional[float] = None):
    """Batched tph.spline_approximation (+ prep_track's min-width inflation) for imported tracks [B, n_raw_max, 4]
    (unclosed; n_raw[b] points each, 0 for an unused slot).  Returns (reftrack_interp [B, n_out_max, 4], n_pts [B],
    smoothing_lambda [B]).  The smoothing spline is the Reinsch formulation with residual budget s_reg
    (csrc/prep_track.cu).  A track the kernel cannot smooth raises ValueError naming the track and the reason."""
    _require_cuda()
    track = _f64(track, "track")
    B, n_raw_max, four = track.shape
    if four != 4:
        raise ValueError("track must be [B, n_raw_max, 4]")
    dev = track.device
    n_raw = _npts(n_raw, B, dev)
    counts = n_raw.cpu().tolist() if n_raw is not None else [n_raw_max] * B
    for b, nr in enumerate(counts):            # (the polygon length below reads n_raw[b] rows: check them first)
        if nr < 0 or nr > n_raw_max:
            raise _prep_refuse(b, f"n_raw = {nr} is outside [0, {n_raw_max}]")
        if 0 < nr < 5:
            raise _prep_refuse(b, f"{nr} raw points, fewer than 5")
    used = torch.arange(n_raw_max, device=dev)[None, :] < torch.tensor(counts, device=dev)[:, None]
    nonfinite = ((~torch.isfinite(track)).any(dim=2) & used).any(dim=1)
    lengths = _closed_polygon_length(track, n_raw)
    nonfinite |= ~torch.isfinite(lengths)
    if bool(nonfinite.any()):
        raise _prep_refuse(int(nonfinite.nonzero()[0, 0]), PREP_REASONS[3])
    lengths = lengths.cpu().tolist()
    for b, length in enumerate(lengths):
        if max(length / float(stepsize_prep), 1.05 * length / float(stepsize_reg), 4.0 * length) + 16 >= PREP_REFUSED:
            raise _prep_refuse(b, f"{PREP_REASONS[4]} (closed length {length:.6g} m)")
    length = max(lengths)
    n_int_max = int(math.ceil(length / float(stepsize_prep))) + 8
    n_out_max = int(math.ceil(1.05 * length / float(stepsize_reg))) + 16
    while True:
        out = torch.zeros((B, n_out_max, 4), dtype=torch.float64, device=dev)
        n_out = torch.zeros((B,), dtype=torch.int32, device=dev)
        lam = torch.zeros((B,), dtype=torch.float64, device=dev)
        ws = _workspace("prep_track", _lib.load().mc_prep_track_workspace_bytes(B, n_raw_max, n_int_max), dev)
        _call("mc_prep_track_batch", B, n_raw_max, n_raw, track, int(k_reg), float(s_reg), float(stepsize_prep),
              float(stepsize_reg), float(min_width) if min_width is not None else 0.0, n_int_max, n_out_max, out, n_out, lam,
              ws=ws)
        codes = n_out.cpu().tolist()
        for b, c in enumerate(codes):
            if c <= -PREP_REFUSED:
                raise _prep_refuse(b, PREP_REASONS.get(-PREP_REFUSED - c, f"unknown reason {-PREP_REFUSED - c}"))
        need = max(-c for c in codes)
        if need <= 0:
            return out, n_out, lam
        n_out_max = max(n_out_max, need + 16)          # (a curve longer than 1.05 x its polygon, or a tiny capacity)
        n_int_max = max(n_int_max, need + 16)


def prep_track_batch(track: torch.Tensor, reg_smooth_opts: dict, stepsize_opts: dict, n_raw: Optional[torch.Tensor] = None,
                     min_width: Optional[float] = None, check_normals: bool = True) -> dict:
    """Batched helper_funcs_glob.src.prep_track.prep_track (helper_funcs_glob/src/prep_track.py): smoothing
    and re-sampling, closed splines of the result, check of the normals, min-width inflation.  Returns dict(reftrack_interp,
    n_pts, normvec_normalized_interp, h (the spline system in moment form), coeffs_x_interp, coeffs_y_interp,
    normals_crossing [B] bool)."""
    rt, n_pts, lam = spline_approximation_batch(track, k_reg=reg_smooth_opts["k_reg"], s_reg=reg_smooth_opts["s_reg"],
                                                stepsize_prep=stepsize_opts["stepsize_prep"],
                                                stepsize_reg=stepsize_opts["stepsize_reg"], n_raw=n_raw, min_width=None)
    cx, cy, nv, h = calc_splines_batch(rt, n_pts=n_pts)
    crossing = check_normals_crossing_batch(rt, nv, 10, n_pts=n_pts) if check_normals else None
    if min_width is not None:                     # (the reference inflates AFTER the normals check: prep_track.py:89-98)
        rt, n_pts, lam = spline_approximation_batch(track, k_reg=reg_smooth_opts["k_reg"], s_reg=reg_smooth_opts["s_reg"],
                                                    stepsize_prep=stepsize_opts["stepsize_prep"],
                                                    stepsize_reg=stepsize_opts["stepsize_reg"], n_raw=n_raw, min_width=min_width)
    return dict(reftrack_interp=rt, n_pts=n_pts, normvec_normalized_interp=nv, h=h, coeffs_x_interp=cx, coeffs_y_interp=cy,
                normals_crossing=crossing, smoothing_lambda=lam)
