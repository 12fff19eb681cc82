"""Quasi-steady-state lap-time refinement of the raceline: batched projected-gradient descent on alpha.

The minimum-curvature raceline is not lap-time optimal (the ggv, the machine limit and drag make the fastest line differ
from the least-curved one).  refine_raceline_batch starts from an alpha inside the box of the QP, normally the
opt_min_curv_batch result, and lowers the lap time that create_raceline_batch followed by vel_profile_batch computes for
it, with the gradient from the device adjoints create_raceline_diff and vel_profile_diff (DESIGN.md section 3.13).  This
is not the reference's 'mintime' problem: the curvature limit is not enforced (unless kappa_bound, below) and the vehicle
model is the QSS one of the velocity profile.

The method is the spectral projected gradient (SPG2) of Birgin, Martinez and Raydan (2000), run per track and in
lockstep over the batch by spg(), which takes the objective as a batched (value, gradient) callable.  Every operation of
spg() is elementwise or a row reduction in a fixed order, so a track's iterates do not depend on the other tracks.

With metric_length = l, the steps are taken in the curvature metric M = I + l^4 H (H = E^T E, the Hessian of the
minimum-curvature QP), applied by CurvatureMetric through the minimum-curvature adjoint's banded solve: the lap-time
gradient is dominated by short wavelengths, which M damps like 1 / (1 + l^4 k^4) while longer ones keep the identity.

With kappa_bound as well, every step is taken inside the minimum-curvature QP's feasible set P = {lb <= alpha <= ub,
|k_ref + E alpha| <= kappa_bound} instead of the box alone: the direction is the scaled projected gradient in M, one
projection QP per iteration on the device (CurvatureProjection, mc_mincurv_solve_batch_ex with prox arguments).
"""
from __future__ import annotations

import contextlib
import math
import os
import re
from typing import Callable, Optional, Union

import torch

from . import _lib, batch as _b
from . import build as _build

# status of a track
CONVERGED = 0          # ||P(x - g) - x||_inf <= pg_tol
ITER_CAP = 1           # max_iters accepted steps without convergence
LINE_SEARCH = 2        # max_halvings halvings found no acceptable step: the last accepted point is kept
NO_GRADIENT = 3        # a non-finite lap time or gradient at the last accepted point, which is kept
EMPTY_BOX = 4          # lb > ub at some point (the track is narrower than w_veh): alpha0 is returned as it is
NO_PROJECTION = 5      # spg(project=...): a projection failed (QP status != 0, non-finite y, or a track the QP does not
                       # take) or gave no descent direction (g^T d >= 0, d != 0): the last accepted point is kept (alpha0,
                       # with NaN lap times, where the projection of alpha0 failed)
INACTIVE = -1          # n_pts[b] == 0
STATUS_TEXT = {CONVERGED: "converged", ITER_CAP: "iteration cap reached", LINE_SEARCH: "line search exhausted",
               NO_GRADIENT: "no usable gradient", EMPTY_BOX: "empty box (track narrower than w_veh)",
               NO_PROJECTION: "projection onto the curvature-limited set failed", INACTIVE: "inactive slot"}

CURV_ERROR_ALLOWED = 0.01     # [1/m] refine_raceline_batch(relinearise=...): the reference's iqp_curverror_allowed

# defaults of the method (Birgin, Martinez and Raydan 2000 use M = 10 and gamma = 1e-4 as well)
MAX_ITERS = 100        # accepted steps per track
PG_TOL = 1e-6          # on ||P(x - g) - x||_inf, x in m and g in s/m
MEMORY = 10            # M: the Armijo test is against the largest of the last M accepted lap times
GAMMA = 1e-4           # sufficient-decrease factor of the Armijo test
LAM_MIN, LAM_MAX = 1e-6, 1e4      # clamp of the Barzilai-Borwein step length [m^2/s]; LAM_MAX where s^T y <= 0
MAX_HALVINGS = 30      # trials per line search (the step goes down to 2^-29 of the spectral one)
ACTIVE_EPS = 1e-2      # [m] the two-metric projection pins the points within min(ACTIVE_EPS, ||P(x - g) - x||_inf) of a
                       # bound that g pushes them against (Bertsekas 1982)
PIN_FACTOR = 1e6       # CurvatureMetric's pin: PIN_FACTOR (mu + 6 / h_min^4), 6 / h^4 the diagonal of E^T E on a straight


def _fix_eps() -> float:
    """FIX_EPS of csrc/common.cuh: the half-width the QP setup gives a collapsed box."""
    src = _lib._c_source(os.path.join(_build.CSRC, "common.cuh"))
    return float(re.search(r"constexpr\s+double\s+FIX_EPS\s*=\s*([0-9.eE+-]+)\s*;", src).group(1))


FIX_EPS = _fix_eps()


def row_sum(v: torch.Tensor) -> torch.Tensor:
    """Sums over the last dimension by pairwise halving (zero-padded to a power of two): elementwise additions only, so
    a row's sum has the same bits whatever the other rows are (a library reduction may pick its order by the shape)."""
    n = v.shape[-1]
    p = 1 << max(0, (n - 1).bit_length())
    if p != n:
        v = torch.nn.functional.pad(v, (0, p - n))
    while v.shape[-1] > 1:
        h = v.shape[-1] // 2
        v = v[..., :h] + v[..., h:]
    return v[..., 0]


def box(reftrack: torch.Tensor, w_veh: Union[float, torch.Tensor], n_pts: Optional[torch.Tensor] = None):
    """(lb, ub, empty) of opt_min_curv's box for every track: ub = w_right - w_veh / 2, lb = -(w_left - w_veh / 2), a
    collapsed box (ub - lb < 2 FIX_EPS) replaced by mid -+ FIX_EPS as in mincurv_setup.cu; empty [B] bool marks the
    tracks with lb > ub at some point.  Beyond n_pts[b] both bounds are 0."""
    B, n_max, _ = reftrack.shape
    wv = w_veh.to(reftrack).reshape(B, 1) if isinstance(w_veh, torch.Tensor) else float(w_veh)
    ub = reftrack[:, :, 2] - 0.5 * wv
    lb = -(reftrack[:, :, 3] - 0.5 * wv)
    valid = _valid(n_pts, B, n_max, reftrack.device)
    empty = ((lb > ub) & valid).any(dim=1)
    mid = 0.5 * (lb + ub)
    collapsed = ub - lb < 2.0 * FIX_EPS
    lb = torch.where(collapsed, mid - FIX_EPS, lb)
    ub = torch.where(collapsed, mid + FIX_EPS, ub)
    zero = torch.zeros_like(lb)
    return torch.where(valid, lb, zero), torch.where(valid, ub, zero), empty


def _valid(n_pts, B, n_max, dev) -> torch.Tensor:
    """bool [B, n_max]: the points below n_pts[b]."""
    if n_pts is None:
        return torch.ones((B, n_max), dtype=torch.bool, device=dev)
    return torch.arange(n_max, device=dev)[None, :] < n_pts.to(device=dev, dtype=torch.int64)[:, None]


def spg(fun: Callable, x0: torch.Tensor, lb: torch.Tensor, ub: torch.Tensor, active: torch.Tensor,
        max_iters: int = MAX_ITERS, pg_tol: float = PG_TOL, memory: int = MEMORY, gamma: float = GAMMA,
        lam_min: float = LAM_MIN, lam_max: float = LAM_MAX, max_halvings: int = MAX_HALVINGS,
        callback: Optional[Callable] = None, metric: Optional[Callable] = None,
        project: Optional[Callable] = None) -> dict:
    """Spectral projected gradient (SPG2 of Birgin, Martinez and Raydan 2000) on the box lb <= x <= ub [B, n] for the
    tracks in active [B] (bool), in lockstep: per iteration and track

      d = P(x - lam g) - x;  t = 1, 1/2, 1/4 ... until f(x + t d) <= max(last `memory` accepted f) + gamma t g^T d;
      s = t d, y = g(x + t d) - g;  lam = clamp(s^T s / s^T y, lam_min, lam_max), lam_max where s^T y <= 0.

    The first lam is 1 / ||P(x0 - g0) - x0||_inf, clamped.  A track converges when ||P(x - g) - x||_inf <= pg_tol.

    metric (None: the above): the steps in a metric M, two-metric projection (Bertsekas 1982).  After every gradient
    evaluation u = M^-1 g on the free points and u = g on the pinned ones, A = {x <= lb + eps, g > 0} u {x >= ub - eps,
    g < 0} with eps = min(ACTIVE_EPS, ||P(x - g) - x||_inf); then d = P(x - lam u) - x, with lam = clamp(s^T y / y^T w)
    (BB2 in M, w = M^-1 y without pins; lam_max where s^T y <= 0 or y^T w <= 0; the first 1 / ||P(x0 - u0) - x0||_inf).
    The line search, the statuses and the stopping rule are the above.  A track takes the above step (u = g and its lam)
    in an iteration whose metric solve failed or whose d has g^T d >= 0, counted in metric_fallbacks [B].
    metric(g, pin, y, mask) -> (u, w, ok): u = M_FF^-1 g_F on the free points of every track in mask (pin [B, n] bool;
    u on the pins is not read), w = M^-1 y (None for y None), ok [B] bool: both are usable.

    project (None: the above): steps inside a convex set P within the box, in the metric project works in.  x0 is first
    replaced by its projection y(x0, 0); then after every gradient evaluation d = y(x, lam g) - x, where
    project(x, q, mask) -> (y, ok) returns y = argmin_{a in P} 1/2 |a - x|^2_M + q^T (a - x) for the tracks in mask and
    ok [B] bool.  lam is BB2 in metric (lam = s^T y / y^T w, w from metric(y, no pins, None, mask); lam_max where that is
    not positive or not usable) or, without metric, the identity BB step above; the first lam is the identity one.  The
    trials x + t d stay in P (convex) up to the box clamp, the pins are not used, the stopping rule is on
    pg_norm = ||d||_inf / lam (the above at lam = 1 with the identity metric and P the box).  A track whose projection fails
    (ok false or a non-finite y) or whose d has g^T d >= 0, d != 0, stops with NO_PROJECTION and keeps its last accepted
    point; where the projection of x0 fails it keeps x0 (box-clamped), is never evaluated and f is NaN.  The result also
    holds projection_failures [B] int32, the failed projections (0 or 1: a failure ends the track).

    fun(x, mask, need_grad) -> (f [B], g [B, n] or None, redo): the objective and, with need_grad, its gradient at
    the rows of x in mask (other rows: anything, they are not read).  redo is None or a bool [B] mask of tracks fun could
    not evaluate at this x for want of buffer space; spg then calls fun.grow() and repeats their trial at the same step
    (such a trial counts neither as one of the track's max_halvings trials nor in evals).  A non-finite f of a trial
    rejects the trial; a non-finite f or g at an accepted point ends the track (NO_GRADIENT).

    One device-to-host read per trial and per iteration (whether any track is still searching / running).  callback(it,
    x, f, status), if given, runs after every iteration (it = 0 after the first evaluation).  Returns dict(x, f, f0,
    status, iters, evals, pg_norm) with the module's status codes (INACTIVE for rows outside active)."""
    if max_iters < 0 or memory < 1 or max_halvings < 1:
        raise ValueError("spg: max_iters >= 0, memory >= 1 and max_halvings >= 1 are required")
    if not (pg_tol >= 0.0 and 0.0 < gamma < 1.0 and 0.0 < lam_min <= lam_max):
        raise ValueError("spg: pg_tol >= 0, 0 < gamma < 1 and 0 < lam_min <= lam_max are required")
    B = x0.shape[0]
    dev = x0.device
    proj = lambda v: torch.minimum(torch.maximum(v, lb), ub)      # noqa: E731
    x = proj(x0)
    started = active
    if project is not None:
        y0, ok0 = project(x, torch.zeros_like(x), active)
        started = active & ok0 & torch.isfinite(y0).all(dim=1)
        x = torch.where(started[:, None], proj(y0), x)
        p_fail = (active & ~started).to(torch.int32)
    f, g, _ = fun(x, started, True)
    evals = started.to(torch.int32)
    usable = started & torch.isfinite(f) & torch.isfinite(g).all(dim=1)
    status = torch.full((B,), INACTIVE, dtype=torch.int32, device=dev)
    status = torch.where(active, torch.where(usable, ITER_CAP, NO_GRADIENT), status).to(torch.int32)
    if project is not None:
        status = torch.where(active & ~started, NO_PROJECTION, status).to(torch.int32)
        f = torch.where(started, f, torch.full_like(f, math.nan))
    running = usable.clone()
    f0 = f.clone()
    hist = f[:, None].repeat(1, int(memory))
    iters = torch.zeros((B,), dtype=torch.int32, device=dev)

    def pg_norm(x, g):
        return (proj(x - g) - x).abs().amax(dim=1)

    def metric_step(x, g, pgn, y, mask):
        """(u, w, ok) of metric at (x, g): u = g on the pins and wherever the solve is not usable."""
        eps = torch.clamp(pgn, max=ACTIVE_EPS)[:, None]
        pin = ((x <= lb + eps) & (g > 0.0)) | ((x >= ub - eps) & (g < 0.0))
        u, w, ok = metric(g, pin, y, mask)
        return torch.where(pin | ~ok[:, None], g, u), w, ok

    def projected_step(x, g, lam, mask):
        """(d, pgn, stop, failed) of project at (x, lam g) for the tracks in mask: d = y - x (0 elsewhere and where the
        projection failed), pgn = ||d||_inf / lam (NaN where it failed), stop: failed or g^T d >= 0 with d != 0."""
        y, ok = project(x, lam[:, None] * g, mask)
        failed = mask & ~(ok & torch.isfinite(y).all(dim=1))
        d = torch.where((mask & ~failed)[:, None], y - x, torch.zeros_like(x))
        pgn = torch.where(failed, torch.full_like(lam, math.nan), d.abs().amax(dim=1) / lam)
        stop = failed | (mask & (row_sum(g * d) >= 0.0) & (d != 0.0).any(dim=1))
        return d, pgn, stop, failed

    pgn = pg_norm(x, g)
    lam = torch.clamp(1.0 / pgn, lam_min, lam_max)          # (pgn = 0: inf, clamped; such a track converges at once)
    if project is not None:
        d_p, pgn, p_stop, failed = projected_step(x, g, lam, running)
        p_fail += failed.to(torch.int32)
    elif metric is not None:
        u, _, m_ok = metric_step(x, g, pgn, None, running)
        lam_m = torch.clamp(1.0 / pg_norm(x, u), lam_min, lam_max)
        fallbacks = torch.zeros((B,), dtype=torch.int32, device=dev)
    if callback is not None:
        callback(0, x, f, status)
    for it in range(1, int(max_iters) + 1):
        conv = running & (pgn <= pg_tol)
        status = torch.where(conv, CONVERGED, status).to(torch.int32)
        running &= ~conv
        if project is not None:
            stop = running & p_stop
            status = torch.where(stop, NO_PROJECTION, status).to(torch.int32)
            running &= ~stop
        if not bool(running.any()):                                         # the iteration's one read
            break
        run2 = running[:, None]
        if project is not None:
            d = torch.where(run2, d_p, torch.zeros_like(x))
        else:
            d = torch.where(run2, proj(x - lam[:, None] * g) - x, torch.zeros_like(x))
        if metric is not None and project is None:
            d_m = torch.where(run2, proj(x - lam_m[:, None] * u) - x, torch.zeros_like(x))
            use_m = m_ok & (row_sum(g * d_m) < 0.0)
            fallbacks += (running & ~use_m).to(torch.int32)
            d = torch.where(use_m[:, None], d_m, d)
        gd = row_sum(g * d)
        f_ref = hist.amax(dim=1)
        t = torch.ones((B,), dtype=x.dtype, device=dev)
        searching = running.clone()
        exhausted = torch.zeros_like(running)
        n_tried = torch.zeros((B,), dtype=torch.int32, device=dev)      # per track: a redo does not use up a trial
        x_new, f_new = x.clone(), f.clone()
        while True:
            xt = proj(x + t[:, None] * d)                                   # (rounding may leave the box by an ulp)
            ft, _, redo = fun(xt, searching, False)
            tried = searching if redo is None else searching & ~redo
            evals += tried.to(torch.int32)
            n_tried += tried.to(torch.int32)
            ok = tried & (ft <= f_ref + gamma * t * gd)
            x_new = torch.where(ok[:, None], xt, x_new)
            f_new = torch.where(ok, ft, f_new)
            searching &= ~ok
            out = searching & (n_tried >= int(max_halvings))
            exhausted |= out
            searching &= ~out
            t = torch.where(tried & ~ok, 0.5 * t, t)
            flags = torch.stack((searching.any(), torch.zeros((), dtype=torch.bool, device=dev) if redo is None
                                 else redo.any())).tolist()                   # the trial's one read
            if flags[1]:
                fun.grow()
            if not flags[0]:
                break
        status = torch.where(exhausted, LINE_SEARCH, status).to(torch.int32)
        acc = running & ~exhausted
        _, g_new, _ = fun(x_new, acc, True)
        evals += acc.to(torch.int32)
        good = acc & torch.isfinite(f_new) & torch.isfinite(g_new).all(dim=1)
        status = torch.where(acc & ~good, NO_GRADIENT, status).to(torch.int32)
        running = good
        s = x_new - x
        sums = row_sum(torch.stack((s * s, s * (g_new - g))))
        lam_bb = torch.where(sums[1] > 0.0, torch.clamp(sums[0] / sums[1], lam_min, lam_max),
                             torch.full_like(lam, lam_max))
        acc2 = acc[:, None]
        y = g_new - g if metric is not None else None
        x = torch.where(acc2, x_new, x)
        f = torch.where(acc, f_new, f)
        g = torch.where(good[:, None], g_new, g)
        lam = torch.where(good, lam_bb, lam)
        hist = torch.where(acc2, torch.cat((hist[:, 1:], f_new[:, None]), dim=1), hist)
        iters += acc.to(torch.int32)
        pgn = torch.where(good, pg_norm(x, g), pgn)
        if project is not None:                     # BB2 in the metric (its row without pins), then the next direction
            if metric is not None:
                w, _, ok_w = metric(y, torch.zeros_like(y, dtype=torch.bool), None, good)
                yw = row_sum(y * w)
                lam_p = torch.where(ok_w & (sums[1] > 0.0) & (yw > 0.0), torch.clamp(sums[1] / yw, lam_min, lam_max),
                                    torch.full_like(lam, lam_max))
                lam = torch.where(good, lam_p, lam)
            d_new, pgn_new, stop_new, failed = projected_step(x, g, lam, good)
            p_fail += failed.to(torch.int32)
            d_p = torch.where(good[:, None], d_new, d_p)
            pgn = torch.where(good, pgn_new, pgn)
            p_stop = torch.where(good, stop_new, p_stop)
        elif metric is not None:                    # the next direction and the metric's BB2 step in one solve
            u_new, w, ok_new = metric_step(x, g, pgn, y, good)
            yw = row_sum(y * w)
            lam_m2 = torch.where((sums[1] > 0.0) & (yw > 0.0), torch.clamp(sums[1] / yw, lam_min, lam_max),
                                 torch.full_like(lam, lam_max))
            u = torch.where(good[:, None], u_new, u)
            m_ok = torch.where(good, ok_new, m_ok)
            lam_m = torch.where(good, lam_m2, lam_m)
        if callback is not None:
            callback(it, x, f, status)
    else:
        conv = running & (pgn <= pg_tol)
        status = torch.where(conv, CONVERGED, status).to(torch.int32)
    ok_pg = (status == CONVERGED) | (status == ITER_CAP) | (status == LINE_SEARCH)
    out = dict(x=x, f=f, f0=f0, status=status, iters=iters, evals=evals,
               pg_norm=torch.where(ok_pg, pgn, torch.full_like(pgn, math.nan)))
    if project is not None:
        out["projection_failures"] = p_fail
    elif metric is not None:
        out["metric_fallbacks"] = fallbacks
    return out


class LapTime:
    """The objective of refine_raceline_batch: the lap time of create_raceline_batch -> vel_profile_batch at alpha, for
    the tracks of a mask (the others get n_pts = 0 for the launch, which every kernel skips), and its gradient from
    create_raceline_diff -> vel_profile_diff (strict=False: n_out and every discrete decision of the forward held).

    No usable gradient (g = NaN for the track) where vel_profile_diff reports grad_status != 0, where the station count
    overflowed (n_out <= 0; f is NaN there too), and where g is exactly zero on every point: with strict=False the two
    adjoints hand on zeros for a track they could not differentiate (the velocity-profile adjoint's own non-finite
    status is not returned), and the lap time of a real raceline never has a zero gradient in every alpha.

    n_out_max is derived as create_raceline_batch derives it, from the start point (unless it was set before); a trial
    that overflows it is reported in redo and grow() enlarges it to what the kernel asked for.  The ggv and machine
    tables are kept on the host (pinned), so that the checks of vel_profile_batch read no device memory and their copy
    does not synchronise the stream; with a vehicle per track (vp_args holds vehicles= and veh_id=) the batch.Vehicles
    object, whose tables are on the device already, is passed through, with veh_id checked and put on the device once
    here.  timer(name), a context manager, brackets the launches of each part ('trial',
    'forward', 'backward'); tools/refine_time.py times them."""

    def __init__(self, reftrack, normvec, n_pts, stepsize_interp, vp_args: dict):
        self.reftrack, self.normvec, self.step = reftrack, normvec, float(stepsize_interp)
        B, n_max, _ = reftrack.shape
        if vp_args.get("vehicles") is not None:
            veh = vp_args["vehicles"]
            self.vp = dict(vp_args, veh_id=veh.veh_id(vp_args.get("veh_id"), B, reftrack.device))
        else:
            host = lambda t: torch.as_tensor(t, dtype=torch.float64).cpu().contiguous()     # noqa: E731
            pin = (lambda t: t.pin_memory()) if reftrack.is_cuda else (lambda t: t)          # noqa: E731
            self.vp = dict(vp_args, ggv=pin(host(vp_args["ggv"])), ax_max_machines=pin(host(vp_args["ax_max_machines"])))
        self.n_pts = n_pts if n_pts is not None else torch.full((B,), n_max, dtype=torch.int32, device=reftrack.device)
        self.n_out_max = None
        self._need = None
        self.timer = lambda name: contextlib.nullcontext()

    def start(self, alpha: torch.Tensor, mask: torch.Tensor) -> None:
        """Derives n_out_max at alpha as create_raceline_batch does (if it is not set yet)."""
        if self.n_out_max is None:
            rl = _b.create_raceline_batch(self.reftrack, self.normvec, alpha, self.step, n_pts=self._masked(mask),
                                          with_head_curv=False)
            self.n_out_max = int(rl["t_values"].shape[1])

    def _masked(self, mask):
        return torch.where(mask, self.n_pts, torch.zeros_like(self.n_pts))

    def _laptime(self, rl):
        return _b.vel_profile_batch(rl["kappa"], rl["el_lengths_interp"], n_pts=rl["n_out"], want_profiles=False,
                                    **self.vp)["laptime"][:, 0]

    def __call__(self, x, mask, need_grad):
        if self.n_out_max is None:                  # (refine_raceline_batch(kappa_bound=...): sized at the projected start)
            self.start(x, mask)
        if not need_grad:
            with self.timer("trial"):
                rl = _b.create_raceline_batch(self.reftrack, self.normvec, x, self.step, n_pts=self._masked(mask),
                                              n_out_max=self.n_out_max)
                f = self._laptime(rl)
                redo = mask & (rl["n_out"] < 0)
                self._need = (-rl["n_out"]).max()
            return f, None, redo
        with self.timer("forward"):
            xg = x.detach().clone().requires_grad_()
            rl = _b.create_raceline_diff(self.reftrack, self.normvec, xg, self.step, n_pts=self._masked(mask),
                                         n_out_max=self.n_out_max, strict=False)
            vp = _b.vel_profile_diff(rl["kappa"], rl["el_lengths_interp"], n_pts=rl["n_out"], strict=False, **self.vp)
        with self.timer("backward"):
            g, = torch.autograd.grad(vp["laptime"].sum(), xg)
        bad = (vp["grad_status"] != 0) | (rl["n_out"] <= 0) | (g == 0.0).all(dim=1)
        f = torch.where(rl["n_out"] > 0, vp["laptime"].detach(), torch.full_like(g[:, 0], math.nan))
        return f, torch.where(bad[:, None], torch.full_like(g, math.nan), g), None

    def grow(self):
        """Enlarges n_out_max to what the last trial's overflowing track asked for (+16, as create_raceline_batch)."""
        self.n_out_max = max(self.n_out_max, int(self._need.item()) + 16)


class CurvatureMetric:
    """The metric of refine_raceline_batch(metric_length=l): M = I + l^4 H, H = E^T E the Hessian of the minimum-curvature
    QP for the track's centre line (DESIGN.md section 3.2), applied through mc_mincurv_adjoint_batch, which assembles H,
    factors H + diag(sens[0] + sens[1]) and returns grad_w_right = sens[0] v, v = (H + diag(sens[0] + sens[1]))^-1 rhs.
    With sens[0] = mu = l^-4 on a point and sens[1] = 0 that is mu v = M^-1 rhs there; a pinned point gets sens[0] = P =
    PIN_FACTOR (mu + 6 / h_min^4), which decouples it (v = rhs / P there), so the free points get M_FF^-1 rhs_F.  The
    widths are replaced by 1 m on each side and w_veh by 0 (H does not depend on them, and no box collapses).

    A call is one launch of 2 B instances: row 2b solves for g with the pins, row 2b + 1 for y without (owned by row 2b
    through centre_id, so it costs a factorisation and no assembly).  Tracks outside the mask, and those with fewer than
    N_MIN points, are not launched (n_pts 0, grad_status -1: not ok); with n_max < N_MIN nothing is.  h, the chunk size
    and the chunk-local centre ids are computed once here, so a call does not synchronise the stream.  timer(name) as
    LapTime's ('metric').  lin_alpha [B, n_max] (None: the centre line): H is that of the QP linearised about the line
    reftrack + lin_alpha * normvec (DESIGN.md section 3.2)."""

    def __init__(self, reftrack, normvec, n_pts, length: float, lin_alpha: Optional[torch.Tensor] = None):
        B, n_max, _ = reftrack.shape
        dev = reftrack.device
        self.mu = float(length) ** -4
        self.n_pts = n_pts if n_pts is not None else torch.full((B,), n_max, dtype=torch.int32, device=dev)
        self.launchable = self.n_pts >= _b.N_MIN
        self.timer = lambda name: contextlib.nullcontext()
        self.chunk = None
        if n_max < _b.N_MIN:
            return
        _, _, _, h = _b.calc_splines_batch(reftrack, n_pts=n_pts, want_coeffs=False)
        valid = _valid(n_pts, B, n_max, dev)
        h_min = torch.where(valid, h, torch.full_like(h, math.inf)).amin(dim=1)
        self.pin = PIN_FACTOR * (self.mu + 6.0 / h_min ** 4)
        two = lambda t: t.repeat_interleave(2, dim=0).contiguous()      # noqa: E731
        self.reftrack = two(torch.cat((reftrack[:, :, :2], torch.ones_like(reftrack[:, :, 2:])), dim=2))
        self.normvec, self.h = two(normvec), two(h)
        self.lin = None if lin_alpha is None else two(lin_alpha.to(torch.float64))
        chunk = _b._chunk(2 * B, _lib.load().mc_mincurv_workspace_bytes(1, n_max), dev)
        self.chunk = max(2, chunk - chunk % 2)                           # (a track's two rows share a launch)
        r = torch.arange(2 * B, dtype=torch.int32, device=dev)
        self.centre_id = r % self.chunk - r % 2                          # row 2b + 1 owned by row 2b, chunk-local

    def __call__(self, g, pin, y, mask):
        B, n_max = g.shape
        if self.chunk is None:
            return g, y, torch.zeros_like(mask)
        with self.timer("metric"):
            go = mask & self.launchable
            n_dir = torch.where(go, self.n_pts, torch.zeros_like(self.n_pts))
            n_pts = torch.stack((n_dir, n_dir if y is not None else torch.zeros_like(n_dir)), dim=1).reshape(2 * B)
            gs = torch.where(n_pts > 0, 0, -1).to(torch.int32)
            sens = torch.zeros((B, 2, 2, n_max), dtype=torch.float64, device=g.device)
            sens[:, 0, 0] = torch.where(pin, self.pin[:, None], self.mu)
            sens[:, 1, 0] = self.mu
            sens = sens.reshape(2 * B, 2, n_max)
            rhs = torch.stack((g, y if y is not None else torch.zeros_like(g)), dim=1).reshape(2 * B, n_max)
            out = torch.empty((2 * B, n_max), dtype=torch.float64, device=g.device)
            gwl = torch.empty_like(out)
            gwv = torch.empty((2 * B,), dtype=torch.float64, device=g.device)
            for s in range(0, 2 * B, self.chunk):
                e = min(2 * B, s + self.chunk)
                _b._mincurv_launch("mc_mincurv_adjoint_batch", e - s, n_pts[s:e], self.reftrack[s:e], self.normvec[s:e],
                                   self.h[s:e], None, 0.0, None, _b.F_SCALE, self.centre_id[s:e], sens[s:e], gs[s:e],
                                   rhs[s:e], out[s:e], gwl[s:e], gwv[s:e], None, None, None, 0,
                                   None if self.lin is None else self.lin[s:e])
            out, gs = out.reshape(B, 2, n_max), gs.reshape(B, 2)
            u, w = out[:, 0], (out[:, 1] if y is not None else None)
            ok = go & (gs[:, 0] == 0) & torch.isfinite(u).all(dim=1)
            if y is not None:
                ok &= (gs[:, 1] == 0) & torch.isfinite(w).all(dim=1)
            return u, w, ok


class CurvatureProjection:
    """The projection of refine_raceline_batch(kappa_bound=kb, metric_length=l) onto the minimum-curvature QP's feasible
    set P = {lb <= alpha <= ub, |k_ref + E alpha| <= kb} (opt_min_curv's, for the same reftrack, w_veh and kb) in the
    curvature metric M = I + l^4 H: spg's project(x, q, mask) -> (y, ok),

      y = argmin_{a in P} 1/2 (a - x)^T M (a - x) + q^T (a - x),

    which is, divided by l^4 with mu = l^-4, the minimum-curvature QP with Hessian H + mu I and linear term
    c = mu q - (H + mu I) x: one mc_mincurv_solve_batch_ex call with prox arguments (the box phase and, where the rows
    bind, the curvature-row phase).  ok: the QP's status is 0 and y is finite.  Tracks outside the mask get n_pts 0, those
    with fewer than N_MIN points are never launched (not ok); with n_max < N_MIN nothing is.  h and the chunk size are
    computed once here, so a call does not synchronise the stream.  kappa_lin(x, mask) -> kappa_lin_max [B], the QP's
    max |k_ref + E x| at x (assembly and the finalize stage); evaluate(x, mask) -> (kappa_lin_max, curv_error_max) [B].
    timer(name) as LapTime's ('projection').  lin_alpha [B, n_max] (None: the centre line): P and H are those of the QP
    linearised about the line reftrack + lin_alpha * normvec (DESIGN.md section 3.2)."""

    def __init__(self, reftrack, normvec, n_pts, w_veh, kappa_bound: float, length: float,
                 lin_alpha: Optional[torch.Tensor] = None):
        B, n_max, _ = reftrack.shape
        dev = reftrack.device
        self.mu, self.kb = float(length) ** -4, float(kappa_bound)
        self.n_pts = n_pts if n_pts is not None else torch.full((B,), n_max, dtype=torch.int32, device=dev)
        self.launchable = self.n_pts >= _b.N_MIN
        self.w_scalar, self.w_batch = _b._wveh(w_veh, B, dev)
        self.timer = lambda name: contextlib.nullcontext()
        self.chunk = None
        self.lin = None if lin_alpha is None else lin_alpha.to(torch.float64).contiguous()
        if n_max < _b.N_MIN:
            return
        self.reftrack, self.normvec = reftrack.contiguous(), normvec.contiguous()
        _, _, _, self.h = _b.calc_splines_batch(self.reftrack, n_pts=n_pts, want_coeffs=False)
        self.chunk = _b._chunk(B, _lib.load().mc_mincurv_workspace_bytes(1, n_max), dev)

    def _n(self, mask):
        return torch.where(mask & self.launchable, self.n_pts, torch.zeros_like(self.n_pts))

    def _ws(self):
        return _b._workspace("mincurv", _lib.load().mc_mincurv_workspace_bytes(self.chunk, self.h.shape[1]), self.h.device)

    def __call__(self, x, q, mask):
        if self.chunk is None:
            return x, torch.zeros_like(mask)
        with self.timer("projection"):
            B, n_max = x.shape
            out = _b._mincurv_results(B, n_max, x.device)
            _b._launch_chunks("mc_mincurv_solve_batch_ex", B, self.chunk, self._ws(), n_max,
                              *map(_b._rows, (self._n(mask), self.reftrack, self.normvec, self.h)), self.kb, self.w_scalar,
                              _b._rows(self.w_batch), _b.F_SCALE, *map(_b._rows, out.values()), self.mu,
                              _b._rows(x.contiguous()), _b._rows(q.contiguous()), _b._rows(self.lin))
            ok = mask & self.launchable & (out["status"] == 0) & torch.isfinite(out["alpha"]).all(dim=1)
            return out["alpha"], ok

    def kappa_lin(self, x, mask):
        return self.evaluate(x, mask)[0]

    def evaluate(self, x, mask):
        B, n_max = x.shape
        kmax = torch.full((B,), math.nan, dtype=torch.float64, device=x.device)
        if self.chunk is None:
            return kmax, kmax.clone()
        out = _b._mincurv_results(B, n_max, x.device)
        n = self._n(mask)
        ws = self._ws()
        x = x.contiguous()
        for s in range(0, B, self.chunk):              # (assembly and finalize share the chunk's workspace)
            e = min(B, s + self.chunk)
            _b._call("mc_mincurv_setup_batch_ex", e - s, n_max, n[s:e], self.reftrack[s:e], self.normvec[s:e], self.h[s:e],
                     self.w_scalar, None if self.w_batch is None else self.w_batch[s:e], _b.F_SCALE, out["status"][s:e],
                     None if self.lin is None else self.lin[s:e], ws=ws)
            _b._call("mc_mincurv_finalize_batch", e - s, n_max, n[s:e], x[s:e], self.kb, out["curv_error_max"][s:e],
                     out["kappa_lin_max"][s:e], out["status"][s:e], int(self.lin is not None), ws=ws)
        ok = mask & self.launchable & (out["status"] != 1) & (out["status"] >= 0)
        return torch.where(ok, out["kappa_lin_max"], kmax), torch.where(ok, out["curv_error_max"], kmax)


def refine_raceline_batch(reftrack: torch.Tensor, normvec: torch.Tensor, alpha0: torch.Tensor,
                          w_veh: Union[float, torch.Tensor], ggv=None, ax_max_machines=None, v_max: Optional[float] = None,
                          drag_coeff: Optional[float] = None, m_veh: Optional[float] = None, stepsize_interp: float = 2.0, n_pts: Optional[torch.Tensor] = None,
                          dyn_model_exp: float = 1.0, filt_window: Optional[int] = None, max_iters: int = MAX_ITERS,
                          pg_tol: float = PG_TOL, memory: int = MEMORY, gamma: float = GAMMA, lam_min: float = LAM_MIN,
                          lam_max: float = LAM_MAX, max_halvings: int = MAX_HALVINGS,
                          callback: Optional[Callable] = None, objective: Optional[LapTime] = None,
                          metric_length: Optional[float] = None, kappa_bound: Optional[float] = None,
                          relinearise: int = 0, curv_error_allowed: float = CURV_ERROR_ALLOWED,
                          vehicles: Optional[_b.Vehicles] = None, veh_id=None) -> dict:
    """Lowers the quasi-steady-state lap time of every track's raceline by moving alpha inside opt_min_curv's box.

    reftrack [B, n_max, 4], normvec [B, n_max, 2] and alpha0 [B, n_max] (normally the opt_min_curv_batch result) as for
    create_raceline_batch; w_veh a float or [B]; the vehicle arguments as for vel_profile_diff (one top speed).  The box
    is ub = w_right - w_veh / 2, lb = -(w_left - w_veh / 2) (collapsed boxes as in the QP); alpha0 is projected onto it.
    The lap time is that of create_raceline_batch(stepsize_interp) followed by vel_profile_batch, each trial with its own
    n_out; the gradient holds n_out and the profile's decisions, and the line search tests the real lap time.  Without
    kappa_bound the curvature limit is not enforced (check_traj_batch reports it).  Method and defaults: spg() and the module constants.

    Returns dict(alpha [B, n_max], laptime [B], laptime_start [B] (at the projected alpha0), iters [B] (accepted steps),
    evals [B] (lap-time evaluations), status [B] int32 (CONVERGED 0, ITER_CAP 1, LINE_SEARCH 2, NO_GRADIENT 3,
    EMPTY_BOX 4, INACTIVE -1), pg_norm [B] (||P(alpha - g) - alpha||_inf at the result; NaN for statuses 3, 4, -1)).
    Statuses 4 and -1, and status 3 for a track with a non-finite reftrack, normal or alpha0 entry, return alpha0
    unchanged; their laptime is NaN.  objective: a LapTime built for these inputs (its
    timer is used, by the metric too), or None.

    metric_length: None (steps in the identity metric), or l > 0 [m]: steps in the curvature metric I + l^4 H
    (CurvatureMetric, spg's metric): wavelengths much longer than l move as with the identity, shorter ones are damped.
    The result then also holds metric_fallbacks [B] int32, the iterations in which the track took the identity step.

    kappa_bound: None (alpha stays in the box only), or kb > 0 [1/m] (metric_length required): alpha stays in opt_min_curv's
    feasible set for this kappa_bound, the box and the linearised curvature rows |k_ref + E alpha| <= kb about the centre
    line.  alpha0 is projected onto it in the metric (replacing the clamp to the box), and every step is the projected
    gradient step in the metric (CurvatureProjection, spg's project: one QP per iteration; no pins, no metric_fallbacks).
    pg_norm is then ||d||_inf / lam of that step.  A track whose projection fails, or gives no descent direction, stops
    with status NO_PROJECTION (5) at its last accepted point; where alpha0's projection fails (e.g. fewer than N_MIN
    points) alpha0 is returned with NaN lap times.  The result also holds kappa_lin_max [B] (the QP's max |k_ref + E alpha|
    at the result), kappa_max [B] (the raceline's max |kappa| from create_raceline_batch at the result; the rows are a
    linearisation, so it may exceed kb by about curv_error_max) and projection_failures [B] int32; kappa_lin_max and
    kappa_max are NaN where alpha0 is returned, and curv_error_max [B] (the QP's linearisation error at the result).

    relinearise: r >= 0 outer rounds after the first (kappa_bound required), as the reference's iterative QP does on a
    fixed grid.  Round 0 is the run above, about the centre line.  Round k >= 1 starts from the previous round's result
    x_k, builds the projection and the metric about the line reftrack + x_k * normvec (DESIGN.md section 3.2), projects
    x_k onto that set and runs spg() for up to max_iters iterations.  A track leaves after a round whose result has
    curv_error_max (against that round's linearisation) <= curv_error_allowed, or after round relinearise; a track whose
    round-start projection fails keeps the previous round's result with status NO_PROJECTION.  The result then also holds
    rounds [B] int32 (the last round whose result is returned); iters, evals and projection_failures add up over the
    rounds, laptime_start is that of round 0, and status, pg_norm, kappa_lin_max and curv_error_max are the last round's.

    vehicles, veh_id: a vehicle per track (batch.Vehicles; veh_id [B], None for one vehicle per track), each track
    driven at its vehicle's v_max; ggv, ax_max_machines, v_max, drag_coeff and m_veh are then None.  Tracks are refined
    independently, so a track's result is that of the track refined alone with its vehicle.  A track whose vehicle the
    kernels refuse gets no gradient (NO_GRADIENT)."""
    if int(relinearise) != relinearise or relinearise < 0:
        raise ValueError("refine_raceline_batch: relinearise must be an integer >= 0")
    if relinearise and kappa_bound is None:
        raise ValueError("refine_raceline_batch: relinearise needs kappa_bound (it re-linearises the curvature rows)")
    if not (math.isfinite(float(curv_error_allowed)) and float(curv_error_allowed) >= 0.0):
        raise ValueError("refine_raceline_batch: curv_error_allowed must be a finite curvature >= 0 [1/m]")
    if metric_length is not None and not (math.isfinite(float(metric_length)) and float(metric_length) > 0.0):
        raise ValueError("refine_raceline_batch: metric_length must be None or a finite length > 0 [m]")
    if kappa_bound is not None:
        if not (math.isfinite(float(kappa_bound)) and float(kappa_bound) > 0.0):
            raise ValueError("refine_raceline_batch: kappa_bound must be None or a finite curvature > 0 [1/m]")
        if metric_length is None:
            raise ValueError("refine_raceline_batch: kappa_bound needs metric_length (the projection runs in the "
                             "curvature metric)")
    _b._require_cuda()
    reftrack, normvec, alpha0 = _b._f64(reftrack, "reftrack"), _b._f64(normvec, "normvec"), _b._f64(alpha0, "alpha0")
    B, n_max, four = reftrack.shape
    if four != 4 or normvec.shape != (B, n_max, 2) or alpha0.shape != (B, n_max):
        raise RuntimeError("refine_raceline_batch: reftrack must be [B, n_max, 4], normvec [B, n_max, 2], alpha0 [B, n_max]")
    if vehicles is None and (isinstance(v_max, torch.Tensor) or hasattr(v_max, "__len__")):
        raise ValueError("refine_raceline_batch: v_max must be one number")
    if not float(stepsize_interp) > 0.0:
        raise ValueError("refine_raceline_batch: stepsize_interp must be positive")
    dev = reftrack.device
    n_pts = _b._npts(n_pts, B, dev)
    if isinstance(w_veh, torch.Tensor) and w_veh.numel() != B:
        raise ValueError("w_veh tensor must have one entry per track")
    lb, ub, empty = box(reftrack, w_veh, n_pts)
    valid = _valid(n_pts, B, n_max, dev)
    lb, ub = torch.where(valid, lb, alpha0), torch.where(valid, ub, alpha0)        # padding stays as it is
    finite = torch.isfinite(reftrack).all(dim=2) & torch.isfinite(normvec).all(dim=2) & torch.isfinite(alpha0)
    broken = (~finite & valid).any(dim=1)
    active = (n_pts > 0 if n_pts is not None else torch.ones((B,), dtype=torch.bool, device=dev)) & ~empty & ~broken
    if vehicles is not None:
        if any(x is not None for x in (ggv, ax_max_machines, v_max, drag_coeff, m_veh)):
            raise ValueError("refine_raceline_batch: with vehicles= the ggv, ax_max_machines, v_max, drag_coeff and m_veh "
                             "arguments must be None (each vehicle has its own)")
        vp = dict(vehicles=vehicles, veh_id=veh_id, dyn_model_exp=float(dyn_model_exp), filt_window=filt_window)
    else:
        if any(x is None for x in (ggv, ax_max_machines, v_max, drag_coeff, m_veh)):
            raise TypeError("refine_raceline_batch needs ggv, ax_max_machines, v_max, drag_coeff and m_veh (or vehicles=)")
        vp = dict(ggv=ggv, ax_max_machines=ax_max_machines, v_max=float(v_max), drag_coeff=float(drag_coeff),
                  m_veh=float(m_veh), dyn_model_exp=float(dyn_model_exp), filt_window=filt_window)
    fun = objective if objective is not None else LapTime(reftrack, normvec, n_pts, stepsize_interp, vp)
    x0 = torch.minimum(torch.maximum(alpha0, lb), ub)
    if kappa_bound is None:
        fun.start(x0, active)                   # (with the projection: at the projected start, by fun's first call)
    metric = project = None
    if metric_length is not None:
        metric = CurvatureMetric(reftrack, normvec, n_pts, float(metric_length))
        metric.timer = fun.timer
    if kappa_bound is not None:
        project = CurvatureProjection(reftrack, normvec, n_pts, w_veh, float(kappa_bound), float(metric_length))
        project.timer = fun.timer
    res = spg(fun, x0, lb, ub, active, max_iters=max_iters, pg_tol=pg_tol, memory=memory, gamma=gamma,
              lam_min=lam_min, lam_max=lam_max, max_halvings=max_halvings, callback=callback, metric=metric,
              project=project)
    status = torch.where(empty, EMPTY_BOX, torch.where(broken, NO_GRADIENT, res["status"])).to(torch.int32)
    kept = ~active
    if project is not None:                     # alpha0 could not be projected: it is returned as it is
        kept = kept | ((res["status"] == NO_PROJECTION) & (res["evals"] == 0))
    nan = torch.full_like(res["f"], math.nan)
    out = dict(alpha=torch.where(kept[:, None], alpha0, res["x"]), laptime=torch.where(kept, nan, res["f"]),
               laptime_start=torch.where(kept, nan, res["f0"]), iters=res["iters"], evals=res["evals"], status=status,
               pg_norm=res["pg_norm"])
    if project is not None:
        nan_b = torch.full_like(res["f"], math.nan)
        kl, ce = project.evaluate(res["x"], ~kept)
        out["kappa_lin_max"], out["curv_error_max"] = torch.where(kept, nan_b, kl), torch.where(kept, nan_b, ce)
        out["projection_failures"] = res["projection_failures"]
        if relinearise:
            _rounds(out, fun, reftrack, normvec, n_pts, w_veh, lb, ub, kept, int(relinearise), float(curv_error_allowed),
                    float(kappa_bound), float(metric_length), dict(max_iters=max_iters, pg_tol=pg_tol, memory=memory,
                    gamma=gamma, lam_min=lam_min, lam_max=lam_max, max_halvings=max_halvings, callback=callback))
        else:
            out["rounds"] = torch.zeros_like(out["iters"])
        rl = _b.create_raceline_batch(reftrack, normvec, out["alpha"], stepsize_interp,
                                      n_pts=torch.where(kept, torch.zeros_like(project.n_pts), project.n_pts))
        k = rl["kappa"].abs()
        k = torch.where(torch.arange(k.shape[1], device=dev)[None, :] < rl["n_out"][:, None], k, torch.zeros_like(k))
        out["kappa_max"] = torch.where(kept | (rl["n_out"] <= 0), nan_b, k.amax(dim=1))
    elif metric is not None:
        out["metric_fallbacks"] = res["metric_fallbacks"]
    return out


def _rounds(out, fun, reftrack, normvec, n_pts, w_veh, lb, ub, kept, relinearise, allowed, kb, length, spg_opts):
    """The outer rounds of refine_raceline_batch(relinearise=...), updating out (round 0's result) in place."""
    B = kept.shape[0]
    rounds = torch.zeros((B,), dtype=torch.int32, device=kept.device)
    done = kept | (out["curv_error_max"] <= allowed)
    for r in range(1, relinearise + 1):
        go = ~done
        if not bool(go.any()):                                              # the round's one read
            break
        x0 = out["alpha"].clone()
        project = CurvatureProjection(reftrack, normvec, n_pts, w_veh, kb, length, lin_alpha=x0)
        metric = CurvatureMetric(reftrack, normvec, n_pts, length, lin_alpha=x0)
        project.timer = metric.timer = fun.timer
        res = spg(fun, x0, lb, ub, go, metric=metric, project=project, **spg_opts)
        failed = go & (res["status"] == NO_PROJECTION) & (res["evals"] == 0)
        ok = go & ~failed
        kl, ce = project.evaluate(res["x"], ok)
        out["alpha"] = torch.where(ok[:, None], res["x"], out["alpha"])
        for k, v in (("laptime", res["f"]), ("pg_norm", res["pg_norm"]), ("kappa_lin_max", kl), ("curv_error_max", ce)):
            out[k] = torch.where(ok, v, out[k])
        out["status"] = torch.where(ok, res["status"], torch.where(failed, NO_PROJECTION, out["status"])).to(torch.int32)
        for k in ("iters", "evals", "projection_failures"):
            out[k] = (out[k] + torch.where(go, res[k], torch.zeros_like(res[k]))).to(torch.int32)
        rounds = torch.where(ok, r, rounds).to(torch.int32)
        done |= failed | (ok & (ce <= allowed))
    out["rounds"] = rounds
