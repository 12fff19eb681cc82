"""Converged float64 reference of the prep_track kernel (csrc/prep_track.cu, DESIGN.md section 3.9): test infrastructure,
not product code.

oracle/tph_prep.py states the same algorithm densely (an O(n^3) solve per smoothing parameter, a bounded scalar search
for the closest points).  This module takes each step to convergence instead, so that the kernel can be held to what
float64 allows:

* fit(sys, lam)     the periodic cubic smoothing spline at a given lam: (R + lam Q^T Q) gamma = Q^T p by a sparse LU
                    (scipy splu), f = p - lam Q gamma, F(lam) = |lam Q gamma|^2 (x and y together);
* root(sys, s)      lam with F(lam) = s by bisection on log lam down to adjacent doubles, and F(inf) = sum |p - mean p|^2
                    (the residual of the best constant, which a budget must stay below);
* closest(...)      the closest curve point of a raw point: a dense scan of the kernel's window (+-4 pre-interpolation
                    steps around the chord-length guess), then Newton until its step is zero in float64, with the
                    stationarity residual |(f(t) - q) . f'(t)| / |f'(t)| in metres;
* outputs(...)      arc length from ceil(L_raw) * 4 samples, re-sampled points, sides, widths (numpy.interp) and the
                    min-width inflation, all at a given lam (so that a test can evaluate the curve at the kernel's lam).
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import scipy.sparse as sps
from scipy.sparse.linalg import splu

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.tph_prep import _interp_track_cl, eval_periodic_cubic  # noqa: E402


def system(track, stepsize_prep=1.0):
    """Pre-interpolation and the sparse matrices of the smoothing problem for a raw track [nr, 4] (unclosed)."""
    track = np.asarray(track, dtype=float)
    ti, dists_cl = _interp_track_cl(track, stepsize_prep)
    pts = ti[:-1, :2]
    ch = np.sqrt(np.sum(np.diff(ti[:, :2], axis=0) ** 2, axis=1))
    ucl = np.insert(np.cumsum(ch), 0, 0.0)
    u = ucl[:-1] / ucl[-1]
    n = u.size
    h = np.diff(np.append(u, 1.0))
    i = np.arange(n)
    im, ip = (i - 1) % n, (i + 1) % n
    # (Q^T y)_i = (y_ip - y_i) / h_i - (y_i - y_im) / h_im; Q[r, c]: column c is node c's stencil
    Q = sps.csc_matrix((np.concatenate((1.0 / h, -1.0 / h - 1.0 / h[im], 1.0 / h[im])),
                        (np.concatenate((ip, i, im)), np.concatenate((i, i, i)))), shape=(n, n))
    R = sps.csc_matrix((np.concatenate(((h[im] + h) / 3.0, h / 6.0, h / 6.0)),
                        (np.concatenate((i, i, ip)), np.concatenate((i, ip, i)))), shape=(n, n))
    return SimpleNamespace(track=track, stepsize_prep=float(stepsize_prep), pts=pts, u=u, n=n, Q=Q, R=R,
                           QtQ=(Q.T @ Q).tocsc(), Qtp=Q.T @ pts, L_raw=float(dists_cl[-1]), dists_cl=dists_cl,
                           F_inf=float(np.sum((pts - pts.mean(axis=0)) ** 2)))


def fit(sys_, lam):
    """(f [n, 2], gamma [n, 2], F) of the smoothing spline at lam."""
    gam = splu((sys_.R + lam * sys_.QtQ).tocsc()).solve(np.ascontiguousarray(sys_.Qtp))
    r = lam * (sys_.Q @ gam)
    return sys_.pts - r, gam, float(np.sum(r * r))


def F(sys_, lam):
    return fit(sys_, lam)[2]


def root(sys_, s):
    """lam with F(lam) = s (F increases from 0 to F(inf)); bisection on log lam until the bracket holds adjacent doubles."""
    if not s < sys_.F_inf:
        raise ValueError(f"s = {s} is not below F(inf) = {sys_.F_inf}")
    lo, hi = 1.0, 1.0
    while F(sys_, hi) < s:
        hi *= 16.0
    while F(sys_, lo) >= s:
        lo /= 16.0
    while True:
        mid = float(np.sqrt(lo) * np.sqrt(hi))
        if not lo < mid < hi:
            break
        if F(sys_, mid) < s:
            lo = mid
        else:
            hi = mid
    return lo if s - F(sys_, lo) <= F(sys_, hi) - s else hi


def eval3(u, f, gam, t):
    """Value, first and second derivative of the periodic cubic spline (period 1) at t (any real: taken mod 1)."""
    t = np.asarray(t, dtype=float) % 1.0
    n = u.size
    ue = np.append(u, 1.0)
    j = np.clip(np.searchsorted(ue, t, side="right") - 1, 0, n - 1)
    jp = (j + 1) % n
    h = (ue[j + 1] - ue[j])[:, None]
    a, b = (ue[j + 1][:, None] - t[:, None]) / h, (t[:, None] - ue[j][:, None]) / h
    x = a * f[j] + b * f[jp] + (a ** 3 - a) * h * h / 6.0 * gam[j] + (b ** 3 - b) * h * h / 6.0 * gam[jp]
    dx = (f[jp] - f[j]) / h - (3.0 * a * a - 1.0) * h / 6.0 * gam[j] + (3.0 * b * b - 1.0) * h / 6.0 * gam[jp]
    ddx = a * gam[j] + b * gam[jp]
    return x, dx, ddx


def closest(u, f, gam, q, t0, span, n_scan=513):
    """Closest curve point of q in the window t0 +- span: dense scan, then Newton to a zero step.
    Returns (t, distance, point, stationarity residual [m])."""
    ts = t0 + np.linspace(-span, span, n_scan)
    x, _, _ = eval3(u, f, gam, ts)
    t = float(ts[int(np.argmin(np.sum((x - q) ** 2, axis=1)))])
    for _ in range(100):
        x, dx, ddx = (v[0] for v in eval3(u, f, gam, [t]))
        g, hs = float((x - q) @ dx), float(dx @ dx + (x - q) @ ddx)
        tn = t - g / hs
        if tn == t:
            break
        t = tn
    x, dx, _ = (v[0] for v in eval3(u, f, gam, [t]))
    return t, float(np.linalg.norm(x - q)), x, abs(float((x - q) @ dx)) / float(np.linalg.norm(dx))


def outputs(sys_, lam, stepsize_reg=3.0, min_width=None):
    """Every output of the kernel for the curve at lam: reftrack_interp [n_reg, 4] and the closest-point data."""
    f, gam, Fv = fit(sys_, lam)
    u, tr = sys_.u, sys_.track
    n_len = int(np.ceil(sys_.L_raw)) * 4
    tmp = eval_periodic_cubic(u, 1.0, f, gam, np.linspace(0.0, 1.0, n_len))
    length = float(np.sum(np.sqrt(np.sum(np.diff(tmp, axis=0) ** 2, axis=1))))
    n_reg_cl = int(np.ceil(length / stepsize_reg)) + 1
    tq = np.linspace(0.0, 1.0, n_reg_cl)
    path = eval3(u, f, gam, tq[:-1])[0]
    tr_cl = np.vstack((tr, tr[0]))
    n_cl = tr_cl.shape[0]
    span = 4.0 * sys_.stepsize_prep / sys_.L_raw
    t_c, d_c, p_c, res = np.zeros(n_cl), np.zeros(n_cl), np.zeros((n_cl, 2)), np.zeros(n_cl)
    for i in range(n_cl):
        t_c[i], d_c[i], p_c[i], res[i] = closest(u, f, gam, tr_cl[i, :2], sys_.dists_cl[i] / sys_.L_raw, span)
    t_w = t_c.copy()
    t_w[0], t_w[-1] = 0.0, 1.0
    e = tr_cl[1:, :2] - tr_cl[:-1, :2]
    sides = np.sign(e[:, 0] * (p_c[:-1, 1] - tr_cl[:-1, 1]) - e[:, 1] * (p_c[:-1, 0] - tr_cl[:-1, 0]))
    sides_cl = np.append(sides, sides[0])
    w_r = tr_cl[:, 2] + sides_cl * d_c
    w_l = tr_cl[:, 3] - sides_cl * d_c
    out = np.column_stack((path, np.interp(tq, t_w, w_r)[:-1], np.interp(tq, t_w, w_l)[:-1]))
    if min_width is not None and min_width > 0.0:
        cur = out[:, 2] + out[:, 3]
        add = np.where(cur < min_width, 0.5 * (min_width - cur), 0.0)
        out[:, 2] += add
        out[:, 3] += add
    return SimpleNamespace(out=out, F=Fv, f=f, gam=gam, length=length, n_reg=n_reg_cl - 1, t_close=t_c, d_close=d_c,
                           p_close=p_c, resid=res, sides=sides_cl)


def spline_approximation(track, s_reg=10.0, stepsize_prep=1.0, stepsize_reg=3.0, min_width=None):
    """The whole stage at the converged root: (outputs, lam, system)."""
    sys_ = system(track, stepsize_prep)
    lam = root(sys_, float(s_reg))
    return outputs(sys_, lam, stepsize_reg, min_width), lam, sys_
