"""Float64 numpy reference of create_raceline's stations, heading and curvature and of one re-linearisation step of
tph.iqp_handler (test infrastructure, not product code).  It follows oracle/tph_dense.py statement for statement where the
result depends on the order of the arithmetic, but solves the moment system with a sparse LU
(mincurv_ref.periodic_spline), so it reaches the track sizes where the device switches to the chunked recurrences
(n > 2048) and to global-memory scratch (n_max > 3488), which the oracle's dense 4N x 4N inverse cannot.

spline_lengths   tph.calc_spline_lengths: polylines through 15 equidistant t samples per spline
create_raceline  tph.create_raceline + tph.calc_head_curv_an at the stations (psi, kappa, dkappa)
relinearise      one pass of tph.iqp_handler's loop body: the raceline re-sampled every stepsize metres becomes the new
                 reference line, the widths shifted by alpha are interpolated in t (the last spline toward row 0), and the
                 new normals come from calc_splines without distance scaling
"""
from __future__ import annotations

import math

import numpy as np

from mincurv_ref import periodic_spline
from oracle import tph_dense as T


def spline_lengths(cx, cy):
    """[n] lengths of the polylines through 15 equidistant t samples of every spline (tph.calc_spline_lengths)."""
    t = np.linspace(0.0, 1.0, 15)
    x = cx[:, 0:1] + cx[:, 1:2] * t + cx[:, 2:3] * np.power(t, 2) + cx[:, 3:4] * np.power(t, 3)
    y = cy[:, 0:1] + cy[:, 1:2] * t + cy[:, 2:3] * np.power(t, 2) + cy[:, 3:4] * np.power(t, 3)
    d = np.diff(np.stack((x, y), axis=2), axis=1)
    return np.sum(np.sqrt(np.sum(np.power(d, 2), axis=2)), axis=1)


def create_raceline(refline, normvec, alpha, stepsize):
    """tph.create_raceline of the closed line refline [n, 2] + alpha [n] * normvec [n, 2], re-sampled every ~stepsize
    metres (the closing point dropped), and tph.calc_head_curv_an at the stations.  Returns a dict:
    coeffs_x, coeffs_y [n, 4], spline_lengths, cum (np.cumsum of the lengths) [n], total (= cum[-1]), no (stations),
    raceline [no, 2], spline_inds, t, s, el [no] (el[-1] closes the loop), psi, kappa, dkappa [no]."""
    P = np.asarray(refline, float)[:, :2] + np.asarray(alpha, float)[:, None] * np.asarray(normvec, float)
    cx, cy, _ = periodic_spline(np.vstack((P, P[0])), use_dist_scaling=False)
    sl = spline_lengths(cx, cy)
    cum = np.cumsum(sl)
    total = cum[-1]
    n_interp = math.ceil(total / stepsize) + 1
    s = np.linspace(0.0, total, n_interp)[:-1]
    inds = np.searchsorted(cum, s, side="right")                 # np.argmax(s_i < cum): the first j with s_i < cum[j]
    t = np.where(inds > 0, s - cum[np.maximum(inds - 1, 0)], s) / sl[inds]
    a, c = cx[inds], cy[inds]
    xy = np.column_stack((a[:, 0] + a[:, 1] * t + a[:, 2] * np.power(t, 2) + a[:, 3] * np.power(t, 3),
                          c[:, 0] + c[:, 1] * t + c[:, 2] * np.power(t, 2) + c[:, 3] * np.power(t, 3)))
    el = np.append(np.diff(s), float(np.sum(sl)) - s[-1])
    psi, kappa, dkappa = T.calc_head_curv_an(cx, cy, inds, t, calc_curv=True, calc_dcurv=True)
    return dict(coeffs_x=cx, coeffs_y=cy, spline_lengths=sl, cum=cum, total=total, no=n_interp - 1, raceline=xy,
                spline_inds=inds, t=t, s=s, el=el, psi=psi, kappa=kappa, dkappa=dkappa)


def interp_widths(w, inds, t):
    """tph.interp_track_widths (incl_last_point=False): w [n, 2] interpolated linearly in t between rows j and j + 1 of
    every station's spline j, the last spline toward row 0."""
    w_cl = np.vstack((w, w[0]))
    w0, w1 = w_cl[inds], w_cl[inds + 1]
    return w0 + (w1 - w0) * t[:, None]                           # np.interp(t, (0, 1), (w0, w1))


def relinearise(reftrack, normvec, alpha, stepsize):
    """One re-linearisation of tph.iqp_handler: dict(reftrack [m, 4], normvec [m, 2], n (= m), raceline (the dict of
    create_raceline))."""
    reftrack = np.asarray(reftrack, float)
    alpha = np.asarray(alpha, float)
    rl = create_raceline(reftrack[:, :2], normvec, alpha, stepsize)
    w = np.column_stack((reftrack[:, 2] - alpha, reftrack[:, 3] + alpha))
    rt = np.column_stack((rl["raceline"], interp_widths(w, rl["spline_inds"], rl["t"])))
    _, _, nv = periodic_spline(np.vstack((rt[:, :2], rt[0, :2])), use_dist_scaling=False)
    return dict(reftrack=rt, normvec=nv, n=rt.shape[0], raceline=rl)
