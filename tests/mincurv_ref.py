"""CPU references for the edge tests of the minimum-curvature path (test infrastructure, not product code).

kkt_certificate   first-order optimality of a point of the full QP of tph.opt_min_curv (oracle/tph_dense.assemble_min_curv),
                  with or without the curvature rows:
                      min 1/2 a^T H a + f^T a   s.t.  lb <= a <= ub,   -kb <= k_ref + E a <= kb
                  The multipliers are recovered from the point alone (non-negative least squares on the near-active
                  constraints), so the certificate does not depend on how the point was found.
periodic_spline   the closed cubic spline of tph.calc_splines from a direct sparse solve of the periodic tridiagonal moment
                  system -- no parallel cyclic reduction, no warm-up recurrences, and cheap at thousands of points, where
                  the oracle's dense 4N x 4N solve is not.
uneven_track      closed test tracks whose point spacing alternates between two steps (ratio 1 : r).
"""
from __future__ import annotations

import numpy as np
import scipy.optimize
import scipy.sparse
import scipy.sparse.linalg


def kkt_certificate(H, f, E, k_ref, lb, ub, kb, alpha, rows=True, act_box=1e-6, act_row=1e-6):
    """Optimality numbers of alpha for the QP above (rows=False: the box-only QP).  Returns a dict:
    box_viol   max violation of the box [m];   row_viol  max(|k_ref + E a| - kb, 0) [1/m] (0 without rows)
    stat       |H a + f + C^T lam|_inf / |f|_inf, lam >= 0 fitted by NNLS on the near-active constraints
               (box slack <= act_box m, row slack <= act_row * kb)
    comp       max lam_i slack_i / (|f|_inf max(ub - lb)) over those constraints
    n_active   number of near-active constraints;  lam_max  largest multiplier / |f|_inf.  Nothing is asserted."""
    H, f, alpha = np.asarray(H, float), np.asarray(f, float), np.asarray(alpha, float)
    lb, ub = np.asarray(lb, float), np.asarray(ub, float)
    n = alpha.size
    g = H @ alpha + f
    cols, slack = [], []
    s_ub, s_lb = ub - alpha, alpha - lb
    eye = np.eye(n)
    for i in np.flatnonzero(s_ub <= act_box):
        cols.append(eye[i]); slack.append(max(s_ub[i], 0.0))
    for i in np.flatnonzero(s_lb <= act_box):
        cols.append(-eye[i]); slack.append(max(s_lb[i], 0.0))
    row_viol = 0.0
    if rows:
        E = np.asarray(E, float)
        k = np.asarray(k_ref, float) + E @ alpha
        s_hi, s_lo = kb - k, kb + k
        row_viol = float(max(0.0, -s_hi.min(), -s_lo.min()))
        for i in np.flatnonzero(s_hi <= act_row * kb):
            cols.append(E[i]); slack.append(max(s_hi[i], 0.0))
        for i in np.flatnonzero(s_lo <= act_row * kb):
            cols.append(-E[i]); slack.append(max(s_lo[i], 0.0))
    scale = np.abs(f).max()
    if cols:
        C = np.array(cols).T
        lam, _ = scipy.optimize.nnls(C, -g, maxiter=50 * C.shape[1])
        r = g + C @ lam
        comp = float((lam * np.array(slack)).max() / (scale * (ub - lb).max()))
    else:
        lam, r, comp = np.zeros(0), g, 0.0
    return dict(box_viol=float(max(0.0, (lb - alpha).max(), (alpha - ub).max())), row_viol=row_viol,
                stat=float(np.abs(r).max() / scale), comp=comp, n_active=len(cols),
                lam_max=float(lam.max() / scale) if lam.size else 0.0)


def periodic_spline(path, use_dist_scaling=True, el_lengths=None):
    """(coeffs_x [n, 4], coeffs_y [n, 4], normvec [n, 2]) of tph.calc_splines for a closed path [n + 1, 2] (last point =
    first).  Spline i runs over t in [0, 1] with parameter scale h_i (its chord length with use_dist_scaling, given by
    el_lengths [n] if not None, 1 otherwise); the moments m = d^2 p / ds^2 at the knots solve
        h_{i-1} m_{i-1} + 2 (h_{i-1} + h_i) m_i + h_i m_{i+1} = 6 ((p_{i+1} - p_i) / h_i - (p_i - p_{i-1}) / h_{i-1})  (cyclic)
    by a sparse LU factorisation."""
    p = np.asarray(path, float)[:-1, :2]
    n = p.shape[0]
    if el_lengths is not None:
        h = np.asarray(el_lengths, float)
    elif use_dist_scaling:
        h = np.linalg.norm(np.roll(p, -1, axis=0) - p, axis=1)
    else:
        h = np.ones(n)
    hm = np.roll(h, 1)
    i = np.arange(n)
    A = scipy.sparse.coo_matrix((np.concatenate((2.0 * (hm + h), hm, h)),
                                 (np.concatenate((i, i, i)), np.concatenate((i, (i - 1) % n, (i + 1) % n)))),
                                shape=(n, n)).tocsc()
    dp = np.roll(p, -1, axis=0) - p
    rhs = 6.0 * (dp / h[:, None] - np.roll(dp, 1, axis=0) / hm[:, None])
    m = scipy.sparse.linalg.splu(A).solve(rhs)
    mp = np.roll(m, -1, axis=0)
    h2 = (h * h)[:, None]
    a1 = dp - h2 * (2.0 * m + mp) / 6.0
    coeffs = [np.column_stack((p[:, c], a1[:, c], 0.5 * h2[:, 0] * m[:, c], h2[:, 0] * (mp[:, c] - m[:, c]) / 6.0))
              for c in range(2)]
    nv = np.column_stack((a1[:, 1], -a1[:, 0]))
    return coeffs[0], coeffs[1], nv / np.linalg.norm(nv, axis=1)[:, None]


def uneven_track(n, ratio, seed=0, step=3.0, run=12):
    """Closed track [n, 4] (x, y, w_right, w_left) on a smooth star-shaped curve whose point spacing alternates between
    runs of `run` short steps and `run` steps `ratio` times as long (measured ratio within a few % of `ratio`)."""
    rng = np.random.default_rng(seed)
    d = np.where((np.arange(n) // run) % 2 == 0, 1.0, float(ratio))
    th = np.concatenate(([0.0], np.cumsum(d)[:-1])) / d.sum() * 2.0 * np.pi
    R = d.sum() * step / (2.0 * np.pi)
    a, k, ph = rng.uniform(0.03, 0.06), int(rng.integers(2, 4)), rng.uniform(0, 2 * np.pi)
    r = R * (1.0 + a * np.cos(k * th + ph))
    w = 3.0 + 1.5 * np.cos(th + rng.uniform(0, 2 * np.pi))
    return np.column_stack((r * np.cos(th), r * np.sin(th), w, w[::-1]))
