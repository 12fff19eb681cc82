"""CPU oracle of the width sensitivities of the minimum-curvature QP with its curvature rows (test infrastructure, not
product code).

    min 1/2 a^T H a + f^T a   s.t.  lb <= a <= ub,   -kappa_bound <= k_ref + E a <= kappa_bound
    ub = w_right - w_veh / 2,  lb = -w_left + w_veh / 2

H, f, E and k_ref come from the dense oracle (oracle/tph_dense.py), the solution from its Goldfarb-Idnani solver.  For
the active set A (the bounds and rows the solution sits on) the exact vector-Jacobian product of L = gbar^T a follows
from the KKT system of the equality-constrained QP on A:
    [H  C_A^T] [p]   [gbar]
    [C_A    0] [q] = [  0 ],      dL/db_A = q,  dL/db = 0 for the inactive constraints,
with C_A the rows +e_i (a_i <= ub_i), -e_i (-a_i <= -lb_i), +E_i (k_ref_i + E_i a <= kappa_bound) and -E_i.  The rows
do not depend on the widths: only the box entries of q reach them, as in qp_sens.width_vjp.
"""
from __future__ import annotations

import numpy as np

import qp_sens as Q
from oracle import quadprog_gi, tph_dense as T


def qp_data(reftrack, normvec, kappa_bound, w_veh) -> dict:
    """dict(H, f, E, k_ref) of one track from the dense oracle (numpy [n, 4] and [n, 2]: the normals the caller uses)."""
    rt = np.asarray(reftrack, dtype=np.float64)
    _, _, A, _ = T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))
    qp = T.assemble_min_curv(rt, normvec, A, kappa_bound, w_veh)
    return dict(H=qp["H"], f=qp["f"], E=qp["E_kappa"], k_ref=qp["k_kappa_ref"])


def _constraints(d, lb, ub, kappa_bound):
    """G a <= h: the upper bounds, the lower bounds, the upper and the lower curvature rows."""
    n = lb.size
    G = np.vstack((np.eye(n), -np.eye(n), d["E"], -d["E"]))
    h = np.concatenate((ub, -lb, kappa_bound - d["k_ref"], kappa_bound + d["k_ref"]))
    return G, h


def solve(d, lb, ub, kappa_bound):
    """(alpha, multipliers [4 n] in the order of _constraints) of the oracle's Goldfarb-Idnani solve."""
    G, h = _constraints(d, lb, ub, kappa_bound)
    out = quadprog_gi.solve_qp(d["H"], -d["f"], -G.T, -h)
    return out[0], out[4][:G.shape[0]]


def width_vjp_rows(d, reftrack, w_veh, kappa_bound, gbar, tol=1e-8) -> dict:
    """dL/dw_right [n], dL/dw_left [n], dL/dw_veh of L = gbar^T alpha, with the solution, the active masks (at_ub, at_lb,
    row_hi, row_lo), the multipliers of the box (lu, ll) and of the rows (l3, l4) and the slacks of the rows."""
    lb, ub, collapsed = Q.bounds(np.asarray(reftrack), w_veh)
    n = lb.size
    alpha, lam = solve(d, lb, ub, kappa_bound)
    G, h = _constraints(d, lb, ub, kappa_bound)
    slack = h - G @ alpha
    act = slack <= tol
    act[n:2 * n] &= ~act[:n]                    # (a collapsed box sits on both of its bounds: one of them is kept)
    C = G[act]
    K = np.block([[d["H"], C.T], [C, np.zeros((C.shape[0], C.shape[0]))]])
    q = np.zeros(4 * n)
    q[act] = np.linalg.solve(K, np.concatenate((gbar, np.zeros(C.shape[0]))))[n:]
    g_ub, g_lb = q[:n], -q[n:2 * n]
    half = 0.5 * (g_ub + g_lb)
    return dict(grad_w_right=np.where(collapsed, half, g_ub), grad_w_left=np.where(collapsed, -half, -g_lb),
                grad_w_veh=float(0.5 * np.sum(np.where(collapsed, 0.0, g_lb - g_ub))), alpha=alpha, lb=lb, ub=ub,
                at_ub=act[:n], at_lb=act[n:2 * n], row_hi=act[2 * n:3 * n], row_lo=act[3 * n:],
                lu=lam[:n], ll=lam[n:2 * n], l3=lam[2 * n:3 * n], l4=lam[3 * n:], row_slack=np.minimum(slack[2 * n:3 * n],
                                                                                                      slack[3 * n:]))


def degenerate(ref, scale):
    """Points where the derivative does not exist or is ill-conditioned at an interior-point solver's tolerance (the
    criterion of DESIGN.md section 3.10, extended to the rows): a bound or row active with a multiplier below 1e-6 scale,
    or inactive with a slack below 1e-6 (m for a bound, 1/m for a row)."""
    a = ref["alpha"]
    box_weak = (ref["at_ub"] & (ref["lu"] < 1e-6 * scale)) | (ref["at_lb"] & (ref["ll"] < 1e-6 * scale))
    box_near = ~(ref["at_ub"] | ref["at_lb"]) & (np.minimum(ref["ub"] - a, a - ref["lb"]) < 1e-6)
    row_weak = (ref["row_hi"] & (ref["l3"] < 1e-6 * scale)) | (ref["row_lo"] & (ref["l4"] < 1e-6 * scale))
    row_near = ~(ref["row_hi"] | ref["row_lo"]) & (ref["row_slack"] < 1e-6)
    return box_weak | box_near | row_weak | row_near
