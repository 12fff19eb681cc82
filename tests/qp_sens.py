"""CPU oracle of the width sensitivities of the box-only min-curvature QP (test infrastructure, not product code).

    min 1/2 a^T H a + f^T a   s.t.  lb <= a <= ub,   ub = w_right - w_veh / 2,  lb = -w_left + w_veh / 2

For a solved instance with the active set A (the bounds the solution sits on), the exact vector-Jacobian product of
L = gbar^T a follows from the KKT system of the equality-constrained QP on A:
    [H  C_A^T] [p]   [gbar]
    [C_A    0] [q] = [  0 ],      dL/db_A = q,  dL/db = 0 for the inactive bounds,
with C_A the rows +e_i (a_i <= ub_i, b = ub) and -e_i (-a_i <= -lb_i, b = -lb).  Widths as in the device kernel
(mincurv_ipm.cu K2d): dL/dw_right = dL/dub, dL/dw_left = -dL/dlb, dL/dw_veh = 1/2 sum (dL/dlb - dL/dub); a collapsed
box (ub - lb < 2 FIX_EPS, replaced by mid -+ FIX_EPS as the device setup does) follows mid = (w_right - w_left) / 2.
"""
from __future__ import annotations

import numpy as np

FIX_EPS = 1e-8          # csrc/common.cuh


def dense_from_band(H_band: np.ndarray) -> np.ndarray:
    """Symmetric cyclic H from its band rows H_band[i][k] = H[i][(i + k) % n], k = 0..32 (the fixtures' H_band)."""
    n, w = H_band.shape
    H = np.zeros((n, n))
    i = np.arange(n)
    for k in range(w):
        H[i, (i + k) % n] = H_band[:, k]
        H[(i + k) % n, i] = H_band[:, k]
    return H


def bounds(reftrack: np.ndarray, w_veh) -> tuple:
    """(lb, ub, collapsed) of the device setup (mincurv_setup.cu P1), collapsed boxes replaced by mid -+ FIX_EPS."""
    ub = reftrack[:, 2] - 0.5 * w_veh
    lb = -(reftrack[:, 3] - 0.5 * w_veh)
    collapsed = ub - lb < 2.0 * FIX_EPS
    mid = 0.5 * (lb + ub)
    return np.where(collapsed, mid - FIX_EPS, lb), np.where(collapsed, mid + FIX_EPS, ub), collapsed


def solve_box_qp(H: np.ndarray, f: np.ndarray, lb: np.ndarray, ub: np.ndarray) -> np.ndarray:
    """The box-only QP by the oracle's Goldfarb-Idnani solver (exact active set)."""
    from oracle.quadprog_gi import solve_qp
    n = H.shape[0]
    C = np.hstack((-np.eye(n), np.eye(n)))          # quadprog: C^T a >= b
    return solve_qp(H, -f, C, np.concatenate((-ub, lb)), 0)[0]


def active_set(H, f, alpha, lb, ub, tol=1e-8):
    """Upper / lower active masks of a solution and the multipliers of the active bounds (lu = -grad, ll = grad)."""
    grad = H @ alpha + f
    at_ub = alpha >= ub - tol
    at_lb = (alpha <= lb + tol) & ~at_ub
    return at_ub, at_lb, np.where(at_ub, -grad, 0.0), np.where(at_lb, grad, 0.0)


def bound_vjp(H, at_ub, at_lb, gbar):
    """(dL/dub, dL/dlb) from the KKT system of the active set."""
    n = H.shape[0]
    act = np.flatnonzero(at_ub | at_lb)
    C = np.zeros((act.size, n))
    C[np.arange(act.size), act] = np.where(at_ub[act], 1.0, -1.0)
    K = np.block([[H, C.T], [C, np.zeros((act.size, act.size))]])
    q = np.linalg.solve(K, np.concatenate((gbar, np.zeros(act.size))))[n:]
    g_ub, g_lb = np.zeros(n), np.zeros(n)
    g_ub[act] = np.where(at_ub[act], q, 0.0)
    g_lb[act] = np.where(at_lb[act], -q, 0.0)
    return g_ub, g_lb


def width_vjp(H, f, reftrack, w_veh, gbar, alpha=None, tol=1e-8) -> dict:
    """dL/dw_right [n], dL/dw_left [n], dL/dw_veh of L = gbar^T alpha.  alpha: the oracle's solution (solved here if None).
    Also returns the active masks and multipliers (for the degenerate-point criterion of the callers)."""
    lb, ub, collapsed = bounds(reftrack, w_veh)
    if alpha is None:
        alpha = solve_box_qp(H, f, lb, ub)
    at_ub, at_lb, lu, ll = active_set(H, f, alpha, lb, ub, tol)
    g_ub, g_lb = bound_vjp(H, at_ub, at_lb, gbar)
    half = 0.5 * (g_ub + g_lb)
    return dict(grad_w_right=np.where(collapsed, half, g_ub), grad_w_left=np.where(collapsed, -half, -g_lb),
                grad_w_veh=float(0.5 * np.sum(np.where(collapsed, 0.0, g_lb - g_ub))), alpha=alpha, lb=lb, ub=ub,
                at_ub=at_ub, at_lb=at_lb, lu=lu, ll=ll, collapsed=collapsed)
