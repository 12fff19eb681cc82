"""CPU oracle of the sensitivities of the shortest-path QP (test infrastructure, not product code).

    min 1/2 a^T H a + f^T a   s.t.  lb <= a <= ub
    H_ii = 4 |n_i|^2,  H_i,i+1 = H_i+1,i = -2 n_i.n_{i+1},  f_i = 2 n_i.(2 p_i - p_{i+1} - p_{i-1})   (cyclic)
    ub = max(w_right - w_veh / 2, 0.001),  lb = -max(w_left - w_veh / 2, 0.001)

(oracle.tph_dense.assemble_shortest_path).  For a solution with the active set A (the bounds it sits on), the exact
vector-Jacobian product of L = gbar^T a follows from the KKT system of the equality-constrained QP on A:
    [H  C_A^T] [p]   [gbar]
    [C_A    0] [q] = [  0 ],
with C_A the rows +e_i (a_i <= ub_i) and -e_i (-a_i <= -lb_i): dL/df = -p, dL/dH_ij = -p_i a_j, dL/dub_A = q,
dL/dlb_A = -q, zero for the inactive bounds.  The chain rule through H and f gives the centre line (at fixed normals) and
the normals; a bound clamped to 0.001 does not depend on the widths, so its width gradients are zero.
"""
from __future__ import annotations

import numpy as np

import qp_sens as Q

CLAMP = 0.001           # tph's lower limit of w - w_veh / 2 (csrc/shortest_path.cu)


def solve(reftrack, normvec, w_veh):
    """The shortest-path QP's alpha by the oracle's Goldfarb-Idnani solver (exact active set)."""
    from oracle import tph_dense as T
    from oracle.quadprog_gi import solve_qp
    qp = T.assemble_shortest_path(reftrack, normvec, w_veh)
    return solve_qp(qp["H"], -qp["f"], -qp["G"].T, -qp["h"], 0)[0]


def vjp(reftrack, normvec, w_veh, gbar, alpha=None, tol=1e-8) -> dict:
    """grad_reftrack [n, 4] (x, y, w_right, w_left), grad_normvec [n, 2] and grad_w_veh of L = gbar^T alpha.  alpha: the
    oracle's solution (solved here if None).  Also returns the bounds, the active masks, the multipliers and the clamp
    masks (for the degenerate-point criterion of the callers)."""
    from oracle import tph_dense as T
    qp = T.assemble_shortest_path(reftrack, normvec, w_veh)
    H, f = qp["H"], qp["f"]
    a = solve(reftrack, normvec, w_veh) if alpha is None else np.asarray(alpha, dtype=float)
    n = a.size
    dr, dl = reftrack[:, 2] - 0.5 * w_veh, reftrack[:, 3] - 0.5 * w_veh
    clamped_r, clamped_l = dr < CLAMP, dl < CLAMP
    ub, lb = np.where(clamped_r, CLAMP, dr), -np.where(clamped_l, CLAMP, dl)
    at_ub, at_lb, lu, ll = Q.active_set(H, f, a, lb, ub, tol)
    act = np.flatnonzero(at_ub | at_lb)
    C = np.zeros((act.size, n))
    C[np.arange(act.size), act] = np.where(at_ub[act], 1.0, -1.0)
    K = np.block([[H, C.T], [C, np.zeros((act.size, act.size))]])
    sol = np.linalg.solve(K, np.concatenate((gbar, np.zeros(act.size))))
    p, q = sol[:n], sol[n:]
    g_ub, g_lb = np.zeros(n), np.zeros(n)
    g_ub[act] = np.where(at_ub[act], q, 0.0)
    g_lb[act] = np.where(at_lb[act], -q, 0.0)
    P, N = reftrack[:, :2], normvec
    ip, im = np.roll(np.arange(n), -1), np.roll(np.arange(n), 1)
    gf = -p
    gd = -p * a                                  # dL/dH_ii
    go = -(p * a[ip] + p[ip] * a)                # dL/dH_i,i+1, both symmetric entries
    g_xy = 4.0 * N * gf[:, None] - 2.0 * N[im] * gf[im, None] - 2.0 * N[ip] * gf[ip, None]
    g_nv = (8.0 * N * gd[:, None] - 2.0 * N[ip] * go[:, None] - 2.0 * N[im] * go[im, None]
            + 2.0 * (2.0 * P - P[ip] - P[im]) * gf[:, None])
    g_wr = np.where(clamped_r, 0.0, g_ub)
    g_wl = np.where(clamped_l, 0.0, -g_lb)
    g_wv = float(0.5 * np.sum(np.where(clamped_l, 0.0, g_lb) - np.where(clamped_r, 0.0, g_ub)))
    return dict(grad_reftrack=np.column_stack((g_xy, g_wr, g_wl)), grad_normvec=g_nv, grad_w_veh=g_wv, alpha=a, f=f, lb=lb,
                ub=ub, at_ub=at_ub, at_lb=at_lb, lu=lu, ll=ll, clamped_r=clamped_r, clamped_l=clamped_l)


def degenerate(ref, scale):
    """Points where the derivative does not exist or is ill-conditioned at a solver's tolerance: a bound active with a
    multiplier below 1e-6 scale, or inactive with a slack below 1e-6 m."""
    weak = (ref["at_ub"] & (ref["lu"] < 1e-6 * scale)) | (ref["at_lb"] & (ref["ll"] < 1e-6 * scale))
    a = ref["alpha"]
    near = ~(ref["at_ub"] | ref["at_lb"]) & (np.minimum(ref["ub"] - a, a - ref["lb"]) < 1e-6)
    return weak | near
