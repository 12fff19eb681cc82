"""Dense float64 reference of the minimum-curvature QP's curvature linearised about a line (DESIGN.md section 3.2): the
closed h-spline of mincurv_setup.cu (moments M = Tri^-1 6 D2 p, Tri cyclic tridiagonal with diagonal 2 (h_{i-1} + h_i)
and off-diagonal h_i), its knot curvature, and tph's linearisation k_ref + E alpha about the line P + a n."""
import numpy as np


def _tri(h):
    n = h.shape[0]
    T = np.zeros((n, n))
    for i in range(n):
        T[i, i] = 2.0 * (h[i - 1] + h[i])
        T[i, (i + 1) % n] += h[i]
        T[(i + 1) % n, i] += h[i]
    return T


def _d2(h):
    """6 D2: (6 D2 p)_i = 6 ((p_{i+1} - p_i) / h_i - (p_i - p_{i-1}) / h_{i-1})."""
    n = h.shape[0]
    D = np.zeros((n, n))
    for i in range(n):
        D[i, (i + 1) % n] += 6.0 / h[i]
        D[i, i] -= 6.0 / h[i] + 6.0 / h[i - 1]
        D[i, i - 1] += 6.0 / h[i - 1]
    return D


def derivatives(p, h):
    """(x', y', x'', y'') at the knots of the closed h-spline through p [n, 2] (per unit of the local parameter)."""
    Z = np.linalg.solve(_tri(h), _d2(h))
    m = Z @ p
    h2 = (h * h)[:, None]
    d1 = (np.roll(p, -1, axis=0) - p) - h2 * (2.0 * m + np.roll(m, -1, axis=0)) / 6.0
    return d1[:, 0], d1[:, 1], h2[:, 0] * m[:, 0], h2[:, 0] * m[:, 1]


def knot_curvature(p, h):
    xp, yp, xpp, ypp = derivatives(p, h)
    return (xp * ypp - yp * xpp) / (xp * xp + yp * yp) ** 1.5


def linearised_curvature(p, nvec, h, a, alpha):
    """k_ref + E alpha about the line p + a n: the first derivatives of that line, the second derivatives of
    p + alpha n (k_ref keeps p's moments, E alpha adds those of alpha n)."""
    xp, yp, _, _ = derivatives(p + a[:, None] * nvec, h)
    _, _, xpp, ypp = derivatives(p + alpha[:, None] * nvec, h)
    return (xp * ypp - yp * xpp) / (xp * xp + yp * yp) ** 1.5


def dense_qp_about(reftrack, normvec, a, kappa_bound, w_veh):
    """The dense QP of oracle/tph_dense.assemble_min_curv linearised about the line P + a n: its algebra with the first
    derivatives x' = T_b (q + M a) in place of T_b q (a None: the oracle's assembly as it is).  dict(H, f, E, k_ref, G, h)
    as the oracle's (min 1/2 a^T H a + f^T a, G a <= h)."""
    from oracle import tph_dense as T
    rt = np.asarray(reftrack, dtype=np.float64)
    _, _, A, _ = T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))
    qp = T.assemble_min_curv(rt, normvec, A, kappa_bound, w_veh)
    if a is None:
        return dict(H=qp["H"], f=qp["f"], E=qp["E_kappa"], k_ref=qp["k_kappa_ref"], G=qp["G"], h=qp["h"])
    a = np.asarray(a, dtype=np.float64)[:, None]
    xp = np.squeeze(qp["T_b"] @ (qp["q_x"] + qp["M_x"] @ a))
    yp = np.squeeze(qp["T_b"] @ (qp["q_y"] + qp["M_y"] @ a))
    c = 1.0 / np.power(xp ** 2 + yp ** 2, 1.5)
    c2 = c ** 2
    Pxx, Pyy, Pxy = np.diag(c2 * yp ** 2), np.diag(c2 * xp ** 2), np.diag(c2 * (-2.0 * xp * yp))
    Tnx, Tny, Tc = qp["T_nx"], qp["T_ny"], qp["T_c"]
    H = Tnx.T @ (Pxx @ Tnx) + Tny.T @ (Pxy @ Tnx) + Tny.T @ (Pyy @ Tny)
    H = (H + H.T) / 2
    half = T.F_SCALE / 2.0                  # (the oracle's order of operations, so that a = 0 is its assembly bit for bit)
    f_x = 2 * half * (qp["q_x"].T @ Tc.T) @ (Pxx @ Tnx)
    f_xy = half * ((qp["q_x"].T @ Tc.T) @ (Pxy @ Tny) + (qp["q_y"].T @ Tc.T) @ (Pxy @ Tnx))
    f = np.squeeze(f_x + f_xy + 2 * half * (qp["q_y"].T @ Tc.T) @ (Pyy @ Tny))
    Qx, Qy = np.diag(c * yp), np.diag(c * xp)
    E = Qy @ Tny - Qx @ Tnx
    k_ref = np.squeeze(Qy @ (Tc @ qp["q_y"]) - Qx @ (Tc @ qp["q_x"]))
    n = rt.shape[0]
    G = np.vstack((np.eye(n), -np.eye(n), E, -E))
    h = np.concatenate((qp["h"][:2 * n], kappa_bound - k_ref, kappa_bound + k_ref))
    return dict(H=H, f=f, E=E, k_ref=k_ref, G=G, h=h)


def solve_dense(d, lb, ub, kappa_bound, rows=True):
    """The QP of dense_qp_about over lb <= alpha <= ub and (rows) |k_ref + E alpha| <= kappa_bound (Goldfarb-Idnani)."""
    from oracle import quadprog_gi
    n = d["H"].shape[0]
    C = [np.eye(n), -np.eye(n)]
    b = [lb, -ub]
    if rows:
        C += [-d["E"].T, d["E"].T]
        b += [d["k_ref"] - kappa_bound, -kappa_bound - d["k_ref"]]
    return quadprog_gi.solve_qp(d["H"], -d["f"], np.hstack(C), np.concatenate(b))[0]
