"""CPU ORACLE (test infrastructure, NOT product code) -- dense numpy restatement of the
``trajectory_planning_helpers==0.76`` functions on the minimum-curvature hot path.

PARITY UNPINNED: the arithmetic restated here lives in the third-party packages
``trajectory_planning_helpers==0.76`` (requirements.txt:3) and ``quadprog``
(Readme.md:40), neither of which is vendored under the reference tree nor
installable offline, and the reference ships no tests or golden vectors (SURVEY.md section 4/8c).
The restatement follows the published algorithm of those packages and is anchored on the
reference's own call sites:

* calc_splines      -- helper_funcs_glob/src/prep_track.py:48-51,
                       main_globaltraj.py:568
* opt_min_curv      -- main_globaltraj.py:264-271, :344-350
* iqp_handler       -- main_globaltraj.py:273-284
* opt_shortest_path -- main_globaltraj.py:286-290
* create_raceline   -- main_globaltraj.py:371-376
* calc_head_curv_an -- main_globaltraj.py:383-387

Everything here deliberately keeps the *dense* structure of the original (4N x 4N spline system,
explicit inverse, dense N x N Hessian) so that it is structurally independent of the banded
O(N b^2) formulation used by the CUDA product path.  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import this module.
"""
from __future__ import annotations

import math

import numpy as np

# Parity-critical constant (SURVEY.md A.3): in tph 0.76 the linear term carries a factor 2
# (f_x = 2 q_x^T T_c^T P_xx T_nx, ...) while H carries none, i.e. the QP solved is
# min 1/2 ||E a + F_SCALE k_ref||^2.  Isolated here so it can be flipped if tph source appears.
F_SCALE = 2.0


# ----------------------------------------------------------------------------------------------
# calc_splines (closed and open), dense 4N x 4N route
# ----------------------------------------------------------------------------------------------
def calc_splines(path, el_lengths=None, psi_s=None, psi_e=None, use_dist_scaling=True):
    path = np.asarray(path, dtype=float)
    if np.all(np.isclose(path[0], path[-1])) and psi_s is None:
        closed = True
    else:
        closed = False

    if not closed and (psi_s is None or psi_e is None):
        raise RuntimeError("Headings must be provided for unclosed spline calculation!")
    if el_lengths is not None and path.shape[0] != el_lengths.size + 1:
        raise RuntimeError("el_lengths input must be one element smaller than path input!")

    if use_dist_scaling and el_lengths is None:
        el_lengths = np.sqrt(np.sum(np.power(np.diff(path, axis=0), 2), axis=1))
    elif el_lengths is not None:
        el_lengths = np.copy(el_lengths)

    if use_dist_scaling and closed:
        el_lengths = np.append(el_lengths, el_lengths[0])

    no_splines = path.shape[0] - 1

    if use_dist_scaling:
        scaling = el_lengths[:-1] / el_lengths[1:]
    else:
        scaling = np.ones(no_splines - 1)

    M = np.zeros((no_splines * 4, no_splines * 4))
    b_x = np.zeros((no_splines * 4, 1))
    b_y = np.zeros((no_splines * 4, 1))

    template_M = np.array([[1, 0, 0, 0, 0, 0, 0, 0],
                           [1, 1, 1, 1, 0, 0, 0, 0],
                           [0, 1, 2, 3, 0, -1, 0, 0],
                           [0, 0, 2, 6, 0, 0, -2, 0]], dtype=float)

    for i in range(no_splines):
        j = i * 4
        if i < no_splines - 1:
            M[j: j + 4, j: j + 8] = template_M
            M[j + 2, j + 5] *= scaling[i]
            M[j + 3, j + 6] *= math.pow(scaling[i], 2)
        else:
            M[j: j + 2, j: j + 4] = [[1, 0, 0, 0],
                                     [1, 1, 1, 1]]
        b_x[j: j + 2] = [[path[i, 0]], [path[i + 1, 0]]]
        b_y[j: j + 2] = [[path[i, 1]], [path[i + 1, 1]]]

    if not closed:
        M[-2, 1] = 1
        el_length_s = 1.0 if el_lengths is None else el_lengths[0]
        b_x[-2] = math.cos(psi_s + math.pi / 2) * el_length_s
        b_y[-2] = math.sin(psi_s + math.pi / 2) * el_length_s
        M[-1, -4:] = [0, 1, 2, 3]
        el_length_e = 1.0 if el_lengths is None else el_lengths[-1]
        b_x[-1] = math.cos(psi_e + math.pi / 2) * el_length_e
        b_y[-1] = math.sin(psi_e + math.pi / 2) * el_length_e
    else:
        M[-2, 1] = scaling[-1]
        M[-2, -3:] = [-1, -2, -3]
        M[-1, 2] = 2 * math.pow(scaling[-1], 2)
        M[-1, -2:] = [-2, -6]

    x_les = np.squeeze(np.linalg.solve(M, b_x))
    y_les = np.squeeze(np.linalg.solve(M, b_y))

    coeffs_x = np.reshape(x_les, (no_splines, 4))
    coeffs_y = np.reshape(y_les, (no_splines, 4))

    normvec = np.stack((coeffs_y[:, 1], -coeffs_x[:, 1]), axis=1)
    norm_factors = 1.0 / np.sqrt(np.sum(np.power(normvec, 2), axis=1))
    normvec_normalized = np.expand_dims(norm_factors, axis=1) * normvec

    return coeffs_x, coeffs_y, M, normvec_normalized


# ----------------------------------------------------------------------------------------------
# opt_min_curv: dense assembly (returns the QP data) + solve through an injected QP solver
# ----------------------------------------------------------------------------------------------
def assemble_min_curv(reftrack, normvectors, A, kappa_bound, w_veh):
    """Dense assembly of the closed-track min-curvature QP exactly as tph does it.

    Returns a dict with H, f, G, h (min 1/2 a^T H a + f^T a  s.t.  G a <= h) plus the pieces
    needed for curv_error_max (T_c, T_nx, T_ny, A_ex_b A_inv, q_x, q_y, M_x, M_y).
    """
    reftrack = np.asarray(reftrack, dtype=float)
    normvectors = np.asarray(normvectors, dtype=float)
    no_points = reftrack.shape[0]
    no_splines = no_points

    if no_points != normvectors.shape[0]:
        raise RuntimeError("Array size of reftrack should be the same as normvectors!")
    if no_points * 4 != A.shape[0] or A.shape[0] != A.shape[1]:
        raise RuntimeError("Spline equation system matrix A has wrong dimensions!")

    A_ex_b = np.zeros((no_points, no_splines * 4))
    A_ex_c = np.zeros((no_points, no_splines * 4))
    for i in range(no_splines):
        A_ex_b[i, i * 4 + 1] = 1
        A_ex_c[i, i * 4 + 2] = 2

    A_inv = np.linalg.inv(A)
    T_c = A_ex_c @ A_inv

    M_x = np.zeros((no_splines * 4, no_points))
    M_y = np.zeros((no_splines * 4, no_points))
    q_x = np.zeros((no_splines * 4, 1))
    q_y = np.zeros((no_splines * 4, 1))
    for i in range(no_splines):
        j = i * 4
        nxt = i + 1 if i < no_points - 1 else 0
        M_x[j, i] = normvectors[i, 0]
        M_x[j + 1, nxt] = normvectors[nxt, 0]
        M_y[j, i] = normvectors[i, 1]
        M_y[j + 1, nxt] = normvectors[nxt, 1]
        q_x[j, 0] = reftrack[i, 0]
        q_x[j + 1, 0] = reftrack[nxt, 0]
        q_y[j, 0] = reftrack[i, 1]
        q_y[j + 1, 0] = reftrack[nxt, 1]

    T_b = A_ex_b @ A_inv
    x_prime = np.squeeze(T_b @ q_x)
    y_prime = np.squeeze(T_b @ q_y)

    curv_den = np.power(x_prime ** 2 + y_prime ** 2, 1.5)
    curv_part = np.divide(1.0, curv_den, out=np.zeros_like(curv_den), where=curv_den != 0)
    curv_part_sq = curv_part ** 2

    P_xx = np.diag(curv_part_sq * y_prime ** 2)
    P_yy = np.diag(curv_part_sq * x_prime ** 2)
    P_xy = np.diag(curv_part_sq * (-2.0 * x_prime * y_prime))

    T_nx = T_c @ M_x
    T_ny = T_c @ M_y

    H_x = T_nx.T @ (P_xx @ T_nx)
    H_xy = T_ny.T @ (P_xy @ T_nx)
    H_y = T_ny.T @ (P_yy @ T_ny)
    H = H_x + H_xy + H_y
    H = (H + H.T) / 2

    half = F_SCALE / 2.0  # tph: f_x, f_y carry "2 *", the two f_xy terms carry "1 *"
    f_x = 2 * half * (q_x.T @ T_c.T) @ (P_xx @ T_nx)
    f_xy = half * ((q_x.T @ T_c.T) @ (P_xy @ T_ny) + (q_y.T @ T_c.T) @ (P_xy @ T_nx))
    f_y = 2 * half * (q_y.T @ T_c.T) @ (P_yy @ T_ny)
    f = np.squeeze(f_x + f_xy + f_y)

    Q_x = np.diag(curv_part * y_prime)
    Q_y = np.diag(curv_part * x_prime)
    E_kappa = Q_y @ T_ny - Q_x @ T_nx
    k_kappa_ref = np.squeeze(Q_y @ (T_c @ q_y) - Q_x @ (T_c @ q_x))

    con_ge = np.ones(no_points) * kappa_bound - k_kappa_ref
    con_le = -(np.ones(no_points) * -kappa_bound - k_kappa_ref)
    con_stack = np.append(con_ge, con_le)

    dev_max_right = reftrack[:, 2] - w_veh / 2
    dev_max_left = reftrack[:, 3] - w_veh / 2

    if np.any(-dev_max_right > dev_max_left) or np.any(-dev_max_left > dev_max_right):
        raise RuntimeError("Problem not solvable, track might be too small to run with current safety distance!")

    G = np.vstack((np.eye(no_points), -np.eye(no_points), E_kappa, -E_kappa))
    h = np.append(dev_max_right, dev_max_left)
    h = np.append(h, con_stack)

    return dict(H=H, f=f, G=G, h=h, E_kappa=E_kappa, k_kappa_ref=k_kappa_ref,
                T_c=T_c, T_b=T_b, T_nx=T_nx, T_ny=T_ny, q_x=q_x, q_y=q_y, M_x=M_x, M_y=M_y,
                x_prime=x_prime, y_prime=y_prime)


def curv_error_max_from(qp, alpha):
    """Linearisation error of tph.opt_min_curv (max |kappa_sol_lin - kappa_orig_lin|)."""
    a = np.expand_dims(np.asarray(alpha, dtype=float), 1)
    q_x_tmp = qp["q_x"] + qp["M_x"] @ a
    q_y_tmp = qp["q_y"] + qp["M_y"] @ a
    x_prime_tmp = np.squeeze(qp["T_b"] @ q_x_tmp)
    y_prime_tmp = np.squeeze(qp["T_b"] @ q_y_tmp)
    x_pp = np.squeeze(qp["T_c"] @ qp["q_x"] + qp["T_nx"] @ a)
    y_pp = np.squeeze(qp["T_c"] @ qp["q_y"] + qp["T_ny"] @ a)
    xp, yp = qp["x_prime"], qp["y_prime"]
    curv_orig_lin = (xp * y_pp - yp * x_pp) / np.power(xp ** 2 + yp ** 2, 1.5)
    curv_sol_lin = (x_prime_tmp * y_pp - y_prime_tmp * x_pp) / np.power(x_prime_tmp ** 2 + y_prime_tmp ** 2, 1.5)
    return float(np.amax(np.abs(curv_sol_lin - curv_orig_lin)))


def _default_solve_qp():
    from . import quadprog_gi
    return quadprog_gi.solve_qp


def opt_min_curv(reftrack, normvectors, A, kappa_bound, w_veh, print_debug=False, plot_debug=False,
                 closed=True, psi_s=None, psi_e=None, fix_s=False, fix_e=False, solve_qp=None):
    if not closed:
        raise NotImplementedError("oracle restates the closed-track branch only (the only one main_globaltraj.py uses)")
    solve_qp = solve_qp or _default_solve_qp()
    qp = assemble_min_curv(reftrack, normvectors, A, kappa_bound, w_veh)
    # quadprog semantics: min 1/2 x^T G x - a^T x  s.t.  C^T x >= b
    alpha = solve_qp(qp["H"], -qp["f"], -qp["G"].T, -qp["h"], 0)[0]
    return alpha, curv_error_max_from(qp, alpha)


# ----------------------------------------------------------------------------------------------
# opt_shortest_path
# ----------------------------------------------------------------------------------------------
def assemble_shortest_path(reftrack, normvectors, w_veh):
    reftrack = np.asarray(reftrack, dtype=float)
    normvectors = np.asarray(normvectors, dtype=float)
    no_points = reftrack.shape[0]
    if no_points != normvectors.shape[0]:
        raise RuntimeError("Array size of reftrack should be the same as normvectors!")
    H = np.zeros((no_points, no_points))
    f = np.zeros(no_points)
    nv, rt = normvectors, reftrack
    for i in range(no_points):
        if i < no_points - 1:
            H[i, i] += 2 * (nv[i, 0] ** 2 + nv[i, 1] ** 2)
            H[i, i + 1] = 0.5 * 2 * (-2 * nv[i, 0] * nv[i + 1, 0] - 2 * nv[i, 1] * nv[i + 1, 1])
            H[i + 1, i] = H[i, i + 1]
            H[i + 1, i + 1] = 2 * (nv[i + 1, 0] ** 2 + nv[i + 1, 1] ** 2)
            f[i] += 2 * nv[i, 0] * rt[i, 0] - 2 * nv[i, 0] * rt[i + 1, 0] \
                + 2 * nv[i, 1] * rt[i, 1] - 2 * nv[i, 1] * rt[i + 1, 1]
            f[i + 1] = -2 * nv[i + 1, 0] * rt[i, 0] - 2 * nv[i + 1, 1] * rt[i, 1] \
                + 2 * nv[i + 1, 0] * rt[i + 1, 0] + 2 * nv[i + 1, 1] * rt[i + 1, 1]
        else:
            H[i, i] += 2 * (nv[i, 0] ** 2 + nv[i, 1] ** 2)
            H[i, 0] = 0.5 * 2 * (-2 * nv[i, 0] * nv[0, 0] - 2 * nv[i, 1] * nv[0, 1])
            H[0, i] = H[i, 0]
            H[0, 0] += 2 * (nv[0, 0] ** 2 + nv[0, 1] ** 2)
            f[i] += 2 * nv[i, 0] * rt[i, 0] - 2 * nv[i, 0] * rt[0, 0] \
                + 2 * nv[i, 1] * rt[i, 1] - 2 * nv[i, 1] * rt[0, 1]
            f[0] += -2 * nv[0, 0] * rt[i, 0] - 2 * nv[0, 1] * rt[i, 1] \
                + 2 * nv[0, 0] * rt[0, 0] + 2 * nv[0, 1] * rt[0, 1]

    dev_max_right = reftrack[:, 2] - w_veh / 2
    dev_max_left = reftrack[:, 3] - w_veh / 2
    dev_max_right = np.where(dev_max_right < 0.001, 0.001, dev_max_right)
    dev_max_left = np.where(dev_max_left < 0.001, 0.001, dev_max_left)

    G = np.vstack((np.eye(no_points), -np.eye(no_points)))
    h = np.ones(2 * no_points) * np.append(dev_max_right, dev_max_left)
    return dict(H=H, f=f, G=G, h=h)


def opt_shortest_path(reftrack, normvectors, w_veh, print_debug=False, solve_qp=None):
    solve_qp = solve_qp or _default_solve_qp()
    qp = assemble_shortest_path(reftrack, normvectors, w_veh)
    return solve_qp(qp["H"], -qp["f"], -qp["G"].T, -qp["h"], 0)[0]


# ----------------------------------------------------------------------------------------------
# create_raceline and helpers
# ----------------------------------------------------------------------------------------------
def calc_spline_lengths(coeffs_x, coeffs_y, quickndirty=False, no_interp_points=15):
    if coeffs_x.shape[0] != coeffs_y.shape[0]:
        raise RuntimeError("Coefficient matrices must have the same length!")
    if coeffs_x.ndim == 1:
        coeffs_x = np.expand_dims(coeffs_x, 0)
        coeffs_y = np.expand_dims(coeffs_y, 0)
    no_splines = coeffs_x.shape[0]
    spline_lengths = np.zeros(no_splines)
    if quickndirty:
        for i in range(no_splines):
            spline_lengths[i] = math.sqrt(math.pow(np.sum(coeffs_x[i]) - coeffs_x[i, 0], 2)
                                          + math.pow(np.sum(coeffs_y[i]) - coeffs_y[i, 0], 2))
    else:
        t_steps = np.linspace(0.0, 1.0, no_interp_points)
        spl_coords = np.zeros((no_interp_points, 2))
        for i in range(no_splines):
            spl_coords[:, 0] = coeffs_x[i, 0] + coeffs_x[i, 1] * t_steps + coeffs_x[i, 2] * np.power(t_steps, 2) \
                + coeffs_x[i, 3] * np.power(t_steps, 3)
            spl_coords[:, 1] = coeffs_y[i, 0] + coeffs_y[i, 1] * t_steps + coeffs_y[i, 2] * np.power(t_steps, 2) \
                + coeffs_y[i, 3] * np.power(t_steps, 3)
            spline_lengths[i] = np.sum(np.sqrt(np.sum(np.power(np.diff(spl_coords, axis=0), 2), axis=1)))
    return spline_lengths


def interp_splines(coeffs_x, coeffs_y, spline_lengths=None, incl_last_point=False, stepsize_approx=None,
                   stepnum_fixed=None):
    if coeffs_x.shape[0] != coeffs_y.shape[0]:
        raise RuntimeError("Coefficient matrices must have the same length!")
    if spline_lengths is not None and coeffs_x.shape[0] != spline_lengths.size:
        raise RuntimeError("coeffs_x/y and spline_lengths must have the same length!")
    if not (coeffs_x.ndim == 2 and coeffs_y.ndim == 2):
        raise RuntimeError("Coefficient matrices do not have two dimensions!")
    if (stepsize_approx is None and stepnum_fixed is None) or (stepsize_approx is not None and stepnum_fixed is not None):
        raise RuntimeError("Provide one of 'stepsize_approx' and 'stepnum_fixed' and set the other to 'None'!")
    if stepnum_fixed is not None:
        raise NotImplementedError("oracle restates the stepsize_approx branch only")

    if spline_lengths is None:
        spline_lengths = calc_spline_lengths(coeffs_x=coeffs_x, coeffs_y=coeffs_y, quickndirty=False)

    dists_cum = np.cumsum(spline_lengths)
    no_interp_points = math.ceil(dists_cum[-1] / stepsize_approx) + 1
    dists_interp = np.linspace(0.0, dists_cum[-1], no_interp_points)

    path_interp = np.zeros((no_interp_points, 2))
    spline_inds = np.zeros(no_interp_points, dtype=int)
    t_values = np.zeros(no_interp_points)

    for i in range(no_interp_points - 1):
        j = int(np.argmax(dists_interp[i] < dists_cum))
        spline_inds[i] = j
        if j > 0:
            t_values[i] = (dists_interp[i] - dists_cum[j - 1]) / spline_lengths[j]
        else:
            t_values[i] = dists_interp[i] / spline_lengths[0]
        t = t_values[i]
        path_interp[i, 0] = coeffs_x[j, 0] + coeffs_x[j, 1] * t + coeffs_x[j, 2] * math.pow(t, 2) + coeffs_x[j, 3] * math.pow(t, 3)
        path_interp[i, 1] = coeffs_y[j, 0] + coeffs_y[j, 1] * t + coeffs_y[j, 2] * math.pow(t, 2) + coeffs_y[j, 3] * math.pow(t, 3)

    if incl_last_point:
        path_interp[-1, 0] = np.sum(coeffs_x[-1])
        path_interp[-1, 1] = np.sum(coeffs_y[-1])
        spline_inds[-1] = coeffs_x.shape[0] - 1
        t_values[-1] = 1.0
    else:
        path_interp = path_interp[:-1]
        spline_inds = spline_inds[:-1]
        t_values = t_values[:-1]
        dists_interp = dists_interp[:-1]

    return path_interp, spline_inds, t_values, dists_interp


def interp_track_widths(w_track, spline_inds, t_values, incl_last_point=False):
    w_track_cl = np.vstack((w_track, w_track[0]))
    no_interp_points = t_values.size
    if incl_last_point:
        w_track_interp = np.zeros((no_interp_points + 1, w_track.shape[1]))
        w_track_interp[-1] = w_track_cl[-1]
    else:
        w_track_interp = np.zeros((no_interp_points, w_track.shape[1]))
    for i in range(no_interp_points):
        ind_spl = spline_inds[i]
        for c in range(w_track.shape[1]):
            w_track_interp[i, c] = np.interp(t_values[i], (0.0, 1.0), w_track_cl[ind_spl:ind_spl + 2, c])
    return w_track_interp


def create_raceline(refline, normvectors, alpha, stepsize_interp):
    raceline = refline + np.expand_dims(alpha, 1) * normvectors
    raceline_cl = np.vstack((raceline, raceline[0]))
    coeffs_x_raceline, coeffs_y_raceline, A_raceline, normvectors_raceline = \
        calc_splines(path=raceline_cl, use_dist_scaling=False)
    spline_lengths_raceline = calc_spline_lengths(coeffs_x=coeffs_x_raceline, coeffs_y=coeffs_y_raceline)
    raceline_interp, spline_inds_raceline_interp, t_values_raceline_interp, s_raceline_interp = \
        interp_splines(spline_lengths=spline_lengths_raceline, coeffs_x=coeffs_x_raceline,
                       coeffs_y=coeffs_y_raceline, incl_last_point=False, stepsize_approx=stepsize_interp)
    s_tot_raceline = float(np.sum(spline_lengths_raceline))
    el_lengths_raceline_interp = np.diff(s_raceline_interp)
    el_lengths_raceline_interp_cl = np.append(el_lengths_raceline_interp, s_tot_raceline - s_raceline_interp[-1])
    return raceline_interp, A_raceline, coeffs_x_raceline, coeffs_y_raceline, spline_inds_raceline_interp, \
        t_values_raceline_interp, s_raceline_interp, spline_lengths_raceline, el_lengths_raceline_interp_cl


# ----------------------------------------------------------------------------------------------
# calc_head_curv_an / normalize_psi
# ----------------------------------------------------------------------------------------------
def normalize_psi(psi):
    psi = np.asarray(psi, dtype=float)
    psi_out = np.sign(psi) * np.mod(np.abs(psi), 2 * math.pi)
    psi_out = np.where(psi_out >= math.pi, psi_out - 2 * math.pi, psi_out)
    psi_out = np.where(psi_out < -math.pi, psi_out + 2 * math.pi, psi_out)
    return psi_out


def calc_head_curv_an(coeffs_x, coeffs_y, ind_spls, t_spls, calc_curv=True, calc_dcurv=False):
    if coeffs_x.shape[0] != coeffs_y.shape[0]:
        raise ValueError("Coefficient matrices must have the same length!")
    if ind_spls.size != t_spls.size:
        raise ValueError("ind_spls and t_spls must have the same length!")
    if not calc_curv and calc_dcurv:
        raise ValueError("dkappa cannot be calculated without kappa!")
    x_d = coeffs_x[ind_spls, 1] + 2 * coeffs_x[ind_spls, 2] * t_spls + 3 * coeffs_x[ind_spls, 3] * np.power(t_spls, 2)
    y_d = coeffs_y[ind_spls, 1] + 2 * coeffs_y[ind_spls, 2] * t_spls + 3 * coeffs_y[ind_spls, 3] * np.power(t_spls, 2)
    x_dd = 2 * coeffs_x[ind_spls, 2] + 6 * coeffs_x[ind_spls, 3] * t_spls
    y_dd = 2 * coeffs_y[ind_spls, 2] + 6 * coeffs_y[ind_spls, 3] * t_spls
    x_ddd = 6 * coeffs_x[ind_spls, 3]
    y_ddd = 6 * coeffs_y[ind_spls, 3]
    psi = normalize_psi(np.arctan2(y_d, x_d) - math.pi / 2)
    if calc_curv:
        kappa = (x_d * y_dd - y_d * x_dd) / np.power(np.power(x_d, 2) + np.power(y_d, 2), 1.5)
    else:
        kappa = 0.0
    if calc_dcurv:
        dkappa = ((np.power(x_d, 2) + np.power(y_d, 2)) * (x_d * y_ddd - y_d * x_ddd)
                  - 3 * (x_d * y_dd - y_d * x_dd) * (x_d * x_dd + y_d * y_dd)) \
            / np.power(np.power(x_d, 2) + np.power(y_d, 2), 3)
        return psi, kappa, dkappa
    return psi, kappa


# ----------------------------------------------------------------------------------------------
# iqp_handler
# ----------------------------------------------------------------------------------------------
def iqp_handler(reftrack, normvectors, A, kappa_bound, w_veh, print_debug, plot_debug, stepsize_interp,
                iters_min=3, curv_error_allowed=0.01, solve_qp=None, max_iters=50, history=None):
    """tph.iqp_handler restated.  Unlike tph the caller's reftrack is copied (tph mutates the
    widths of the caller's array on the first iteration through aliasing)."""
    reftrack_tmp = np.array(reftrack, dtype=float, copy=True)
    normvectors_tmp = normvectors
    A_tmp = A
    iter_cur = 0
    while True:
        iter_cur += 1
        alpha_mincurv_tmp, curv_error_max_tmp = opt_min_curv(
            reftrack=reftrack_tmp, normvectors=normvectors_tmp, A=A_tmp, kappa_bound=kappa_bound, w_veh=w_veh,
            print_debug=print_debug, plot_debug=plot_debug, solve_qp=solve_qp)
        if history is not None:
            history.append(dict(iter=iter_cur, n=reftrack_tmp.shape[0], curv_error_max=curv_error_max_tmp))
        if iter_cur < iters_min:
            alpha_mincurv_tmp = alpha_mincurv_tmp * (iter_cur * 1.0 / iters_min)
        if (iter_cur >= iters_min and curv_error_max_tmp <= curv_error_allowed) or iter_cur >= max_iters:
            break
        refline_tmp, _, _, _, spline_inds_tmp, t_values_tmp, _, spline_lengths_tmp = create_raceline(
            refline=reftrack_tmp[:, :2], normvectors=normvectors_tmp, alpha=alpha_mincurv_tmp,
            stepsize_interp=stepsize_interp)[:8]
        if history is not None:
            history[-1]["s_total"] = float(np.sum(spline_lengths_tmp))      # (the lap length that sets the next point count)
        reftrack_tmp[:, 2] -= alpha_mincurv_tmp
        reftrack_tmp[:, 3] += alpha_mincurv_tmp
        ws_track_tmp = interp_track_widths(w_track=reftrack_tmp[:, 2:], spline_inds=spline_inds_tmp,
                                           t_values=t_values_tmp, incl_last_point=False)
        reftrack_tmp = np.column_stack((refline_tmp, ws_track_tmp))
        refline_tmp_cl = np.vstack((reftrack_tmp[:, :2], reftrack_tmp[0, :2]))
        _, _, A_tmp, normvectors_tmp = calc_splines(path=refline_tmp_cl, use_dist_scaling=False)
    return alpha_mincurv_tmp, reftrack_tmp, normvectors_tmp
