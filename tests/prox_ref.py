"""Dense float64 reference of the projection QP of mc_mincurv_solve_batch_ex (raceline_refine.CurvatureProjection): H, E
and k_ref from the dense oracle (oracle/tph_dense.py), the box as the setup kernel builds it, solved with the
Goldfarb-Idnani oracle (test infrastructure, not product code)."""
import numpy as np
import torch

from oracle import quadprog_gi, tph_dense as T
from global_racetrajectory_optimization_b200 import raceline_refine as R


def qp_data(reftrack, normvec, w_veh):
    """dict(H, E, k_ref, lb, ub) of one track (numpy [n, 4] and [n, 2]; the normals the device used)."""
    rt = np.asarray(reftrack, dtype=np.float64)
    _, _, A, _ = T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))
    qp = T.assemble_min_curv(rt, normvec, A, 0.12, w_veh)
    lb, ub, _ = R.box(torch.tensor(rt)[None], float(w_veh))
    return dict(H=qp["H"], E=qp["E_kappa"], k_ref=qp["k_kappa_ref"], lb=lb[0].numpy(), ub=ub[0].numpy())


def prox_qp(d, kappa_bound, mu, x, q, rows=True):
    """argmin 1/2 a^T (H + mu I) a + c^T a,  c = mu q - (H + mu I) x,  over lb <= a <= ub and (rows)
    |k_ref + E a| <= kappa_bound; d from qp_data."""
    n = d["H"].shape[0]
    G = d["H"] + mu * np.eye(n)
    c = mu * np.asarray(q) - G @ np.asarray(x)
    C = [np.eye(n), -np.eye(n)]
    b = [d["lb"], -d["ub"]]
    if rows:
        C += [-d["E"].T, d["E"].T]
        b += [d["k_ref"] - kappa_bound, -kappa_bound - d["k_ref"]]
    return quadprog_gi.solve_qp(G, -c, np.hstack(C), np.concatenate(b))[0]
