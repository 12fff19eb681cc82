"""CPU tests of tests/mincurv_ref.py: the KKT certificate accepts the oracle's quadprog solutions of the full
minimum-curvature QP and rejects perturbed or under-constrained ones; the sparse periodic spline reproduces the oracle's
dense calc_splines."""
import numpy as np
import pytest

import mincurv_ref as R
import qp_sens as Q
from global_racetrajectory_optimization_b200 import synth
from oracle import tph_dense as T
from oracle.quadprog_gi import solve_qp


def _closed(rt):
    return np.vstack((rt[:, :2], rt[0, :2]))


def _qp(rt, kb, w_veh=2.0):
    _, _, A, nv = T.calc_splines(_closed(rt))
    qp = T.assemble_min_curv(rt, nv, A, kb, w_veh)
    lb, ub, _ = Q.bounds(rt, w_veh)
    return qp, lb, ub, T.opt_min_curv(rt, nv, A, kb, w_veh)[0]


def _cert(qp, lb, ub, kb, alpha, rows=True):
    return R.kkt_certificate(qp["H"], qp["f"], qp["E_kappa"], qp["k_kappa_ref"], lb, ub, kb, alpha, rows=rows)


def _ok(c):
    return c["box_viol"] <= 1e-9 and c["row_viol"] <= 1e-9 and c["stat"] <= 1e-9 and c["comp"] <= 1e-12


# (seed, n, kappa_bound, rows active at the optimum)
CASES = [(5, 100, 0.12, False), (31, 150, 0.12, False), (3, 87, 0.04, True), (4, 96, 0.03, True)]


@pytest.mark.parametrize("seed,n,kb,active", CASES)
def test_certificate_accepts_the_oracle_and_rejects_perturbations(seed, n, kb, active):
    qp, lb, ub, alpha = _qp(synth.make_track(seed, n), kb)
    c = _cert(qp, lb, ub, kb, alpha)
    assert _ok(c) and c["n_active"] > 0, c
    box = Q.solve_box_qp(qp["H"], qp["f"], lb, ub)
    assert (np.abs(alpha - box).max() > 1e-3) == active
    rng = np.random.default_rng(seed)
    # 1e-4 m in random directions: leaves the box, or (kept inside it) breaks stationarity
    bad = _cert(qp, lb, ub, kb, alpha + 1e-4 * rng.choice([-1.0, 1.0], n))
    assert bad["box_viol"] > 5e-5 and not _ok(bad), bad
    inside = np.clip(alpha + 1e-4 * rng.choice([-1.0, 1.0], n), lb, ub)
    bad = _cert(qp, lb, ub, kb, inside)
    assert bad["box_viol"] == 0.0 and bad["stat"] > 1e-4, bad


@pytest.mark.parametrize("seed,n,kb", [(3, 87, 0.04), (4, 96, 0.03)])
def test_certificate_rejects_solutions_of_a_qp_with_a_row_dropped(seed, n, kb):
    qp, lb, ub, alpha = _qp(synth.make_track(seed, n), kb)
    # the certificate needs the rows: without them the rows' multipliers are missing from stationarity
    assert _cert(qp, lb, ub, kb, alpha, rows=False)["stat"] > 1e-2
    # drop the row constraint (one of the 2n) whose multiplier is largest, and solve again
    G, h = qp["G"], qp["h"]
    rows = np.arange(2 * n, 4 * n)
    slack = h[rows] - G[rows] @ alpha
    drop = rows[np.argmin(slack)]
    keep = np.delete(np.arange(4 * n), drop)
    a2 = solve_qp(qp["H"], -qp["f"], -G[keep].T, -h[keep], 0)[0]
    assert np.abs(a2 - alpha).max() > 1e-4
    c = _cert(qp, lb, ub, kb, a2)
    assert c["row_viol"] > 1e-6 and not _ok(c), c
    # ... and the box-only optimum is not a solution of the full QP either
    c = _cert(qp, lb, ub, kb, Q.solve_box_qp(qp["H"], qp["f"], lb, ub))
    assert c["row_viol"] > 1e-4, c


def _spline_cases():
    out = [(f"uneven n={n}", R.uneven_track(n, 1.0, n)) for n in range(3, 66)]
    out += [(f"synth n={n}", synth.make_track(n, n)) for n in (80, 129, 200, 350)]
    out += [("spacing 1:5", R.uneven_track(300, 5.0, 1)), ("spacing 1:20", R.uneven_track(340, 20.0, 2))]
    return out


def test_periodic_spline_matches_the_dense_oracle():
    worst = 0.0
    for name, rt in _spline_cases():
        for ds in (False, True):
            ox, oy, _, onv = T.calc_splines(_closed(rt), use_dist_scaling=ds)
            cx, cy, nv = R.periodic_spline(_closed(rt), ds)
            e = max(np.abs(cx - ox).max(), np.abs(cy - oy).max(), np.abs(nv - onv).max())
            worst = max(worst, e)
            assert e < 1e-11, (name, ds, e)
        if ds:
            el = np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1)
            cx, cy, nv = R.periodic_spline(_closed(rt), el_lengths=el)
            assert np.abs(cx - ox).max() < 1e-11
    el = np.linalg.norm(np.diff(_closed(_spline_cases()[-1][1]), axis=0), axis=1)
    assert el.max() / el.min() > 18.0
    print(f"periodic_spline vs dense calc_splines: worst abs err {worst:.1e}")


def test_periodic_spline_is_usable_at_3600_points():
    rt = R.uneven_track(3600, 20.0, 7)
    cx, cy, nv = R.periodic_spline(_closed(rt))
    # interpolation, C1 and C2 continuity in the arc-length parameter at every knot
    h = np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1)
    for c, col in ((cx, 0), (cy, 1)):
        end = c.sum(axis=1)
        assert np.abs(end - np.roll(rt[:, col], -1)).max() < 1e-9
        d1 = (c[:, 1] + 2 * c[:, 2] + 3 * c[:, 3]) / h
        assert np.abs(d1 - np.roll(c[:, 1] / h, -1)).max() < 1e-9
        d2 = (2 * c[:, 2] + 6 * c[:, 3]) / h ** 2
        assert np.abs(d2 - np.roll(2 * c[:, 2] / h ** 2, -1)).max() < 1e-9
    assert np.allclose(np.linalg.norm(nv, axis=1), 1.0, rtol=0, atol=1e-15)
