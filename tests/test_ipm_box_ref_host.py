"""CPU tests of the replay of the box-phase interior-point iteration (tests/ipm_box_ref.py) that
tests/test_gpu_ipm_box_edges.py measures mincurv_pdip_kernel against: its bordered band factor against a dense
long-double Cholesky, its end point against Goldfarb-Idnani, the rotation symmetry, the iteration count of the bench's
CPU arm (oracle/banded_cpu.c), every exit reached by a named case with the test that decided it, and the gap between
the carried and the exact dual residual.

A non-positive pivot (status 3) is not reached: the band of E^T E cut to half-width 32 stays positive definite on the
candidates (1:5 and 1:20 spacing, n = 80 .. 96, where truncation drops the most), so H_32 + D has no non-positive pivot
for any D >= 0 at these sizes, and the iteration keeps D > 0."""
import numpy as np
import pytest

import ipm_box_ref as X
import ipm_rows_ref as IR
from conftest import load_golden
from oracle import banded_cpu as BC
from oracle import quadprog_gi as QG

GOLDEN = ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth1000", "synth128",
          "synth160_kappa", "synth200", "synth2000", "synth333", "synth333_kappa", "synth500", "synth500_narrow"]
# the fixtures on which the step test decides the exit (the mu and r_d tests already pass one iteration earlier)
STEP_DECIDES = ("berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth200", "synth500",
                "synth500_narrow")
# factor: long-double solve against the dense _chol solve, relative: <= 4.0e-19; backward residual <= 3.9e-27
FACTOR_TOL = 1e-17
RESID_TOL = 1e-25
# the replay at mu_rel = 1e-16 against quadprog on the same banded QP, max |d alpha| / max |alpha|: <= 2.5e-10 (1:20
# spacing), <= 2.6e-11 elsewhere
QP_TOL = 1e-9
# rotated against unrotated long-double replay, max |d alpha| / max |alpha|: <= 2.4e-15.  Same status and count; the
# alpha differ by more than long-double rounding because the stopping iterate amplifies it (mu_rel = 1e-10)
ROT_TOL = 3e-14
# carried against exact |r_d| / rd_tol, any iteration of any fixture: long double <= 2.7e-8, float64 <= 4.7e-5 (both on
# synth160_kappa)
GAP_TOL = dict(ld=3e-7, f64=5e-4)


@pytest.fixture(scope="module")
def fixtures():
    out = {}
    for nm in GOLDEN:
        g = load_golden(nm)
        q = X.qp_of_fixture(g)
        out[nm] = (g, q, X.stability(q))
    return out


@pytest.fixture(scope="module")
def exits():
    return {nm: (t, kw, X.stability(X.qp_of_track(t), **kw)) for nm, (t, kw) in X.exit_cases().items()}


@pytest.mark.parametrize("n", [80, 83, 87, 96, 113, 130])
def test_band_factor_against_dense_cholesky(n):
    q = X.qp_of_track(X.synth_track(n))
    rng = np.random.default_rng(n)
    D = (10.0 ** rng.uniform(-8.0, 8.0, n)).astype(X.LD)
    M = X.dense(q["hb"], D)
    L = IR._chol(M)
    f = X.BandFactor(q["hb"], D)
    assert f.ok and L is not None
    g = rng.standard_normal(n).astype(X.LD)
    x, xd = f.solve(g), IR._chol_solve(L, g)
    e = float(np.abs(x - xd).max() / np.abs(xd).max())
    res = float(np.abs(M @ x - g).max() / (np.abs(M).max() * np.abs(x).max()))
    print(f"n {n}: against dense {e:.1e} (bound {FACTOR_TOL:.0e}), residual {res:.1e} (bound {RESID_TOL:.0e})")
    assert e <= FACTOR_TOL and res <= RESID_TOL


def test_band_factor_reports_a_non_positive_pivot():
    q = X.qp_of_track(X.synth_track(90))
    D = np.full(90, 1e-3, dtype=X.LD)
    D[40] = -10.0
    assert not X.BandFactor(q["hb"], D).ok
    D[40] = 1e-3
    D[75] = -10.0                      # in the separator
    assert not X.BandFactor(q["hb"], D).ok


def _quadprog(q):
    H = X.dense(q["hb"]).astype(np.float64)
    n = q["n"]
    C = np.hstack((np.eye(n), -np.eye(n)))
    b = np.concatenate((q["lb"].astype(np.float64), -q["ub"].astype(np.float64)))
    return QG.solve_qp(H, -q["f"].astype(np.float64), C, b)[0]


@pytest.mark.parametrize("name", ["handling", "synth128", "synth160_kappa", "synth200", "collapsed96", "uneven96_r20",
                                  "floor_narrow", "fscale1_n100"])
def test_the_replay_solves_the_banded_qp(name):
    if name in GOLDEN:
        q = X.qp_of_fixture(load_golden(name))
    elif name == "collapsed96":
        q = X.qp_of_track(IR.track(IR.collapsed(96)))
    elif name == "uneven96_r20":
        q = X.qp_of_track(X.uneven(96, 20.0))
    elif name == "fscale1_n100":
        q = X.qp_of_track(X.synth_track(100, f_scale=1.0))
    else:
        q = X.qp_of_track(X.exit_cases()[name][0])
    r = X.replay(q, mu_rel=1e-16)
    a = _quadprog(q)
    e = float(np.abs(r["alpha"].astype(np.float64) - a).max() / max(np.abs(a).max(), 1e-3))
    print(f"{name}: status {r['status']} after {r['iters']} ({r['exit']}), against quadprog {e:.1e} (bound {QP_TOL:.0e})")
    assert r["status"] == 0 and e <= QP_TOL


@pytest.mark.parametrize("name", ["handling", "synth128", "synth333"])
def test_rotation_is_a_symmetry(name):
    q = X.qp_of_fixture(load_golden(name))
    r = X.replay(q)
    for k in (1, q["n"] // 3, q["n"] - 5):
        rr = X.replay(q, rotate=k)
        e = float(np.abs(rr["alpha"] - r["alpha"]).max() / np.abs(r["alpha"]).max())
        print(f"{name} rotated by {k}: status {rr['status']} after {rr['iters']}, alpha {e:.1e} (bound {ROT_TOL:.0e})")
        assert (rr["status"], rr["iters"]) == (r["status"], r["iters"]) and e <= ROT_TOL


def test_fixture_counts_and_the_cpu_arm(fixtures):
    """every fixture is count-stable, converges, and oracle/banded_cpu.c takes the float64 replay's iteration count"""
    for nm, (g, q, (r, stable, runs)) in fixtures.items():
        _, it_cpu = BC.opt_min_curv_banded(g["reftrack"], g["normvec"], float(g["w_veh"]))
        print(f"{nm} (n {q['n']}): {X.outcomes(runs)} stable {stable}, banded_cpu {it_cpu}, decided by {r['decided']}")
        assert stable and r["status"] == 0 and r["exit"] == "converged", nm
        assert it_cpu == runs[1]["iters"], nm
        assert 9 <= r["iters"] <= 16, nm
    step = sorted(nm for nm, (_, _, (r, _, _)) in fixtures.items() if r["decided"] == ("step",))
    print(f"the step test alone decides {len(step)} of {len(fixtures)} fixtures: {step}")
    assert step == sorted(STEP_DECIDES)


def test_constructed_counts_and_the_cpu_arm():
    """constructed tracks: banded_cpu.c takes the float64 replay's count wherever the case is count-stable"""
    tally = [0, 0]
    for name, t in (("synth80", X.synth_track(80)), ("synth97", X.synth_track(97)), ("uneven96_r5", X.uneven(96, 5.0)),
                    ("uneven96_r20", X.uneven(96, 20.0)), ("collapsed96", IR.track(IR.collapsed(96))),
                    ("wveh1.5_n130", X.synth_track(130, w_veh=1.5)), ("fscale1_n100", X.synth_track(100, f_scale=1.0))):
        r, stable, runs = X.stability(X.qp_of_track(t))
        try:
            _, it_cpu = BC.opt_min_curv_banded(t["rt"], t["nv"], t["w_veh"], f_scale=t["f_scale"], h=t["h"])
        except (ValueError, RuntimeError):
            it_cpu = None
        print(f"{name}: {X.outcomes(runs)} stable {stable}, banded_cpu {it_cpu}")
        tally[0 if stable else 1] += 1
        if stable:
            assert it_cpu == runs[1]["iters"], name
    assert tally[0] >= 5, tally


def test_every_exit_is_reached(fixtures, exits):
    r = fixtures["synth128"][2][0]
    assert (r["exit"], r["status"], r["decided"]) == ("converged", 0, ("rd",))
    r = fixtures["handling"][2][0]
    assert (r["exit"], r["status"], r["decided"]) == ("converged", 0, ("step",))
    step_margin = r["trace"][-2]["step"]
    print(f"handling: the step test fails one iteration before the exit by {step_margin:.3f}")
    assert 1.0 < step_margin < 1.1
    for nm, (t, kw, (r, stable, runs)) in exits.items():
        tr = r["trace"][-1]
        print(f"{nm} {kw}: {X.outcomes(runs)} stable {stable}, {r['exit']} status {r['status']} after {r['iters']}, "
              f"last |r_d| {tr['rd']:.2e} rd_tol, step ratio {tr['step']:.2f}, max|a| {tr['amax']:.2e}")
        assert stable, nm
    r = exits["floor_narrow"][2][0]
    tr = r["trace"][-1]
    assert (r["exit"], r["status"]) == ("converged", 0) and tr["floor"]
    assert tr["step"] <= 1.0 < tr["step"] * 0.01 / tr["amax"], "the 1 cm floor must decide the step test"
    r = exits["mu_floor_0"][2][0]
    assert (r["exit"], r["status"]) == ("mu_floor", 0) and 1.0 < r["trace"][-1]["rd"] <= 1e3
    r = exits["mu_floor_2"][2][0]
    assert (r["exit"], r["status"]) == ("mu_floor", 2) and r["trace"][-1]["rd"] > 1e3
    r = exits["cap"][2][0]
    assert (r["exit"], r["status"], r["iters"]) == ("cap", 2, X.MAX_ITER)


@pytest.mark.parametrize("ratio", [5.0, 20.0])
def test_no_non_positive_pivot_from_band_truncation(ratio):
    """the truncated band stays positive definite where truncation drops the most (uneven spacing, small n)"""
    worst = np.inf
    for n in range(80, 97):
        hb = X.qp_of_track(X.uneven(n, ratio))["hb"]
        ev = np.linalg.eigvalsh(X.dense(hb.astype(np.float64)))
        worst = min(worst, ev[0] / ev[-1])
    print(f"1:{ratio:g} spacing, n 80 .. 96: smallest lambda_min / lambda_max of H_32 {worst:.1e}")
    assert worst > 0.0


def test_carried_residual_gap(fixtures):
    worst = dict(ld=0.0, f64=0.0)
    for nm, (_, q, (r, _, runs)) in fixtures.items():
        for key, run in (("ld", r), ("f64", runs[1])):
            gap = max(abs(t["rd"] - t["rd_exact"]) for t in run["trace"])
            worst[key] = max(worst[key], gap)
    kap = fixtures["synth160_kappa"][2]
    for key, run in (("ld", kap[0]), ("f64", kap[2][1])):
        tr = run["trace"][-1]
        print(f"synth160_kappa {key}: last carried |r_d| {tr['rd']:.1e} rd_tol, exact {tr['rd_exact']:.1e} rd_tol")
    print("largest |carried - exact| / rd_tol over the fixtures:", {k: f"{v:.1e}" for k, v in worst.items()},
          "bounds", GAP_TOL)
    assert worst["ld"] <= GAP_TOL["ld"] and worst["f64"] <= GAP_TOL["f64"]
    tr = kap[0]["trace"][-1]
    assert tr["rd_exact"] > 1e3 * tr["rd"], "the gap on synth160_kappa is what shows the bound is not vacuous"
