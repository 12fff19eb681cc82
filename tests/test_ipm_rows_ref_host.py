"""CPU tests of the replay of the curvature-row interior-point iteration (tests/ipm_rows_ref.py) that
tests/test_gpu_ipm_rows_edges.py measures the kernels against: its QP against the dense oracle, its solution against
Goldfarb-Idnani and a long-double KKT certificate, which of the device cases are count-stable (long double, float64
and float64 with permuted reductions give the same status and iteration count), that every exit of the iteration is
reached by a named case, and the feasibility boundary kb_min by LP.

Reached: exit 1 (converged); exit 2 with status 0 and with status 2 (f_scale 1e-12: the dual residual test sits at
the edge of rounding); a non-positive pivot with late-accept 0 and with status 3 (likewise); the cap and a pivot
failure under status 4 on rows that cannot be met (long double runs to the cap, float64 stops at a pivot); clamped
start slacks; full and damped primal affine steps.  A full dual affine step cannot happen: its ratio takes the max of
1 - dx_i / s_u,i and 1 + dx_i / s_l,i, one of which exceeds 1 wherever dx_i != 0, so ad_aff = 1 only if the predictor's
dx is exactly zero everywhere."""
import numpy as np
import pytest

import ipm_rows_ref as IR
import lin_ref
from global_racetrajectory_optimization_b200 import synth
from oracle import tph_dense as T

# the long-double QP against the oracle's float64 assembly (its dense 4N x 4N inverse), relative to the largest entry:
# E <= 2.2e-14, k_ref and f <= 1.1e-12 (f, n 79 about a given line)
ASSEMBLY_TOL = 1e-11
# the replay run to mu <= 1e-16 mu0 against quadprog, max |d alpha| / max |alpha|: <= 1.2e-12 (bound 1e-9), and 2.0e-9
# on the collapsed boxes (bound 1e-8: quadprog's own accuracy on a 2e-8 wide box); at the kernels' stopping rule
# (mu <= 1e-11 mu0) the stopping iterate is up to 2.5e-7 from the optimum on these cases.  KKT in long double:
# stationarity <= 3.2e-12 of |f|.
QP_TOL = 1e-9
QP_TOL_COLLAPSED = 1e-8
RULE_TOL = 2e-6


@pytest.fixture(scope="module")
def dense():
    cases = IR.dense_cases()
    return cases, [IR.stability(t["d"], kb) for _, t, kb in cases]


@pytest.mark.parametrize("n", [3, 5, 16, 33, 79])
@pytest.mark.parametrize("lin", [False, True])
def test_assembly_against_the_oracle(n, lin):
    rt = synth.make_track(n, n)
    a = IR.lin_line(n) if lin else None
    t = IR.track(rt, w_veh=min(2.0, 0.5 * float((rt[:, 2] + rt[:, 3]).min())), lin_alpha=a)
    ref = lin_ref.dense_qp_about(rt, t["nv"], a, 0.1, t["w_veh"])
    for k, want in (("E", ref["E"]), ("k_ref", ref["k_ref"]), ("f", ref["f"])):
        e = np.abs(t["d"][k].astype(np.float64) - want).max() / np.abs(want).max()
        print(f"n {n} lin {lin}: {k} {e:.2e} (bound {ASSEMBLY_TOL:.0e})")
        assert e <= ASSEMBLY_TOL, (n, lin, k)


@pytest.mark.parametrize("name", ["synth16_rows", "synth33_feasible", "synth64_rows", "collapsed31_rows",
                                  "uneven40_r20_feasible", "synth31_infeasible", "synth8_infeasible"])
def test_the_replay_solves_the_qp(dense, name):
    cases, _ = dense
    _, t, kb = next(c for c in cases if c[0] == name)
    d = t["d"]
    _, _, A, _ = T.calc_splines(np.vstack((t["rt"][:, :2], t["rt"][:1, :2])))
    try:
        a_qp, _ = T.opt_min_curv(t["rt"], t["nv"], A, kb, t["w_veh"])
    except ValueError:
        assert IR.replay(d, kb)["status"] == 4
        return
    tight, rule = IR.replay(d, kb, mu_rel=1e-16), IR.replay(d, kb)
    scale = np.abs(a_qp).max()
    e_t = float(np.abs(tight["alpha"].astype(np.float64) - a_qp).max() / scale)
    e_r = float(np.abs(rule["alpha"].astype(np.float64) - a_qp).max() / scale)
    # long-double KKT certificate at the replay's own iterate and multipliers
    a, m = tight["alpha"], tight["mult"]
    E, k = d["E"], d["k_ref"] + d["E"] @ tight["alpha"]
    stat = np.abs(E.T @ (E @ a) + d["f"] + m["lu"] - m["ll"] + E.T @ (m["l3"] - m["l4"])).max() / np.abs(d["f"]).max()
    comp = max(float(np.abs(m["lu"] * (d["ub"] - a)).max()), float(np.abs(m["ll"] * (a - d["lb"])).max()),
               float(np.abs(m["l3"] * (kb - k)).max()), float(np.abs(m["l4"] * (kb + k)).max())) / float(np.abs(d["f"]).max())
    feas = max(float((d["lb"] - a).max()), float((a - d["ub"]).max()), float((np.abs(k) - kb).max() / kb), 0.0)
    tol = QP_TOL_COLLAPSED if name.startswith("collapsed") else QP_TOL
    print(f"{name}: tight {e_t:.2e} (bound {tol:.0e})  stopping rule {e_r:.2e} (bound {RULE_TOL:.0e})  "
          f"KKT stat {stat:.1e} comp {comp:.1e} feas {feas:.1e}")
    assert tight["status"] == 0 and rule["status"] == 0
    assert e_t <= tol and e_r <= RULE_TOL
    assert stat <= 3e-11 and comp <= 1e-11 and feas <= 1e-15


def test_count_stable_cases_per_path(dense):
    cases, refs = dense
    tally = dict(dense=[0, 0], banded=[0, 0], projection=[0, 0])
    for (_, _, _), (_, stable, _) in zip(cases, refs):
        tally["dense"][0 if stable else 1] += 1
    for _, t, kb in IR.banded_cases():
        tally["banded"][0 if IR.stability(t["d"], kb, band=IR.HBW, override="banded")[1] else 1] += 1
    for _, t, kb, mu, x, q in IR.prox_cases():
        st = IR.stability(t["d"], kb, band=IR.HBW, override="banded", prox_mu=mu, prox_x=x, prox_q=q)[1]
        tally["projection"][0 if st else 1] += 1
    for path, (s, u) in tally.items():
        print(f"{path}: {s} count-stable cases, {u} not (long double factored by hand at every n; the permuted float64 run "
              f"factors in another elimination order above {IR.DENSE_LD_MAX} points)")
        assert s >= 1, path


def _run(cases, refs, name):
    i = next(i for i, c in enumerate(cases) if c[0] == name)
    return refs[i]


def test_every_exit_is_reached(dense):
    cases, refs = dense
    r, _, _ = _run(cases, refs, "synth33_rows")
    assert r["exit"] == "converged" and r["status"] == 0
    r, _, _ = _run(cases, refs, "exit_mu_floor_0")
    assert (r["exit"], r["result"], r["status"]) == ("mu_floor", 0, 0)
    assert r["trace"][-1]["margin"]["floor"] <= 1.0 and r["trace"][-1]["margin"]["rd"] > 1.0
    r, _, _ = _run(cases, refs, "exit_mu_floor_2")
    assert (r["exit"], r["result"], r["status"]) == ("mu_floor", 2, 2)
    assert r["trace"][-1]["margin"]["rd"] > 1e3 or r["trace"][-1]["margin"]["rp"] > 1e2
    r, _, _ = _run(cases, refs, "exit_pivot_late0")
    assert (r["exit"], r["result"], r["status"]) == ("pivot", 0, 0)
    r, _, _ = _run(cases, refs, "exit_pivot_3")
    assert (r["exit"], r["result"], r["status"]) == ("pivot", 3, 3)
    r, _, runs = _run(cases, refs, "synth31_infeasible")
    assert (r["exit"], r["status"]) == ("cap", 4) and r["iters"] == IR.MAX_ITER + 20
    assert (runs[1]["exit"], runs[1]["result"], runs[1]["status"]) == ("pivot", 3, 4)
    assert any(c[0] == "synth31_infeasible" for c in cases)
    r, _, _ = _run(cases, refs, "synth64_feasible")
    assert r["clamped"] > 0
    steps = [s for (r, _, _) in refs for s in r["trace"]]
    assert any(s["aff_full"][0] for s in steps) and any(not s["aff_full"][0] for s in steps)
    assert any(s["full"][0] for s in steps) and any(not s["full"][0] for s in steps)
    exits = {}
    for (name, _, _), (r, _, _) in zip(cases, refs):
        exits.setdefault((r["exit"], r["status"]), name)
    print("first case per (exit, status):", exits)


@pytest.mark.parametrize("n", [5, 16, 40, 79])
def test_the_feasibility_boundary(n):
    t = IR.track(synth.make_track(1, n))
    kmin, a = IR.kappa_min(t["d"])
    d = t["d"]
    assert (a >= d["lb"] - 1e-12).all() and (a <= d["ub"] + 1e-12).all()
    below = IR.replay(d, float(kmin) * (1 - 1e-3))
    assert below["status"] == 4, below["exit"]
    for f in (1 + 1e-6, 1 + 1e-3):
        r = IR.replay(d, float(kmin) * f)
        tr = r["trace"][-1]["margin"]
        print(f"n {n} kb_min {float(kmin):.6g} x (1 + {f - 1:.0e}): status {r['status']} after {r['iters']} ({r['exit']}); "
              f"last margins mu {tr['mu']:.1e} rd {tr['rd']:.1e} rp {tr['rp']:.1e}")
        assert r["status"] in (0, 2, 3, 4)
        if r["status"] == 0:
            assert r["kappa_lin_max"] <= float(kmin) * f * (1 + 1e-7)
