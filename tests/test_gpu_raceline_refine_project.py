"""GPU tests of the lap-time refinement under the curvature limit (raceline_refine.CurvatureProjection,
refine_raceline_batch(kappa_bound=...); DESIGN.md section 3.13): mc_mincurv_solve_batch_ex without prox arguments is
opt_min_curv_batch bit for bit; the projection QP against the dense float64 reference (tests/prox_ref.py) with the rows
inactive and active; the refinement on the golden tracks at curvlim and a tight limit (the rows hold at every accepted
iterate, the lap time falls, a fresh evaluation bit for bit, descent and Armijo at every accepted step), batch
independence, no stream synchronisation, and the NO_PROJECTION of a track the QP does not take."""
import numpy as np
import pytest
import torch

import prox_ref
from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine as R, synth
from test_gpu_raceline_refine_metric import _Recording, _accepted_steps_descend_and_pass_armijo, _batch, _fresh, _veh

pytestmark = pytest.mark.gpu
DEV = "cuda"
STEP = 2.0
NAMES = ["berlin", "handling", "modena", "synth1000"]
ELL = 10.0                  # [m] the metric length the refinement tests run with
CURVLIM = 0.12              # tests/golden/racecar_ini.json veh_params.curvlim
TIGHT_CURVLIM = 0.05        # tight_curvlim of the tests/golden/refback_* fixtures
KAPPA_REL = 1e-7            # the finalize stage's acceptance of |k_ref + E alpha| <= kappa_bound (status 4 beyond it)
# max |y - y_ref| [m] of the projection against the dense float64 reference, set from the H100 (80GB HBM3, 700 W;
# DESIGN.md 3.13): with the rows inactive 3.4e-5 m at most (the box phase's step criterion); with them active 3.2e-4 m at
# l = 10 m and 3.0e-3 m at l = 40 m (handling: H + l^-4 I is nearly singular along the long wavelengths the active rows
# leave free, and the curvature-row phase stops at its complementarity tolerance)
PROX_TOL = 1e-4
PROX_TOL_ROWS = 1e-2


def test_the_extended_entry_without_prox_is_opt_min_curv(golden):
    rt, nv, _, npts, wv = _batch(golden, NAMES)
    wv = wv.to(torch.float64)
    B, n_max = rt.shape[:2]
    _, _, _, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    for kb in (CURVLIM, TIGHT_CURVLIM):
        ref = B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts, max_chunk=B)
        out = B_._mincurv_results(B, n_max, rt.device)
        ws = B_._workspace("mincurv", B_._lib.load().mc_mincurv_workspace_bytes(B, n_max), rt.device)
        B_._call("mc_mincurv_solve_batch_ex", B, n_max, npts, rt, nv, h, kb, 0.0, wv, B_.F_SCALE, *out.values(), 0.0, None,
                 None, ws=ws)
        print(f"PROJECT null prox kb {kb}: status {out['status'].tolist()}, iters {out['iters'].tolist()}")
        valid = torch.arange(n_max, device=DEV)[None] < npts[:, None]          # (the padding is not written)
        assert torch.equal(torch.where(valid, out["alpha"], 0.0), torch.where(valid, ref["alpha"], 0.0)), kb
        for k in ("status", "iters", "kappa_lin_max", "curv_error_max"):
            assert torch.equal(out[k], ref[k]), (kb, k)


def _pushed(d, x, kb):
    """x moved along the curvature rows' normal until max |k_ref + E x| is 1.5 kb (then clipped to the box)."""
    k = d["k_ref"] + d["E"] @ x
    v = np.linalg.lstsq(d["E"], np.sign(k) * 1.5 * kb - k, rcond=None)[0]
    return np.clip(x + v, d["lb"], d["ub"])


@pytest.mark.parametrize("name", ["synth128", "handling", "berlin", "synth1000"])
def test_the_projection_matches_the_dense_reference(golden, name):
    """y of CurvatureProjection against the dense QP for l in {5, 10, 40} m (10 m above 300 points), at curvlim and the
    tight limit, from the minimum-curvature alpha with a smooth random q of 5 cm, and from a point pushed against the rows
    with q = 0."""
    g0 = golden(name)
    rt = torch.tensor(g0["reftrack"], device=DEV)[None]
    n, wv = rt.shape[1], float(g0["w_veh"])
    _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
    d = prox_ref.qp_data(g0["reftrack"], nv[0].cpu().numpy(), wv)
    rng = np.random.default_rng(7)
    mask = torch.ones(1, dtype=torch.bool, device=DEV)
    errs = []
    ells = (5.0, 10.0, 40.0) if n <= 300 else (10.0,)
    for kb in (CURVLIM, TIGHT_CURVLIM):
        x_in = np.clip(g0["alpha_mincurv"], d["lb"], d["ub"])
        s = 2.0 * np.pi * np.arange(n) / n
        q = 0.05 * sum(np.sin(k * s + p) for k, p in zip(rng.integers(1, 12, 4), rng.uniform(0.0, 6.28, 4))) / 4.0
        cases = dict(start=(x_in, q), pushed=(_pushed(d, x_in, kb), np.zeros(n)))
        for ell in ells:
            prj = R.CurvatureProjection(rt, nv, None, wv, kb, ell)
            for case, (x, q) in cases.items():
                y, ok = prj(torch.tensor(x, device=DEV)[None], torch.tensor(q, device=DEV)[None], mask)
                try:
                    y_ref = prox_ref.prox_qp(d, kb, ell ** -4, x, q)
                except ValueError:                            # the rows and the box have no common point
                    print(f"PROJECT prox {name} kb {kb} l {ell} {case}: infeasible, device ok {ok.tolist()}")
                    assert ok.tolist() == [False]
                    continue
                assert ok.tolist() == [True], (kb, ell, case)
                e = float(np.abs(y[0].cpu().numpy() - y_ref).max())
                kl = float(prj.kappa_lin(y, mask)[0])
                rows = float(np.abs(d["k_ref"] + d["E"] @ y_ref).max())
                errs.append(e)
                print(f"PROJECT prox {name} (n {n}) kb {kb} l {ell} {case}: max |y - y_ref| {e:.2e} m, "
                      f"kappa_lin {kl:.6f} (reference {rows:.6f}), rows active {rows >= kb * (1 - 1e-6)}")
                assert kl <= kb * (1.0 + KAPPA_REL)
                assert e <= (PROX_TOL_ROWS if rows >= kb * (1 - 1e-6) else PROX_TOL), (kb, ell, case)
    assert errs


def _kappa_checks(prj, xs, kb):
    return max(float(prj.kappa_lin(x, torch.isfinite(x).all(dim=1)).nan_to_num(0.0).max()) for x in xs) / kb - 1.0


@pytest.mark.parametrize("kb", [CURVLIM, TIGHT_CURVLIM])
def test_refinement_under_the_curvature_limit_on_the_golden_tracks(golden, kb):
    veh = _veh(golden)
    rt, nv, al, npts, wv = _batch(golden, NAMES)
    _, _, _, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    qp = B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts)
    qp_ok = qp["status"] == 0
    qp_slack = float((qp["kappa_lin_max"][qp_ok] / kb - 1.0).max()) if bool(qp_ok.any()) else 0.0
    vp = dict(veh, dyn_model_exp=1.0, filt_window=None)
    obj = _Recording(rt, nv, npts, STEP, vp)
    xs = []
    res = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, objective=obj, metric_length=ELL,
                                  kappa_bound=kb, max_iters=40, callback=lambda it, x, f, st: xs.append(x.clone()),
                                  **veh)
    free = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, metric_length=ELL, max_iters=40,
                                   **veh)
    prj = R.CurvatureProjection(rt, nv, npts, wv, kb, ELL)
    ran = res["evals"] > 0                                # (the others: alpha0 could not be projected)
    slack = _kappa_checks(prj, [torch.where(ran[:, None], x, torch.full_like(x, np.nan)) for x in xs], kb)
    rl_free = B_.create_raceline_batch(rt, nv, free["alpha"], STEP, n_pts=npts)
    for b, nm in enumerate(NAMES):
        no = int(rl_free["n_out"][b])
        print(f"PROJECT REFINE {nm} kb {kb} (l {ELL} m): qp status {int(qp['status'][b])}, laptime "
              f"{float(res['laptime_start'][b]):.6f} -> {float(res['laptime'][b]):.6f} s (unconstrained "
              f"{float(free['laptime'][b]):.6f}), iters {int(res['iters'][b])}, status {int(res['status'][b])}, pg_norm "
              f"{float(res['pg_norm'][b]):.3e}, kappa_lin_max {float(res['kappa_lin_max'][b]):.6f}, kappa_max "
              f"{float(res['kappa_max'][b]):.6f} (unconstrained {float(rl_free['kappa'][b, :no].abs().max()):.6f}), "
              f"projection failures {int(res['projection_failures'][b])}")
    print(f"PROJECT REFINE kb {kb}: the QP's own slack {qp_slack:.2e}, the iterates' {slack:.2e}")
    # a track starts exactly where the QP itself has a solution at this kappa_bound
    assert torch.equal(ran, qp_ok)
    assert torch.equal(res["status"][~ran], torch.full_like(res["status"][~ran], R.NO_PROJECTION))
    assert bool(ran.any())
    assert qp_slack <= KAPPA_REL and slack <= KAPPA_REL
    assert bool((res["kappa_lin_max"][ran] <= kb * (1.0 + KAPPA_REL)).all())
    assert bool((res["laptime"][ran] <= res["laptime_start"][ran]).all())
    lb, ub, _ = R.box(rt, wv, npts)
    for b, nm in enumerate(NAMES):
        n = int(npts[b])
        if not bool(ran[b]):
            assert torch.equal(res["alpha"][b], al[b]) and bool(torch.isnan(res["laptime"][b])), nm
            continue
        a = res["alpha"][b, :n]
        assert bool(((a >= lb[b, :n]) & (a <= ub[b, :n])).all()), nm
        assert _accepted_steps_descend_and_pass_armijo(obj.grads, b) == int(res["iters"][b]), nm
    assert bool(torch.isin(res["status"][ran], torch.tensor([R.CONVERGED, R.ITER_CAP, R.LINE_SEARCH, R.NO_PROJECTION],
                                                             device=DEV)).all())
    assert int(res["projection_failures"][ran].sum()) == 0
    lap, rl = _fresh(rt, nv, res["alpha"], npts, veh)
    assert torch.equal(lap[ran], res["laptime"][ran])
    k = torch.where(torch.arange(rl["kappa"].shape[1], device=DEV)[None] < rl["n_out"][:, None], rl["kappa"].abs(), 0.0)
    assert torch.equal(k.amax(dim=1)[ran], res["kappa_max"][ran])


def test_a_tracks_result_under_the_limit_does_not_depend_on_its_batch(golden):
    veh = _veh(golden)
    g = golden("handling")
    slot = 17

    def run(B):
        rt = torch.tensor(g["reftrack"], device=DEV)[None].repeat(B, 1, 1)
        rt[:, :, 2:] *= torch.linspace(0.9, 1.2, B, device=DEV, dtype=torch.float64)[:, None, None]
        rt[min(slot, B - 1), :, 2:] = torch.tensor(g["reftrack"][:, 2:], device=DEV)
        _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
        al = torch.tensor(g["alpha_mincurv"], device=DEV)[None].repeat(B, 1)
        res = R.refine_raceline_batch(rt, nv, al, 2.0, stepsize_interp=STEP, max_iters=10, metric_length=ELL,
                                      kappa_bound=CURVLIM, **veh)
        return {k: v[min(slot, B - 1)] for k, v in res.items()}
    alone, many = run(1), run(300)
    for k in ("alpha", "laptime", "laptime_start", "iters", "status", "evals", "pg_norm", "kappa_lin_max", "kappa_max",
              "projection_failures"):
        assert torch.equal(alone[k], many[k]), k


def test_a_short_track_beside_long_ones_keeps_alpha0(golden):
    veh = _veh(golden)
    g = golden("handling")
    n_long = g["reftrack"].shape[0]
    rt = torch.zeros((3, n_long, 4), dtype=torch.float64, device=DEV)
    rt[0] = torch.tensor(g["reftrack"], device=DEV)
    rt[1, :70] = torch.tensor(synth.make_track(5, 70), device=DEV)
    rt[2] = rt[0]
    npts = torch.tensor([n_long, 70, n_long], dtype=torch.int32, device=DEV)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    al = torch.zeros((3, n_long), dtype=torch.float64, device=DEV)
    al[0], al[2] = torch.tensor(g["alpha_mincurv"], device=DEV), torch.tensor(g["alpha_mincurv"], device=DEV)
    al[1, :70] = 0.01
    res = R.refine_raceline_batch(rt, nv, al, 2.0, n_pts=npts, stepsize_interp=STEP, max_iters=5, metric_length=ELL,
                                  kappa_bound=CURVLIM, **veh)
    assert res["status"].tolist()[1] == R.NO_PROJECTION and int(res["projection_failures"][1]) == 1
    assert torch.equal(res["alpha"][1], al[1]) and int(res["evals"][1]) == 0
    for k in ("laptime", "laptime_start", "kappa_lin_max", "kappa_max", "pg_norm"):
        assert bool(torch.isnan(res[k][1])), k
    assert int(res["iters"][0]) > 0 and int(res["iters"][2]) > 0
    assert torch.equal(res["alpha"][0], res["alpha"][2])


def test_the_projection_does_not_synchronise_the_stream(golden):
    rt, nv, al, npts, wv = _batch(golden, ["handling", "modena"])
    prj = R.CurvatureProjection(rt, nv, npts, wv, CURVLIM, ELL)
    mask = torch.ones(2, dtype=torch.bool, device=DEV)
    first = torch.tensor([True, False], device=DEV)
    q = 1e-3 * torch.randn(al.shape, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    prj(al, q, mask)                                          # (warm: the workspace allocated)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y, ok = prj(al, q, mask)
        y2, ok2 = prj(al, q, first)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert ok.tolist() == [True, True] and ok2.tolist() == [True, False]
    assert torch.equal(y[0], y2[0])
