"""GPU tests of the lap-time refinement in the curvature metric (raceline_refine.CurvatureMetric,
refine_raceline_batch(metric_length=...); DESIGN.md section 3.13): the metric's solve through mc_mincurv_adjoint_batch
against dense numpy with H from the dense oracle (truncated to the band the device keeps), with and without pinned
points; the refinement in the metric on the golden tracks (lower lap time, the box, a fresh evaluation bit for bit, the
oracle chain, descent and Armijo at every accepted step, batch independence); the identity fallback of a track the
banded solver does not take; no stream synchronisation in the metric's call."""
import numpy as np
import pytest
import torch

import raceline_ref as RR
from oracle import tph_dense as T, tph_velprofile as VP
from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine as R, synth

pytestmark = pytest.mark.gpu
DEV = "cuda"
STEP = 2.0
NAMES = ["berlin", "handling", "modena", "synth1000"]
ELL = 20.0                  # [m] the metric length the refinement tests run with
BAND = 32                   # half-width of the cyclic band of H the device keeps (DESIGN.md section 3.2)
# max |u - u_ref| / max |u_ref| of the metric's solve against dense numpy, set from the H100 (80GB HBM3, 700 W): without
# pins 1.7e-11 at most (u and w); with pins the pinned points leak ~1 / PIN_FACTOR of their right-hand side into the free
# ones: 3.9e-7 for runs of pins, 5.9e-5 for a single free point among pins (its u is the smallest)
SOLVE_TOL = 1e-10
PINNED_TOL = 1e-6
ONE_FREE_TOL = 2e-4
ORACLE_TOL = 1e-9


def _veh(golden):
    v = golden("velprofile")
    return dict(ggv=v["ggv"], ax_max_machines=v["ax_max_machines"], v_max=float(v["v_max"]),
                drag_coeff=float(v["dragcoeff"]), m_veh=float(v["mass"]))


def _batch(golden, names, key="alpha_mincurv"):
    gs = [golden(nm) for nm in names]
    n = [g["reftrack"].shape[0] for g in gs]
    rt = np.zeros((len(gs), max(n), 4))
    al = np.zeros((len(gs), max(n)))
    for b, g in enumerate(gs):
        rt[b, :n[b]], al[b, :n[b]] = g["reftrack"], g[key]
    rt, al = torch.tensor(rt, device=DEV), torch.tensor(al, device=DEV)
    npts = torch.tensor(n, dtype=torch.int32, device=DEV)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    wv = torch.tensor([float(g["w_veh"]) for g in gs], device=DEV)
    return rt, nv, al, npts, wv


def _fresh(rt, nv, alpha, npts, veh):
    rl = B_.create_raceline_batch(rt, nv, alpha, STEP, n_pts=npts)
    return B_.vel_profile_batch(rl["kappa"], rl["el_lengths_interp"], n_pts=rl["n_out"], **veh)["laptime"][:, 0], rl


def _banded_h(rt, nv):
    """H of the dense oracle for one track (its normals: the device's), outside the cyclic band of half-width BAND 0."""
    n = rt.shape[0]
    _, _, A, _ = T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))
    H = T.assemble_min_curv(rt, nv, A, 0.12, 0.0)["H"]
    i = np.arange(n)
    dist = np.abs(i[:, None] - i[None, :])
    return np.where(np.minimum(dist, n - dist) <= BAND, H, 0.0)


@pytest.mark.parametrize("name", ["synth128", "handling", "berlin", "synth1000"])
def test_the_metric_solve_matches_dense_numpy(golden, name):
    """u = (I + l^4 H)_FF^-1 g_F on the free points and w = (I + l^4 H)^-1 y, H the oracle's band, for no pins, a run
    of pins across the seam, the separator nodes of the band factor (the last 32), random pins, every point pinned and
    one point free."""
    g0 = golden(name)
    rt = torch.tensor(g0["reftrack"], device=DEV)[None]
    n = rt.shape[1]
    _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
    Hb = _banded_h(g0["reftrack"], nv[0].cpu().numpy())
    rng = np.random.default_rng(11)
    M = np.eye(n) + ELL ** 4 * Hb
    met = R.CurvatureMetric(rt, nv, None, ELL)
    mask = torch.ones(1, dtype=torch.bool, device=DEV)
    pins = dict(none=[], seam=list(range(n - 6, n)) + list(range(6)), separator=list(range(n - 32, n)),
                random=sorted(rng.choice(n, n // 5, replace=False).tolist()), all=list(range(n)),
                one_free=[i for i in range(n) if i != n // 2])
    errs = {}
    for case, idx in pins.items():
        g = rng.standard_normal(n) * 0.01
        y = rng.standard_normal(n) * 0.01
        pin = np.zeros(n, dtype=bool)
        pin[idx] = True
        u, w, ok = met(torch.tensor(g, device=DEV)[None], torch.tensor(pin, device=DEV)[None],
                       torch.tensor(y, device=DEV)[None], mask)
        assert ok.tolist() == [True], case
        free = ~pin
        u_ref = np.zeros(n)
        if free.any():
            u_ref[free] = np.linalg.solve(M[np.ix_(free, free)], g[free])
        w_ref = np.linalg.solve(M, y)
        u = u[0].cpu().numpy()
        eu = float(np.abs(u - u_ref)[free].max() / np.abs(u_ref[free]).max()) if free.any() else 0.0
        ew = float(np.abs(w[0].cpu().numpy() - w_ref).max() / np.abs(w_ref).max())
        errs[case] = (eu, ew)
    print(f"METRIC solve {name} (n {n}, l {ELL} m): max rel. error (u, w) " +
          ", ".join(f"{k} ({a:.1e}, {b:.1e})" for k, (a, b) in errs.items()))
    assert max(errs["none"][0], max(e[1] for e in errs.values())) <= SOLVE_TOL
    assert max(errs[k][0] for k in ("seam", "separator", "random")) <= PINNED_TOL
    assert errs["one_free"][0] <= ONE_FREE_TOL


class _Recording(R.LapTime):
    """The lap-time objective that records every gradient evaluation (x, f, g, mask) on the host."""

    def __init__(self, *args):
        super().__init__(*args)
        self.grads = []

    def __call__(self, x, mask, need_grad):
        f, g, redo = super().__call__(x, mask, need_grad)
        if need_grad:
            self.grads.append((x.cpu(), f.cpu(), g.cpu(), mask.cpu()))
        return f, g, redo


def _accepted_steps_descend_and_pass_armijo(grads, b):
    pts = [(x[b], f[b], g[b]) for x, f, g, m in grads if bool(m[b])]
    hist = [float(pts[0][1])]
    for (x0, _, g0), (x1, f1, _) in zip(pts, pts[1:]):
        gs = float((g0 * (x1 - x0)).sum())
        assert gs < 0.0
        assert float(f1) <= max(hist[-R.MEMORY:]) + R.GAMMA * gs + 1e-12 * abs(float(f1))
        hist.append(float(f1))
    return len(pts) - 1


def test_refinement_in_the_metric_on_the_golden_tracks(golden):
    veh = _veh(golden)
    rt, nv, al, npts, wv = _batch(golden, NAMES)
    vp = dict(veh, dyn_model_exp=1.0, filt_window=None)
    obj = _Recording(rt, nv, npts, STEP, vp)
    res = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, objective=obj, metric_length=ELL,
                                  **veh)
    ident = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, **veh)
    lb, ub, _ = R.box(rt, wv, npts)
    for b, nm in enumerate(NAMES):
        n = int(npts[b])
        print(f"METRIC REFINE {nm} (l {ELL} m): laptime {float(res['laptime_start'][b]):.6f} -> "
              f"{float(res['laptime'][b]):.6f} s (identity {float(ident['laptime'][b]):.6f}), iters "
              f"{int(res['iters'][b])}, status {int(res['status'][b])}, pg_norm {float(res['pg_norm'][b]):.3e}, "
              f"fallbacks {int(res['metric_fallbacks'][b])}, largest move "
              f"{float((res['alpha'][b, :n] - al[b, :n]).abs().max()):.4f} m")
        a = res["alpha"][b, :n]
        assert bool(((a >= lb[b, :n]) & (a <= ub[b, :n])).all()), nm
        assert _accepted_steps_descend_and_pass_armijo(obj.grads, b) == int(res["iters"][b]), nm
    assert bool((res["laptime"] < res["laptime_start"]).all())
    assert res["metric_fallbacks"].dtype == torch.int32
    assert bool(torch.isin(res["status"], torch.tensor([R.CONVERGED, R.ITER_CAP, R.LINE_SEARCH], device=DEV)).all())
    lap0, _ = _fresh(rt, nv, torch.clamp(al, lb, ub), npts, veh)
    lap, rl = _fresh(rt, nv, res["alpha"], npts, veh)
    assert torch.equal(lap0, res["laptime_start"]) and torch.equal(lap, res["laptime"])
    v = golden("velprofile")
    errs = []
    for b, nm in enumerate(NAMES):
        n, no = int(npts[b]), int(rl["n_out"][b])
        rr = RR.create_raceline(rt[b, :n, :2].cpu(), nv[b, :n].cpu(), res["alpha"][b, :n].cpu(), STEP, no=no,
                                seg=rl["spline_inds"][b, :no].cpu().long())
        k, e = rr["kappa"].numpy(), rr["el_lengths"].numpy()
        vx = VP.calc_vel_profile(ggv=v["ggv"], ax_max_machines=v["ax_max_machines"], v_max=veh["v_max"], kappa=k,
                                 el_lengths=e, closed=True, dyn_model_exp=1.0, drag_coeff=veh["drag_coeff"], m_veh=veh["m_veh"])
        ax = VP.calc_ax_profile(np.append(vx, vx[0]), e)
        t = VP.calc_t_profile(vx, e, ax_profile=ax)
        errs.append(abs(float(res["laptime"][b]) - t[-1]) / t[-1])
    print("METRIC REFINE oracle relative errors:", dict(zip(NAMES, errs)))
    assert max(errs) <= ORACLE_TOL


def test_a_tracks_result_in_the_metric_does_not_depend_on_its_batch(golden):
    veh = _veh(golden)
    g = golden("handling")
    slot = 17

    def run(B):
        rt = torch.tensor(g["reftrack"], device=DEV)[None].repeat(B, 1, 1)
        rt[:, :, 2:] *= torch.linspace(0.9, 1.2, B, device=DEV, dtype=torch.float64)[:, None, None]
        rt[min(slot, B - 1), :, 2:] = torch.tensor(g["reftrack"][:, 2:], device=DEV)
        _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
        al = torch.tensor(g["alpha_mincurv"], device=DEV)[None].repeat(B, 1)
        res = R.refine_raceline_batch(rt, nv, al, 2.0, stepsize_interp=STEP, max_iters=10, metric_length=ELL, **veh)
        return {k: v[min(slot, B - 1)] for k, v in res.items()}
    alone, many = run(1), run(300)
    for k in ("alpha", "laptime", "iters", "status", "metric_fallbacks", "evals"):
        assert torch.equal(alone[k], many[k]), k


def test_a_track_the_banded_solver_does_not_take_refines_as_without_the_metric(golden):
    """A 70-point track (fewer than N_MIN) next to long ones takes the identity step in every iteration: its result is
    that of the refinement without the metric, bit for bit, while the long tracks use the metric."""
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
    kw = dict(n_pts=npts, stepsize_interp=STEP, max_iters=25, **veh)
    res = R.refine_raceline_batch(rt, nv, al, 2.0, metric_length=ELL, **kw)
    plain = R.refine_raceline_batch(rt, nv, al, 2.0, **kw)
    print(f"METRIC short track: iters {res['iters'].tolist()}, fallbacks {res['metric_fallbacks'].tolist()}, "
          f"status {res['status'].tolist()}")
    assert int(res["iters"][1]) > 0 and int(res["metric_fallbacks"][1]) >= int(res["iters"][1])
    for k in ("alpha", "laptime", "iters", "evals", "status", "pg_norm"):
        assert torch.equal(res[k][1], plain[k][1]), k
    assert int(res["metric_fallbacks"][0]) < int(res["iters"][0])


def test_the_metric_does_not_synchronise_the_stream(golden):
    rt, nv, al, npts, wv = _batch(golden, ["handling", "modena"])
    met = R.CurvatureMetric(rt, nv, npts, ELL)
    mask = torch.ones(2, dtype=torch.bool, device=DEV)
    g = torch.randn(al.shape, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
    pin = g > 1.5
    met(g, pin, g, mask), met(g, pin, None, mask)            # (warm: the workspace allocated)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        u, w, ok = met(g, pin, -g, mask)
        u2, w2, ok2 = met(g, pin, None, mask)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert bool(ok.all()) and bool(ok2.all()) and w2 is None
    assert torch.equal(u, u2) and torch.isfinite(w).all()
