"""GPU tests of the lap-time refinement (raceline_refine.refine_raceline_batch; DESIGN.md section 3.13) from the
minimum-curvature alpha of the golden tracks with the stock ggv and machine tables of the fixtures: the lap time falls,
alpha stays in the QP's box, the reported lap time is a fresh create_raceline_batch -> vel_profile_batch bit for bit and
the oracle chain's to 1e-9; the stopping rule, and the descent of the device lap time along the projected direction; a
track's result does not depend on its batch; capacity overflows, inactive slots, tracks without a gradient (reported by
the library or made unusable); no stream synchronisation inside the objective; globaltraj_batch(refine=...)."""
import numpy as np
import pytest
import torch

import raceline_ref as RR
from oracle import tph_velprofile as VP
from global_racetrajectory_optimization_b200 import batch as B_, globaltraj, raceline_refine as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
STEP = 2.0
NAMES = ["berlin", "handling", "modena", "synth1000"]
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


def test_refinement_lowers_the_lap_time_inside_the_box_and_reports_a_fresh_evaluation(golden):
    veh = _veh(golden)
    rt, nv, al, npts, wv = _batch(golden, NAMES)
    res = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, **veh)
    lb, ub, empty = R.box(rt, wv, npts)
    assert not empty.any()
    for b, nm in enumerate(NAMES):
        n = int(npts[b])
        print(f"REFINE {nm}: laptime {float(res['laptime_start'][b]):.6f} -> {float(res['laptime'][b]):.6f} s "
              f"({100.0 * (1.0 - float(res['laptime'][b] / res['laptime_start'][b])):.3f} %), iters {int(res['iters'][b])}, "
              f"evals {int(res['evals'][b])}, status {int(res['status'][b])}, pg_norm {float(res['pg_norm'][b]):.3e}")
        a = res["alpha"][b, :n]
        assert bool(((a >= lb[b, :n]) & (a <= ub[b, :n])).all()), nm
    assert bool((res["laptime"] < res["laptime_start"]).all())
    assert bool(torch.isin(res["status"], torch.tensor([R.CONVERGED, R.ITER_CAP, R.LINE_SEARCH], device=DEV)).all())
    # the start is the mincurv line's lap time, the result a fresh evaluation at the returned alpha, bit for bit
    lap0, _ = _fresh(rt, nv, torch.clamp(al, lb, ub), npts, veh)
    lap, rl = _fresh(rt, nv, res["alpha"], npts, veh)
    assert torch.equal(lap0, res["laptime_start"]) and torch.equal(lap, res["laptime"])
    # the oracle chain: the torch restatement of create_raceline at the device's station count and segments, then the
    # oracle's velocity, acceleration and time profiles
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
    print("REFINE oracle relative errors:", dict(zip(NAMES, errs)))
    assert max(errs) <= ORACLE_TOL


def _lap_and_grad(rt, nv, x, npts, veh, n_out_max):
    xg = x.clone().requires_grad_()
    rl = B_.create_raceline_diff(rt, nv, xg, STEP, n_pts=npts, n_out_max=n_out_max)
    vp = B_.vel_profile_diff(rl["kappa"], rl["el_lengths_interp"], n_pts=rl["n_out"], **veh)
    g, = torch.autograd.grad(vp["laptime"].sum(), xg)
    return vp["laptime"].detach(), g, rl


def test_the_stopping_rule_and_the_descent_of_the_device_lap_time_along_the_projected_direction(golden):
    """On the golden tracks no iterate reaches a small ||P(x - g) - x||_inf within a test's budget (it is still 7-10
    after 100 iterations, DESIGN.md section 3.13; real convergence to a KKT point is tested on the CPU with functions
    whose solution is known).  This test checks the stopping rule at a refined point: with pg_tol just above its
    ||P(x - g) - x||_inf the call stops at once with status 0, just below it the call takes a step; and d = P(x - g) - x
    there lowers the device lap time (a central difference at a delta that holds n_out and the station segments)."""
    veh = _veh(golden)
    rt, nv, al, npts, wv = _batch(golden, ["handling"])
    first = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, max_iters=15, **veh)
    pg = float(first["pg_norm"][0])
    res = R.refine_raceline_batch(rt, nv, first["alpha"], wv, n_pts=npts, stepsize_interp=STEP, pg_tol=1.01 * pg, **veh)
    assert res["status"].tolist() == [R.CONVERGED] and res["iters"].tolist() == [0]
    assert torch.equal(res["alpha"], first["alpha"]) and torch.equal(res["laptime"], first["laptime"])
    below = R.refine_raceline_batch(rt, nv, first["alpha"], wv, n_pts=npts, stepsize_interp=STEP, pg_tol=0.99 * pg,
                                    max_iters=1, **veh)
    assert below["status"].tolist() != [R.CONVERGED] or below["iters"].tolist() == [1]
    assert below["evals"].tolist()[0] >= 2
    lb, ub, _ = R.box(rt, wv, npts)
    x = res["alpha"]
    _, rl0 = _fresh(rt, nv, x, npts, veh)
    lap, g, rl = _lap_and_grad(rt, nv, x, npts, veh, int(rl0["kappa"].shape[1]))
    d = torch.clamp(x - g, lb, ub) - x
    dmax = float(d.abs().max())
    assert abs(dmax - pg) <= 1e-12 * pg
    gd = float((g * d).sum())
    no = int(rl["n_out"][0])
    for move in (1e-3, 3e-4, 1e-4, 3e-5, 1e-5):             # the largest point move [m]
        delta = move / dmax
        laps, held = [], True
        for s in (1.0, -1.0):
            lp, r2 = _fresh(rt, nv, x + s * delta * d, npts, veh)
            laps.append(float(lp[0]))
            held = held and int(r2["n_out"][0]) == no and torch.equal(r2["spline_inds"][0, :no], rl["spline_inds"][0, :no])
        if held:
            break
    assert held
    fd = (laps[0] - laps[1]) / (2.0 * delta)
    print(f"DESCENT handling: pg {pg:.3e}, largest move {move:.0e} m, central difference {fd:.6e}, g^T d {gd:.6e}")
    assert gd < 0.0 and fd < 0.0


def test_a_tracks_result_does_not_depend_on_its_batch(golden):
    veh = _veh(golden)
    g = golden("handling")
    slot = 17

    def run(B):
        rt = torch.tensor(g["reftrack"], device=DEV)[None].repeat(B, 1, 1)
        rt[:, :, 2:] *= torch.linspace(0.9, 1.2, B, device=DEV, dtype=torch.float64)[:, None, None]
        rt[min(slot, B - 1), :, 2:] = torch.tensor(g["reftrack"][:, 2:], device=DEV)
        _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
        al = torch.tensor(g["alpha_mincurv"], device=DEV)[None].repeat(B, 1)
        res = R.refine_raceline_batch(rt, nv, al, 2.0, stepsize_interp=STEP, max_iters=10, **veh)
        return {k: v[min(slot, B - 1)] for k, v in res.items()}
    alone, many = run(1), run(300)
    assert int(alone["iters"]) == int(many["iters"]) and int(alone["status"]) == int(many["status"])
    assert float((alone["alpha"] - many["alpha"]).abs().max()) <= 1e-12
    assert abs(float(alone["laptime"] - many["laptime"])) <= 1e-12 * float(alone["laptime"])


class _NoGradientFrom(R.LapTime):
    """The lap-time objective with the gradient of one track made unusable from its k-th gradient evaluation on."""

    def __init__(self, *args, track, k):
        super().__init__(*args)
        self.track, self.k, self.calls = track, k, 0

    def __call__(self, x, mask, need_grad):
        f, g, redo = super().__call__(x, mask, need_grad)
        if need_grad:
            self.calls += 1
            if self.calls >= self.k:
                g = g.clone()
                g[self.track] = float("nan")
        return f, g, redo


def test_overflow_regrowth_inactive_slots_and_tracks_without_a_gradient(golden):
    """From the shortest path every move lengthens the raceline, so an n_out_max fixed at the start's station count
    overflows; the capacity grows and the result is that of the run with room to spare.  An n_pts = 0 slot is never
    touched; a track whose gradient turns unusable keeps its last accepted point."""
    veh = _veh(golden)
    rt, nv, al, npts, wv = _batch(golden, ["handling", "handling", "handling"], key="alpha_shpath")
    npts[1] = 0
    kw = dict(n_pts=npts, stepsize_interp=STEP, max_iters=6, **veh)
    plain = R.refine_raceline_batch(rt, nv, al, wv, **kw)
    assert plain["status"][1] == R.INACTIVE and plain["evals"][1] == 0 and torch.equal(plain["alpha"][1], al[1])
    _, rl0 = _fresh(rt, nv, al, npts, veh)
    vp = dict(veh, dyn_model_exp=1.0, filt_window=None)
    tight = R.LapTime(rt, nv, npts, STEP, vp)
    tight.n_out_max = int(rl0["n_out"].max())
    res = R.refine_raceline_batch(rt, nv, al, wv, objective=tight, **kw)
    assert tight.n_out_max > int(rl0["n_out"].max())
    for k in ("alpha", "laptime", "iters", "status"):                 # (the inactive slot's lap time is NaN)
        assert torch.allclose(res[k], plain[k], rtol=0.0, atol=0.0, equal_nan=True), k
    # the library itself reports it: a station capacity below berlin's need at the start makes create_raceline report
    # n_out < 0 and the velocity profile grad_status != 0 for it; handling refines as it does alone
    rt2, nv2, al2, np2, wv2 = _batch(golden, ["handling", "berlin"])
    alone = R.refine_raceline_batch(rt2[:1, :208], nv2[:1, :208], al2[:1, :208], wv2[:1], n_pts=np2[:1],
                                    stepsize_interp=STEP, max_iters=6, **veh)
    _, rl2 = _fresh(rt2, nv2, al2, np2, veh)
    short = R.LapTime(rt2, nv2, np2, STEP, vp)
    short.n_out_max = int(rl2["n_out"][0]) + 16
    assert short.n_out_max < int(rl2["n_out"][1])
    res = R.refine_raceline_batch(rt2, nv2, al2, wv2, objective=short, n_pts=np2, stepsize_interp=STEP, max_iters=6, **veh)
    assert res["status"].tolist() == [int(alone["status"][0]), R.NO_GRADIENT] and res["iters"].tolist()[1] == 0
    lb2, ub2, _ = R.box(rt2, wv2, np2)
    assert bool(torch.isnan(res["laptime_start"][1])) and torch.equal(res["alpha"][1], torch.clamp(al2, lb2, ub2)[1])
    assert float((res["alpha"][0, :208] - alone["alpha"][0]).abs().max()) <= 1e-12
    assert abs(float(res["laptime"][0] - alone["laptime"][0])) <= 1e-12 * float(alone["laptime"][0])
    forced = _NoGradientFrom(rt, nv, npts, STEP, vp, track=2, k=3)
    res = R.refine_raceline_batch(rt, nv, al, wv, objective=forced, **kw)
    assert res["status"].tolist() == [int(plain["status"][0]), R.INACTIVE, R.NO_GRADIENT]
    assert res["iters"].tolist() == [int(plain["iters"][0]), 0, 2]
    assert torch.equal(res["alpha"][0], plain["alpha"][0])
    lap, _ = _fresh(rt, nv, res["alpha"], npts, veh)
    assert lap[2] == res["laptime"][2] and res["laptime"][2] < res["laptime_start"][2]


def test_globaltraj_batch_with_refine(golden):
    v = golden("velprofile")
    names = ["handling", "berlin"]
    gs = [golden(nm) for nm in names]
    n = [g["reftrack"].shape[0] for g in gs]
    rt = np.zeros((2, max(n), 4))
    for b, g in enumerate(gs):
        rt[b, :n[b]] = g["reftrack"]
    rt = torch.tensor(rt, device=DEV)
    npts = torch.tensor(n, dtype=torch.int32, device=DEV)
    pars = globaltraj.default_pars()
    pars["optim_opts"]["width_opt"] = 2.0
    base = globaltraj.globaltraj_batch(rt, "mincurv", pars, v["ggv"], v["ax_max_machines"], n_pts=npts)
    ref = globaltraj.globaltraj_batch(rt, "mincurv", pars, v["ggv"], v["ax_max_machines"], n_pts=npts,
                                      refine=dict(max_iters=20))
    assert torch.equal(ref["qp_alpha"], base["alpha"]) and torch.equal(ref["laptime_start"], base["laptime"])
    assert ref["trajectory"].shape[0] == base["trajectory"].shape[0] and ref["trajectory"].shape[2] == 7
    assert ref["vx"].shape[1] + 1 == ref["trajectory"].shape[1]
    assert bool((ref["laptime"] < base["laptime"]).all())
    assert bool((ref["vel_status"] == 0).all()) and torch.equal(ref["n_out"] > 0, base["n_out"] > 0)
    for b in range(2):                       # the lap closes at the raceline's length, the last row's time the lap time
        no = int(ref["n_out"][b])
        assert float(ref["trajectory"][b, no, 0]) == pytest.approx(float(ref["spline_lengths"][b, :n[b]].sum()), rel=1e-12)
        assert float(ref["t"][b, no]) == float(ref["laptime"][b])


def test_the_objective_does_not_synchronise_the_stream(golden):
    """A trial and a gradient evaluation of the lap-time objective queue their work without a device-to-host read or a
    stream synchronisation (the tables go through pinned memory): the one read per trial or iteration is spg's."""
    veh = _veh(golden)
    rt, nv, al, npts, wv = _batch(golden, ["handling", "modena"])
    obj = R.LapTime(rt, nv, npts, STEP, dict(veh, dyn_model_exp=1.0, filt_window=None))
    mask = torch.ones(2, dtype=torch.bool, device=DEV)
    obj.start(al, mask)
    obj(al, mask, False), obj(al, mask, True)                 # (warm: workspaces and pinned blocks allocated)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        f, _, redo = obj(al, mask, False)
        f2, g, _ = obj(al, mask, True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(f, f2) and not redo.any() and bool(torch.isfinite(g).all())
