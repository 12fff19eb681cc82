"""CPU tests of the lap-time refinement (raceline_refine.py; DESIGN.md section 3.13): the SPG core on functions with a
known solution (box-constrained quadratics, a non-convex double well), its statuses by construction and its batch
independence; refine_raceline_batch and globaltraj_batch(refine=...) against the recording stand-in of the library."""
import ctypes

import numpy as np
import pytest
import torch

from fake_lib import FakeLib, fake  # noqa: F401  (fake: the fixture)
from global_racetrajectory_optimization_b200 import globaltraj, raceline_refine as R

F64 = dict(dtype=torch.float64)
GGV = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.0], [80.0, 5.0]])


class Recorder:
    """A batched objective (value, gradient) that records every point it is asked for and every gradient it gives."""

    def __init__(self, f, g, lb, ub):
        self.f, self.g, self.lb, self.ub = f, g, lb, ub
        self.grads = []                 # (x, g) of every gradient evaluation

    def __call__(self, x, mask, need_grad):
        inside = (x >= self.lb) & (x <= self.ub)
        assert bool(inside[mask].all()), "a point outside the box was evaluated"
        f = self.f(x)
        if not need_grad:
            return f, None, None
        g = self.g(x)
        self.grads.append((x.clone(), g.clone()))
        return f, g, None


def _quadratic(B=6, n=40, seed=0):
    """0.5 sum a_i (x_i - c_i)^2 per track: the solution is clamp(c, lb, ub)."""
    rng = np.random.default_rng(seed)
    a = torch.tensor(rng.uniform(0.5, 20.0, (B, n)), **F64)
    c = torch.tensor(rng.uniform(-3.0, 3.0, (B, n)), **F64)
    lb = torch.tensor(rng.uniform(-2.0, -0.5, (B, n)), **F64)
    ub = torch.tensor(rng.uniform(0.5, 2.0, (B, n)), **F64)
    x0 = torch.tensor(rng.uniform(-4.0, 4.0, (B, n)), **F64)
    rec = Recorder(lambda x: 0.5 * (a * (x - c) ** 2).sum(1), lambda x: a * (x - c), lb, ub)
    return rec, x0, lb, ub, torch.clamp(c, lb, ub)


def _double_well(B=5, n=30, seed=1):
    """sum (x_i^2 - 1)^2 + 0.1 x_i per track, separable.  Its KKT points that are local minima, per coordinate: the
    roots near -1.012 and +0.987 of 4x^3 - 4x + 0.1, the latter replaced by the upper bound where it lies outside the
    box.  Returns them as [2, B, n]."""
    rng = np.random.default_rng(seed)
    lb = torch.full((B, n), -2.0, **F64)
    ub = torch.tensor(rng.choice([0.9, 1.5], (B, n)), **F64)
    x0 = torch.tensor(rng.uniform(0.3, 1.4, (B, n)), **F64)
    rec = Recorder(lambda x: ((x * x - 1.0) ** 2 + 0.1 * x).sum(1), lambda x: 4.0 * x * (x * x - 1.0) + 0.1, lb, ub)
    roots = sorted(r.real for r in np.roots([4.0, 0.0, -4.0, 0.1]))
    return rec, x0, lb, ub, torch.stack((torch.full_like(ub, roots[0]), torch.minimum(torch.full_like(ub, roots[2]), ub)))


def _accepted_steps_pass_the_armijo_test(rec, res, memory, gamma, x0_proj):
    """Every accepted step, from the recorded gradient evaluations (one per accepted point): f_new <= max of the last
    `memory` accepted values + gamma g^T s."""
    B = x0_proj.shape[0]
    for b in range(B):
        pts = [(x[b], g[b]) for x, g in rec.grads]
        hist = [float(rec.f(x0_proj)[b])]
        x_prev, g_prev = x0_proj[b], pts[0][1]
        for x, g in pts[1:]:
            if torch.equal(x, x_prev):
                continue                                  # (the track was not running in this evaluation)
            f_new = float(rec.f(x[None].expand(B, -1))[b])
            s = x - x_prev
            assert f_new <= max(hist[-memory:]) + gamma * float((g_prev * s).sum()) + 1e-12 * abs(f_new)
            hist.append(f_new)
            x_prev, g_prev = x, g


@pytest.mark.parametrize("problem", [_quadratic, _double_well])
def test_spg_converges_to_the_kkt_point_inside_the_box(problem):
    rec, x0, lb, ub, x_star = problem()
    seen = []
    res = R.spg(rec, x0, lb, ub, torch.ones(x0.shape[0], dtype=torch.bool), max_iters=500, pg_tol=1e-10,
                callback=lambda it, x, f, st: seen.append(x.clone()))
    assert res["status"].tolist() == [R.CONVERGED] * x0.shape[0]
    assert all(bool(((x >= lb) & (x <= ub)).all()) for x in seen)
    assert float(res["pg_norm"].max()) <= 1e-10
    assert float((res["x"] - x_star).abs().reshape(-1, *x0.shape).amin(dim=0).max()) <= 1e-9
    assert bool((res["f"] <= res["f0"]).all()) and bool((res["iters"] > 0).all())
    assert bool((res["evals"] >= res["iters"] + 1).all())
    _accepted_steps_pass_the_armijo_test(rec, res, R.MEMORY, R.GAMMA, torch.clamp(x0, lb, ub))


def test_spg_statuses_by_construction():
    rec, x0, lb, ub, _ = _quadratic(B=5)
    active = torch.tensor([True, True, True, True, False])
    calls = {"grad": 0}

    def fun(x, mask, need_grad):
        f, g, redo = rec(x, mask, need_grad)
        f = f.clone()
        f[3] = float("nan")                                   # track 3: a non-finite lap time from the start
        if need_grad:
            g = g.clone()
            g[1] = -g[1]                                      # track 1: an ascent direction -> no step is ever accepted
            calls["grad"] += 1
            if calls["grad"] == 3:
                g[2, 7] = float("inf")                        # track 2: a non-finite gradient at its second accepted point
        return f, g, redo
    res = R.spg(fun, x0, lb, ub, active, max_iters=4, pg_tol=0.0, max_halvings=8)
    assert res["status"].tolist() == [R.ITER_CAP, R.LINE_SEARCH, R.NO_GRADIENT, R.NO_GRADIENT, R.INACTIVE]
    assert res["iters"].tolist() == [4, 0, 2, 0, 0]
    x0p = torch.clamp(x0, lb, ub)
    assert torch.equal(res["x"][1], x0p[1]) and torch.equal(res["x"][3], x0p[3])     # frozen at the last accepted point
    assert res["evals"][1] == 1 + 8                          # one gradient evaluation and eight trials
    assert torch.isnan(res["pg_norm"][2:]).all() and bool(torch.isfinite(res["pg_norm"][:2]).all())


def test_spg_repeats_a_trial_that_asked_for_more_room():
    rec, x0, lb, ub, _ = _quadratic(B=3)
    state = {"trials": 0, "grown": 0}

    def fun(x, mask, need_grad):
        f, g, _ = rec(x, mask, need_grad)
        if need_grad:
            return f, g, None
        state["trials"] += 1
        redo = mask & (torch.arange(3) == 1) if state["trials"] == 2 else torch.zeros(3, dtype=torch.bool)
        return torch.where(redo, torch.full_like(f, -1e300), f), None, redo       # (a redo value must not be accepted)
    fun.grow = lambda: state.__setitem__("grown", state["grown"] + 1)
    res = R.spg(fun, x0, lb, ub, torch.ones(3, dtype=torch.bool), max_iters=30, pg_tol=1e-10)
    plain = R.spg(rec, x0, lb, ub, torch.ones(3, dtype=torch.bool), max_iters=30, pg_tol=1e-10)
    assert state["grown"] == 1
    for k in ("x", "iters", "evals", "status"):
        assert torch.equal(res[k], plain[k]), k


def test_a_repeated_trial_does_not_use_up_the_tracks_halvings():
    """Track 0 passes the Armijo test only on its last allowed trial of the first line search; an overflow reported on
    its first trial must not turn that into an exhausted line search (nor change evals)."""
    rec, x0, lb, ub, _ = _quadratic(B=2)

    def make(with_redo):
        state = {"calls": 0, "tried0": 0}

        def fun(x, mask, need_grad):
            f, g, _ = rec(x, mask, need_grad)
            if need_grad:
                return f, g, None
            state["calls"] += 1
            redo = torch.tensor([with_redo and state["calls"] == 1, False]) & mask
            if bool(mask[0]) and not bool(redo[0]):
                state["tried0"] += 1
                if state["tried0"] < 3:
                    f = f.clone()
                    f[0] = float("inf")                     # rejected: the step is halved
            return f, None, redo
        fun.grow = lambda: None
        return fun
    kw = dict(max_iters=1, pg_tol=0.0, max_halvings=3)
    plain = R.spg(make(False), x0, lb, ub, torch.ones(2, dtype=torch.bool), **kw)
    res = R.spg(make(True), x0, lb, ub, torch.ones(2, dtype=torch.bool), **kw)
    assert plain["status"].tolist() == [R.ITER_CAP, R.ITER_CAP] and plain["iters"].tolist() == [1, 1]
    for k in ("x", "iters", "evals", "status"):
        assert torch.equal(res[k], plain[k]), k


def test_a_tracks_iterates_do_not_depend_on_its_batch():
    rec, x0, lb, ub, _ = _double_well(B=7, n=33)
    hist = {}

    def run(idx):
        r = Recorder(rec.f, rec.g, lb[idx], ub[idx])
        xs = []
        out = R.spg(r, x0[idx], lb[idx], ub[idx], torch.ones(len(idx), dtype=torch.bool), max_iters=40, pg_tol=1e-13,
                    callback=lambda it, x, f, st: xs.append(x[idx.index(4)].clone()))
        hist[len(idx)] = xs
        return out, idx.index(4)
    alone, a = run([4])
    many, m = run([0, 1, 2, 3, 4, 5, 6])
    assert torch.equal(alone["x"][a], many["x"][m]) and alone["iters"][a] == many["iters"][m]
    assert alone["f"][a] == many["f"][m] and alone["evals"][a] == many["evals"][m]
    k = int(alone["iters"][a])
    assert k > 5 and all(torch.equal(u, v) for u, v in zip(hist[1][:k + 1], hist[7][:k + 1]))


def test_row_sum_and_the_box():
    v = torch.tensor(np.random.default_rng(3).standard_normal((4, 37)), **F64)
    assert torch.allclose(R.row_sum(v), v.sum(1), rtol=1e-13, atol=1e-13)
    assert torch.equal(R.row_sum(v[2:3]), R.row_sum(v)[2:3])
    rt = torch.zeros((3, 5, 4), **F64)
    rt[:, :, 2:] = 2.0
    rt[1, 3, 2:] = torch.tensor([1.0, 1.0 + 5e-9], **F64)    # ub - lb = 5e-9 < 2 FIX_EPS: collapsed onto its centre
    rt[2, 1, 2:] = 0.5                                  # lb > ub: empty
    lb, ub, empty = R.box(rt, 2.0, n_pts=torch.tensor([5, 5, 4]))
    assert empty.tolist() == [False, False, True]
    assert float(ub[0, 0]) == 1.0 and float(lb[0, 0]) == -1.0
    mid = 0.5 * ((1.0 - 1.0) - (1.0 + 5e-9 - 1.0))
    assert abs(float(lb[1, 3]) - (mid - R.FIX_EPS)) < 1e-15 and abs(float(ub[1, 3]) - (mid + R.FIX_EPS)) < 1e-15
    assert float(ub[2, 4]) == 0.0 and float(lb[2, 4]) == 0.0          # beyond n_pts


def test_spg_rejects_bad_parameters():
    rec, x0, lb, ub, _ = _quadratic(B=2)
    act = torch.ones(2, dtype=torch.bool)
    for kw in (dict(max_iters=-1), dict(memory=0), dict(max_halvings=0), dict(gamma=1.0), dict(lam_min=0.0),
               dict(lam_min=2.0, lam_max=1.0), dict(pg_tol=-1.0)):
        with pytest.raises(ValueError, match="spg"):
            R.spg(rec, x0, lb, ub, act, **kw)


# ------------------------------------------------------------------------------------------------
# refine_raceline_batch and globaltraj_batch(refine=...) against the recording stand-in
# ------------------------------------------------------------------------------------------------
def _names(lib):
    return [c[0] for c in lib.calls if not c[0].endswith("_workspace_bytes")]


def _inputs(B=4, n=120):
    rt = torch.rand((B, n, 4), **F64) + 3.0
    return rt, torch.rand((B, n, 2), **F64), torch.zeros((B, n), **F64)


@pytest.fixture()
def lapfake(fake, monkeypatch):
    """The stand-in with two things written: n_out = 10 for every track create_raceline is launched for (n_pts > 0),
    and, with unit_gradient set, dL/dalpha = 1 from the create_raceline adjoint.  The n_pts of every create_raceline
    launch are recorded (in n_pts)."""
    real = FakeLib.__getattr__
    fake.unit_gradient, fake.n_pts = False, []
    i32 = lambda ptr, k: (ctypes.c_int32 * k).from_address(ptr.value)          # noqa: E731

    def patched(self, name):
        fn = real(self, name)
        if name == "mc_create_raceline_batch":
            def rl(*a):
                fn(*a)
                bq = a[0]
                npts = list(i32(a[2], bq)) if a[2] is not None else [a[1]] * bq
                self.n_pts.append(npts)
                i32(a[12], bq)[:] = [10 if k > 0 else 0 for k in npts]
                return 0
            return rl
        if name == "mc_create_raceline_adjoint_batch" and self.unit_gradient:
            def adj(*a):
                fn(*a)
                m = a[0] * a[1]
                ctypes.memmove(a[15].value, (ctypes.c_double * m)(*([1.0] * m)), 8 * m)
                return 0
            return adj
        return fn
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    return fake


def test_refine_raceline_batch_runs_the_entries_in_order(lapfake):
    """With dL/dalpha = 1 and lap times of 0 (the stand-in writes none), no trial passes the Armijo test: after the first
    gradient evaluation every track takes max_halvings trials (create_raceline, profile) and ends with its line search
    exhausted, so the last gradient evaluation launches for no track."""
    lapfake.unit_gradient = True
    rt, nv, a0 = _inputs()
    npts = torch.tensor([120, 100, 0, 120], dtype=torch.int32)
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, n_pts=npts, max_halvings=2)
    grad = ["mc_create_raceline_batch", "mc_vel_profile_batch_ex", "mc_vel_profile_adjoint_batch",
            "mc_create_raceline_adjoint_batch"]
    trial = ["mc_create_raceline_batch", "mc_vel_profile_batch_ex"]
    staged = _names(lapfake)
    stages = [nm for k, nm in enumerate(staged) if k == 0 or staged[k - 1] != nm]   # (chunked launches collapse, and so
    assert stages == ["mc_polygon_length_batch"] + grad + trial + trial + grad      # does the capacity's create_raceline)
    assert res["status"].tolist() == [R.LINE_SEARCH, R.LINE_SEARCH, R.INACTIVE, R.LINE_SEARCH]
    assert res["iters"].tolist() == [0, 0, 0, 0] and res["evals"].tolist() == [3, 3, 0, 3]
    assert res["alpha"].shape == (4, 120) and bool(torch.isnan(res["laptime"][2]))
    assert lapfake.n_pts[0] == [120, 100, 0, 120] and lapfake.n_pts[-1] == [0, 0, 0, 0]


def test_refine_raceline_batch_checks_its_arguments(lapfake):
    rt, nv, a0 = _inputs()
    args = (GGV, MACH, 70.0, 0.75, 1200.0)
    with pytest.raises(RuntimeError, match="refine_raceline_batch"):
        R.refine_raceline_batch(rt, nv[:, :10], a0, 2.0, *args)
    with pytest.raises(RuntimeError, match="refine_raceline_batch"):
        R.refine_raceline_batch(rt, nv, a0[:, :10], 2.0, *args)
    with pytest.raises(ValueError, match="v_max"):
        R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, [60.0, 70.0], 0.75, 1200.0)
    with pytest.raises(ValueError, match="stepsize_interp"):
        R.refine_raceline_batch(rt, nv, a0, 2.0, *args, stepsize_interp=0.0)
    with pytest.raises(ValueError, match="w_veh"):
        R.refine_raceline_batch(rt, nv, a0, torch.ones(3, **F64), *args)
    with pytest.raises(ValueError, match="spg"):
        R.refine_raceline_batch(rt, nv, a0, 2.0, *args, max_iters=-1)


def test_refine_leaves_empty_boxes_and_non_finite_tracks_untouched(lapfake):
    rt, nv, a0 = _inputs()
    rt[1, 5, 2:] = 0.2                                      # narrower than w_veh = 2: lb > ub
    a0[1] = 7.0
    nv[3, 17, 0] = float("nan")                             # a non-finite normal
    a0[3, 4] = 9.0
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, max_iters=3)
    assert res["status"].tolist()[1:] == [R.EMPTY_BOX, R.NO_GRADIENT, R.NO_GRADIENT]
    assert lapfake.n_pts[0] == [120, 0, 120, 0]                                     # neither is ever launched
    for b in (1, 3):
        assert torch.equal(res["alpha"][b], a0[b]) and bool(torch.isnan(res["laptime"][b])) and res["evals"][b] == 0


def test_a_gradient_the_library_could_not_give_is_no_gradient(lapfake):
    """With strict=False the adjoints hand on zeros for a track they could not differentiate (the velocity-profile
    adjoint's non-finite status is not returned): the stand-in's adjoints write no gradient, i.e. exactly zero, and
    that is status 3 at the start point, not convergence."""
    rt, nv, a0 = _inputs()
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0)
    assert res["status"].tolist() == [R.NO_GRADIENT] * 4 and res["iters"].tolist() == [0] * 4
    assert torch.equal(res["alpha"], a0) and bool(torch.isnan(res["pg_norm"]).all())
    lapfake.unit_gradient = True                          # a gradient: the same tracks search (and fail, lap times 0)
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, max_halvings=1)
    assert res["status"].tolist() == [R.LINE_SEARCH] * 4


@pytest.mark.parametrize("opt_type", ["mincurv", "shortest_path"])
def test_globaltraj_batch_refines_between_the_qp_and_the_raceline(lapfake, opt_type):
    rt, _, _ = _inputs(B=3, n=150)
    out = globaltraj.globaltraj_batch(rt, opt_type, globaltraj.default_pars(), GGV, MACH, refine=dict(max_iters=3))
    order = _names(lapfake)
    qp = "mc_mincurv_solve_batch_shared" if opt_type == "mincurv" else "mc_shortest_path_solve_batch"
    want = ["mc_calc_splines_batch", qp, "mc_create_raceline_adjoint_batch", "mc_create_raceline_batch",
            "mc_vel_profile_batch_ex", "mc_assemble_trajectory_batch", "mc_interp_track_batch", "mc_min_bound_dists_batch",
            "mc_traj_extrema_batch"]
    pos = [max(k for k, nm in enumerate(order) if nm == w) if w in ("mc_create_raceline_batch", "mc_vel_profile_batch_ex")
           else order.index(w) for w in want]
    assert pos == sorted(pos)                       # the raceline and the profile of the result follow the refinement
    assert {"qp_alpha", "laptime_start", "refine_status", "refine_iters", "refine_evals"} <= set(out)
    assert out["refine_status"].tolist() == [R.NO_GRADIENT] * 3 and out["trajectory"].shape[2] == 7   # (no gradient)
    with pytest.raises(NotImplementedError, match="mincurv_iqp"):
        globaltraj.globaltraj_batch(rt, "mincurv_iqp", globaltraj.default_pars(), GGV, MACH, refine={})
    with pytest.raises(TypeError, match="refine"):
        globaltraj.globaltraj_batch(rt, opt_type, globaltraj.default_pars(), GGV, MACH, refine=3)


def test_globaltraj_batch_does_not_refine_a_track_whose_qp_failed(lapfake, monkeypatch):
    real = FakeLib.__getattr__

    def patched(self, name):
        fn = real(self, name)
        if name != "mc_shortest_path_solve_batch":
            return fn

        def solve(*a):
            fn(*a)
            ctypes.memmove(a[8].value, (ctypes.c_int32 * 3)(0, 2, 0), 12)          # status: track 1 failed
            ctypes.memmove(a[7].value + 8 * a[1], (ctypes.c_double * a[1])(*([0.25] * a[1])), 8 * a[1])   # its alpha
            return 0
        return solve
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    lapfake.unit_gradient = True
    rt, _, _ = _inputs(B=3, n=150)
    out = globaltraj.globaltraj_batch(rt, "shortest_path", globaltraj.default_pars(), GGV, MACH, refine=dict(max_iters=2))
    assert lapfake.n_pts[0] == [150, 0, 150] and lapfake.n_pts[1] == [150, 0, 150]          # the refinement leaves it out
    assert out["refine_status"][1] == R.INACTIVE and torch.equal(out["alpha"][1], out["qp_alpha"][1])
    assert bool((out["alpha"][1] == 0.25).all()) and out["status"].tolist() == [0, 2, 0]
