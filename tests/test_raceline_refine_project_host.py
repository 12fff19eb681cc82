"""CPU tests of the lap-time refinement under the curvature limit (raceline_refine.spg(project=...),
refine_raceline_batch(kappa_bound=...); DESIGN.md section 3.13): convergence on cyclic quadratics with a box and general
linear inequality rows against the Goldfarb-Idnani oracle, with a dense projection honouring spg's project contract;
NO_PROJECTION; batch independence; CurvatureProjection's launches against the recording stand-in of the library; the
extended C entry's argument checks; the dense reference of the projection QP."""
import ctypes

import numpy as np
import pytest
import torch

import prox_ref
from fake_lib import FakeLib, fake  # noqa: F401  (fake: the fixture)
from oracle import quadprog_gi, tph_dense as T
from global_racetrajectory_optimization_b200 import _lib, batch as B_, globaltraj, raceline_refine as R, synth

from test_raceline_refine_metric_host import DenseMetric, Quadratic

F64 = dict(dtype=torch.float64)
GGV = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.0], [80.0, 5.0]])


class DenseProjection:
    """spg's project contract with dense matrices: y = argmin 1/2 (a - x)^T M (a - x) + q^T (a - x) over
    lb <= a <= ub, C a <= r (per track, Goldfarb-Idnani).  fail(call, b) -> True makes track b's projection fail."""

    def __init__(self, M, C, r, lb, ub, fail=None):
        self.M, self.C, self.r, self.lb, self.ub, self.fail = M, C, r, lb, ub, fail
        self.calls, self.masks = 0, []

    def __call__(self, x, q, mask):
        self.masks.append(mask.clone())
        y = torch.full_like(x, float("nan"))
        ok = torch.zeros_like(mask)
        for b in range(x.shape[0]):
            if not bool(mask[b]) or (self.fail is not None and self.fail(self.calls, b)):
                continue
            M, n = self.M[b].numpy(), x.shape[1]
            a = M @ x[b].numpy() - q[b].numpy()
            Cq = np.hstack((np.eye(n), -np.eye(n), -self.C[b].numpy().T))
            bq = np.concatenate((self.lb[b].numpy(), -self.ub[b].numpy(), -self.r[b].numpy()))
            y[b] = torch.tensor(quadprog_gi.solve_qp(M, a, Cq, bq)[0], **F64)
            ok[b] = True
        self.calls += 1
        return y, ok


def _rows_problem(B=3, n=120, delta=1e-2, seed=0):
    """0.5 x^T Q x - c^T x on -1 <= x <= 1 and |D2 x| <= kb, Q = delta I + D2^T D2 (D2 the cyclic second difference),
    c = Q x_t for a smooth x_t that leaves the box; kb = 0.6 max |D2 x_box| of the box-only optimum, so that rows bind.
    Returns (objective, x0, lb, ub, Q, C, r, x*) with x* from the Goldfarb-Idnani oracle."""
    rng = np.random.default_rng(seed)
    D2 = -2.0 * np.eye(n) + np.roll(np.eye(n), 1, axis=1) + np.roll(np.eye(n), -1, axis=1)
    Q = delta * np.eye(n) + D2.T @ D2
    s = 2.0 * np.pi * np.arange(n) / n
    xt = np.stack([1.2 * np.sin(s * k + p) + 0.4 * np.cos(5 * s + p) for k, p in zip(rng.integers(1, 4, B),
                                                                                    rng.uniform(0, 6.28, B))])
    c = xt @ Q
    lb, ub = -np.ones((B, n)), np.ones((B, n))
    box = np.hstack((np.eye(n), -np.eye(n)))
    xs, rs = [], []
    for b in range(B):
        xb = quadprog_gi.solve_qp(Q, c[b], box, np.concatenate((lb[b], -ub[b])))[0]
        kb = 0.6 * np.abs(D2 @ xb).max()
        rs.append(np.full(2 * n, kb))
        Cq = np.hstack((box, -D2.T, D2.T))
        xs.append(quadprog_gi.solve_qp(Q, c[b], Cq, np.concatenate((lb[b], -ub[b], -rs[-1])))[0])
    C = np.vstack((D2, -D2))
    x0 = np.clip(rng.uniform(-0.3, 0.3, (B, n)), lb, ub)
    Qt = torch.tensor(Q, **F64)[None].repeat(B, 1, 1)
    return (Quadratic(Qt, torch.tensor(c, **F64)), torch.tensor(x0, **F64), torch.tensor(lb, **F64),
            torch.tensor(ub, **F64), Qt, torch.tensor(C, **F64)[None].repeat(B, 1, 1), torch.tensor(np.stack(rs), **F64),
            torch.tensor(np.stack(xs), **F64))


def test_projected_steps_converge_to_the_oracles_kkt_point():
    """With rows binding at the optimum, spg(project=...) in the metric Q / delta converges (status 0) to the oracle's
    solution; every accepted iterate satisfies the rows; one projection for x0, then one per gradient evaluation."""
    fun, x0, lb, ub, Q, C, r, xs = _rows_problem()
    B, n = x0.shape
    act = torch.ones(B, dtype=torch.bool)
    prj = DenseProjection(Q / 1e-2, C, r, lb, ub)
    viol = []
    res = R.spg(fun, x0, lb, ub, act, max_iters=100, pg_tol=1e-9, metric=DenseMetric(Q / 1e-2), project=prj,
                callback=lambda it, x, f, st: viol.append(float((torch.einsum("bij,bj->bi", C, x) - r).max())))
    n_rows = int(((torch.einsum("bij,bj->bi", C, xs) - r).abs() <= 1e-9).sum())
    print(f"PROJECT quadratic n={n}: iters {res['iters'].tolist()}, evals {res['evals'].tolist()}, pg "
          f"{res['pg_norm'].tolist()}, binding rows {n_rows}, max row violation {max(viol):.1e}")
    assert n_rows > 0
    assert res["status"].tolist() == [R.CONVERGED] * B
    assert float((res["x"] - xs).abs().max()) <= 1e-7
    assert max(viol) <= 1e-10
    assert res["projection_failures"].tolist() == [0] * B and "metric_fallbacks" not in res
    assert prj.calls == 2 + int(res["iters"].max())
    assert not bool(prj.masks[0].logical_not().any()) and bool((res["pg_norm"] <= 1e-9).all())


def test_a_failed_projection_ends_the_track_at_its_last_accepted_point():
    """Track 1's fourth projection fails: it stops with NO_PROJECTION at the point accepted before (the callback's), the
    other tracks run on unchanged; a track whose first projection (of x0) fails keeps x0 (clamped to the box), is never
    evaluated and has f = NaN; an ascent 'projection' (g^T d >= 0) stops a track before its first step."""
    fun, x0, lb, ub, Q, C, r, _ = _rows_problem(B=3, n=64, seed=3)
    act = torch.ones(3, dtype=torch.bool)
    seen = []
    prj = DenseProjection(Q / 1e-2, C, r, lb, ub, fail=lambda call, b: (b == 1 and call == 3) or (b == 2 and call == 0))
    res = R.spg(fun, x0, lb, ub, act, max_iters=30, pg_tol=1e-12, metric=DenseMetric(Q / 1e-2), project=prj,
                callback=lambda it, x, f, st: seen.append(x.clone()))
    ref = R.spg(fun, x0, lb, ub, act, max_iters=30, pg_tol=1e-12, metric=DenseMetric(Q / 1e-2),
                project=DenseProjection(Q / 1e-2, C, r, lb, ub))
    assert res["status"].tolist()[1:] == [R.NO_PROJECTION, R.NO_PROJECTION]
    assert res["projection_failures"].tolist() == [0, 1, 1]
    assert int(res["iters"][1]) == 2 and torch.equal(res["x"][1], seen[2][1])
    assert torch.equal(res["x"][2], x0[2]) and int(res["evals"][2]) == 0 and bool(torch.isnan(res["f"][2]))
    assert bool(torch.isnan(res["pg_norm"][1:]).all())
    for k in ("x", "f", "iters", "evals", "status"):
        assert torch.equal(res[k][0], ref[k][0]), k
    ascent = lambda x, q, mask: (torch.clamp(x + q, lb, ub), mask.clone())       # noqa: E731
    asc = R.spg(fun, x0, lb, ub, act, max_iters=30, project=ascent)
    assert asc["status"].tolist() == [R.NO_PROJECTION] * 3 and asc["iters"].tolist() == [0] * 3
    assert asc["projection_failures"].tolist() == [0] * 3


def test_a_tracks_projected_iterates_do_not_depend_on_its_batch():
    """(In the identity metric with identity BB steps: many iterations.)"""
    fun, x0, lb, ub, Q, C, r, _ = _rows_problem(B=4, n=80, seed=5)
    eye = torch.eye(80, **F64)[None].repeat(4, 1, 1)

    def run(idx):
        xs = []
        out = R.spg(Quadratic(fun.Q[idx], fun.c[idx]), x0[idx], lb[idx], ub[idx], torch.ones(len(idx), dtype=torch.bool),
                    max_iters=25, pg_tol=1e-13, project=DenseProjection(eye[idx], C[idx], r[idx], lb[idx], ub[idx]),
                    callback=lambda it, x, f, st: xs.append(x[idx.index(2)].clone()))
        return {k: v[idx.index(2)] for k, v in out.items()}, xs
    (alone, ha), (many, hm) = run([2]), run([0, 1, 2, 3])
    for k in ("x", "f", "iters", "evals", "status", "projection_failures"):
        assert torch.equal(alone[k], many[k]), k
    assert int(alone["iters"]) > 2 and all(torch.equal(u, v) for u, v in zip(ha, hm))


# ------------------------------------------------------------------------------------------------
# CurvatureProjection against the recording stand-in
# ------------------------------------------------------------------------------------------------
def _names(lib):
    return [c[0] for c in lib.calls if not c[0].endswith("_workspace_bytes")]


@pytest.fixture()
def projfake(fake, monkeypatch):
    """The stand-in with n_out = 10 per launched create_raceline track, dL/dalpha = 1 from the create_raceline adjoint,
    a lap time that falls by 1 s with every forward velocity-profile launch (every trial passes Armijo at t = 1), and a
    'projection' y = x - q (the unconstrained identity step); the inputs of every mc_mincurv_solve_batch_ex launch are
    recorded in prox (dicts of numpy arrays)."""
    real = FakeLib.__getattr__
    fake.prox, fake.lap = [], [0.0]

    def arr(ptr, ct, k):
        return np.array((ct * k).from_address(ptr.value))

    def patched(self, name):
        fn = real(self, name)
        if name == "mc_create_raceline_batch":
            def rl(*a):
                fn(*a)
                bq = a[0]
                npts = list(arr(a[2], ctypes.c_int32, bq)) if a[2] is not None else [a[1]] * bq
                (ctypes.c_int32 * bq).from_address(a[12].value)[:] = [10 if k > 0 else 0 for k in npts]
                return 0
            return rl
        if name == "mc_create_raceline_adjoint_batch":
            def adj(*a):
                fn(*a)
                m = a[0] * a[1]
                ctypes.memmove(a[15].value, (ctypes.c_double * m)(*([1.0] * m)), 8 * m)
                return 0
            return adj
        if name == "mc_vel_profile_batch_ex":
            def vp(*a):
                fn(*a)
                if a[24] is None and a[22] is not None:
                    self.lap[0] -= 1.0
                    m = a[0] * a[6]
                    ctypes.memmove(a[22].value, (ctypes.c_double * m)(*([self.lap[0]] * m)), 8 * m)
                return 0
            return vp
        if name == "mc_mincurv_solve_batch_ex":
            def solve(*a):
                fn(*a)
                bq, n = a[0], a[1]
                x, q = arr(a[16], ctypes.c_double, bq * n), arr(a[17], ctypes.c_double, bq * n)
                self.prox.append(dict(B=bq, n_pts=arr(a[2], ctypes.c_int32, bq), kb=a[6], w_veh=a[7], f_scale=a[9],
                                      mu=a[15], x=x.reshape(bq, n), q=q.reshape(bq, n)))
                ctypes.memmove(a[10].value, (ctypes.c_double * (bq * n))(*(x - q)), 8 * bq * n)
                return 0
            return solve
        return fn
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    return fake


def _inputs(B=4, n=120):
    rt = torch.rand((B, n, 4), **F64) + 3.0
    return rt, torch.rand((B, n, 2), **F64), torch.zeros((B, n), **F64)


def test_the_projection_launches_once_for_alpha0_and_once_per_gradient_evaluation(projfake):
    """One mc_mincurv_solve_batch_ex call (two launches: the stand-in halves the batch) with prox_q = 0 for alpha0, then
    one per gradient evaluation with prox_q = lam g; mu = l^-4, kappa_bound and w_veh as given, n_pts 0 for a track the
    QP does not take (it keeps alpha0 with NaN lap times and status NO_PROJECTION) and for the tracks that have
    finished; then the assembly and finalize stages once for kappa_lin_max at the result."""
    rt, nv, a0 = _inputs()
    npts = torch.tensor([120, 100, 60, 120], dtype=torch.int32)
    iters = 3
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, n_pts=npts, max_iters=iters,
                                  pg_tol=0.0, metric_length=10.0, kappa_bound=0.12)
    calls = projfake.prox
    assert len(calls) == 2 * (2 + iters) and all(c["B"] == 2 for c in calls)
    assert all(c["mu"] == 10.0 ** -4 and c["kb"] == 0.12 and c["w_veh"] == 2.0 and c["f_scale"] == B_.F_SCALE
               for c in calls)
    for k in range(0, len(calls), 2):
        n_call = np.concatenate((calls[k]["n_pts"], calls[k + 1]["n_pts"]))
        q = np.concatenate((calls[k]["q"], calls[k + 1]["q"]))
        assert n_call.tolist() == [120, 100, 0, 120]
        if k == 0:
            assert np.all(q == 0.0)                                        # alpha0: lam = 0
        else:
            for b in (0, 1, 3):                                            # lam g with g = 1
                lam = q[b, 0]
                assert lam > 0.0 and np.all(q[b, :int(npts[b])] == lam), (k, b)
    assert res["status"].tolist() == [R.ITER_CAP, R.ITER_CAP, R.NO_PROJECTION, R.ITER_CAP]
    assert res["iters"].tolist() == [iters, iters, 0, iters] and res["projection_failures"].tolist() == [0, 0, 1, 0]
    assert torch.equal(res["alpha"][2], a0[2]) and bool(torch.isnan(res["laptime"][2]))
    assert bool(torch.isnan(res["kappa_lin_max"][2])) and bool(torch.isnan(res["kappa_max"][2]))
    assert "metric_fallbacks" not in res and res["projection_failures"].dtype == torch.int32
    names = _names(projfake)
    tail = names[names.index("mc_mincurv_setup_batch_ex"):]
    assert tail[:4] == ["mc_mincurv_setup_batch_ex", "mc_mincurv_finalize_batch"] * 2


def test_finished_tracks_are_not_launched(projfake):
    """pg_tol = inf: every track converges at its first test, so the only launches are alpha0's and the first direction's
    (the direction is computed after every gradient evaluation); none follows for a finished track."""
    rt, nv, a0 = _inputs()
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, max_iters=5, pg_tol=float("inf"),
                                  metric_length=10.0, kappa_bound=0.12)
    assert res["status"].tolist() == [R.CONVERGED] * 4 and len(projfake.prox) == 4


def test_argument_errors_and_globaltraj_passes_kappa_bound_through(projfake):
    rt, nv, a0 = _inputs()
    with pytest.raises(ValueError, match="metric_length"):
        R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, kappa_bound=0.12)
    for bad in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="kappa_bound"):
            R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, metric_length=10.0, kappa_bound=bad)
    assert not projfake.prox
    rt3, _, _ = _inputs(B=3, n=150)
    globaltraj.globaltraj_batch(rt3, "mincurv", globaltraj.default_pars(), GGV, MACH,
                                refine=dict(max_iters=1, max_halvings=1, metric_length=15.0, kappa_bound=0.1))
    assert projfake.prox and projfake.prox[0]["kb"] == 0.1 and projfake.prox[0]["mu"] == 15.0 ** -4
    assert projfake.prox[0]["w_veh"] == globaltraj.default_pars()["optim_opts"]["width_opt"]


def test_the_extended_entry_refuses_bad_prox_arguments():
    """mc_mincurv_solve_batch_ex refuses mu <= 0 or non-finite and a missing prox_q before any launch (no device needed:
    the checks come first)."""
    lib = _lib.load()
    dummy = ctypes.c_void_p(8)
    args = lambda mu, q: (1, 130, None, dummy, dummy, dummy, 0.12, 2.0, None, 2.0, dummy, dummy, None, dummy, None,  # noqa
                          mu, dummy, q, dummy, 1 << 30, None)
    for mu, q, what in ((0.0, dummy, "prox_mu"), (-1.0, dummy, "prox_mu"), (float("nan"), dummy, "prox_mu"),
                        (float("inf"), dummy, "prox_mu"), (1e-4, None, "NULL argument")):
        assert lib.mc_mincurv_solve_batch_ex(*args(mu, q)) == -1
        msg = lib.mc_last_error().decode()
        assert msg.startswith("mc_mincurv_solve_batch_ex") and what in msg, msg


# ------------------------------------------------------------------------------------------------
# the dense reference of the projection QP
# ------------------------------------------------------------------------------------------------
def test_the_dense_prox_reference():
    """On a synthetic 140-point track: the solution lies in P, a point inside P projects onto itself with q = 0, with
    inactive rows the result is the box-only solution, and a point pushed against the rows is moved onto them."""
    rt = synth.make_track(2, 140)
    _, _, _, nv = T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))
    d = prox_ref.qp_data(rt, nv, 2.0)
    n, mu = rt.shape[0], 10.0 ** -4
    kb = 1.5 * np.abs(d["k_ref"]).max()
    x_in = np.zeros(n)                                                      # the centre line
    assert np.abs(d["k_ref"] + d["E"] @ x_in).max() < kb
    y = prox_ref.prox_qp(d, kb, mu, x_in, np.zeros(n))
    assert np.abs(y - x_in).max() <= 1e-9
    q = np.random.default_rng(1).standard_normal(n) * 1e-3
    y_rows = prox_ref.prox_qp(d, 10.0, mu, x_in, q)
    y_box = prox_ref.prox_qp(d, 10.0, mu, x_in, q, rows=False)
    assert np.abs(y_rows - y_box).max() <= 1e-9
    tight = 0.5 * np.abs(d["k_ref"]).max()
    y_t = prox_ref.prox_qp(d, tight, mu, x_in, np.zeros(n))
    k_t = d["k_ref"] + d["E"] @ y_t
    assert np.all(np.abs(k_t) <= tight * (1 + 1e-9)) and np.abs(k_t).max() >= tight * (1 - 1e-9)
    assert np.all(y_t >= d["lb"] - 1e-12) and np.all(y_t <= d["ub"] + 1e-12)

