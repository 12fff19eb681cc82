"""CPU tests of the lap-time refinement in a metric (raceline_refine.spg(metric=...), refine_raceline_batch(metric_length=...);
DESIGN.md section 3.13): convergence on a box-constrained quadratic against the Goldfarb-Idnani oracle with a dense
metric honouring spg's metric contract, the descent safeguard, batch independence; CurvatureMetric's launches against
the recording stand-in of the library."""
import ctypes

import numpy as np
import pytest
import torch

from fake_lib import FakeLib, fake  # noqa: F401  (fake: the fixture)
from oracle import quadprog_gi
from global_racetrajectory_optimization_b200 import batch as B_, globaltraj, raceline_refine as R

F64 = dict(dtype=torch.float64)
GGV = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.0], [80.0, 5.0]])


class DenseMetric:
    """spg's metric contract with dense matrices M [B, n, n]: u_F = M_FF^-1 g_F, w = M^-1 y."""

    def __init__(self, M):
        self.M, self.calls = M, 0

    def __call__(self, g, pin, y, mask):
        self.calls += 1
        u = torch.zeros_like(g)
        w = None if y is None else torch.zeros_like(y)
        for b in range(g.shape[0]):
            if not bool(mask[b]):
                continue
            free = ~pin[b]
            u[b, free] = torch.linalg.solve(self.M[b][free][:, free], g[b, free])
            if y is not None:
                w[b] = torch.linalg.solve(self.M[b], y[b])
        return u, w, mask.clone()


class Quadratic:
    def __init__(self, Q, c):
        self.Q, self.c = Q, c

    def __call__(self, x, mask, need_grad):
        Qx = torch.stack([self.Q[b] @ x[b] for b in range(x.shape[0])])      # (per track: independent of the batch)
        f = R.row_sum(0.5 * x * Qx - self.c * x)
        return f, (Qx - self.c) if need_grad else None, None


def _cyclic_problem(B=3, n=200, delta=1e-2, seed=0):
    """0.5 x^T Q x - c^T x on -1 <= x <= 1, Q = delta I + D2^T D2 (D2 the cyclic second difference): c = Q x_t for a
    smooth x_t that leaves the box on about a fifth of the points.  Returns (objective, x0, lb, ub, Q, x*) with x* from
    the Goldfarb-Idnani oracle."""
    rng = np.random.default_rng(seed)
    D2 = -2.0 * np.eye(n) + np.roll(np.eye(n), 1, axis=1) + np.roll(np.eye(n), -1, axis=1)
    Q = delta * np.eye(n) + D2.T @ D2
    s = 2.0 * np.pi * np.arange(n) / n
    xt = np.stack([1.2 * np.sin(s * k + p) + 0.1 * np.cos(3 * s + p) for k, p in zip(rng.integers(1, 4, B),
                                                                                    rng.uniform(0, 6.28, B))])
    c = xt @ Q
    lb, ub = -np.ones((B, n)), np.ones((B, n))
    xs = np.stack([quadprog_gi.solve_qp(Q, c[b], np.hstack((np.eye(n), -np.eye(n))), np.concatenate((lb[b], -ub[b])))[0]
                   for b in range(B)])
    x0 = np.clip(rng.uniform(-0.3, 0.3, (B, n)), lb, ub)
    Qt = torch.tensor(Q, **F64)[None].repeat(B, 1, 1)
    return (Quadratic(Qt, torch.tensor(c, **F64)), torch.tensor(x0, **F64), torch.tensor(lb, **F64),
            torch.tensor(ub, **F64), Qt, torch.tensor(xs, **F64))


def test_the_metric_converges_where_the_identity_does_not():
    """M = I + l^4 D2^T D2 with l^4 = 1 / delta (M = Q / delta): status 0 at pg_tol 1e-9 within 50 iterations and the
    oracle's solution to 1e-7; the identity metric has not converged after 50."""
    fun, x0, lb, ub, Q, xs = _cyclic_problem()
    B, n = x0.shape
    act = torch.ones(B, dtype=torch.bool)
    frac = float(((xs <= -1 + 1e-9) | (xs >= 1 - 1e-9)).double().mean())
    assert 0.1 <= frac <= 0.35                              # bounds active on about a fifth of the points
    met = DenseMetric(Q / 1e-2)
    res = R.spg(fun, x0, lb, ub, act, max_iters=50, pg_tol=1e-9, metric=met)
    ident = R.spg(fun, x0, lb, ub, act, max_iters=50, pg_tol=1e-9)
    print(f"METRIC quadratic n={n}: active {frac:.2f}, metric iters {res['iters'].tolist()} "
          f"(fallbacks {res['metric_fallbacks'].tolist()}), identity status {ident['status'].tolist()} "
          f"pg {ident['pg_norm'].tolist()}")
    assert res["status"].tolist() == [R.CONVERGED] * B and bool((res["iters"] <= 50).all())
    assert float((res["x"] - xs).abs().max()) <= 1e-7
    assert bool(((res["x"] >= lb) & (res["x"] <= ub)).all())
    assert ident["status"].tolist() == [R.ITER_CAP] * B and "metric_fallbacks" not in ident
    assert met.calls == 1 + int(res["iters"].max())          # one per gradient evaluation


def _separable(B=4, n=30, seed=2):
    rng = np.random.default_rng(seed)
    a = torch.tensor(rng.uniform(0.5, 20.0, (B, n)), **F64)
    c = torch.tensor(rng.uniform(-3.0, 3.0, (B, n)), **F64)
    lb = torch.tensor(rng.uniform(-2.0, -0.5, (B, n)), **F64)
    ub = torch.tensor(rng.uniform(0.5, 2.0, (B, n)), **F64)
    x0 = torch.tensor(rng.uniform(-4.0, 4.0, (B, n)), **F64)

    def fun(x, mask, need_grad):
        return 0.5 * (a * (x - c) ** 2).sum(1), (a * (x - c)) if need_grad else None, None
    return fun, x0, lb, ub, torch.clamp(c, lb, ub)


def test_an_ascent_metric_falls_back_to_the_identity_step_every_iteration():
    """u = -g: every direction fails g^T d < 0, every iteration takes the identity step (bit for bit the identity run)
    and the run converges."""
    fun, x0, lb, ub, xs = _separable()
    act = torch.ones(x0.shape[0], dtype=torch.bool)
    bad = lambda g, pin, y, mask: (-g, None if y is None else -y, mask.clone())       # noqa: E731
    res = R.spg(fun, x0, lb, ub, act, max_iters=500, pg_tol=1e-10, metric=bad)
    ident = R.spg(fun, x0, lb, ub, act, max_iters=500, pg_tol=1e-10)
    assert res["status"].tolist() == [R.CONVERGED] * x0.shape[0]
    assert torch.equal(res["metric_fallbacks"], res["iters"])
    for k in ("x", "f", "iters", "evals", "status", "pg_norm"):
        assert torch.equal(res[k], ident[k]), k
    assert float((res["x"] - xs).abs().max()) <= 1e-9


def test_a_tracks_iterates_in_the_metric_do_not_depend_on_its_batch():
    fun, x0, lb, ub, Q, _ = _cyclic_problem(B=4, n=96, seed=5)

    def run(idx):
        xs = []
        f = Quadratic(fun.Q[idx], fun.c[idx])
        out = R.spg(f, x0[idx], lb[idx], ub[idx], torch.ones(len(idx), dtype=torch.bool), max_iters=30, pg_tol=1e-13,
                    metric=DenseMetric(Q[idx] / 1e-2), callback=lambda it, x, f, st: xs.append(x[idx.index(2)].clone()))
        return {k: v[idx.index(2)] for k, v in out.items()}, xs
    (alone, ha), (many, hm) = run([2]), run([0, 1, 2, 3])
    for k in ("x", "f", "iters", "evals", "status", "metric_fallbacks"):
        assert torch.equal(alone[k], many[k]), k
    assert int(alone["iters"]) > 2 and all(torch.equal(u, v) for u, v in zip(ha, hm))


# ------------------------------------------------------------------------------------------------
# CurvatureMetric against the recording stand-in
# ------------------------------------------------------------------------------------------------
def _names(lib):
    return [c[0] for c in lib.calls if not c[0].endswith("_workspace_bytes")]


def _stages(lib):
    names = _names(lib)
    return [nm for k, nm in enumerate(names) if k == 0 or names[k - 1] != nm]


@pytest.fixture()
def metricfake(fake, monkeypatch):
    """The stand-in with n_out = 10 for every launched create_raceline track, dL/dalpha = 1 from the create_raceline
    adjoint, and the inputs of every mc_mincurv_adjoint_batch launch recorded in adj (dicts of numpy arrays)."""
    real = FakeLib.__getattr__
    fake.adj = []

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
        if name == "mc_mincurv_adjoint_batch":
            def mc(*a):
                fn(*a)
                bq, n = a[0], a[1]
                self.adj.append(dict(B=bq, n_pts=arr(a[2], ctypes.c_int32, bq),
                                     reftrack=arr(a[3], ctypes.c_double, bq * n * 4).reshape(bq, n, 4), w_veh=a[6],
                                     w_veh_batch=a[7], centre_id=arr(a[9], ctypes.c_int32, bq),
                                     sens=arr(a[10], ctypes.c_double, bq * 2 * n).reshape(bq, 2, n),
                                     grad_status=arr(a[11], ctypes.c_int32, bq),
                                     grad_alpha=arr(a[12], ctypes.c_double, bq * n).reshape(bq, n)))
                return 0
            return mc
        return fn
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    return fake


def _inputs(B=4, n=120):
    rt = torch.rand((B, n, 4), **F64) + 3.0
    return rt, torch.rand((B, n, 2), **F64), torch.zeros((B, n), **F64)


def test_the_metric_launches_one_adjoint_per_gradient_evaluation(metricfake):
    """One calc_splines; after every gradient evaluation one mc_mincurv_adjoint_batch call (two launches: the stand-in
    halves the batch of 2 B rows) with widths 1 / 1, w_veh 0, sens[:, 1] = 0, interleaved chunk-local centre ids and
    the gradient as the direction rows' right-hand side; a track shorter than N_MIN is never launched.  Lap times of 0
    (the stand-in writes none) pass no Armijo test: every line search is exhausted after the first gradient evaluation,
    so the second evaluation, and its metric call, launch for no track."""
    rt, nv, a0 = _inputs()
    npts = torch.tensor([120, 100, 60, 120], dtype=torch.int32)
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, n_pts=npts, max_halvings=2,
                                  metric_length=20.0)
    names = _names(metricfake)
    assert names.count("mc_calc_splines_batch") == 1
    stages = _stages(metricfake)
    grads = [k for k, nm in enumerate(stages) if nm == "mc_create_raceline_adjoint_batch"]
    assert len(grads) == 2 and [stages[k + 1] for k in grads] == ["mc_mincurv_adjoint_batch"] * 2
    assert stages.count("mc_mincurv_adjoint_batch") == 2
    assert len(metricfake.adj) == 4 and all(c["B"] == 4 for c in metricfake.adj)
    mu, pin = 20.0 ** -4, R.PIN_FACTOR * (20.0 ** -4 + 6.0)          # (the stand-in leaves h = 1)
    for k, c in enumerate(metricfake.adj):
        assert np.all(c["reftrack"][:, :, 2:] == 1.0) and c["w_veh"] == 0.0 and c["w_veh_batch"] is None
        assert np.array_equal(c["centre_id"], [0, 0, 2, 2])
        assert np.all(c["sens"][:, 1] == 0.0)
        first = k < 2                                    # the first call solves for g0 alone (no y rows)
        tracks = [2 * k, 2 * k + 1]
        for j, b in enumerate(tracks):
            want = int(npts[b]) if first and int(npts[b]) >= B_.N_MIN else 0
            assert c["n_pts"][2 * j] == want and c["n_pts"][2 * j + 1] == (0 if first else want)
            assert c["grad_status"][2 * j] == (0 if want else -1)
            assert np.all(c["sens"][2 * j + 1, 0] == mu)
            if want:
                assert np.all(c["grad_alpha"][2 * j, :want] == 1.0)
                assert set(np.unique(c["sens"][2 * j, 0, :want]).tolist()) <= {mu, pin}
    # the stand-in's solve writes zeros: u = 0 is no descent direction, every step is the identity one
    assert torch.equal(res["metric_fallbacks"], torch.tensor([1, 1, 1, 1], dtype=torch.int32))
    assert res["metric_fallbacks"].dtype == torch.int32


def test_no_launch_below_n_min_and_argument_errors(metricfake):
    rt, nv, a0 = _inputs(n=60)
    res = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, max_iters=2, max_halvings=1,
                                  metric_length=10.0)
    names = _names(metricfake)
    assert "mc_calc_splines_batch" not in names and "mc_mincurv_adjoint_batch" not in names
    assert res["metric_fallbacks"].tolist() == [1, 1, 1, 1]
    rt, nv, a0 = _inputs()
    for bad in (0.0, -5.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="metric_length"):
            R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, metric_length=bad)
    plain = R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, max_iters=1)
    assert "metric_fallbacks" not in plain


def test_globaltraj_batch_passes_metric_length_through(metricfake):
    rt, _, _ = _inputs(B=3, n=150)
    globaltraj.globaltraj_batch(rt, "mincurv", globaltraj.default_pars(), GGV, MACH,
                                refine=dict(max_iters=1, max_halvings=1, metric_length=15.0))
    assert "mc_mincurv_adjoint_batch" in _names(metricfake)
    assert np.all(metricfake.adj[0]["sens"][1::2, 0] == 15.0 ** -4)
    with pytest.raises(ValueError, match="metric_length"):
        globaltraj.globaltraj_batch(rt, "mincurv", globaltraj.default_pars(), GGV, MACH, refine=dict(metric_length=-1.0))
