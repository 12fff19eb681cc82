"""GPU tests of the lap-time refinement on closed tracks below N_MIN points (refine_raceline_batch(small_tracks=True);
DESIGN.md sections 3.13 and 3.14): the dense projection (mc_mincurv_solve_batch_ex(prox_x, prox_dense_below)) against
the long-double replay of its iteration (tests/ipm_rows_ref.py) and against the Goldfarb-Idnani KKT point; dense against
banded projection, metric and evaluation on 80 .. 108 points (_dense_below); the dense metric solve (the dense adjoint of
mc_mincurv_adjoint_batch, about the linearisation line), with pins, against an extended-precision solve of the QP's own
linearised E; the dense evaluation (mc_mincurv_finalize_batch(dense_below)) against the long-double finalize; the refinement end to end on karting tracks (synthetic
ones and the handling track thinned below 80 points) in the metric, under a curvature limit and with re-linearisation;
batch independence in a ragged batch of short and long tracks; no stream synchronisation; globaltraj_batch with the
flag on both stages."""
import numpy as np
import pytest
import torch

import ipm_rows_ref as IR
from global_racetrajectory_optimization_b200 import batch as B_, globaltraj, raceline_refine as R, synth
from test_gpu_ipm_rows_edges import _check_counts, _pack, _rel
from test_gpu_raceline_refine_metric import _fresh, _veh
from test_raceline_refine_small_host import _gi, small_prox_cases

pytestmark = pytest.mark.gpu
DEV = "cuda"
STEP = 2.0
ELL = 10.0
KAPPA_REL = 1e-7            # the finalize stage's acceptance of |k_ref + E alpha| <= kappa_bound
DENSE_BELOW = B_.N_DENSE_MAX + 1
# Bounds, about ten times the values measured on an H100 80GB HBM3 (700 W power limit) over the cases below (pytest -s
# prints each next to its bound):
ALPHA_TOL = 1e-5            # projection alpha against the replay, max |d alpha| / max |alpha| (the stopping iterate)
GI_TOL = 1e-5               # ... against the Goldfarb-Idnani solution, relative to max(|y|, 1e-3 m)
FIN_TOL = dict(klin=1e-13, cerr=3e-13)      # the device's kappa_lin_max / curv_error_max at its alpha, long double
METRIC_TOL = 1e-10          # the metric solve against long double, relative to max |v|
SPLIT_TOL = dict(alpha=2e-5, metric=1e-9, klin=1e-12, cerr=1e-11)     # dense against banded on 80 .. 108 points


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def _rows(vals, n_max):
    out = np.zeros((len(vals), n_max))
    for b, v in enumerate(vals):
        out[b, :len(v)] = v
    return _dev(out)


def _dense_prox(tracks, kbs, mu, xs, qs, lin):
    rt, nv, h, npts, la = _pack(tracks)
    B, n_max = h.shape
    out = B_._mincurv_results(B, n_max, h.device)
    B_._call("mc_mincurv_solve_batch_ex", B, n_max, npts, rt, nv, h, 0.0, 0.0, _dev([t["w_veh"] for t in tracks]),
             B_.F_SCALE, *out.values(), mu, _rows(xs, n_max), _rows(qs, n_max), la if lin else None, _dev(kbs),
             *(None,) * 5, 0, DENSE_BELOW, None, 0)
    return {k: v.cpu().numpy() for k, v in out.items()}


# ------------------------------------------------------------------------------------------------
# the projection QP against its replay and the KKT point
# ------------------------------------------------------------------------------------------------
def test_the_dense_projection_against_the_replay_and_the_kkt_point():
    cases = small_prox_cases()
    groups = {}
    for i, c in enumerate(cases):
        groups.setdefault((c[3], c[1]["lin_alpha"] is not None), []).append(i)
    tally, bad, worst = [0, 0, 0], [], dict(alpha=0.0, gi=0.0, klin=0.0, cerr=0.0)
    for (mu, lin), idx in groups.items():
        cs = [cases[i] for i in idx]
        res = _dense_prox([c[1] for c in cs], [c[2] for c in cs], mu, [c[4] for c in cs], [c[5] for c in cs], lin)
        for b, (name, t, kb, _, x, q) in enumerate(cs):
            n = t["d"]["n"]
            r, stable, runs = IR.stability(t["d"], kb, prox_mu=mu, prox_x=x, prox_q=q)
            st, it, a = int(res["status"][b]), int(res["iters"][b]), res["alpha"][b, :n]
            print(f"{name}: status {st} iters {it}  replay {[(y['status'], y['iters'], y['exit']) for y in runs]}"
                  f"{'  count-stable' if stable else ''}")
            assert not res["alpha"][b, n:].any()
            _check_counts(name, st, it, runs, stable, tally, bad)
            assert st == 0, name
            e = _rel(a, r["alpha"])
            y = _gi(t, kb, mu, x, q)
            e_gi = float(np.abs(a - y).max() / max(np.abs(y).max(), 1e-3))
            kl, ce, _ = IR.finalize(t["d"], a)
            e_k = abs(float(res["kappa_lin_max"][b]) - float(kl)) / float(kl)
            e_c = abs(float(res["curv_error_max"][b]) - float(ce)) / max(float(ce), 1e-3 * float(kl))
            print(f"    alpha {e:.2e} (bound {ALPHA_TOL:.0e})  GI {e_gi:.2e} (bound {GI_TOL:.0e})  kappa_lin_max "
                  f"{e_k:.2e}  curv_error_max {e_c:.2e}")
            for k, v, tol in (("alpha", e, ALPHA_TOL), ("gi", e_gi, GI_TOL), ("klin", e_k, FIN_TOL["klin"]),
                              ("cerr", e_c, FIN_TOL["cerr"])):
                worst[k] = max(worst[k], v)
                if not v <= tol:
                    bad.append((name, k, v))
            assert float(res["kappa_lin_max"][b]) <= kb * (1 + KAPPA_REL)
    print(f"dense projection: exact counts on {tally[0]} count-stable cases, within one on {tally[1]}; worst {worst}")
    assert not bad, bad


def test_the_dense_evaluation_against_the_long_double_finalize():
    """mc_mincurv_finalize_batch(dense_below) at alpha off the solution (a line through the box, with and without LIN) against the
    long-double finalize, the status-4 rule at a limit just below and above kappa_lin_max, and its refusals."""
    cases = [("synth5", IR.track(synth.make_track(2, 5), w_veh=0.5)), ("synth40", IR.track(synth.make_track(3, 40))),
             ("lin_n33", IR.track(synth.make_track(4, 33), lin_alpha=IR.lin_line(33))),
             ("collapsed64", IR.track(IR.collapsed(64)))]
    worst = [0.0, 0.0]
    for name, t in cases:
        d = t["d"]
        n = d["n"]
        x = np.clip(0.4 * np.sin(np.arange(n) * 0.7), d["lb"].astype(np.float64), d["ub"].astype(np.float64))
        kl, ce, _ = IR.finalize(d, x)
        rt, nv, h, npts, la = _pack([t, t, t, t])
        kbs = _dev([float(kl) * (1 - 1e-6), float(kl) * (1 + 1e-6), -1.0, float("nan")])
        cerr, kmax = torch.empty(4, dtype=torch.float64, device=DEV), torch.empty(4, dtype=torch.float64, device=DEV)
        st = torch.full((4,), 77, dtype=torch.int32, device=DEV)
        lin = t["lin_alpha"] is not None
        B_._call("mc_mincurv_finalize_batch", 4, n, npts, _rows([x] * 4, n), 0.0, cerr, kmax, st, int(lin), kbs, rt, nv,
                 h, 0.0, _dev([t["w_veh"]] * 4), la if lin else None, DENSE_BELOW, None, 0)
        e_k = abs(float(kmax[0]) - float(kl)) / float(kl)
        e_c = abs(float(cerr[0]) - float(ce)) / max(float(ce), 1e-3 * float(kl))
        print(f"EVAL {name}: kappa_lin_max {e_k:.2e} (bound {FIN_TOL['klin']:.0e}), curv_error_max {e_c:.2e} "
              f"(bound {FIN_TOL['cerr']:.0e}), status {st.tolist()}")
        assert e_k <= FIN_TOL["klin"] and e_c <= FIN_TOL["cerr"], name
        assert st.tolist() == [4, 0, -1, -1] and kmax[2:].tolist() == [0.0, 0.0] and cerr[2:].tolist() == [0.0, 0.0]
        assert torch.equal(kmax[0], kmax[1]) and torch.equal(cerr[0], cerr[1])
        worst = [max(worst[0], e_k), max(worst[1], e_c)]
    print(f"EVAL worst {worst}")


# ------------------------------------------------------------------------------------------------
# the metric solve
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lin", [False, True])
def test_the_dense_metric_solve_against_long_double(lin):
    """v = (E^T E + diag(d))^-1 r on 3 .. 79 points through the call CurvatureMetric makes (the dense adjoint with zero
    row weights; with lin_alpha about the line P + lin_alpha n as the centre line) against the long-double Cholesky solve
    with the QP's own E (linearised about lin_alpha), with d = l^-4 (no pins), with random pins (d = CurvatureMetric's
    pin value there) and with a single free point."""
    worst = 0.0
    rng = np.random.default_rng(5)
    for n in (3, 4, 7, 16, 33, 64, 79):
        t = IR.track(synth.make_track(50 + n, n), lin_alpha=IR.lin_line(n) if lin else None)
        d = t["d"]
        E = d["E"]
        mu = ELL ** -4
        pin = R.PIN_FACTOR * (mu + 6.0 / float(np.min(t["h"])) ** 4)
        diags = dict(none=np.full(n, mu), random=np.where(rng.random(n) < 0.3, pin, mu),
                     one_free=np.where(np.arange(n) == n // 2, mu, pin))
        rs = [rng.standard_normal(n) for _ in diags]
        line = t["rt"][:, :2] + (0.0 if t["lin_alpha"] is None else t["lin_alpha"][:, None] * t["nv"])
        rt, nv, h, npts, _ = _pack([dict(t, rt=np.hstack((line, np.ones((n, 2))))) for _ in diags])
        k = len(diags)
        dg = _rows(list(diags.values()), n)
        sens = torch.stack((dg, torch.zeros_like(dg)), dim=1).contiguous()
        gs = torch.zeros((k,), dtype=torch.int32, device=DEV)
        u, gwl = torch.empty((k, n), dtype=torch.float64, device=DEV), torch.empty((k, n), dtype=torch.float64, device=DEV)
        gwv = torch.empty((k,), dtype=torch.float64, device=DEV)
        B_._call("mc_mincurv_adjoint_batch", k, n, npts, rt, nv, h, 0.0, None, B_.F_SCALE, None, sens, gs, _rows(rs, n), u,
                 gwl, gwv, torch.zeros_like(dg), torch.zeros((k,), dtype=torch.int32, device=DEV),
                 torch.zeros((1,), dtype=torch.float64, device=DEV), 0, None, DENSE_BELOW, None, 0)
        assert gs.tolist() == [0] * k
        v = u / dg
        for k, (name, dg) in enumerate(diags.items()):
            K = E.T @ E + np.diag(IR.S.ld(dg))
            ref = IR._chol_solve(IR._chol(K), IR.S.ld(rs[k])).astype(np.float64)
            e = _rel(v[k].cpu().numpy(), ref)
            print(f"METRIC n {n} lin {lin} {name}: {e:.2e} (bound {METRIC_TOL:.0e})")
            assert e <= METRIC_TOL, (n, name)
            worst = max(worst, e)
    print(f"METRIC worst {worst:.2e}")


# ------------------------------------------------------------------------------------------------
# dense against banded on 80 .. 108 points
# ------------------------------------------------------------------------------------------------
def _split_tracks():
    n_all = (80, 93, 108)
    rts = [synth.make_track(70 + n, n) for n in n_all]
    rt = torch.zeros((3, max(n_all), 4), dtype=torch.float64, device=DEV)
    for b, r in enumerate(rts):
        rt[b, :r.shape[0]] = _dev(r)
    npts = torch.tensor(n_all, dtype=torch.int32, device=DEV)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    lb, ub, _ = R.box(rt, 2.0, npts)
    i = torch.arange(rt.shape[1], device=DEV, dtype=torch.float64)[None]
    x = torch.where(i < npts[:, None], 0.5 * (lb + ub) + 0.45 * (ub - lb) * torch.sin(0.9 * i), 0.0)
    q = torch.where(i < npts[:, None], 1e-3 * torch.cos(0.21 * i), 0.0)
    return rt, nv, npts, x, q


@pytest.mark.parametrize("lin", [False, True])
def test_dense_against_banded_on_80_to_108_points(lin):
    rt, nv, npts, x, q = _split_tracks()
    la = (0.2 * torch.sin(0.37 * torch.arange(rt.shape[1], device=DEV, dtype=torch.float64)))[None].repeat(3, 1) \
        if lin else None
    mask = torch.ones(3, dtype=torch.bool, device=DEV)
    _, _, _, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    a_box = B_.opt_min_curv_batch(rt, nv, h, 1e3, 2.0, n_pts=npts, lin_alpha=la)["alpha"]
    kb = 1.2 * R.CurvatureProjection(rt, nv, npts, 2.0, 1e3, ELL, lin_alpha=la).kappa_lin(a_box, mask)  # (x is beyond)
    out = {}
    for db in (0, DENSE_BELOW):
        prj = R.CurvatureProjection(rt, nv, npts, 2.0, kb, ELL, lin_alpha=la, dense_below=db)
        met = R.CurvatureMetric(rt, nv, npts, ELL, lin_alpha=la, dense_below=db)
        pin = torch.rand(x.shape, device=DEV, generator=torch.Generator(DEV).manual_seed(2)) < 0.2
        y, ok = prj(x, q, mask)
        u, w, okm = met(q, pin, x, mask)
        out[db] = dict(y=y, ok=ok, u=torch.where(pin, 0.0, u), w=w, okm=okm, prj=prj)
    a, b = out[0], out[DENSE_BELOW]
    for r in (a, b):                                    # (the evaluations at one alpha: the banded projection's)
        r["kl"], r["ce"] = r["prj"].evaluate(a["y"], mask)
    assert a["ok"].tolist() == b["ok"].tolist() == [True] * 3 and a["okm"].tolist() == b["okm"].tolist() == [True] * 3
    for k in range(3):
        n = int(npts[k])
        e = dict(alpha=_rel(b["y"][k, :n].cpu(), a["y"][k, :n].cpu()),
                 metric=max(_rel(b["u"][k, :n].cpu(), a["u"][k, :n].cpu()), _rel(b["w"][k, :n].cpu(), a["w"][k, :n].cpu())),
                 klin=abs(float(b["kl"][k] / a["kl"][k]) - 1.0), cerr=abs(float(b["ce"][k] / a["ce"][k]) - 1.0))
        print(f"SPLIT n {n} lin {lin}: " + ", ".join(f"{k2} {v:.2e} (bound {SPLIT_TOL[k2]:.0e})" for k2, v in e.items()))
        assert all(v <= SPLIT_TOL[k2] for k2, v in e.items()), (n, e)
        assert float(b["prj"].kappa_lin(b["y"], mask)[k]) <= float(kb[k]) * (1 + KAPPA_REL)


# ------------------------------------------------------------------------------------------------
# the refinement end to end
# ------------------------------------------------------------------------------------------------
def _karting(golden):
    """Five short closed tracks: synthetic ones of 24, 40, 64 and 79 points (widths at least 2 m a side) and the handling
    track thinned to fewer than 80 points.  Returns (rt, nv, npts, names)."""
    tracks = []
    for n in (24, 40, 64, 79):
        r = synth.make_track(80 + n, n)
        r[:, 2:] = np.maximum(r[:, 2:], 2.0)
        tracks.append((f"synth{n}", r))
    hd = golden("handling")["reftrack"]
    step = -(-hd.shape[0] // 70)
    tracks.append((f"handling/{step}", hd[::step]))
    n_max = max(r.shape[0] for _, r in tracks)
    rt = torch.zeros((len(tracks), n_max, 4), dtype=torch.float64, device=DEV)
    for b, (_, r) in enumerate(tracks):
        rt[b, :r.shape[0]] = _dev(r)
    npts = torch.tensor([r.shape[0] for _, r in tracks], dtype=torch.int32, device=DEV)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    return rt, nv, npts, [nm for nm, _ in tracks]


def _start(rt, nv, npts, kb):
    _, _, _, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    return B_.opt_min_curv_batch(rt, nv, h, kb, 2.0, n_pts=npts, small_tracks=True)


@pytest.mark.parametrize("form", ["metric", "kappa", "relinearise"])
def test_the_refinement_on_karting_tracks(golden, form):
    veh = _veh(golden)
    rt, nv, npts, names = _karting(golden)
    B = rt.shape[0]
    mask = torch.ones(B, dtype=torch.bool, device=DEV)
    box_k = R.CurvatureProjection(rt, nv, npts, 2.0, 1e3, ELL, small_tracks=True).kappa_lin(
        _start(rt, nv, npts, 1e3)["alpha"], mask)
    kb = 0.97 * box_k                                          # (binding at the QP's own optimum)
    qp = _start(rt, nv, npts, kb if form != "metric" else 1e3)
    assert qp["status"].tolist() == [0] * B, qp["status"].tolist()
    al = qp["alpha"]
    xs = []
    kw = dict(metric_length=ELL, max_iters=25)
    if form != "metric":
        kw["kappa_bound"] = kb
    if form == "relinearise":
        kw["relinearise"] = 2
    res = R.refine_raceline_batch(rt, nv, al, 2.0, n_pts=npts, stepsize_interp=STEP, small_tracks=True,
                                  callback=lambda it, x, f, st: xs.append(x.clone()), **kw, **veh)
    ident = R.refine_raceline_batch(rt, nv, al, 2.0, n_pts=npts, stepsize_interp=STEP, max_iters=25, **veh)
    for b, nm in enumerate(names):
        print(f"SMALL REFINE {form} {nm} (n {int(npts[b])}): laptime {float(res['laptime_start'][b]):.6f} -> "
              f"{float(res['laptime'][b]):.6f} s (identity {float(ident['laptime'][b]):.6f}), iters "
              f"{int(res['iters'][b])}, status {int(res['status'][b])}, "
              + (f"metric_fallbacks {int(res['metric_fallbacks'][b])}" if form == "metric" else
                 f"kappa_lin_max / kb {float(res['kappa_lin_max'][b] / kb[b]):.9f}, rounds {int(res['rounds'][b])}, "
                 f"curv_error_max {float(res['curv_error_max'][b]):.2e}"))
    assert bool((res["iters"] > 0).all())
    assert bool((res["laptime"] <= res["laptime_start"]).all())
    assert bool((res["laptime"] < res["laptime_start"]).any())
    # (after a re-linearisation a track may stop with NO_PROJECTION: the set about the new line may hold no descent
    # direction, or not its start, whose round is then not taken; the banded path does the same)
    done = [R.CONVERGED, R.ITER_CAP, R.LINE_SEARCH] + ([R.NO_PROJECTION] if form == "relinearise" else [])
    assert bool(torch.isin(res["status"], torch.tensor(done, device=DEV)).all())
    lb, ub, _ = R.box(rt, 2.0, npts)
    valid = torch.arange(rt.shape[1], device=DEV)[None] < npts[:, None]
    for x in xs + [res["alpha"]]:
        assert bool(((x >= lb) & (x <= ub) | ~valid).all())
    if form == "metric":
        assert res["metric_fallbacks"].tolist() == [0] * B
    else:
        assert bool((res["kappa_lin_max"] <= kb * (1 + KAPPA_REL)).all())
        if form == "kappa":                                   # every accepted iterate in P about the centre line
            assert int(res["projection_failures"].sum()) == 0
            prj = R.CurvatureProjection(rt, nv, npts, 2.0, kb, ELL, small_tracks=True)
            worst = max(float((prj.kappa_lin(x, mask) / kb).max()) for x in xs) - 1.0
            print(f"SMALL REFINE kappa: the iterates' largest kappa_lin_max / kb - 1 {worst:.2e}")
            assert worst <= KAPPA_REL
        else:
            assert bool((res["rounds"] >= 1).any())
    lap, _ = _fresh(rt, nv, res["alpha"], npts, veh)
    assert torch.equal(lap, res["laptime"])


def test_a_ragged_batch_of_short_and_long_tracks(golden):
    """Each short track bit for bit as refined alone, each long one bit for bit as with small_tracks=False."""
    veh = _veh(golden)
    rt_s, nv_s, np_s, _ = _karting(golden)
    g = golden("handling")
    n_long = g["reftrack"].shape[0]
    B = rt_s.shape[0] + 2
    rt = torch.zeros((B, n_long, 4), dtype=torch.float64, device=DEV)
    rt[0] = rt[B - 1] = _dev(g["reftrack"])
    rt[B - 1, :, 2:] *= 1.1
    rt[1:B - 1, :rt_s.shape[1]] = rt_s
    npts = torch.cat((torch.tensor([n_long], device=DEV, dtype=torch.int32), np_s,
                      torch.tensor([n_long], device=DEV, dtype=torch.int32)))
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    qp = _start(rt, nv, npts, 1e3)
    box_k = R.CurvatureProjection(rt, nv, npts, 2.0, 1e3, ELL, small_tracks=True).kappa_lin(
        qp["alpha"], torch.ones(B, dtype=torch.bool, device=DEV))
    kb = 0.97 * box_k
    al = _start(rt, nv, npts, kb)["alpha"]
    kw = dict(n_pts=npts, stepsize_interp=STEP, metric_length=ELL, max_iters=8, relinearise=1, **veh)
    res = R.refine_raceline_batch(rt, nv, al, 2.0, kappa_bound=kb, small_tracks=True, **kw)
    old = R.refine_raceline_batch(rt, nv, al, 2.0, kappa_bound=kb, **kw)
    keys = ("alpha", "laptime", "laptime_start", "iters", "status", "evals", "pg_norm", "kappa_lin_max", "kappa_max",
            "curv_error_max", "projection_failures", "rounds")
    for b in (0, B - 1):
        for k in keys:
            assert torch.equal(res[k][b], old[k][b]), (b, k)
    for b in range(1, B - 1):
        n = int(npts[b])
        one = R.refine_raceline_batch(rt[b:b + 1, :n].contiguous(), nv[b:b + 1, :n].contiguous(), al[b:b + 1, :n].contiguous(),
                                      2.0, kappa_bound=kb[b:b + 1], small_tracks=True,
                                      **dict(kw, n_pts=npts[b:b + 1]))
        assert int(old["status"][b]) == R.NO_PROJECTION
        for k in keys:
            got = res[k][b, :n] if k == "alpha" else res[k][b]
            assert torch.equal(got, one[k][0]), (b, k)
        assert not bool(res["alpha"][b, n:].any())
    print(f"RAGGED: short tracks {res['status'][1:B - 1].tolist()} iters {res['iters'][1:B - 1].tolist()}")


def test_the_metric_and_the_projection_do_not_synchronise_the_stream(golden):
    for n_max_long in (False, True):
        rt_s, nv_s, npts, _ = _karting(golden)
        if n_max_long:                                      # a mixed batch: banded and dense launches
            g = golden("handling")
            n_long = g["reftrack"].shape[0]
            rt = torch.zeros((rt_s.shape[0] + 1, n_long, 4), dtype=torch.float64, device=DEV)
            rt[0] = _dev(g["reftrack"])
            rt[1:, :rt_s.shape[1]] = rt_s
            npts = torch.cat((torch.tensor([n_long], device=DEV, dtype=torch.int32), npts))
            _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
        else:
            rt, nv = rt_s, nv_s
        B, n_max = rt.shape[:2]
        mask = torch.ones(B, dtype=torch.bool, device=DEV)
        x = _start(rt, nv, npts, 1e3)["alpha"]
        q = 1e-3 * torch.randn(x.shape, dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(3))
        q = torch.where(torch.arange(n_max, device=DEV)[None] < npts[:, None], q, 0.0)
        prj = R.CurvatureProjection(rt, nv, npts, 2.0, 0.5, ELL, small_tracks=True)
        met = R.CurvatureMetric(rt, nv, npts, ELL, small_tracks=True)
        pin = torch.zeros_like(x, dtype=torch.bool)
        prj(x, q, mask), met(q, pin, q, mask), prj.evaluate(x, mask)         # (warm)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y, ok = prj(x, q, mask)
            u, w, okm = met(q, pin, q, mask)
            kl, _ = prj.evaluate(y, mask)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert ok.tolist() == okm.tolist() == [True] * B and bool(torch.isfinite(kl).all())


def test_globaltraj_batch_refines_short_tracks_with_both_flags(golden):
    g = golden("velprofile")
    rts = []
    for n in (30, 50, 70):
        r = synth.make_track(120 + n, n)
        r[:, 2:] = np.maximum(r[:, 2:], 2.5)
        rts.append(r)
    rt = torch.zeros((3, 70, 4), dtype=torch.float64, device=DEV)
    for b, r in enumerate(rts):
        rt[b, :r.shape[0]] = _dev(r)
    npts = torch.tensor([30, 50, 70], dtype=torch.int32, device=DEV)
    pars = globaltraj.default_pars()
    base = globaltraj.globaltraj_batch(rt, "mincurv", pars, g["ggv"], g["ax_max_machines"], n_pts=npts,
                                       small_tracks=True, check=False)
    opts = dict(max_iters=10, metric_length=ELL, kappa_bound=0.12)
    res = globaltraj.globaltraj_batch(rt, "mincurv", pars, g["ggv"], g["ax_max_machines"], n_pts=npts, small_tracks=True,
                                      check=False, refine=dict(opts, small_tracks=True))
    without = globaltraj.globaltraj_batch(rt, "mincurv", pars, g["ggv"], g["ax_max_machines"], n_pts=npts,
                                          small_tracks=True, check=False, refine=opts)
    print(f"GLOBALTRAJ small: qp status {base['status'].tolist()}, laptime {base['laptime'].tolist()} -> "
          f"{res['laptime'].tolist()}, refine_status {res['refine_status'].tolist()} iters {res['refine_iters'].tolist()}"
          f"; without the refinement's flag {without['refine_status'].tolist()}")
    assert base["status"].tolist() == [0, 0, 0]
    assert torch.equal(res["qp_alpha"], base["alpha"])
    assert bool((res["refine_iters"] > 0).all())
    assert bool((res["laptime"] <= res["laptime_start"]).all()) and bool((res["laptime"] < res["laptime_start"]).any())
    assert without["refine_status"].tolist() == [R.NO_PROJECTION] * 3
