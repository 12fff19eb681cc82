"""GPU tests (-m gpu) of the curvature-row interior-point iteration against its long-double replay (tests/ipm_rows_ref.py):
not only where the iteration ends but how it gets there, through the status and the iteration count.

A  the dense small-track kernel (mincurv_dense_kernel, opt_min_curv_batch(small_tracks=True) and _dense_below = 109) on
   3 .. 108 points (odd and even n, the ring wrap of n = 3 and 4, the trailing-update and warp-row boundaries at 16, 32,
   64) in four regimes (only the box binds, the rows bind, just feasible, just infeasible), uneven spacing, collapsed
   boxes, a narrower vehicle, f_scale 1, the LIN form and the named cases that reach each exit; per-track kb and w_veh.
   The same cases again in a ragged batch with n_max = 1000 (m < n_max) and with _dense_below = 90 (the banded path in
   the same launch): bit for bit.  Separately, kappa_lin_max and curv_error_max recomputed in long double at the
   device's own alpha (the finalize apart from the solve).
B  the banded curvature-row phase (mincurv_pdip_kappa_kernel<false>) on 80 .. 333 points against the replay with the
   cyclic band of half-width 32; its iteration count is the difference from the same batch at kb = 1e3 (the box phase
   is the same), and on 80 .. 108 points the dense kernel's count where band truncation does not move it.
C  the projection variant (mincurv_pdip_kappa_kernel<true>) through the call CurvatureProjection makes, at two mu.
Status: one of the replay runs' statuses, and also 0 or 2 where the last step was taken on a normal matrix that float64
cannot resolve (ipm_rows_ref.statuses).  Iterations: exact on the
count-stable cases (the three runs agree), within one of one of the runs elsewhere.  Every measured error is printed
next to its bound (pytest -s), and the number of exact iteration matches per section."""
import numpy as np
import pytest

import ipm_rows_ref as IR
import mincurv_ref as R

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402

# Bounds, about ten times the values measured on an H100 80GB HBM3 (700 W power limit) over the cases below:
# alpha against the long-double replay, max |d alpha| / max |alpha| over the status-0 cases: 7.8e-7 dense, 1.5e-6
# banded and projection (the replay stops where the kernels stop, at mu <= 1e-11 mu0, so this is the spread of the
# stopping iterate, not of the optimum); kappa_lin_max relative 1.4e-14 and curv_error_max relative to
# max(|curv_error_max|, 1e-3 kappa_lin_max) 3.3e-14, recomputed in long double at the device's alpha.
ALPHA_TOL = dict(dense=1e-5, banded=2e-5, prox=2e-5)
FIN_TOL = dict(klin=1e-13, cerr=3e-13)
DENSE_BELOW = B_.N_DENSE_MAX + 1


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def _pack(tracks, n_max=None):
    n = [t["rt"].shape[0] for t in tracks]
    n_max = n_max or max(n)
    rt, nv, h = np.zeros((len(tracks), n_max, 4)), np.zeros((len(tracks), n_max, 2)), np.ones((len(tracks), n_max))
    la = np.zeros((len(tracks), n_max))
    for b, t in enumerate(tracks):
        rt[b, :n[b]], nv[b, :n[b]], h[b, :n[b]] = t["rt"], t["nv"], t["h"]
        if t.get("lin_alpha") is not None:
            la[b, :n[b]] = t["lin_alpha"]
    return _dev(rt), _dev(nv), _dev(h), _dev(n, torch.int32), _dev(la)


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items()}


def _solve(tracks, kbs, n_max=None, **kw):
    rt, nv, h, npts, la = _pack(tracks, n_max)
    lin = tracks[0].get("lin_alpha") is not None
    return _np(B_.opt_min_curv_batch(rt, nv, h, _dev(kbs), _dev([t["w_veh"] for t in tracks]), n_pts=npts,
                                     f_scale=tracks[0]["f_scale"], lin_alpha=la if lin else None, **kw))


def _groups(cases):
    """case indices by (f_scale, LIN): one launch each"""
    g = {}
    for i, (_, t, _) in enumerate(cases):
        g.setdefault((t["f_scale"], t["lin_alpha"] is not None), []).append(i)
    return g.values()


def _dense_run(cases, pad=None, **kw):
    """per case dict(status, iters, alpha, klin, cerr); pad: a track appended to every launch"""
    out = [None] * len(cases)
    for idx in _groups(cases):
        tracks, kbs = [cases[i][1] for i in idx], [cases[i][2] for i in idx]
        if pad is not None:
            lin = None if tracks[0]["lin_alpha"] is None else np.zeros(pad["rt"].shape[0])
            tracks, kbs = tracks + [dict(pad, f_scale=tracks[0]["f_scale"], lin_alpha=lin)], kbs + [0.12]
        res = _solve(tracks, kbs, **kw)
        for b, i in enumerate(idx):
            n = cases[i][1]["rt"].shape[0]
            out[i] = dict(status=int(res["status"][b]), iters=int(res["iters"][b]), alpha=res["alpha"][b, :n],
                          rest=res["alpha"][b, n:], klin=float(res["kappa_lin_max"][b]), cerr=float(res["curv_error_max"][b]))
    return out


def _check_counts(name, got_status, got_iters, runs, stable, tally, bad):
    """the status and the iteration count of one case against the replay's three runs; a mismatch goes into bad"""
    st = {r["status"] for r in runs}
    ok = got_status in IR.statuses(runs)
    if stable:
        ok = ok and got_iters == runs[0]["iters"]
        tally[0] += ok
    elif st == {4} and runs[0]["exit"] == "cap":
        # rows that cannot be met: the long-double iterate diverges (mu beyond 1e30 mu0) and runs to the cap, and
        # float64 stops at a non-positive pivot some iterations later, when rounding has broken the growing weights;
        # that iteration is no decision of the method, so the count must only lie past the divergence
        div = next((k + 1 for k, t in enumerate(runs[0]["trace"]) if not t["mu"] < 1e30), IR.MAX_ITER + 20)
        ok = ok and got_iters >= div
        tally[2] += ok
    else:
        ok = ok and min(abs(got_iters - r["iters"]) for r in runs) <= 1
        tally[1] += ok
    if not ok:
        bad.append((name, got_status, got_iters, [(r["status"], r["iters"], r["exit"]) for r in runs], stable))


def _rel(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max() /
                 max(float(np.abs(np.asarray(b, dtype=np.float64)).max()), 1e-300))


@pytest.fixture(scope="module")
def dense():
    cases = IR.dense_cases()
    return cases, [IR.stability(t["d"], kb) for _, t, kb in cases]


def test_dense_kernel_against_the_replay(dense):
    cases, refs = dense
    got = _dense_run(cases, _dense_below=DENSE_BELOW)
    tally, worst, bad = [0, 0, 0], dict(alpha=0.0, klin=0.0, cerr=0.0), []
    for (name, t, kb), (r, stable, runs), g in zip(cases, refs, got):
        assert not g["rest"].any()
        print(f"{name}: status {g['status']} iters {g['iters']}  replay {[(x['status'], x['iters'], x['exit']) for x in runs]}"
              f"{'  count-stable' if stable else ''}")
        _check_counts(name, g["status"], g["iters"], runs, stable, tally, bad)
        if g["status"] == 0 and r["status"] == 0:
            e = _rel(g["alpha"], r["alpha"])
            print(f"    alpha {e:.2e} (bound {ALPHA_TOL['dense']:.0e})")
            if not e <= ALPHA_TOL["dense"]:
                bad.append((name, "alpha", e))
            worst["alpha"] = max(worst["alpha"], e)
        if np.isfinite(g["alpha"]).all():
            kl, ce, _ = IR.finalize(t["d"], g["alpha"])
            e_k = abs(g["klin"] - float(kl)) / float(kl)
            e_c = abs(g["cerr"] - float(ce)) / max(float(ce), 1e-3 * float(kl))
            print(f"    finalize: kappa_lin_max {e_k:.2e} (bound {FIN_TOL['klin']:.0e})  curv_error_max {e_c:.2e} "
                  f"(bound {FIN_TOL['cerr']:.0e})")
            if not (e_k <= FIN_TOL["klin"] and e_c <= FIN_TOL["cerr"]):
                bad.append((name, "finalize", e_k, e_c))
            worst["klin"], worst["cerr"] = max(worst["klin"], e_k), max(worst["cerr"], e_c)
    print(f"dense: exact iteration counts on {tally[0]} count-stable cases, within one on {tally[1]} others, past the divergence on {tally[2]}; worst {worst}")
    assert not bad, bad


def test_dense_kernel_in_ragged_and_mixed_batches(dense):
    cases, _ = dense
    base = _dense_run(cases, _dense_below=DENSE_BELOW)
    rt = synth.make_track(90, 1000)
    _, _, nv = R.periodic_spline(np.vstack((rt[:, :2], rt[:1, :2])))
    pad = dict(rt=rt, nv=nv, h=np.linalg.norm(np.diff(np.vstack((rt[:, :2], rt[:1, :2])), axis=0), axis=1), w_veh=2.0)
    for kw, keep in ((dict(_dense_below=DENSE_BELOW), lambda n: True), (dict(_dense_below=90), lambda n: n < 90)):
        other = _dense_run(cases, pad=pad, **kw)
        same = 0
        for (name, t, _), a, b in zip(cases, base, other):
            if not keep(t["rt"].shape[0]):
                continue
            assert a["status"] == b["status"] and a["iters"] == b["iters"], (name, kw)
            assert np.array_equal(a["alpha"], b["alpha"], equal_nan=True) and not b["rest"].any(), (name, kw)
            assert np.array_equal([a["klin"], a["cerr"]], [b["klin"], b["cerr"]], equal_nan=True), (name, kw)
            same += 1
        print(f"n_max 1000, {kw}: {same} cases bit for bit")


def test_banded_row_phase_against_the_replay():
    cases = IR.banded_cases()
    tracks, kbs = [t for _, t, _ in cases], [kb for _, _, kb in cases]
    res = _solve(tracks, kbs)
    box = _solve(tracks, [1e3] * len(cases))
    small = [i for i, t in enumerate(tracks) if t["rt"].shape[0] <= B_.N_DENSE_MAX]
    den = _solve([tracks[i] for i in small], [kbs[i] for i in small], _dense_below=DENSE_BELOW)
    tally, same_dense, bad = [0, 0, 0], 0, []
    for b, (name, t, kb) in enumerate(cases):
        r, stable, runs = IR.stability(t["d"], kb, band=IR.HBW, override="banded")
        rows_it = int(res["iters"][b]) - int(box["iters"][b])
        print(f"{name}: status {res['status'][b]} row iterations {rows_it} (box {box['iters'][b]})  replay "
              f"{[(x['status'], x['iters'], x['exit']) for x in runs]}{'  count-stable' if stable else ''}")
        assert box["status"][b] == 0
        _check_counts(name, int(res["status"][b]), rows_it, runs, stable, tally, bad)
        n = t["rt"].shape[0]
        if res["status"][b] == 0 and r["status"] == 0:
            e = _rel(res["alpha"][b, :n], r["alpha"])
            print(f"    alpha {e:.2e} (bound {ALPHA_TOL['banded']:.0e})")
            if not e <= ALPHA_TOL["banded"]:
                bad.append((name, "alpha", e))
        if b in small:
            full = IR.replay(t["d"], kb)
            k = small.index(b)
            if stable and full["iters"] == r["iters"] and full["status"] == r["status"]:
                if int(den["iters"][k]) != rows_it:
                    bad.append((name, "dense", int(den["iters"][k]), rows_it))
                same_dense += 1
    print(f"banded: exact row-phase counts on {tally[0]} count-stable cases, within one on {tally[1]} others; "
          f"dense = banded on {same_dense}")
    assert not bad, bad


def _prox(tracks, kbs, mu, xs, qs):
    rt, nv, h, npts, _ = _pack(tracks)
    B, n_max = h.shape
    kb, kbb = B_._kappa_bound(_dev(kbs), B, h.device)
    x, q = np.zeros((B, n_max)), np.zeros((B, n_max))
    for b, t in enumerate(tracks):
        n = t["rt"].shape[0]
        x[b, :n], q[b, :n] = xs[b], qs[b]
    out = B_._mincurv_results(B, n_max, h.device)
    chunk = B_._chunk(B, _lib.load().mc_mincurv_workspace_bytes(1, n_max), h.device)
    ws = B_._workspace("mincurv", _lib.load().mc_mincurv_workspace_bytes(chunk, n_max), h.device)
    B_._launch_chunks("mc_mincurv_solve_batch_ex", B, chunk, ws, n_max, *map(B_._rows, (npts, rt, nv, h)), kb, 2.0,
                      None, B_.F_SCALE, *map(B_._rows, out.values()), mu, B_._rows(_dev(x)), B_._rows(_dev(q)), None,
                      B_._rows(kbb), *(None,) * 5, 0)
    return _np(out)


# On the 200-point cases the last step is taken on a normal matrix with lambda_min / lambda_max ~ 4e-17 (below the
# float64 epsilon): the kernel ends at the replay's count with status 2 (mu floor, |r_d| 5.5e3 rd_tol) where the
# replay's factorisations leave |r_d| at 1.7e-2 rd_tol (IR.statuses admits both).
@pytest.mark.parametrize("n", [120, 200])
def test_projection_row_phase_against_the_replay(n):
    cases = [c for c in IR.prox_cases() if c[1]["rt"].shape[0] == n]
    tally, bad = [0, 0, 0], []
    for mu in sorted({c[3] for c in cases}):
        cs = [c for c in cases if c[3] == mu]
        tracks, kbs, xs, qs = [c[1] for c in cs], [c[2] for c in cs], [c[4] for c in cs], [c[5] for c in cs]
        res = _prox(tracks, kbs, mu, xs, qs)
        box = _prox(tracks, [1e3] * len(cs), mu, xs, qs)
        for b, (name, t, kb, _, x, q) in enumerate(cs):
            r, stable, runs = IR.stability(t["d"], kb, band=IR.HBW, override="banded", prox_mu=mu, prox_x=x, prox_q=q)
            rows_it = int(res["iters"][b]) - int(box["iters"][b])
            print(f"{name} (mu {mu:.2e}): status {res['status'][b]} row iterations {rows_it}  replay "
                  f"{[(y['status'], y['iters'], y['exit']) for y in runs]}{'  count-stable' if stable else ''}")
            assert box["status"][b] == 0
            _check_counts(name, int(res["status"][b]), rows_it, runs, stable, tally, bad)
            n = t["rt"].shape[0]
            if res["status"][b] == 0 and r["status"] == 0:
                e = _rel(res["alpha"][b, :n], r["alpha"])
                print(f"    alpha {e:.2e} (bound {ALPHA_TOL['prox']:.0e})")
                if not e <= ALPHA_TOL["prox"]:
                    bad.append((name, "alpha", e))
    print(f"projection: exact row-phase counts on {tally[0]} count-stable cases, within one on {tally[1]} others")
    assert not bad, bad
