"""CPU tests (-m "not gpu") of the lap-time refinement on closed tracks below N_MIN points (refine_raceline_batch(
small_tracks=True)): the MC_OPTIONAL6 groups of mc_mincurv_solve_batch_ex and mc_mincurv_finalize_batch as the
binding reads them, their argument checks in the real library before any CUDA call, the calls of CurvatureMetric,
CurvatureProjection and refine_raceline_batch against the recording stand-in of the library (only the dense calls below
N_MIN, banded then dense in a mixed batch, today's calls without the flag), and the long-double replay of the projection QP
(tests/ipm_rows_ref.py) on short tracks against the Goldfarb-Idnani solution of tests/prox_ref.py."""
import ctypes

import numpy as np
import pytest
import torch

import ipm_rows_ref as IR
import prox_ref
from fake_lib import FakeLib, fake  # noqa: F401  (fake: the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_, raceline_refine as R, synth

F64 = dict(dtype=torch.float64)
GGV = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.0], [80.0, 5.0]])
ENTRIES = ("mc_mincurv_solve_batch_ex", "mc_mincurv_adjoint_batch", "mc_mincurv_setup_batch_ex", "mc_mincurv_finalize_batch")


def test_the_dense_groups_are_parsed_from_the_header():
    """prox_dense_below on mc_mincurv_solve_batch_ex and the dense evaluation's group on mc_mincurv_finalize_batch, both
    MC_OPTIONAL6 after every earlier group; no new entry point, and the adjoint keeps its 25 parameters."""
    i, d, p = ctypes.c_int, ctypes.c_double, ctypes.c_void_p
    assert _lib._OPTIONAL6 == {"mc_mincurv_solve_batch_ex": (26, 1), "mc_mincurv_finalize_batch": (10, 7)}
    assert _lib._SIGS["mc_mincurv_solve_batch_ex"][1][25:] == [i, i, p, ctypes.c_size_t, p]
    assert _lib._SIGS["mc_mincurv_finalize_batch"][1][8:] == [i, p, p, p, p, d, p, p, i, p, ctypes.c_size_t, p]
    assert len(_lib._SIGS["mc_mincurv_adjoint_batch"][1]) == 25 and not any("dense" in k for k in _lib.EXPORTED_SYMBOLS)


def _ex(d, **kw):
    """mc_mincurv_solve_batch_ex's arguments for the dense projection (ws NULL)"""
    a = dict(B=1, n_max=40, n_pts=None, rt=d, nv=d, h=d, kb=0.12, wv=2.0, wvb=None, fs=2.0, alpha=d, cerr=d, kmax=None,
             status=d, iters=None, mu=1e-4, x=d, q=d, lin=None, kbb=None, cid=None, sens=None, gs=None, srows=None,
             nrows=None, dense=0, prox_dense=B_.N_MIN, ws=None, wsb=0, stream=None)
    a.update(kw)
    return list(a.values())


def _fin(d, **kw):
    """mc_mincurv_finalize_batch's arguments for the dense evaluation (ws NULL)"""
    a = dict(B=1, n_max=40, n_pts=None, alpha=d, kb=0.12, cerr=d, kmax=d, status=d, lin_flag=0, kbb=None, rt=d, nv=d, h=d,
             wv=2.0, wvb=None, lin=None, dense=B_.N_MIN, ws=None, wsb=0, stream=None)
    a.update(kw)
    return list(a.values())


@pytest.mark.parametrize("entry", ["mc_mincurv_solve_batch_ex", "mc_mincurv_finalize_batch"])
def test_the_real_library_refuses_before_any_cuda_call(entry):
    """The dense groups outside [N_MIN, MC_DENSE_N_MAX + 1], B or n_max <= 0 and NULL inputs or outputs are refused with
    MC_EINVAL and a message naming the entry (no device is touched: the checks come first); the earlier refusals stay."""
    lib = _lib.load()
    d = ctypes.c_void_p(4096)
    fn, args, key = ((lib.mc_mincurv_solve_batch_ex, _ex, "prox_dense") if entry == "mc_mincurv_solve_batch_ex" else
                     (lib.mc_mincurv_finalize_batch, _fin, "dense"))

    def refused(what, **kw):
        assert fn(*args(d, **kw)) == -1, kw
        msg = lib.mc_last_error().decode()
        assert msg.startswith(entry) and what in msg, msg

    for bad in (1, B_.N_MIN - 1, B_.N_DENSE_MAX + 2, -80):
        refused("dense_below", **{key: bad})
    refused("B <= 0", B=0)
    refused("n_max <= 0", n_max=0)
    nulls = ("rt", "nv", "h", "alpha", "cerr", "status") + (("q",) if key == "prox_dense" else ("kmax",))
    for k in nulls:
        refused("NULL argument", **{k: None})
    if key == "prox_dense":
        for mu in (0.0, -1.0, float("nan"), float("inf")):
            refused("prox_mu", mu=mu)
        refused("needs prox_x", x=None)
        refused("dense_below does not take prox_x", dense=B_.N_MIN)
        # the MC_OPTIONAL4 form: dense_below with prox_x refused as before, whatever prox_dense_below is
        assert lib.mc_mincurv_solve_batch_ex(*_ex(d, dense=B_.N_MIN)[:26], None, 0, None) == -1
    else:
        refused("linearised", lin_flag=1)
        refused("linearised", lin=d)


# ------------------------------------------------------------------------------------------------
# ------------------------------------------------------------------------------------------------
# launches against the recording stand-in
# ------------------------------------------------------------------------------------------------
def _inputs(n_max, B=4):
    g = torch.Generator().manual_seed(5)
    return torch.rand((B, n_max, 4), generator=g, **F64) + 3.0, torch.rand((B, n_max, 2), generator=g, **F64)


@pytest.fixture()
def rec(fake, monkeypatch):
    """The stand-in, with the n_pts of every minimum-curvature call read when it is made (the buffers are temporaries)."""
    real = FakeLib.__getattr__
    fake.npts = {}

    def patched(self, name):
        fn = real(self, name)
        if name not in ENTRIES:
            return fn

        def call(*a):
            rc = fn(*a)
            self.npts[len(self.calls) - 1] = (None if a[2] is None else
                                              np.array((ctypes.c_int32 * a[0]).from_address(a[2].value)).tolist())
            return rc
        return call
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    return fake


def _dense(c, a):
    """is a recorded call one of the dense refinement's?"""
    return {"mc_mincurv_solve_batch_ex": 26, "mc_mincurv_adjoint_batch": 21, "mc_mincurv_finalize_batch": 16}.get(c) \
        is not None and a[{"mc_mincurv_solve_batch_ex": 26, "mc_mincurv_adjoint_batch": 21,
                           "mc_mincurv_finalize_batch": 16}[c]] != 0


def _calls(fake):
    """[(entry, args, n_pts, dense)] of the minimum-curvature calls"""
    return [(c, a, fake.npts[k], _dense(c, a)) for k, (c, a) in enumerate(fake.calls) if c in ENTRIES]


def _use(metric, project, x, mask):
    B, n = x.shape
    g = torch.ones_like(x)
    metric(g, torch.zeros_like(x, dtype=torch.bool), g, mask)
    project(x, g, mask)
    project.evaluate(x, mask)


def test_below_n_min_only_the_dense_calls_run(rec):
    fake = rec
    rt, nv = _inputs(40)
    npts = torch.tensor([40, 12, 3, 0], dtype=torch.int32)
    m = R.CurvatureMetric(rt, nv, npts, 10.0, small_tracks=True)
    p = R.CurvatureProjection(rt, nv, npts, 2.0, 0.12, 10.0, small_tracks=True)
    fake.calls.clear()
    mask = torch.tensor([True, True, True, False])
    _use(m, p, torch.zeros((4, 40), **F64), mask)
    calls = _calls(fake)
    assert [(c, dn) for c, _, _, dn in calls] == [("mc_mincurv_adjoint_batch", True), ("mc_mincurv_solve_batch_ex", True),
                                                  ("mc_mincurv_finalize_batch", True)]
    adj, prox, fin = (a for _, a, _, _ in calls)
    assert calls[0][2] == [40, 40, 12, 12, 3, 3, 0, 0]                # both rows of every track, one call
    assert calls[1][2] == calls[2][2] == [40, 12, 3, 0]
    assert adj[1] == 40 and adj[21] == B_.N_MIN and adj[20] is None and adj[22] is None and adj[19] == 0
    assert prox[25] == 0 and prox[26] == B_.N_MIN and prox[15] == 10.0 ** -4 and prox[6] == 0.12 and prox[27] is None
    assert fin[16] == B_.N_MIN and fin[8] == 0 and fin[15] is None and fin[17] is None
    # without the flag the short tracks are never launched, as before
    m0, p0 = R.CurvatureMetric(rt, nv, npts, 10.0), R.CurvatureProjection(rt, nv, npts, 2.0, 0.12, 10.0)
    fake.calls.clear()
    _use(m0, p0, torch.zeros((4, 40), **F64), mask)
    assert not _calls(fake)


@pytest.mark.parametrize("lin", [False, True])
def test_a_mixed_batch_runs_banded_then_dense(rec, lin):
    """n_max 120, tracks of 120, 40, 100 and 60 points: every banded call as without the flag but with the short tracks
    at n_pts 0, then one dense call with only the short tracks (the metric's on their first N_MIN - 1 points, about the
    shifted line with lin_alpha); lin_alpha reaches the others."""
    rt, nv = _inputs(120)
    npts = torch.tensor([120, 40, 100, 60], dtype=torch.int32)
    la = torch.full((4, 120), 0.1, **F64) if lin else None
    mask = torch.tensor([True, True, True, True])
    x = torch.zeros((4, 120), **F64)
    runs = {}
    for flag in (False, True):
        m = R.CurvatureMetric(rt, nv, npts, 10.0, lin_alpha=la, small_tracks=flag)
        p = R.CurvatureProjection(rt, nv, npts, 2.0, 0.12, 10.0, lin_alpha=la, small_tracks=flag)
        rec.calls.clear()
        _use(m, p, x, mask)
        runs[flag] = _calls(rec)
    old, new = runs[False], runs[True]
    assert not any(dn for *_, dn in old)
    assert [(c, dn) for c, _, _, dn in new] == (
        [("mc_mincurv_adjoint_batch", False)] * 2 + [("mc_mincurv_adjoint_batch", True)]
        + [("mc_mincurv_solve_batch_ex", False)] * 2 + [("mc_mincurv_solve_batch_ex", True)]
        + [("mc_mincurv_setup_batch_ex", False), ("mc_mincurv_finalize_batch", False)] * 2
        + [("mc_mincurv_finalize_batch", True)])
    for (c0, a0, n0, _), (c1, a1, n1, _) in zip(old, [x for x in new if not x[3]]):
        assert c0 == c1 and len(a0) == len(a1)
        assert n1 == [k if k >= B_.N_MIN else 0 for k in n0], c0
    dense = {c: (a, n) for c, a, n, dn in new if dn}
    adj, prox, fin = dense["mc_mincurv_adjoint_batch"], dense["mc_mincurv_solve_batch_ex"], dense["mc_mincurv_finalize_batch"]
    assert adj[1] == [0, 0, 40, 40, 0, 0, 60, 60] and adj[0][1] == B_.N_MIN - 1 and adj[0][20] is None
    assert prox[1] == fin[1] == [0, 40, 0, 60] and prox[0][1] == fin[0][1] == 120
    assert (prox[0][18] is not None) == lin and (fin[0][15] is not None) == lin and fin[0][8] == int(lin)


def test_the_metric_takes_the_linearisation_line_as_its_centre_line(rec):
    """The dense metric's reftrack holds the points P + lin_alpha n (widths 1 m), both rows of a track alike."""
    rt, nv = _inputs(40)
    la = torch.linspace(-0.3, 0.3, 40, **F64)[None].repeat(4, 1)
    m = R.CurvatureMetric(rt, nv, None, 10.0, lin_alpha=la, small_tracks=True)
    want = rt[:, :, :2] + la[:, :, None] * nv
    assert torch.equal(m.d_rt[0::2, :, :2], want) and torch.equal(m.d_rt[1::2, :, :2], want)
    assert bool((m.d_rt[:, :, 2:] == 1.0).all())


def test_the_dense_below_override_moves_the_split(rec):
    fake = rec
    rt, nv = _inputs(120)
    npts = torch.tensor([120, 40, 100, 108], dtype=torch.int32)
    p = R.CurvatureProjection(rt, nv, npts, 2.0, 0.12, 10.0, dense_below=B_.N_DENSE_MAX + 1)
    fake.calls.clear()
    p(torch.zeros((4, 120), **F64), torch.zeros((4, 120), **F64), torch.ones(4, dtype=torch.bool))
    calls = _calls(fake)
    assert [n for c, _, n, dn in calls if not dn] == [[120, 0], [0, 0]]
    assert calls[-1][2] == [0, 40, 100, 108] and calls[-1][1][26] == B_.N_DENSE_MAX + 1


@pytest.mark.parametrize("n_max", [40, 120])
def test_refine_raceline_batch_passes_the_flag_through(rec, n_max):
    """refine_raceline_batch(small_tracks=True) with the metric, kappa_bound and relinearise reaches the dense projection
    and evaluation (the stand-in gives no gradient, so no step and no metric solve follows) and, below N_MIN, nothing
    banded; without the flag no dense call is made.  A bad _dense_below is refused."""
    fake = rec
    rt, nv = _inputs(n_max)
    npts = torch.tensor([n_max, 30, n_max, 20], dtype=torch.int32)
    a0 = torch.zeros((4, n_max), **F64)
    kw = dict(n_pts=npts, max_iters=1, max_halvings=1, metric_length=10.0, kappa_bound=0.12, relinearise=1,
              curv_error_allowed=-0.0)
    for flag in (False, True):
        fake.calls.clear()
        R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, small_tracks=flag, **kw)
        calls = _calls(fake)
        dense = {c for c, _, _, dn in calls if dn}
        assert dense == ({"mc_mincurv_solve_batch_ex", "mc_mincurv_finalize_batch"} if flag else set())
        if n_max < B_.N_MIN:
            assert all(dn for *_, dn in calls)
    with pytest.raises(ValueError, match="_dense_below"):
        R.refine_raceline_batch(rt, nv, a0, 2.0, GGV, MACH, 70.0, 0.75, 1200.0, _dense_below=B_.N_DENSE_MAX + 2, **kw)


# ------------------------------------------------------------------------------------------------
# the replay of the projection QP on short tracks against Goldfarb-Idnani
# ------------------------------------------------------------------------------------------------
def small_prox_cases():
    """[(name, track dict, kb, mu, x, q)]: the projection QP on short tracks at two mu = l^-4, with the rows slack
    ('slack': 3x the box-only projection's largest |k|) and binding (half way between the smallest limit the box allows
    and that value); x a line through the box, q a smooth linear term.  Also collapsed boxes and the LIN form."""
    out = []
    tracks = [(f"synth{n}", IR.track(rt, w_veh=min(2.0, 0.5 * float((rt[:, 2] + rt[:, 3]).min()))))
              for n, rt in ((n, synth.make_track(20 + n, n)) for n in (3, 4, 5, 8, 16, 17, 31, 32, 33, 64, 79))]
    tracks += [("collapsed31", IR.track(IR.collapsed(31))), ("lin_n17", IR.track(synth.make_track(43, 17),
                lin_alpha=IR.lin_line(17))), ("lin_n64", IR.track(synth.make_track(44, 64), lin_alpha=IR.lin_line(64)))]
    for name, t in tracks:
        d = t["d"]
        n = d["n"]
        lb, ub = d["lb"].astype(np.float64), d["ub"].astype(np.float64)
        x = 0.5 * (lb + ub) + 0.45 * (ub - lb) * np.sin(np.arange(n) * 0.9)
        q = 1e-3 * np.cos(np.arange(n) * 0.21)
        kmin, _ = IR.kappa_min(d)
        for length in (5.0, 12.0):
            mu = length ** -4
            kbox = IR.replay(d, 1e3, prox_mu=mu, prox_x=x, prox_q=q)["kappa_lin_max"]
            out.append((f"{name}_l{length:g}_slack", t, float(3.0 * kbox), mu, x, q))
            if kbox > kmin * (1 + 1e-2):
                out.append((f"{name}_l{length:g}_binding", t, float(0.5 * (kmin + kbox)), mu, x, q))
    return out


def _gi(t, kb, mu, x, q):
    """prox_ref's Goldfarb-Idnani solution of the same QP (its E, k_ref and box from the long-double data, rounded)"""
    d = t["d"]
    E = d["E"].astype(np.float64)
    dd = dict(H=E.T @ E, E=E, k_ref=d["k_ref"].astype(np.float64), lb=d["lb"].astype(np.float64),
              ub=d["ub"].astype(np.float64))
    return prox_ref.prox_qp(dd, kb, mu, x, q)


def test_the_replay_of_the_dense_projection_on_short_tracks_reaches_the_kkt_point():
    """The dense iteration with prox (override 'dense': the kernel's status rule) converges (status 0) on every case and
    its alpha is the Goldfarb-Idnani projection to 1e-6 relative; the rows hold to kb (1 + 1e-7) and bind where meant."""
    worst, binding = 0.0, 0
    for name, t, kb, mu, x, q in small_prox_cases():
        r = IR.replay(t["d"], kb, prox_mu=mu, prox_x=x, prox_q=q, override="dense")
        y = _gi(t, kb, mu, x, q)
        e = float(np.abs(r["alpha"].astype(np.float64) - y).max() / max(np.abs(y).max(), 1e-3))
        k = np.abs(t["d"]["k_ref"].astype(np.float64) + t["d"]["E"].astype(np.float64) @ y)
        print(f"{name}: status {r['status']} iters {r['iters']} exit {r['exit']}  |alpha - GI| {e:.1e}  "
              f"max|k| / kb {k.max() / kb:.4f}")
        assert r["status"] == 0, name
        assert e <= 1e-6, (name, e)
        assert float(r["kappa_lin_max"]) <= kb * (1 + 1e-7)
        if name.endswith("binding"):
            assert k.max() >= kb * (1 - 1e-6), name
            binding += 1
        worst = max(worst, e)
    print(f"worst {worst:.1e} over the cases, {binding} with binding rows")
    assert binding >= 10
