"""CPU tests (-m "not gpu") of the width sensitivities of small closed tracks: the MC_OPTIONAL5 parameter of
mc_mincurv_adjoint_batch as the binding reads it, the argument checks of the real library before any CUDA call, the
launches of opt_min_curv_diff(small_tracks=True) against the recording stand-in of the library, and the oracle's
active-set VJP with rows (tests/qp_sens_rows.py) against central differences of its Goldfarb-Idnani solves on tracks
below N_MIN points."""
import ctypes

import numpy as np
import pytest
import torch

import qp_sens_rows as QR
from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth


def test_the_dense_adjoint_parameter_is_parsed_from_the_header():
    assert _lib._OPTIONAL5 == {"mc_mincurv_adjoint_batch": (21, 1)}
    assert _lib._SIGS["mc_mincurv_adjoint_batch"][1][21] is ctypes.c_int
    assert len(_lib._SIGS["mc_mincurv_adjoint_batch"][1]) == 25


def _adjoint(lib, d, **kw):
    a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, h=d, wv=2.0, wvb=None, fs=2.0, cid=None, sens=d, gs=d, ga=d, gwr=d,
             gwl=d, gwv=d, srows=d, nrows=d, schur=d, cap=4, lin=None, dense=B_.N_MIN, ws=None, wsb=0, stream=None)
    a.update(kw)
    return lib.mc_mincurv_adjoint_batch(*a.values())


def test_the_real_library_refuses_before_any_cuda_call():
    lib = _lib.load()
    d = ctypes.c_void_p(4096)
    # the full row export with dense_below and n_max >= N_MIN passes the checks to the banded stage's workspace check
    assert _adjoint(lib, d) == -3 and b"workspace too small" in lib.mc_last_error()
    assert _adjoint(lib, d, dense=B_.N_DENSE_MAX + 1) == -3
    for bad in (1, B_.N_MIN - 1, B_.N_DENSE_MAX + 2, -80):
        assert _adjoint(lib, d, dense=bad) == -1 and b"dense_below" in lib.mc_last_error()
    assert _adjoint(lib, d, srows=None, nrows=None, schur=None) == -1 and b"sens_rows" in lib.mc_last_error()
    assert _adjoint(lib, d, schur=None) == -1 and b"schur" in lib.mc_last_error()
    assert _adjoint(lib, d, lin=d) == -1 and b"lin_alpha" in lib.mc_last_error()
    assert _adjoint(lib, d, rt=None) == -1
    assert _adjoint(lib, d, B=0) == -1
    # without the dense adjoint: n_max below N_MIN is refused as before
    assert _adjoint(lib, d, dense=0, n_max=10) == -1
    # the solve: the full row export goes with dense_below (refused only for its workspace), sens alone does not
    ex = [1, 100, None, d, d, d, 0.12, 2.0, None, 2.0, d, d, None, d, None, 0.0, None, None, None, None, None]
    assert lib.mc_mincurv_solve_batch_ex(*ex, d, d, d, d, B_.N_MIN, None, 0, None) == -3
    assert lib.mc_mincurv_solve_batch_ex(*ex, d, d, None, None, B_.N_MIN, None, 0, None) == -1
    assert b"sens_rows" in lib.mc_last_error()


def _diff(n=120, B=4, **kw):
    g = torch.Generator().manual_seed(3)
    centre = torch.rand((B, n, 2), dtype=torch.float64, generator=g)
    widths = (torch.rand((B, n, 2), dtype=torch.float64, generator=g) + 3.0).requires_grad_()
    nv, h = torch.rand((B, n, 2), dtype=torch.float64, generator=g), torch.ones((B, n), dtype=torch.float64)
    res = B_.opt_min_curv_diff(centre, widths, nv, h, 0.12, 2.0, **kw)
    res["alpha"].sum().backward()
    return widths


def _calls(fake, name):
    return [a for c, a in fake.calls if c == name]


@pytest.mark.parametrize("n", [120, 40])
@pytest.mark.parametrize("kb", ["scalar", "batch"])
def test_small_tracks_wiring(fake, n, kb):
    """The forward goes through mc_mincurv_solve_batch_ex with the four export tensors and dense_below = N_MIN; the
    backward passes dense_below to mc_mincurv_adjoint_batch; both on the same chunks."""
    B = 4
    g = torch.Generator().manual_seed(3)
    centre = torch.rand((B, n, 2), dtype=torch.float64, generator=g)
    widths = (torch.rand((B, n, 2), dtype=torch.float64, generator=g) + 3.0).requires_grad_()
    nv, h = torch.rand((B, n, 2), dtype=torch.float64, generator=g), torch.ones((B, n), dtype=torch.float64)
    kappa = 0.12 if kb == "scalar" else torch.full((B,), 0.12, dtype=torch.float64)
    res = B_.opt_min_curv_diff(centre, widths, nv, h, kappa, 2.0, curvature_rows=True, small_tracks=True)
    res["alpha"].sum().backward()
    assert widths.grad.shape == (B, n, 2)
    fwd, bwd = _calls(fake, "mc_mincurv_solve_batch_ex"), _calls(fake, "mc_mincurv_adjoint_batch")
    assert not _calls(fake, "mc_mincurv_solve_batch_sens")
    assert [a[0] for a in fwd] == [a[0] for a in bwd] == [2, 2]           # the stand-in's chunks: B // 2
    for a in fwd:
        assert a[25] == B_.N_MIN and all(p is not None for p in a[21:25]) and a[16] is None
        assert (a[6] == 0.12 and a[19] is None) if kb == "scalar" else a[19] is not None
    for f, a in zip(fwd, bwd):
        assert a[21] == B_.N_MIN and a[20] is None
        assert a[10].value == f[21].value and a[16].value == f[23].value and a[17].value == f[24].value
        assert a[18] is not None
    fake.calls.clear()
    _diff(n=n, curvature_rows=True, small_tracks=True, _dense_below=B_.N_DENSE_MAX + 1)
    assert all(a[25] == B_.N_DENSE_MAX + 1 for a in _calls(fake, "mc_mincurv_solve_batch_ex"))
    assert all(a[21] == B_.N_DENSE_MAX + 1 for a in _calls(fake, "mc_mincurv_adjoint_batch"))


def test_small_tracks_need_the_curvature_rows(fake):
    with pytest.raises(ValueError, match="curvature_rows"):
        _diff(small_tracks=True)
    with pytest.raises(ValueError, match="curvature_rows"):
        _diff(_dense_below=B_.N_MIN)
    assert not fake.calls


@pytest.mark.parametrize("rows", [False, True])
def test_without_the_flag_nothing_changes(fake, rows):
    """The forward is mc_mincurv_solve_batch_sens and the backward passes dense_below 0; n_max < N_MIN is refused."""
    _diff(curvature_rows=rows)
    fwd, bwd = _calls(fake, "mc_mincurv_solve_batch_sens"), _calls(fake, "mc_mincurv_adjoint_batch")
    assert [a[0] for a in fwd] == [a[0] for a in bwd] == [2, 2]
    assert not _calls(fake, "mc_mincurv_solve_batch_ex")
    assert all(a[21] == 0 and a[20] is None for a in bwd)
    assert all((a[16] is not None) == rows for a in bwd)
    with pytest.raises(NotImplementedError):
        _diff(n=40, curvature_rows=True)


def _short_track(n, seed):
    rt = synth.make_track(seed, n)
    rt[:, 2:] = np.maximum(rt[:, 2:], 1.6)            # (the widths of tiny tracks fit a 2 m car)
    _, _, _, nv = QR.T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))
    return rt, nv


def _kb_binding(d, rt, wv):
    """A curvature limit at which the rows bind but can be met: 0.9 of the box-only optimum's largest |k|, raised to the
    smallest limit the box allows (bisection on the oracle's solves) if that is above it."""
    lb, ub, _ = QR.Q.bounds(rt, wv)
    a0 = QR.solve(d, lb, ub, 1e6)[0]
    kmax = float(np.abs(d["k_ref"] + d["E"] @ a0).max())
    lo, hi = 0.0, kmax
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        try:
            QR.solve(d, lb, ub, mid)
            hi = mid
        except ValueError:
            lo = mid
    return max(0.9 * kmax, 1.02 * hi), kmax


@pytest.mark.parametrize("n,seed", [(5, 1), (8, 2), (16, 3), (31, 4), (40, 5), (64, 6), (79, 7)])
@pytest.mark.parametrize("regime", ["slack", "binding"])
def test_oracle_vjp_on_short_tracks_matches_central_differences(n, seed, regime):
    """The exact active-set VJP with rows on tracks below N_MIN points: rows slack (a limit far above the box-only
    optimum's curvature) and rows binding (below it); the perturbation keeps the active set."""
    rt, nv = _short_track(n, seed)
    wv = 2.0
    d0 = QR.qp_data(rt, nv, 1.0, wv)
    kb_bind, kmax = _kb_binding(d0, rt, wv)
    kb = 10.0 * kmax if regime == "slack" else kb_bind
    d = QR.qp_data(rt, nv, kb, wv)
    rng = np.random.default_rng(n)
    gbar = rng.standard_normal(n)
    ref = QR.width_vjp_rows(d, rt, wv, kb, gbar)
    rows = ref["row_hi"] | ref["row_lo"]
    assert rows.any() == (regime == "binding")
    delta = 1e-6

    def loss(rt_, wv_):
        out = QR.width_vjp_rows(d, rt_, wv_, kb, gbar)
        for k in ("at_ub", "at_lb", "row_hi", "row_lo"):
            assert np.array_equal(out[k], ref[k]), k
        return gbar @ out["alpha"]

    for _ in range(3):
        dw = rng.uniform(-1.0, 1.0, (n, 2))
        dv = rng.uniform(-1.0, 1.0)
        rp, rm = rt.copy(), rt.copy()
        rp[:, 2:] += delta * dw
        rm[:, 2:] -= delta * dw
        fd = (loss(rp, wv + delta * dv) - loss(rm, wv - delta * dv)) / (2 * delta)
        ad = ref["grad_w_right"] @ dw[:, 0] + ref["grad_w_left"] @ dw[:, 1] + ref["grad_w_veh"] * dv
        assert abs(fd - ad) <= 1e-6 * max(abs(ad), 1e-3), (fd, ad)
