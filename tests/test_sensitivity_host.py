"""CPU tests (-m "not gpu") of the width sensitivities: the oracle's exact active-set VJP (tests/qp_sens.py) against
central finite differences of the oracle's own Goldfarb-Idnani solves, the argument validation of the two C entries
without a GPU, and the host logic of batch.opt_min_curv_diff against the recording stand-in of the library (fake_lib.py)."""
import ctypes

import numpy as np
import pytest
import torch

import qp_sens as Q
from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_


def _fd_case(golden, name):
    g = golden(name)
    return g["reftrack"], float(g["w_veh"]), Q.dense_from_band(g["H_band"]), g["f"]


@pytest.mark.parametrize("name", ["synth128", "synth200"])
def test_oracle_vjp_matches_central_differences_of_the_qp(golden, name):
    rt, wv, H, f = _fd_case(golden, name)
    n = rt.shape[0]
    rng = np.random.default_rng(11)
    gbar = rng.standard_normal(n)
    ref = Q.width_vjp(H, f, rt, wv, gbar)
    assert ref["at_ub"].any() and ref["at_lb"].any() and (~(ref["at_ub"] | ref["at_lb"])).any()
    delta = 1e-5

    def loss(rt_, wv_):
        out = Q.width_vjp(H, f, rt_, wv_, gbar)
        # the perturbation keeps the active set: the solution is affine in the bounds on it
        assert np.array_equal(out["at_ub"], ref["at_ub"]) and np.array_equal(out["at_lb"], ref["at_lb"])
        return gbar @ out["alpha"]

    # whole-gradient directions (widths and w_veh together) and single coordinates of each kind of point
    for k in range(3):
        d = rng.uniform(-1.0, 1.0, (n, 2))
        dv = rng.uniform(-1.0, 1.0)
        rp, rm = rt.copy(), rt.copy()
        rp[:, 2:] += delta * d
        rm[:, 2:] -= delta * d
        fd = (loss(rp, wv + delta * dv) - loss(rm, wv - delta * dv)) / (2 * delta)
        ad = ref["grad_w_right"] @ d[:, 0] + ref["grad_w_left"] @ d[:, 1] + ref["grad_w_veh"] * dv
        assert abs(fd - ad) <= 1e-6 * abs(ad)
    picks = [int(np.flatnonzero(ref["at_ub"])[0]), int(np.flatnonzero(ref["at_lb"])[0])]
    for i in picks:
        for col, key in ((2, "grad_w_right"), (3, "grad_w_left")):
            rp, rm = rt.copy(), rt.copy()
            rp[i, col] += delta
            rm[i, col] -= delta
            fd = (loss(rp, wv) - loss(rm, wv)) / (2 * delta)
            assert abs(fd - ref[key][i]) <= 1e-6 * np.abs(ref[key]).max()
    fd = (loss(rt, wv + delta) - loss(rt, wv - delta)) / (2 * delta)
    assert abs(fd - ref["grad_w_veh"]) <= 1e-6 * abs(ref["grad_w_veh"])
    # an inactive bound has no influence
    free = np.flatnonzero(~(ref["at_ub"] | ref["at_lb"]))
    assert np.all(ref["grad_w_right"][free] == 0.0) and np.all(ref["grad_w_left"][free] == 0.0)


def test_oracle_collapsed_boxes_follow_the_box_centre(golden):
    rt, wv, H, f = _fd_case(golden, "synth128")
    rt = rt.copy()
    for i in (10, 60, 61):
        rt[i, 3] = wv - rt[i, 2] + 1e-9            # ub - lb = 1e-9 < 2 FIX_EPS: the box collapses onto its centre
    gbar = np.random.default_rng(3).standard_normal(rt.shape[0])
    ref = Q.width_vjp(H, f, rt, wv, gbar)
    assert ref["collapsed"].sum() == 3
    c = ref["collapsed"]
    assert np.allclose(ref["grad_w_right"][c], -ref["grad_w_left"][c], rtol=0, atol=0)
    # moving the centre of a collapsed box moves alpha_i with it: d/dw_right at fixed ub - lb
    i, delta = 60, 1e-5
    rp, rm = rt.copy(), rt.copy()
    rp[i, 2] += delta
    rp[i, 3] -= delta
    rm[i, 2] -= delta
    rm[i, 3] += delta
    fd = (gbar @ Q.width_vjp(H, f, rp, wv, gbar)["alpha"] - gbar @ Q.width_vjp(H, f, rm, wv, gbar)["alpha"]) / (2 * delta)
    assert abs(fd - (ref["grad_w_right"][i] - ref["grad_w_left"][i])) <= 1e-6 * np.abs(ref["grad_w_right"]).max()


def test_sensitivity_entries_validate_their_arguments_without_gpu():
    lib = _lib.load()
    d = ctypes.c_void_p(4096)

    def solve(**kw):
        a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, h=d, kb=0.12, wv=2.0, wvb=None, fs=2.0, cid=None, alpha=d, cerr=d,
                 kmax=None, st=d, it=None, sens=d, gs=d, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_mincurv_solve_batch_sens(*a.values())

    def adjoint(**kw):
        a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, h=d, wv=2.0, wvb=None, fs=2.0, cid=None, sens=d, gs=d, ga=d, gwr=d,
                 gwl=d, gwv=d, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_mincurv_adjoint_batch(*a.values())

    for call in (solve, adjoint):
        assert call() == -3 and b"workspace too small" in lib.mc_last_error()
        assert call(n_max=10) == -1                                   # below N_MIN
        assert call(B=0) == -1
        assert call(fs=0.0) == -1
        assert call(sens=None) == -1 and b"NULL argument" in lib.mc_last_error()
        assert call(gs=None) == -1
    assert solve(alpha=None) == -1 and solve(st=None) == -1
    for k in ("ga", "gwr", "gwl", "gwv", "rt", "nv", "h"):
        assert adjoint(**{k: None}) == -1


def test_opt_min_curv_diff_chunks_forward_and_backward_alike(fake):
    B, n = 5, 120
    centre = torch.rand((B, n, 2), dtype=torch.float64)
    widths = (torch.rand((B, n, 2), dtype=torch.float64) + 3.0).requires_grad_()
    nv, h = torch.rand((B, n, 2), dtype=torch.float64), torch.ones((B, n), dtype=torch.float64)
    wv = torch.full((B,), 2.0, dtype=torch.float64, requires_grad=True)
    cid = torch.tensor([0, 0, 2, 2, 0], dtype=torch.int32)
    res = B_.opt_min_curv_diff(centre, widths, nv, h, 0.12, wv, centre_id=cid, max_chunk=2)
    assert set(res) == {"alpha", "curv_error_max", "kappa_lin_max", "status", "iters", "grad_status"}
    assert res["alpha"].requires_grad and not res["status"].requires_grad
    (res["alpha"] * 2.0).sum().backward()
    fwd = [c[1] for c in fake.calls if c[0] == "mc_mincurv_solve_batch_sens"]
    bwd = [c[1] for c in fake.calls if c[0] == "mc_mincurv_adjoint_batch"]
    assert [c[0] for c in fwd] == [c[0] for c in bwd] == [2, 2, 1]          # same chunks both ways
    assert widths.grad.shape == (B, n, 2) and wv.grad.shape == (B,)
    with pytest.raises(ValueError, match="centre is a constant"):
        B_.opt_min_curv_diff(centre.clone().requires_grad_(), widths, nv, h, 0.12, 2.0)
    with pytest.raises(ValueError, match="normvec is a constant"):
        B_.opt_min_curv_diff(centre, widths, nv.clone().requires_grad_(), h, 0.12, 2.0)
    with pytest.raises(ValueError, match="h is a constant"):
        B_.opt_min_curv_diff(centre, widths, nv, h.clone().requires_grad_(), 0.12, 2.0)
    # a scalar w_veh is a constant: only the widths get a gradient
    w2 = widths.detach().clone().requires_grad_()
    B_.opt_min_curv_diff(centre, w2, nv, h, 0.12, 2.0)["alpha"].sum().backward()
    assert w2.grad is not None
