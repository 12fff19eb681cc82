"""GPU tests (-m gpu) of the width sensitivities (batch.opt_min_curv_diff, mincurv_adjoint_kernel): device gradients
against the oracle's exact active-set VJP (tests/qp_sens.py) on every box-only golden fixture, against finite differences
through the device solver itself, their invariances, the forward pass against opt_min_curv_batch, the unsupported
instances, and the whole chain through torch autograd."""
import numpy as np
import pytest

import qp_sens as Q
from conftest import rel_max

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402

BOX = ["berlin", "modena", "handling", "synth128", "synth200", "synth333", "synth500", "synth500_narrow", "synth1000",
       "synth2000", "berlin500_jitter_a", "berlin500_jitter_b"]
GRAD_TOL = 1e-5
# The device differentiates the interior-point iterate at which the solver stops (relative step 1e-5), not the exact active
# set: a weakly active bound (multiplier ~1e-5 .. 1e-3 |f|_inf) still has a finite d = l / s there, and the gradient around
# it is damped by about H_ii / d.  The fixtures with such bounds are held to what was measured on them (DESIGN.md 3.10).
WEAK_TOL = {"berlin": 1e-4, "modena": 1e-4, "synth333": 5e-4, "synth500_narrow": 1e-4, "synth2000": 2e-1}
COLLAPSED = (10, 60, 61)          # points of the collapsed-box variant of synth128


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _device_batch(rts, dev):
    """Ragged batch [B, n_max, 4] + n_pts + the device's normals and spline scales."""
    n = [r.shape[0] for r in rts]
    rt = np.zeros((len(rts), max(n), 4))
    for b, r in enumerate(rts):
        rt[b, :n[b]] = r
    rt = torch.tensor(rt, device=dev)
    npts = torch.tensor(n, dtype=torch.int32, device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    return rt, npts, nv, h


def _cases(golden):
    """(name, reftrack, w_veh, H, f, alpha of the oracle or None) of every box-only fixture, and synth128 with three
    collapsed boxes (w_right + w_left = w_veh + 1e-9)."""
    out = []
    for name in BOX:
        g = golden(name)
        out.append((name, g["reftrack"], float(g["w_veh"]), Q.dense_from_band(g["H_band"]), g["f"], g["alpha_mincurv_boxonly"]))
    g = golden("synth128")
    rt = g["reftrack"].copy()
    for i in COLLAPSED:
        rt[i, 3] = float(g["w_veh"]) - rt[i, 2] + 1e-9
    out.append(("synth128_collapsed", rt, float(g["w_veh"]), Q.dense_from_band(g["H_band"]), g["f"], None))
    return out


def _degenerate(ref, scale):
    """Points where the derivative does not exist or is ill-conditioned at the solver's tolerance: a bound active with a
    multiplier below 1e-6 |f|_inf, or inactive with a slack below 1e-6 m."""
    weak = (ref["at_ub"] & (ref["lu"] < 1e-6 * scale)) | (ref["at_lb"] & (ref["ll"] < 1e-6 * scale))
    a = ref["alpha"]
    near = ~(ref["at_ub"] | ref["at_lb"]) & (np.minimum(ref["ub"] - a, a - ref["lb"]) < 1e-6)
    return weak | near


def device_vs_oracle(golden, seed=0):
    """Per case: max|diff| / max|ref| of grad_w_right, grad_w_left, grad_w_veh (degenerate points excluded) and the number
    of excluded points.  One ragged batch through opt_min_curv_diff and torch.autograd.grad."""
    dev = torch.device("cuda")
    cases = _cases(golden)
    rt, npts, nv, h = _device_batch([c[1] for c in cases], dev)
    B, n_max = rt.shape[:2]
    widths = rt[:, :, 2:].clone().requires_grad_()
    wv = torch.tensor([c[2] for c in cases], dtype=torch.float64, device=dev, requires_grad=True)
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, wv, n_pts=npts)
    rng = np.random.default_rng(seed)
    gbar = np.zeros((B, n_max))
    for b, c in enumerate(cases):
        gbar[b, :c[1].shape[0]] = rng.standard_normal(c[1].shape[0])
    gw, gv = torch.autograd.grad(res["alpha"], (widths, wv), torch.tensor(gbar, device=dev))
    gw, gv = gw.cpu().numpy(), gv.cpu().numpy()
    out = {}
    for b, (name, r, w, H, f, alpha) in enumerate(cases):
        n = r.shape[0]
        ref = Q.width_vjp(H, f, r, w, gbar[b, :n], alpha=alpha)
        bad = _degenerate(ref, np.abs(f).max())
        keep = ~bad
        errs = {}
        for key, dv in (("grad_w_right", gw[b, :n, 0]), ("grad_w_left", gw[b, :n, 1])):
            errs[key] = float(np.abs(dv - ref[key])[keep].max() / np.abs(ref[key]).max())
        errs["grad_w_veh"] = abs(float(gv[b]) - ref["grad_w_veh"]) / abs(ref["grad_w_veh"])
        out[name] = dict(errs, excluded=int(bad.sum()), grad_status=int(res["grad_status"][b]), status=int(res["status"][b]),
                         collapsed=int(ref["collapsed"].sum()))
    return out


def test_device_gradients_match_the_oracle_on_every_box_only_fixture(golden):
    out = device_vs_oracle(golden)
    for name, o in out.items():
        assert o["status"] == 0 and o["grad_status"] == 0, (name, o)
        worst = max(o["grad_w_right"], o["grad_w_left"], o["grad_w_veh"])
        assert worst <= WEAK_TOL.get(name, GRAD_TOL), (name, o)
    assert out["synth128_collapsed"]["collapsed"] == len(COLLAPSED)


def _n1000_batch(dev, B=6):
    base = synth.make_batch(4242, 3, 1000)
    rts = [base[i % 3] if i < 3 else synth.jitter_widths(base[i % 3], 77 + i) for i in range(B)]
    return _device_batch(rts, dev)


def test_directional_finite_difference_through_the_device_solver():
    dev = torch.device("cuda")
    rt, npts, nv, h = _n1000_batch(dev)
    B, n = rt.shape[:2]
    gen = torch.Generator(device="cpu").manual_seed(5)
    gbar = torch.randn((B, n), generator=gen, dtype=torch.float64).to(dev)
    # a smooth direction: widths change by at most delta, w_veh by delta
    s = torch.linspace(0.0, 2.0 * np.pi, n + 1, dtype=torch.float64)[:n]
    ph = torch.rand((B, 2, 2), generator=gen, dtype=torch.float64) * 2.0 * np.pi
    d = torch.stack([torch.sin(3.0 * s[None] + ph[:, k, 0, None]) * torch.cos(2.0 * s[None] + ph[:, k, 1, None]) for k in range(2)],
                    dim=2).to(dev)
    dv = torch.rand((B,), generator=gen, dtype=torch.float64).to(dev) * 2.0 - 1.0
    widths = rt[:, :, 2:].clone().requires_grad_()
    wv = torch.full((B,), 2.0, dtype=torch.float64, device=dev, requires_grad=True)
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, wv, n_pts=npts)
    gw, gv = torch.autograd.grad(res["alpha"], (widths, wv), gbar)
    ad = (gw * d).sum(dim=(1, 2)) + gv * dv
    delta = 1e-2

    def loss(sign):
        r = rt.clone()
        r[:, :, 2:] += sign * delta * d
        out = B_.opt_min_curv_batch(r, nv, h, 0.12, 2.0 + sign * delta * dv, n_pts=npts)
        assert bool((out["status"] == 0).all())
        return (out["alpha"] * gbar).sum(dim=1)
    fd = (loss(1.0) - loss(-1.0)) / (2.0 * delta)
    rel = ((fd - ad).abs() / ad.abs()).max().item()
    assert rel <= 2e-2, (fd.tolist(), ad.tolist())      # (the stopping rule, and bounds that change state within +-delta)


def _grads(rt, npts, nv, h, wv, gbar, **kw):
    widths = rt[:, :, 2:].clone().requires_grad_()
    wvt = wv.clone().requires_grad_() if isinstance(wv, torch.Tensor) else wv
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, wvt, n_pts=npts, **kw)
    (res["alpha"] * gbar).sum().backward()
    return res, widths.grad, (wvt.grad if isinstance(wvt, torch.Tensor) else None)


def test_gradients_are_invariant_to_sharing_chunking_and_the_form_of_w_veh():
    dev = torch.device("cuda")
    rt, npts, nv, h = _n1000_batch(dev, B=8)
    rt[7], nv[7], h[7] = rt[1], nv[1], h[1]                         # an exact duplicate of instance 1
    B, n = rt.shape[:2]
    gbar = torch.randn((B, n), generator=torch.Generator(device="cpu").manual_seed(9), dtype=torch.float64).to(dev)
    gbar[7] = gbar[1]
    cid = B_.shared_centre_ids(torch.arange(B, device=dev) % 3)
    wv = torch.full((B,), 2.0, dtype=torch.float64, device=dev)
    _, g0, v0 = _grads(rt, npts, nv, h, wv, gbar)
    _, g1, v1 = _grads(rt, npts, nv, h, wv, gbar, centre_id=cid)
    _, g2, v2 = _grads(rt, npts, nv, h, wv, gbar, centre_id=cid, max_chunk=3)
    _, g3, _ = _grads(rt, npts, nv, h, 2.0, gbar)
    assert g0.abs().max() > 0 and v0.abs().max() > 0
    assert torch.equal(g0, g1) and torch.equal(v0, v1)
    assert torch.equal(g0, g2) and torch.equal(v0, v2)
    assert torch.equal(g0, g3)
    assert torch.equal(g0[7], g0[1]) and torch.equal(v0[7], v0[1])


def test_forward_is_bit_identical_to_opt_min_curv_batch(golden):
    dev = torch.device("cuda")
    rt, npts, nv, h = _device_batch([c[1] for c in _cases(golden)], dev)
    wv = torch.tensor([c[2] for c in _cases(golden)], dtype=torch.float64, device=dev)
    ref = B_.opt_min_curv_batch(rt, nv, h, 0.12, wv, n_pts=npts)
    res = B_.opt_min_curv_diff(rt[:, :, :2], rt[:, :, 2:].clone().requires_grad_(), nv, h, 0.12, wv.clone().requires_grad_(),
                               n_pts=npts)
    for k in ("alpha", "curv_error_max", "kappa_lin_max", "status", "iters"):
        assert torch.equal(res[k].detach(), ref[k]), k
    assert bool((res["grad_status"] == res["status"]).all())


def test_unsupported_instances_get_zero_gradients_or_raise(golden):
    dev = torch.device("cuda")
    g = golden("synth160_kappa")
    ok = golden("synth128")["reftrack"]
    narrow = ok.copy()
    narrow[40:44, 2:] = 0.5                                           # 1 m wide for a 2 m vehicle: infeasible
    for rts, kb, expect in (([g["reftrack"]], float(g["kappa_bound"]), [4]), ([narrow, ok], 0.12, [1, 0])):
        rt, npts, nv, h = _device_batch(rts, dev)
        gbar = torch.ones(rt.shape[:2], dtype=torch.float64, device=dev)
        for strict in (True, False):
            widths = rt[:, :, 2:].clone().requires_grad_()
            res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, 2.0, n_pts=npts, strict=strict)
            assert res["grad_status"].tolist() == expect
            if strict:
                with pytest.raises(_lib.MinCurvLibError, match="grad_status"):
                    (res["alpha"] * gbar).sum().backward()
                continue
            (res["alpha"] * gbar).sum().backward()
            for b, e in enumerate(expect):
                assert (widths.grad[b] == 0).all() if e != 0 else (widths.grad[b] != 0).any()
    # an instance with a zero upstream gradient does not need one
    rt, npts, nv, h = _device_batch([narrow, ok], dev)
    widths = rt[:, :, 2:].clone().requires_grad_()
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, 2.0, n_pts=npts)
    res["alpha"][1].sum().backward()
    assert (widths.grad[0] == 0).all() and (widths.grad[1] != 0).any()


def test_loss_backward_reaches_widths_and_w_veh(golden):
    dev = torch.device("cuda")
    cases = [c for c in _cases(golden) if c[0] in ("handling", "synth200", "berlin500_jitter_a")]
    rt, npts, nv, h = _device_batch([c[1] for c in cases], dev)
    widths = rt[:, :, 2:].clone().requires_grad_()
    wv = torch.tensor([c[2] for c in cases], dtype=torch.float64, device=dev, requires_grad=True)
    c = torch.tensor(np.random.default_rng(21).uniform(-1.0, 1.0, rt.shape[:2]), device=dev)
    loss = (B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, wv, n_pts=npts)["alpha"] * c).sum()
    loss.backward()
    for b, (name, r, w, H, f, alpha) in enumerate(cases):
        n = r.shape[0]
        ref = Q.width_vjp(H, f, r, w, c[b, :n].cpu().numpy(), alpha=alpha)
        keep = ~_degenerate(ref, np.abs(f).max())
        got = widths.grad[b, :n].cpu().numpy()
        assert rel_max(got[keep, 0], ref["grad_w_right"][keep]) <= GRAD_TOL, name
        assert rel_max(got[keep, 1], ref["grad_w_left"][keep]) <= GRAD_TOL, name
        assert abs(wv.grad[b].item() - ref["grad_w_veh"]) <= GRAD_TOL * abs(ref["grad_w_veh"]), name
