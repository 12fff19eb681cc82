"""GPU tests (-m gpu) of the shortest-path sensitivities (batch.opt_shortest_path_diff, shortest_path_adjoint_kernel):
device gradients against the oracle's exact active-set VJP (tests/sp_sens.py) on every golden fixture, against a
directional finite difference through the device solver itself, their invariances, the forward pass against
opt_shortest_path_batch, the unsupported instances, and the whole chain through torch autograd."""
import numpy as np
import pytest

import sp_sens as S

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402

FIXTURES = ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth1000", "synth128",
            "synth160_kappa", "synth200", "synth2000", "synth333", "synth333_kappa", "synth500", "synth500_narrow"]
CLAMPED = {"berlin": 7, "modena": 4, "berlin500_jitter_b": 3}
KINDS = ("x", "y", "w_right", "w_left", "normal_x", "normal_y", "w_veh")
# Worst error over the seven kinds, measured on an H100 (seed 0) -> the bound, 4-6x above it.  The device differentiates
# the interior-point iterate at which the solver stops (mu <= 1e-11 mu0).  A bound that is nearly active (slack ~1e-4 m)
# or weakly active (multiplier ~1e-4 |f|_inf) is not resolved there: its d = l / s is neither large nor small next to
# H_ii = 4, and the error of v spreads along the free stretch around it.  The fixtures with such bounds are held to what
# was measured on them (DESIGN.md 3.11).
GRAD_TOL = {
    "synth128": 5e-8,               # 9.2e-9
    "synth160_kappa": 2e-7,         # 3.6e-8
    "synth333": 3e-7,               # 5.4e-8
    "synth500_narrow": 4e-6,        # 6.7e-7
    "synth333_kappa": 1e-5,         # 1.9e-6
    "synth200": 1e-5,               # 2.0e-6
    "synth500": 4e-5,               # 7.2e-6
    "synth1000": 1e-4,              # 2.2e-5
    "berlin": 5e-4,                 # 9.0e-5
    "synth2000": 1e-3,              # 1.8e-4
    "handling": 2e-3,               # 3.9e-4   (inactive bound 1.5e-4 m from its limit)
    "modena": 1e-2,                 # 1.7e-3   (active bound with multiplier 3e-4 |f|_inf)
    "berlin500_jitter_a": 5e-2,     # 9.4e-3   (inactive bound 2.2e-4 m from its limit)
    "berlin500_jitter_b": 1.0,      # 2.3e-1   (inactive bound 5.9e-5 m from its limit)
}
FD_TOL = 1e-3                       # directional finite difference through the device solver: 1.6e-4 measured
E2E_TOL = {"synth128": 2e-8, "synth333": 2e-6}      # uniform upstream gradient: 3.4e-9, 3.4e-7 measured


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _device_batch(golden, names, dev):
    """Ragged batch of the fixtures: reftrack [B, n_max, 4], normvec [B, n_max, 2] (the fixtures' own), n_pts, w_veh [B]."""
    gs = [golden(nm) for nm in names]
    n = [g["reftrack"].shape[0] for g in gs]
    rt, nv = np.zeros((len(gs), max(n), 4)), np.zeros((len(gs), max(n), 2))
    for b, g in enumerate(gs):
        rt[b, :n[b]], nv[b, :n[b]] = g["reftrack"], g["normvec"]
    return (torch.tensor(rt, device=dev), torch.tensor(nv, device=dev), torch.tensor(n, dtype=torch.int32, device=dev),
            torch.tensor([float(g["w_veh"]) for g in gs], dtype=torch.float64, device=dev))


def _err(got, ref, keep):
    return float(np.abs(got - ref)[keep].max() / max(np.abs(ref).max(), 1e-300))


def device_vs_oracle(golden, seed=0):
    """Per fixture: max|diff| / max|ref| of every input kind (degenerate points and their neighbours excluded; the widths
    normalised by the larger of their two gradients), the excluded and the clamped points, and the device's width
    gradients at the clamped bounds.  One ragged batch through opt_shortest_path_diff and torch.autograd.grad."""
    dev = torch.device("cuda")
    rt, nv, npts, wv = _device_batch(golden, FIXTURES, dev)
    rt.requires_grad_(), nv.requires_grad_(), wv.requires_grad_()
    res = B_.opt_shortest_path_diff(rt, nv, wv, n_pts=npts)
    rng = np.random.default_rng(seed)
    gbar = np.zeros(rt.shape[:2])
    for b, m in enumerate(npts.tolist()):
        gbar[b, :m] = rng.standard_normal(m)
    grt, gnv, gwv = (t.cpu().numpy() for t in torch.autograd.grad(res["alpha"], (rt, nv, wv), torch.tensor(gbar, device=dev)))
    out = {}
    for b, name in enumerate(FIXTURES):
        g = golden(name)
        n = g["reftrack"].shape[0]
        ref = S.vjp(g["reftrack"], g["normvec"], float(g["w_veh"]), gbar[b, :n], alpha=g["alpha_shpath"])
        bad = S.degenerate(ref, np.abs(ref["f"]).max())
        keep = ~(bad | np.roll(bad, 1) | np.roll(bad, -1))      # (the centre line and normals see v at the neighbours)
        r, d = ref["grad_reftrack"], grt[b, :n]
        wscale = np.abs(r[:, 2:]).max()
        errs = dict(x=_err(d[:, 0], r[:, 0], keep), y=_err(d[:, 1], r[:, 1], keep),
                    w_right=float(np.abs(d[:, 2] - r[:, 2])[keep].max() / wscale),
                    w_left=float(np.abs(d[:, 3] - r[:, 3])[keep].max() / wscale),
                    normal_x=_err(gnv[b, :n, 0], ref["grad_normvec"][:, 0], keep),
                    normal_y=_err(gnv[b, :n, 1], ref["grad_normvec"][:, 1], keep),
                    w_veh=abs(float(gwv[b]) - ref["grad_w_veh"]) / abs(ref["grad_w_veh"]))
        clamped_grads = np.concatenate((d[ref["clamped_r"], 2], d[ref["clamped_l"], 3]))
        out[name] = dict(errs, excluded=int(bad.sum()), clamped=int((ref["clamped_r"] | ref["clamped_l"]).sum()),
                         clamped_grad_max=float(np.abs(clamped_grads).max()) if clamped_grads.size else 0.0,
                         status=int(res["status"][b]), grad_status=int(res["grad_status"][b]),
                         padding_zero=bool((grt[b, n:] == 0).all() and (gnv[b, n:] == 0).all()))
    return out


def test_device_gradients_match_the_oracle_on_every_fixture(golden):
    out = device_vs_oracle(golden)
    for name, o in out.items():
        assert o["status"] == 0 and o["grad_status"] == 0 and o["padding_zero"], (name, o)
        assert max(o[k] for k in KINDS) <= GRAD_TOL[name], (name, o)
        assert o["clamped"] == CLAMPED.get(name, 0) and o["clamped_grad_max"] == 0.0, (name, o)


def test_forward_is_bit_identical_to_opt_shortest_path_batch(golden):
    dev = torch.device("cuda")
    rt, nv, npts, wv = _device_batch(golden, FIXTURES, dev)
    ref = B_.opt_shortest_path_batch(rt, nv, wv, n_pts=npts)
    res = B_.opt_shortest_path_diff(rt.clone().requires_grad_(), nv, wv, n_pts=npts)
    for k in ("alpha", "status", "iters"):
        assert torch.equal(res[k].detach(), ref[k]), k
    assert torch.equal(res["grad_status"], ref["status"])


def _n1000_batch(dev, B=6):
    base = synth.make_batch(4242, 3, 1000)
    rt = torch.tensor(np.stack([base[i % 3] if i < 3 else synth.jitter_widths(base[i % 3], 77 + i) for i in range(B)]),
                      device=dev)
    _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
    return rt, nv


def test_directional_finite_difference_through_the_device_solver():
    dev = torch.device("cuda")
    rt, nv = _n1000_batch(dev)
    B, n = rt.shape[:2]
    gen = torch.Generator(device="cpu").manual_seed(5)
    gbar = torch.randn((B, n), generator=gen, dtype=torch.float64).to(dev)
    # a smooth direction in every input: the centre line and the widths by at most delta (m), the normals by delta, w_veh
    s = torch.linspace(0.0, 2.0 * np.pi, n + 1, dtype=torch.float64)[:n]
    ph = torch.rand((B, 6, 2), generator=gen, dtype=torch.float64) * 2.0 * np.pi
    d = torch.stack([torch.sin(3.0 * s[None] + ph[:, k, 0, None]) * torch.cos(2.0 * s[None] + ph[:, k, 1, None])
                     for k in range(6)], dim=2).to(dev)
    dv = (torch.rand((B,), generator=gen, dtype=torch.float64) * 2.0 - 1.0).to(dev)
    wv = torch.full((B,), 2.0, dtype=torch.float64, device=dev)
    r, v, w = rt.clone().requires_grad_(), nv.clone().requires_grad_(), wv.clone().requires_grad_()
    res = B_.opt_shortest_path_diff(r, v, w)
    grt, gnv, gwv = torch.autograd.grad(res["alpha"], (r, v, w), gbar)
    ad = (grt * d[:, :, :4]).sum(dim=(1, 2)) + (gnv * d[:, :, 4:]).sum(dim=(1, 2)) + gwv * dv
    delta = 1e-4

    def loss(sign):
        out = B_.opt_shortest_path_batch(rt + sign * delta * d[:, :, :4], nv + sign * delta * d[:, :, 4:], wv + sign * delta * dv)
        assert bool((out["status"] == 0).all())
        return (out["alpha"] * gbar).sum(dim=1)
    fd = (loss(1.0) - loss(-1.0)) / (2.0 * delta)
    rel = ((fd - ad).abs() / ad.abs()).max().item()
    assert rel <= FD_TOL, (rel, fd.tolist(), ad.tolist())


def _grads(rt, nv, wv, gbar, n_pts=None):
    r, v = rt.clone().requires_grad_(), nv.clone().requires_grad_()
    w = wv.clone().requires_grad_() if isinstance(wv, torch.Tensor) else wv
    res = B_.opt_shortest_path_diff(r, v, w, n_pts=n_pts)
    (res["alpha"] * gbar).sum().backward()
    return r.grad, v.grad, (w.grad if isinstance(w, torch.Tensor) else None)


def test_gradients_are_invariant_to_the_form_of_w_veh_duplicates_and_the_batch():
    dev = torch.device("cuda")
    rt, nv = _n1000_batch(dev, B=8)
    rt[7], nv[7] = rt[1], nv[1]                                      # an exact duplicate of instance 1
    B, n = rt.shape[:2]
    gbar = torch.randn((B, n), generator=torch.Generator(device="cpu").manual_seed(9), dtype=torch.float64).to(dev)
    gbar[7] = gbar[1]
    g0, n0, v0 = _grads(rt, nv, torch.full((B,), 2.0, dtype=torch.float64, device=dev), gbar)
    g1, n1, _ = _grads(rt, nv, 2.0, gbar)
    assert g0.abs().max() > 0 and n0.abs().max() > 0 and v0.abs().max() > 0
    assert torch.equal(g0, g1) and torch.equal(n0, n1)
    assert torch.equal(g0[7], g0[1]) and torch.equal(n0[7], n0[1]) and torch.equal(v0[7], v0[1])
    # instance 3 alone and inside a batch of 4096 (more blocks than SMs)
    reps = 4096
    idx = torch.arange(reps, device=dev) % B
    gb = gbar[idx].clone()
    gl, nl, vl = _grads(rt[idx], nv[idx], torch.full((reps,), 2.0, dtype=torch.float64, device=dev), gb)
    gs, ns, vs = _grads(rt[3:4], nv[3:4], torch.full((1,), 2.0, dtype=torch.float64, device=dev), gbar[3:4])
    k = 3 + B * 300
    assert torch.equal(gl[k], gs[0]) and torch.equal(nl[k], ns[0]) and torch.equal(vl[k], vs[0])


def test_unsupported_instances_get_zero_gradients_or_raise(golden):
    dev = torch.device("cuda")
    rt, nv, _, _ = _device_batch(golden, ["synth128", "synth128"], dev)
    npts = torch.tensor([2, 128], dtype=torch.int32, device=dev)             # fewer than 3 points: not a closed track
    gbar = torch.ones(rt.shape[:2], dtype=torch.float64, device=dev)
    for strict in (True, False):
        r = rt.clone().requires_grad_()
        res = B_.opt_shortest_path_diff(r, nv, 2.0, n_pts=npts, strict=strict)
        assert res["grad_status"].tolist() == [-1, 0] and res["status"].tolist() == [-1, 0]
        if strict:
            with pytest.raises(_lib.MinCurvLibError, match="grad_status"):
                (res["alpha"] * gbar).sum().backward()
            continue
        (res["alpha"] * gbar).sum().backward()
        assert (r.grad[0] == 0).all() and (r.grad[1] != 0).any()
    # an instance with a zero upstream gradient does not need one
    r = rt.clone().requires_grad_()
    B_.opt_shortest_path_diff(r, nv, 2.0, n_pts=npts)["alpha"][1].sum().backward()
    assert (r.grad[0] == 0).all() and (r.grad[1] != 0).any()


def test_loss_backward_reaches_reftrack_normvec_and_w_veh(golden):
    dev = torch.device("cuda")
    names = ["synth128", "synth333"]
    rt, nv, npts, wv = _device_batch(golden, names, dev)
    rt.requires_grad_(), nv.requires_grad_(), wv.requires_grad_()
    c = torch.tensor(np.random.default_rng(21).uniform(-1.0, 1.0, rt.shape[:2]), device=dev)
    loss = (B_.opt_shortest_path_diff(rt, nv, wv, n_pts=npts)["alpha"] * c).sum()
    loss.backward()
    for b, name in enumerate(names):
        g = golden(name)
        n = g["reftrack"].shape[0]
        ref = S.vjp(g["reftrack"], g["normvec"], float(g["w_veh"]), c[b, :n].cpu().numpy(), alpha=g["alpha_shpath"])
        tol = E2E_TOL[name]
        assert np.abs(rt.grad[b, :n].cpu().numpy() - ref["grad_reftrack"]).max() <= tol * np.abs(ref["grad_reftrack"]).max()
        assert np.abs(nv.grad[b, :n].cpu().numpy() - ref["grad_normvec"]).max() <= tol * np.abs(ref["grad_normvec"]).max()
        assert abs(wv.grad[b].item() - ref["grad_w_veh"]) <= tol * abs(ref["grad_w_veh"]), name
        assert (rt.grad[b, n:] == 0).all() and (nv.grad[b, n:] == 0).all()
