"""GPU tests of the create_raceline adjoint (batch.create_raceline_diff, create_raceline_adjoint_kernel) and of the whole
chain widths / reftrack -> alpha -> raceline -> lap time (DESIGN.md section 3.12): the forward is create_raceline_batch's
bit for bit; the adjoint agrees with autograd of the torch restatement tests/raceline_ref.py on a ragged batch that takes
every regime of the forward's moment solve (PCR, chunked, shared and global scratch); the chain's gradient agrees with a
directional central difference through the device chain; unsupported tracks raise (strict) or get zeros."""
import numpy as np
import pytest
import torch

import raceline_ref as R
from vp_adj_ref import Harness
from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth

pytestmark = pytest.mark.gpu
DEV = "cuda"
VEH = dict(drag_coeff=0.75, m_veh=1200.0)
REF_TOL = 1e-10         # |device - reference| / max |reference| per gradient; measured 7.1e-12 (n = 4000) on an H100 80GB HBM3
STEP = 2.0
# |central difference - chain gradient| / |chain gradient| per track.  The difference runs through the QP solvers, whose
# active sets are not held (the raceline's station segments and the profile's decisions are): measured on the H100,
# shortest path <= 2e-2, min-curvature 6.3e-2 on synth333 (a bound changes inside +-delta), 1.6e-3 on handling
CHAIN_TOL = dict(mincurv=0.15, shortest=0.05)


def _batch(rts, alphas):
    n = [r.shape[0] for r in rts]
    rt = np.zeros((len(rts), max(n), 4))
    al = np.zeros((len(rts), max(n)))
    for b, (r, a) in enumerate(zip(rts, alphas)):
        rt[b, :n[b]], al[b, :n[b]] = r, a
    rt, al = torch.tensor(rt, device=DEV), torch.tensor(al, device=DEV)
    npts = torch.tensor(n, dtype=torch.int32, device=DEV)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    return rt, nv, al, npts


def _tracks(golden, big):
    rts = [golden(nm)["reftrack"] for nm in ("synth333", "handling", "berlin")]
    als = [golden(nm)["alpha_mincurv"] for nm in ("synth333", "handling", "berlin")]
    rng = np.random.default_rng(6)
    for n in big:                        # n > 2048: the chunked moment solve; n_max > 3490: global scratch
        rts.append(synth.make_track(11 + n, n))
        als.append(0.3 * np.sin(np.linspace(0.0, 12.0 * np.pi, n, endpoint=False)) + 0.05 * rng.standard_normal(n))
    return rts, als


def _reference_errors(golden, big):
    rts, als = _tracks(golden, big)
    rt, nv, al, npts = _batch(rts, als)
    ref = B_.create_raceline_batch(rt, nv, al, STEP, n_pts=npts)
    r_, n_, a_ = rt.clone().requires_grad_(), nv.clone().requires_grad_(), al.clone().requires_grad_()
    rl = B_.create_raceline_diff(r_, n_, a_, STEP, n_pts=npts)
    for k in B_._RL_KEYS:
        assert torch.equal(rl[k].detach(), ref[k]), k
    gen = torch.Generator(device="cpu").manual_seed(3)
    wr = torch.randn(tuple(rl["raceline_interp"].shape), generator=gen, dtype=torch.float64).to(DEV)
    wk = torch.randn(tuple(rl["kappa"].shape), generator=gen, dtype=torch.float64).to(DEV)
    we = torch.randn(tuple(rl["kappa"].shape), generator=gen, dtype=torch.float64).to(DEV)
    ((rl["raceline_interp"] * wr).sum() + 100.0 * (rl["kappa"] * wk).sum() + (rl["el_lengths_interp"] * we).sum()).backward()
    errs = []
    for b, r in enumerate(rts):
        n, no = r.shape[0], int(ref["n_out"][b])
        xs = [torch.tensor(np.asarray(x, dtype=float)).requires_grad_() for x in (r[:, :2], nv[b, :n].cpu(), als[b])]
        rr = R.create_raceline(*xs, STEP, no=no, seg=ref["spline_inds"][b, :no].cpu().long())
        loss = ((rr["raceline"] * wr[b, :no].cpu()).sum() + 100.0 * (rr["kappa"] * wk[b, :no].cpu()).sum()
                + (rr["el_lengths"] * we[b, :no].cpu()).sum())
        gr, gn, ga = torch.autograd.grad(loss, xs)
        e = []
        for got, want in ((r_.grad[b, :n, :2], gr), (n_.grad[b, :n], gn), (a_.grad[b, :n], ga)):
            e.append(float((got.cpu() - want).abs().max() / want.abs().max()))
        assert not r_.grad[b, :, 2:].any() and not a_.grad[b, n:].any() and not n_.grad[b, n:].any()
        errs.append((n, e))
    return errs


def test_adjoint_matches_the_torch_reference_in_every_regime_of_the_moment_solve(golden):
    for n, e in _reference_errors(golden, (2500, 4000)):
        print(f"  n={n}: measured {max(e):.3e}, bound {REF_TOL:.0e}")
        assert max(e) <= REF_TOL, (n, e)


def _chain(src, kind, rt, nv, h, npts, no_max, strict=True):
    """lap time [B] of the chain from the widths (kind 'mincurv') or the reftrack (kind 'shortest')."""
    v = np.load(__import__("conftest").GOLD + "/velprofile.npz")
    if kind == "mincurv":
        al = B_.opt_min_curv_diff(rt[:, :, :2], src, nv, h, 0.12, 2.0, n_pts=npts, strict=strict)["alpha"]
        rl = B_.create_raceline_diff(rt[:, :, :2], nv, al, STEP, n_pts=npts, n_out_max=no_max, strict=strict)
    else:
        al = B_.opt_shortest_path_diff(src, nv, 2.0, n_pts=npts, strict=strict)["alpha"]
        rl = B_.create_raceline_diff(src, nv, al, STEP, n_pts=npts, n_out_max=no_max, strict=strict)
    lap = B_.vel_profile_diff(rl["kappa"], rl["el_lengths_interp"], v["ggv"], v["ax_max_machines"], 70.0, n_pts=rl["n_out"],
                              strict=strict, **VEH)["laptime"]
    return lap, rl


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return Harness(tmp_path_factory.mktemp("vp_adj_chain"))


def _codes(harness, rl, b):
    """The velocity profile's decisions (branch codes, fixed-point iterations) on track b of a raceline batch."""
    v = np.load(__import__("conftest").GOLD + "/velprofile.npz")
    no = int(rl["n_out"][b])
    a = harness.adjoint(rl["kappa"][b, :no].detach().cpu().numpy(), rl["el_lengths_interp"][b, :no].detach().cpu().numpy(),
                        v["ggv"], v["ax_max_machines"], 70.0, g_lap=1.0, **VEH)
    return a["codes"] & ~(16 | 64), a["iters"]


@pytest.mark.parametrize("kind", ["mincurv", "shortest"])
def test_chain_gradient_matches_a_directional_difference_through_the_device_chain(golden, harness, kind):
    rts = [golden(nm)["reftrack"] for nm in ("synth333", "handling")]
    rt, nv, _, npts = _batch(rts, [np.zeros(r.shape[0]) for r in rts])
    _, _, _, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    src0 = rt[:, :, 2:].clone() if kind == "mincurv" else rt.clone()
    src = src0.clone().requires_grad_()
    lap, rl = _chain(src, kind, rt, nv, h, npts, None)
    no_max = rl["kappa"].shape[1]
    lap.sum().backward()
    g = src.grad.clone()
    gen = torch.Generator(device="cpu").manual_seed(8)
    d = (torch.rand(tuple(src0.shape), generator=gen, dtype=torch.float64) - 0.5).to(DEV)
    mask = torch.arange(rt.shape[1], device=DEV)[None, :] < npts[:, None]
    d = d * mask[:, :, None]
    if kind == "shortest":
        d[:, :, :2] *= 0.01                       # move the line a centimetre, the widths up to half a metre
    an = (g * d).sum(dim=(1, 2))
    base = [_codes(harness, rl, b) for b in range(rt.shape[0])]
    # per track the largest delta at which n_out, the station segments and every decision of the velocity profile are
    # those of the unperturbed chain (the lap time is only piecewise smooth in the inputs)
    for b in range(rt.shape[0]):
        for delta in (1e-3, 3e-4, 1e-4, 3e-5):
            laps, held = [], True
            for s in (1.0, -1.0):
                with torch.no_grad():
                    lp, r2 = _chain(src0 + s * delta * d, kind, rt, nv, h, npts, no_max)
                laps.append(float(lp[b]))
                c2 = _codes(harness, r2, b)
                held = held and int(r2["n_out"][b]) == int(rl["n_out"][b]) and \
                    torch.equal(r2["spline_inds"][b], rl["spline_inds"][b]) and \
                    np.array_equal(c2[0], base[b][0]) and c2[1] == base[b][1]
            if held:
                break
        assert held, (kind, b)
        fd = (laps[0] - laps[1]) / (2.0 * delta)
        assert abs(fd - float(an[b])) <= CHAIN_TOL[kind] * abs(float(an[b])), (kind, b, delta, fd, float(an[b]))


def test_unsupported_tracks_raise_or_get_zeros(golden):
    rts = [golden(nm)["reftrack"] for nm in ("synth333", "handling")]
    rt, nv, al, npts = _batch(rts, [golden(nm)["alpha_mincurv"] for nm in ("synth333", "handling")])
    ref = B_.create_raceline_batch(rt, nv, al, STEP, n_pts=npts)
    cap = int(ref["n_out"].min())                # the larger track overflows an explicit n_out_max
    for strict in (True, False):
        a = al.clone().requires_grad_()
        rl = B_.create_raceline_diff(rt, nv, a, STEP, n_pts=npts, n_out_max=cap, strict=strict)
        assert (rl["n_out"] < 0).sum() == 1
        if strict:
            with pytest.raises(_lib.MinCurvLibError, match="n_out <= 0"):
                rl["kappa"].sum().backward()
        else:
            rl["kappa"].sum().backward()
            bad = int((rl["n_out"] < 0).nonzero()[0])
            assert not a.grad[bad].any() and a.grad[1 - bad].abs().max() > 0.0
    # a mincurv instance solved with the curvature rows (grad_status 4): the chain refuses it, or gives zeros
    g = golden("synth160_kappa")
    rt, nv, _, npts = _batch([g["reftrack"]], [np.zeros(g["reftrack"].shape[0])])
    _, _, _, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    v = np.load(__import__("conftest").GOLD + "/velprofile.npz")
    for strict in (True, False):
        w = rt[:, :, 2:].clone().requires_grad_()
        res = B_.opt_min_curv_diff(rt[:, :, :2], w, nv, h, float(g["kappa_bound"]), 2.0, n_pts=npts, strict=strict)
        assert res["grad_status"].tolist() == [4]
        rl = B_.create_raceline_diff(rt[:, :, :2], nv, res["alpha"], STEP, n_pts=npts, strict=strict)
        lap = B_.vel_profile_diff(rl["kappa"], rl["el_lengths_interp"], v["ggv"], v["ax_max_machines"], 70.0,
                                  n_pts=rl["n_out"], strict=strict, **VEH)["laptime"]
        if strict:
            with pytest.raises(_lib.MinCurvLibError, match="opt_min_curv_diff"):
                lap.sum().backward()
        else:
            lap.sum().backward()
            assert not w.grad.any()


def test_a_tracks_raceline_gradient_does_not_depend_on_its_batch(golden):
    g = golden("handling")
    rts, als = [g["reftrack"]] * 40, [g["alpha_mincurv"] * s for s in np.linspace(0.9, 1.1, 40)]
    als[17] = g["alpha_mincurv"]
    out = []
    for idx in ([17], list(range(40))):
        rt, nv, al, npts = _batch([rts[i] for i in idx], [als[i] for i in idx])
        a = al.clone().requires_grad_()
        B_.create_raceline_diff(rt, nv, a, STEP, n_pts=npts, n_out_max=800)["kappa"].sum().backward()
        out.append(a.grad[idx.index(17)])
    assert torch.equal(out[0], out[1])
