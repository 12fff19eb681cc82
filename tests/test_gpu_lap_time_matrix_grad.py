"""GPU tests of the lap-time matrix's sensitivities (batch.lap_time_matrix_diff; vel_profile_adjoint_kernel over B * V
profiles and vel_profile_adjoint_sum_kernel; DESIGN.md section 3.12): the forward is lap_time_matrix_batch's bit for bit;
the device agrees with the host build of the same statements (tests/vp_matrix_ref.py) for every cell of a small matrix;
one cell at scale 1 is vel_profile_diff bit for bit, and every cell agrees with vel_profile_diff on a pre-scaled ggv;
the chain from the widths agrees with a directional difference; a track's gradient does not depend on its batch or
the chunking; unsupported tracks raise (strict) or get zeros."""
import numpy as np
import pytest
import torch

from global_racetrajectory_optimization_b200 import _lib, batch as B_
from vp_matrix_ref import MatrixHarness

pytestmark = pytest.mark.gpu
DEV = "cuda"
VEH = dict(drag_coeff=0.75, m_veh=1200.0)
SCALES = [0.6, 1.0, 1.3]
SPEEDS = [30.0, 50.0, 70.0]
NAMES = ["berlin", "handling", "synth333"]
# Bounds at 4-10x what was measured on an H100 80GB HBM3 (700 W power limit; DESIGN.md 3.12):
# |device - host| / max |host gradient| per track (the same statements; the device contracts products into FMAs):
# <= 2.9e-16 with dyn_model_exp 1, <= 4.0e-12 for kappa with dyn_model_exp 1.5 (pow)
HOST_TOL = 2e-11
# |cell of lap_time_matrix_diff - vel_profile_diff on ggv[:, 1:] * scale| / max |gradient|: measured 0 (the products
# of the scale with the table entries round as the pre-scaled table does), bounded in case a contraction differs
PRESCALED_TOL = 1e-12
# |central difference - chain gradient| / |chain gradient| per track, through the QP solver (its active set is not held):
# 6.0e-2 on synth333 (a bound changes inside +-delta), 3.8e-6 on handling
CHAIN_TOL = 0.3
STEP = 2.0


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return MatrixHarness(tmp_path_factory.mktemp("vp_matrix_gpu"))


def _ragged(golden, names=NAMES):
    rows = [(golden(nm)["rl_kappa"], golden(nm)["rl_el_lengths"]) for nm in names]
    n_max = max(k.size for k, _ in rows) + 7
    kap = np.zeros((len(rows) + 1, n_max))
    el = np.ones((len(rows) + 1, n_max))
    npts = np.zeros(len(rows) + 1, dtype=np.int32)               # the last slot is inactive (n_pts 0)
    for b, (k, e) in enumerate(rows):
        kap[b, :k.size], el[b, :k.size], npts[b] = k, e, k.size
    t = lambda a: torch.tensor(a, device=DEV)
    return t(kap), t(el), t(npts), rows


def _rel(got, want):
    return float(np.abs(got - want).max() / np.abs(want).max())


@pytest.mark.parametrize("kw", [dict(), dict(filt_window=5, dyn_model_exp=1.5), dict(decel_slice_upper=0)])
def test_every_cell_matches_the_host_build_and_the_forward_is_the_matrix(golden, harness, kw):
    v = golden("velprofile")
    kap, el, npts, rows = _ragged(golden)
    k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
    res = B_.lap_time_matrix_diff(k, e, v["ggv"], v["ax_max_machines"], SCALES, SPEEDS, n_pts=npts, **kw, **VEH)
    if "decel_slice_upper" not in kw:
        ref = B_.lap_time_matrix_batch(kap, el, v["ggv"], v["ax_max_machines"], SCALES, SPEEDS, n_pts=npts,
                                       dyn_model_exp=kw.get("dyn_model_exp", 1.0), filt_window=kw.get("filt_window"), **VEH)
        assert torch.equal(res["laptime"].detach(), ref)
    assert not res["status"].any() and not res["grad_status"].any()
    w = torch.tensor(np.random.default_rng(2).uniform(0.5, 2.0, tuple(res["laptime"].shape)), device=DEV)
    (res["laptime"] * w).sum().backward()
    gk, ge = k.grad.cpu().numpy(), e.grad.cpu().numpy()
    upper = kw.get("decel_slice_upper", B_.VP_DECEL_SLICE_UPPER)
    errs = []
    for b, (kk, ee) in enumerate(rows):
        n = kk.size
        h = harness.matrix_adjoint(kk, ee, v["ggv"], v["ax_max_machines"], SCALES, SPEEDS, w[b].cpu().numpy(),
                                   exp=kw.get("dyn_model_exp", 1.0), filt=kw.get("filt_window", 0), upper=upper, **VEH)
        assert not h["status"].any()
        assert np.abs(h["laptime"] - res["laptime"][b].detach().cpu().numpy()).max() <= 1e-12 * h["laptime"].max()
        errs.append((_rel(gk[b, :n], h["g_kappa"]), _rel(ge[b, :n], h["g_el"])))
        assert max(errs[-1]) <= HOST_TOL, (NAMES[b], kw, errs[-1])
        assert not gk[b, n:].any() and not ge[b, n:].any()                       # zeros in the padding
    assert not gk[-1].any() and not ge[-1].any()                                 # the inactive slot
    print(f"measured device vs host {kw}: kappa {max(x[0] for x in errs):.2e}, el {max(x[1] for x in errs):.2e}")


def test_one_cell_at_scale_one_and_v_max_is_vel_profile_diff_bit_for_bit(golden):
    v = golden("velprofile")
    kap, el, npts, _ = _ragged(golden)
    w = torch.tensor(np.random.default_rng(7).uniform(0.5, 2.0, kap.shape[0]), device=DEV)
    k1, e1 = kap.clone().requires_grad_(), el.clone().requires_grad_()
    m = B_.lap_time_matrix_diff(k1, e1, v["ggv"], v["ax_max_machines"], [1.0], [70.0], n_pts=npts, **VEH)
    (m["laptime"][:, 0, 0] * w).sum().backward()
    k2, e2 = kap.clone().requires_grad_(), el.clone().requires_grad_()
    d = B_.vel_profile_diff(k2, e2, v["ggv"], v["ax_max_machines"], 70.0, n_pts=npts, **VEH)
    (d["laptime"] * w).sum().backward()
    assert torch.equal(m["laptime"][:, 0, 0], d["laptime"])
    assert torch.equal(k1.grad, k2.grad) and torch.equal(e1.grad, e2.grad)


def test_each_cell_agrees_with_vel_profile_diff_on_a_prescaled_ggv(golden):
    v = golden("velprofile")
    kap, el, npts, _ = _ragged(golden)
    k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
    m = B_.lap_time_matrix_diff(k, e, v["ggv"], v["ax_max_machines"], SCALES, SPEEDS, n_pts=npts, **VEH)
    worst = 0.0
    for t, vm in enumerate(SPEEDS):
        for s, sc in enumerate(SCALES):
            gk, ge = torch.autograd.grad(m["laptime"][:, t, s].sum(), (k, e), retain_graph=True)
            ggv = v["ggv"].copy()
            ggv[:, 1:] *= sc
            k2, e2 = kap.clone().requires_grad_(), el.clone().requires_grad_()
            d = B_.vel_profile_diff(k2, e2, ggv, v["ax_max_machines"], vm, n_pts=npts, **VEH)
            d["laptime"].sum().backward()
            lap, lap_ref = m["laptime"][:, t, s].detach(), d["laptime"].detach()
            assert float((lap - lap_ref).abs().max()) <= 1e-12 * float(lap_ref.max())
            for got, want in ((gk, k2.grad), (ge, e2.grad)):
                err = float((got - want).abs().max() / want.abs().max())
                worst = max(worst, err)
                assert err <= PRESCALED_TOL, (vm, sc, err)
    print(f"measured cell vs pre-scaled ggv: {worst:.2e}")


def _chain(widths, rt, nv, h, npts, no_max, w):
    v = np.load(__import__("conftest").GOLD + "/velprofile.npz")
    al = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, 2.0, n_pts=npts)["alpha"]
    rl = B_.create_raceline_diff(rt[:, :, :2], nv, al, STEP, n_pts=npts, n_out_max=no_max)
    m = B_.lap_time_matrix_diff(rl["kappa"], rl["el_lengths_interp"], v["ggv"], v["ax_max_machines"], [0.8, 1.0],
                                [50.0, 70.0], n_pts=rl["n_out"], **VEH)
    return (m["laptime"] * w).sum(dim=(1, 2)), rl


def _codes(harness, rl, b, w):
    """The decisions (branch codes, fixed-point iterations) of every cell's profile on track b of a raceline batch."""
    v = np.load(__import__("conftest").GOLD + "/velprofile.npz")
    no = int(rl["n_out"][b])
    m = harness.matrix_adjoint(rl["kappa"][b, :no].detach().cpu().numpy(), rl["el_lengths_interp"][b, :no].detach().cpu().numpy(),
                               v["ggv"], v["ax_max_machines"], [0.8, 1.0], [50.0, 70.0], w, **VEH)
    return [(c["codes"] & ~(16 | 64), c["iters"]) for c in m["cells"]]


def test_a_weighted_sum_of_cells_matches_a_directional_difference_from_the_widths(golden, harness):
    rts = [golden(nm)["reftrack"] for nm in ("synth333", "handling")]
    n = [r.shape[0] for r in rts]
    rt = np.zeros((2, max(n), 4))
    for b, r in enumerate(rts):
        rt[b, :n[b]] = r
    rt, npts = torch.tensor(rt, device=DEV), torch.tensor(n, dtype=torch.int32, device=DEV)
    _, _, nv, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    w = torch.tensor([[0.5, 1.0], [1.5, 2.0]], device=DEV, dtype=torch.float64)
    src0 = rt[:, :, 2:].clone()
    src = src0.clone().requires_grad_()
    lap, rl = _chain(src, rt, nv, h, npts, None, w)
    no_max = rl["kappa"].shape[1]
    lap.sum().backward()
    gen = torch.Generator(device="cpu").manual_seed(8)
    d = (torch.rand(tuple(src0.shape), generator=gen, dtype=torch.float64) - 0.5).to(DEV)
    d = d * (torch.arange(rt.shape[1], device=DEV)[None, :] < npts[:, None])[:, :, None]
    an = (src.grad * d).sum(dim=(1, 2))
    wn = w.cpu().numpy()
    base = [_codes(harness, rl, b, wn) for b in range(2)]
    for b in range(2):
        # the largest delta at which n_out, the station segments and every cell's decisions are held
        for delta in (1e-3, 3e-4, 1e-4, 3e-5):
            laps, held = [], True
            for s in (1.0, -1.0):
                with torch.no_grad():
                    lp, r2 = _chain(src0 + s * delta * d, rt, nv, h, npts, no_max, w)
                laps.append(float(lp[b]))
                held = held and int(r2["n_out"][b]) == int(rl["n_out"][b]) and \
                    torch.equal(r2["spline_inds"][b], rl["spline_inds"][b]) and \
                    all(np.array_equal(c[0], c0[0]) and c[1] == c0[1] for c, c0 in zip(_codes(harness, r2, b, wn), base[b]))
            if held:
                break
        assert held, b
        fd = (laps[0] - laps[1]) / (2.0 * delta)
        err = abs(fd - float(an[b])) / abs(float(an[b]))
        print(f"measured chain track {b}: delta {delta:g}, relative error {err:.2e}")
        assert err <= CHAIN_TOL, (b, delta, fd, float(an[b]))


def _grads(k0, e0, B, slot, ggv, mach, chunk=None, monkeypatch=None):
    scale = torch.linspace(0.8, 1.2, B, device=DEV, dtype=torch.float64)[:, None]
    k = (k0[None] * scale).clone()
    k[slot] = k0
    k.requires_grad_()
    e = e0[None].repeat(B, 1).requires_grad_()
    if chunk is not None:
        monkeypatch.setattr(B_, "_chunk", lambda B, per_item, dev: chunk)
    B_.lap_time_matrix_diff(k, e, ggv, mach, [0.6, 1.3], [30.0, 70.0], **VEH)["laptime"].sum().backward()
    return k.grad[slot], e.grad[slot]


def test_a_tracks_gradient_does_not_depend_on_its_batch_or_the_chunking(golden, monkeypatch):
    v = golden("velprofile")
    g = golden("synth333")
    k0 = torch.tensor(g["rl_kappa"], device=DEV)
    e0 = torch.tensor(g["rl_el_lengths"], device=DEV)
    alone = _grads(k0, e0, 1, 0, v["ggv"], v["ax_max_machines"])
    assert alone[0].abs().max() > 0.0
    for B, slot, chunk in ((300, 0, None), (1000, 517, None), (1000, 517, 7), (300, 299, 64)):
        many = _grads(k0, e0, B, slot, v["ggv"], v["ax_max_machines"], chunk, monkeypatch)
        assert torch.equal(alone[0], many[0]) and torch.equal(alone[1], many[1]), (B, slot, chunk)


def test_non_finite_and_inactive_tracks_raise_or_give_zeros(golden):
    v = golden("velprofile")
    g = golden("handling")
    k = torch.tensor(np.stack([g["rl_kappa"]] * 5), device=DEV)
    e = torch.tensor(np.stack([g["rl_el_lengths"]] * 5), device=DEV)
    e[1, 5] = float("nan")
    n = k.shape[1]
    npts = torch.tensor([n, n, n, 0, -3], dtype=torch.int32, device=DEV)   # an inactive slot, a reported overflow
    args = (v["ggv"], v["ax_max_machines"], [0.6, 1.0], [30.0, 70.0])
    for strict in (True, False):
        kk, ee = k.clone().requires_grad_(), e.clone().requires_grad_()
        res = B_.lap_time_matrix_diff(kk, ee, *args, n_pts=npts, strict=strict, **VEH)
        assert res["grad_status"].flatten(1).tolist() == [[0] * 4, [3] * 4, [0] * 4, [0] * 4, [3] * 4]
        assert torch.equal(res["status"], res["grad_status"])
        if strict:
            with pytest.raises(_lib.MinCurvLibError, match="lap_time_matrix_diff"):
                res["laptime"].sum().backward()
        else:
            res["laptime"].sum().backward()
            assert not kk.grad[1].any() and not ee.grad[1].any() and not kk.grad[3:].any() and not ee.grad[3:].any()
            assert torch.equal(kk.grad[0], kk.grad[2]) and kk.grad[0].abs().max() > 0.0
    # cells without upstream gradient are not refused
    kk = k.clone().requires_grad_()
    res = B_.lap_time_matrix_diff(kk, e, *args, n_pts=npts, **VEH)
    res["laptime"][0, 1, 0].backward()
    assert kk.grad[0].abs().max() > 0.0 and not kk.grad[1:].any()
