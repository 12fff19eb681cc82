"""GPU tests of the lap-time sensitivities of the velocity profile (batch.vel_profile_diff, vel_profile_adjoint_kernel;
DESIGN.md section 3.12): the forward is vel_profile_batch's bit for bit, the device adjoint agrees with the host build of
the same statements (tests/vp_adj_ref.py) on a ragged batch with zeros in the padding, a track's gradient does not depend
on its batch, and unsupported instances raise (strict) or get zeros."""
import numpy as np
import pytest
import torch

from global_racetrajectory_optimization_b200 import _lib, batch as B_
from vp_adj_ref import Harness

pytestmark = pytest.mark.gpu
DEV = "cuda"
VEH = dict(drag_coeff=0.75, m_veh=1200.0)
# |device - host| / max |host gradient|: the same statements, the device contracts the adjoint's products into FMAs.
# Measured on an H100 (700 W): <= 3.2e-16 with dyn_model_exp 1, <= 2.3e-12 for kappa with dyn_model_exp 1.5 (pow).
HOST_TOL = 2e-11
NAMES = ["berlin", "handling", "modena", "synth333", "synth1000"]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return Harness(tmp_path_factory.mktemp("vp_adj_gpu"))


def _ragged(golden):
    rows = [(golden(nm)["rl_kappa"], golden(nm)["rl_el_lengths"]) for nm in NAMES]
    n_max = max(k.size for k, _ in rows) + 7
    kap = np.zeros((len(rows) + 1, n_max))
    el = np.ones((len(rows) + 1, n_max))
    npts = np.zeros(len(rows) + 1, dtype=np.int32)               # the last slot is inactive (n_pts 0)
    for b, (k, e) in enumerate(rows):
        kap[b, :k.size], el[b, :k.size], npts[b] = k, e, k.size
    t = lambda a: torch.tensor(a, device=DEV)
    return t(kap), t(el), t(npts), rows


@pytest.mark.parametrize("kw", [dict(v_max=70.0), dict(v_max=40.0, filt_window=5, dyn_model_exp=1.5),
                                dict(v_max=70.0, decel_slice_upper=0)])
def test_forward_and_adjoint_match_the_batch_forward_and_the_host_adjoint(golden, harness, kw):
    v = golden("velprofile")
    kap, el, npts, rows = _ragged(golden)
    ref = B_.vel_profile_batch(kap, el, v["ggv"], v["ax_max_machines"], kw["v_max"], dyn_model_exp=kw.get("dyn_model_exp", 1.0),
                               filt_window=kw.get("filt_window"), n_pts=npts, decel_slice_upper=kw.get("decel_slice_upper"),
                               **VEH)
    k = kap.clone().requires_grad_()
    e = el.clone().requires_grad_()
    res = B_.vel_profile_diff(k, e, v["ggv"], v["ax_max_machines"], n_pts=npts, **kw, **VEH)
    assert torch.equal(res["laptime"], ref["laptime"][:, 0]) and torch.equal(res["vx"], ref["vx"][:, 0])
    assert torch.equal(res["ax"], ref["ax"][:, 0]) and torch.equal(res["t"], ref["t"][:, 0])
    assert torch.equal(res["status"], ref["status"][:, 0]) and not res["grad_status"].any()
    rng = np.random.default_rng(2)
    gl = torch.tensor(rng.uniform(0.5, 2.0, k.shape[0]), device=DEV)
    gv = torch.tensor(0.01 * rng.standard_normal(tuple(k.shape)), device=DEV)
    ((res["laptime"] * gl).sum() + (res["vx"] * gv).sum()).backward()
    gk, ge = k.grad.cpu().numpy(), e.grad.cpu().numpy()
    upper = kw.get("decel_slice_upper", B_.VP_DECEL_SLICE_UPPER)
    for b, (kk, ee) in enumerate(rows):
        n = kk.size
        h = harness.adjoint(kk, ee, v["ggv"], v["ax_max_machines"], kw["v_max"], g_lap=float(gl[b]),
                            g_vx=gv[b, :n].cpu().numpy(), exp=kw.get("dyn_model_exp", 1.0), filt=kw.get("filt_window", 0),
                            upper=upper, **VEH)
        assert h["status"] == 0 and abs(h["laptime"] - float(res["laptime"][b].detach())) <= 1e-12 * h["laptime"]
        for got, want in ((gk[b, :n], h["g_kappa"]), (ge[b, :n], h["g_el"])):
            assert np.abs(got - want).max() <= HOST_TOL * np.abs(want).max(), (NAMES[b], kw)
        assert not gk[b, n:].any() and not ge[b, n:].any()                       # zeros in the padding
    assert not gk[-1].any() and not ge[-1].any()                                 # the inactive slot


def test_a_tracks_gradient_does_not_depend_on_its_batch(golden):
    v = golden("velprofile")
    g = golden("synth333")
    k0 = torch.tensor(g["rl_kappa"], device=DEV)
    e0 = torch.tensor(g["rl_el_lengths"], device=DEV)

    def grads(B, slot):
        scale = torch.linspace(0.8, 1.2, B, device=DEV, dtype=torch.float64)[:, None]
        k = (k0[None] * scale).clone()
        k[slot] = k0
        k.requires_grad_()
        e = e0[None].repeat(B, 1).requires_grad_()
        B_.vel_profile_diff(k, e, v["ggv"], v["ax_max_machines"], 70.0, **VEH)["laptime"].sum().backward()
        return k.grad[slot], e.grad[slot]

    alone = grads(1, 0)
    for B, slot in ((300, 0), (1000, 517)):
        many = grads(B, slot)
        assert torch.equal(alone[0], many[0]) and torch.equal(alone[1], many[1])


def test_non_finite_lap_times_raise_or_give_zeros(golden):
    v = golden("velprofile")
    g = golden("handling")
    k = torch.tensor(np.stack([g["rl_kappa"]] * 3), device=DEV)
    e = torch.tensor(np.stack([g["rl_el_lengths"]] * 3), device=DEV)
    e[1, 5] = float("nan")
    for strict in (True, False):
        kk, ee = k.clone().requires_grad_(), e.clone().requires_grad_()
        res = B_.vel_profile_diff(kk, ee, v["ggv"], v["ax_max_machines"], 70.0, strict=strict, **VEH)
        assert res["grad_status"].tolist() == [0, 3, 0]
        if strict:
            with pytest.raises(_lib.MinCurvLibError, match="vel_profile_diff"):
                res["laptime"].sum().backward()
        else:
            res["laptime"].sum().backward()
            assert not kk.grad[1].any() and not ee.grad[1].any()
            assert torch.equal(kk.grad[0], kk.grad[2]) and kk.grad[0].abs().max() > 0.0
    # an instance without upstream gradient is not refused
    kk = k.clone().requires_grad_()
    res = B_.vel_profile_diff(kk, e, v["ggv"], v["ax_max_machines"], 70.0, **VEH)
    res["laptime"][0].backward()
    assert kk.grad[0].abs().max() > 0.0 and not kk.grad[1:].any()
