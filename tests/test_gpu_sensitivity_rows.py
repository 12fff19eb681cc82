"""GPU tests (-m gpu) of the width sensitivities with the curvature rows (batch.opt_min_curv_diff(curvature_rows=True),
mincurv_sens_rows_export_kernel, mincurv_adjoint_rows_kernel; DESIGN.md section 3.10): device gradients against the
oracle's exact active-set VJP with rows (tests/qp_sens_rows.py), against a central difference through the device solver,
what must not move (the forward, the box-only gradients, sharing, chunking, w_veh as a float, the batch around an
instance), and the lap-time chain on an instance whose rows bind."""
import numpy as np
import pytest

import qp_sens_rows as QR

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import batch as B_  # noqa: E402
from test_gpu_edges import KB_MIXED, _mixed_cases, _pack  # noqa: E402

DEV = "cuda"
GRAD_TOL = 1e-5
# The device differentiates the curvature-row phase's final iterate, not the exact active set: a weakly active bound or
# row keeps a finite weight there and damps the gradient around it.  Fixtures held to what was measured on them, with
# the cause, in DESIGN.md section 3.10 (curvature rows).
WEAK_TOL = {"synth333_kappa": 5e-4, "handling": 5e-5, "N1000": 0.25, "collapsed": 5e-4}
FD_TOL = 0.05            # directional central difference through the device solver (delta 1 cm)
CHAIN_TOL = 0.05         # lap-time central difference against the chain gradient
VEH = dict(drag_coeff=0.75, m_veh=1200.0)
STEP = 2.0


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _golden_case(golden, name, kb):
    g = golden(name)
    return dict(name=name, rt=g["reftrack"], nv=g["normvec"], h=g["el_lengths"], w_veh=float(g["w_veh"]), kb=kb)


def _fixture_cases(golden):
    return [_golden_case(golden, "synth160_kappa", 0.02), _golden_case(golden, "synth333_kappa", 0.03),
            _golden_case(golden, "handling", 0.06)]


def _grads(cases, kb, gbar, **kw):
    """(result dict, dL/dwidths [B, n_max, 2], dL/dw_veh [B]) of L = sum gbar * alpha."""
    rt, nv, h, npts, wv = _pack(cases)
    widths = rt[:, :, 2:].clone().requires_grad_()
    wvg = wv.clone().requires_grad_()
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, wvg, n_pts=npts, strict=False, **kw)
    gw, gv = torch.autograd.grad(res["alpha"], (widths, wvg), torch.as_tensor(gbar, device=DEV))
    return res, gw.cpu().numpy(), gv.cpu().numpy()


def _gbar(cases, seed):
    n_max = max(c["rt"].shape[0] for c in cases)
    rng = np.random.default_rng(seed)
    g = np.zeros((len(cases), n_max))
    for b, c in enumerate(cases):
        g[b, :c["rt"].shape[0]] = rng.standard_normal(c["rt"].shape[0])
    return g


def _errors(cases, kb, gbar, res, gw, gv):
    out = {}
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        d = QR.qp_data(c["rt"], c["nv"], kb, c["w_veh"])
        ref = QR.width_vjp_rows(d, c["rt"], c["w_veh"], kb, gbar[b, :n])
        scale = np.abs(d["f"]).max()
        keep = ~QR.degenerate(ref, scale)
        top = max(np.abs(ref["grad_w_right"]).max(), np.abs(ref["grad_w_left"]).max())      # (one side may have no bound)
        e = {k: float(np.abs(dv - ref[k])[keep].max() / top)
             for k, dv in (("grad_w_right", gw[b, :n, 0]), ("grad_w_left", gw[b, :n, 1]))}
        e["grad_w_veh"] = abs(float(gv[b]) - ref["grad_w_veh"]) / max(abs(ref["grad_w_veh"]), 1e-300)
        act = np.concatenate((np.where(ref["at_ub"], ref["lu"], np.inf), np.where(ref["at_lb"], ref["ll"], np.inf),
                              np.where(ref["row_hi"], ref["l3"], np.inf), np.where(ref["row_lo"], ref["l4"], np.inf)))
        out[c["name"]] = dict(e, rows=int((ref["row_hi"] | ref["row_lo"]).sum()), excluded=int((~keep).sum()),
                              weakest=float(act.min() / scale), status=int(res["status"][b]),
                              grad_status=int(res["grad_status"][b]))
    return out


def _check(out, tag):
    for name, o in out.items():
        print(tag, name, {k: (f"{v:.1e}" if isinstance(v, float) else v) for k, v in o.items()})
    for name, o in out.items():
        assert o["status"] == 0 and o["grad_status"] == 0, (name, o)
        worst = max(o["grad_w_right"], o["grad_w_left"], o["grad_w_veh"])
        assert worst <= WEAK_TOL.get(name, GRAD_TOL), (name, o)


@pytest.mark.parametrize("seed", [0, 1])
def test_device_gradients_match_the_oracle_with_rows(golden, seed):
    for c in _fixture_cases(golden):
        gbar = _gbar([c], seed)
        res, gw, gv = _grads([c], c["kb"], gbar, curvature_rows=True)
        out = _errors([c], c["kb"], gbar, res, gw, gv)
        assert out[c["name"]]["rows"] > 0
        _check(out, f"seed {seed}")


@pytest.mark.parametrize("seed", [0, 1])
def test_mixed_batch_matches_the_oracle_unshared_and_shared(golden, seed):
    cases, centre_id, rows = _mixed_cases(golden)
    keep = [b for b in range(len(cases)) if b != 7]                  # (7: infeasible)
    gbar = _gbar(cases, seed)
    res0, gw0, gv0 = _grads(cases, KB_MIXED, gbar, curvature_rows=True)
    res1, gw1, gv1 = _grads(cases, KB_MIXED, gbar, curvature_rows=True, centre_id=torch.tensor(centre_id, device=DEV))
    assert res0["grad_status"].tolist() == [0] * 7 + [1, 0, 0]
    assert np.array_equal(gw0, gw1) and np.array_equal(gv0, gv1)      # sharing changes nothing
    assert not gw0[7].any() and gv0[7] == 0.0
    sub = [cases[b] for b in keep]
    _check(_errors(sub, KB_MIXED, gbar[keep], {k: v[keep] for k, v in res0.items()}, gw0[keep], gv0[keep]),
           f"mixed seed {seed}")


def test_directional_difference_through_the_device_solver(golden):
    """The N = 1000 row instance of the mixed batch: gbar^T (alpha(w + delta d) - alpha(w - delta d)) / (2 delta) against
    the gradient, delta 1 cm on the widths along a smooth direction and on w_veh."""
    cases, _, _ = _mixed_cases(golden)
    c = cases[2]
    n = c["rt"].shape[0]
    gbar = _gbar([c], 3)
    res, gw, gv = _grads([c], KB_MIXED, gbar, curvature_rows=True)
    assert int(res["grad_status"][0]) == 0 and int(B_.opt_min_curv_batch(*_pack([c])[:3], KB_MIXED, 2.0)["status"][0]) == 0
    s = np.linspace(0.0, 2.0 * np.pi, n, endpoint=False)
    d = np.stack((np.sin(3.0 * s), np.cos(5.0 * s)), axis=1)
    delta = 0.01
    rt, nv, h, npts, wv = _pack([c])

    def alpha(sign):
        r = rt.clone()
        r[0, :, 2:] += sign * delta * torch.tensor(d, device=DEV)
        return B_.opt_min_curv_batch(r, nv, h, KB_MIXED, wv + sign * delta, n_pts=npts)["alpha"][0].cpu().numpy()
    fd = gbar[0] @ (alpha(1.0) - alpha(-1.0)) / (2.0 * delta)
    ad = float(gw[0, :, 0] @ d[:, 0] + gw[0, :, 1] @ d[:, 1] + gv[0])
    print(f"N=1000 row instance: central difference {fd:.6e}, gradient {ad:.6e}, rel {abs(fd - ad) / abs(ad):.2e}")
    assert abs(fd - ad) <= FD_TOL * abs(ad)


def test_nothing_else_moves(golden):
    """Flag on against off: the forward bit for bit, the gradients of the box-only instances bit for bit.  With the
    flag on: the same gradients with sharing, in chunks of three, with w_veh as a float."""
    cases, centre_id, rows = _mixed_cases(golden)
    rt, nv, h, npts, wv = _pack(cases)
    gbar = torch.tensor(_gbar(cases, 4), device=DEV)
    cid = torch.tensor(centre_id, device=DEV)

    def run(w_veh, **kw):
        widths = rt[:, :, 2:].clone().requires_grad_()
        res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, KB_MIXED, w_veh, n_pts=npts, strict=False, **kw)
        (gw,) = torch.autograd.grad(res["alpha"], (widths,), gbar)
        return res, gw
    off, gw_off = run(wv, centre_id=cid)
    on, gw_on = run(wv, centre_id=cid, curvature_rows=True)
    for k in ("alpha", "curv_error_max", "kappa_lin_max", "status", "iters"):
        assert torch.equal(off[k], on[k]), k
    box = [b for b in range(len(cases)) if b not in rows]
    assert off["grad_status"].tolist() == [4 if b in rows else (1 if b == 7 else 0) for b in range(len(cases))]
    assert torch.equal(gw_on[box], gw_off[box])
    assert gw_on[rows].abs().amax(dim=(1, 2)).min() > 0.0 and not gw_off[rows].any()
    for kw in (dict(), dict(centre_id=cid, max_chunk=3), dict(max_chunk=1)):
        assert torch.equal(run(wv, curvature_rows=True, **kw)[1], gw_on), kw
    assert torch.equal(run(2.0, curvature_rows=True, centre_id=cid)[1], gw_on)       # every w_veh of the batch is 2.0


def test_one_instance_alone_and_in_a_batch_larger_than_the_resident_ctas(golden):
    cases, _, _ = _mixed_cases(golden)
    picks = [0, 1, 3, 4]                                           # two row instances, a box-only one, a row follower
    sub = [cases[b] for b in picks]
    gbar = _gbar(sub, 5)
    alone = [_grads([c], KB_MIXED, gbar[b:b + 1, :c["rt"].shape[0]], curvature_rows=True)[1:] for b, c in enumerate(sub)]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    reps = -(-2 * sms * 8 // len(sub))
    big = sub * reps
    _, gw, gv = _grads(big, KB_MIXED, np.tile(gbar, (reps, 1)), curvature_rows=True)
    print(f"{len(big)} instances ({sms} SMs)")
    for b in range(len(big)):
        n = big[b]["rt"].shape[0]
        a_gw, a_gv = alone[b % len(sub)]
        assert np.array_equal(gw[b, :n], a_gw[0, :n]) and gv[b] == a_gv[0], b


def test_lap_time_chain_through_the_curvature_rows(golden):
    """widths -> opt_min_curv_diff(curvature_rows=True) -> create_raceline_diff -> vel_profile_diff on synth160_kappa:
    finite, nonzero width gradients that a central difference of the device lap time confirms."""
    g = golden("synth160_kappa")
    v = golden("velprofile")
    c = _golden_case(golden, "synth160_kappa", float(g["kappa_bound"]))
    rt, nv, h, npts, wv = _pack([c])

    def lap(widths, want_grad):
        res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, c["kb"], 2.0, n_pts=npts, curvature_rows=True)
        rl = B_.create_raceline_diff(rt[:, :, :2], nv, res["alpha"], STEP, n_pts=npts)
        out = B_.vel_profile_diff(rl["kappa"], rl["el_lengths_interp"], v["ggv"], v["ax_max_machines"], 70.0,
                                  n_pts=rl["n_out"], **VEH)
        assert int(res["grad_status"][0]) == 0 and int(out["grad_status"][0]) == 0
        return out["laptime"], int(rl["n_out"][0])
    w = rt[:, :, 2:].clone().requires_grad_()
    t0, n_out = lap(w, True)
    (gw,) = torch.autograd.grad(t0.sum(), (w,))
    gw = gw.cpu().numpy()[0]
    assert np.isfinite(gw).all() and np.abs(gw).max() > 0.0
    n = c["rt"].shape[0]
    s = np.linspace(0.0, 2.0 * np.pi, n, endpoint=False)
    d = np.stack((np.sin(2.0 * s), np.cos(3.0 * s)), axis=1)
    delta = 1e-4
    lp, np_ = lap(rt[:, :, 2:] + delta * torch.tensor(d, device=DEV)[None], False)
    lm, nm = lap(rt[:, :, 2:] - delta * torch.tensor(d, device=DEV)[None], False)
    assert np_ == nm == n_out
    fd = float((lp - lm).sum()) / (2.0 * delta)
    ad = float((gw * d).sum())
    print(f"lap-time chain on synth160_kappa: central difference {fd:.6e}, gradient {ad:.6e}, rel {abs(fd - ad) / abs(ad):.2e}")
    assert abs(fd - ad) <= CHAIN_TOL * abs(ad)
