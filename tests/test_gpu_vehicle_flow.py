"""GPU tests (-m gpu) of a vehicle per track through the whole flow: a [B] curvature limit in the minimum-curvature QPs
(mincurv_finalize_kernel<., true>, the curvature-row phase with kb_batch), a vehicle size, drag and mass per trajectory in
check_traj (min_bound_dists_kernel<true>, traj_extrema_kernel<true>), and globaltraj_batch(vehicles=, veh_id=).

The contract: each track of a per-track call is bit for bit that track in the scalar call over the same whole batch, with
the same chunking, at the track's own value (one scalar call per distinct value), so that batch composition stays out
of the comparison."""
import numpy as np
import pytest
import torch

import mincurv_ref as R
import qp_sens as Q
from global_racetrajectory_optimization_b200 import batch as B_, globaltraj, raceline_refine as RR, synth
from oracle import tph_dense as T

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = ["berlin", "handling", "modena", "synth1000", "synth333", "synth333_kappa", "synth160_kappa", "synth500"]
QP_KEYS = ("alpha", "status", "iters", "curv_error_max", "kappa_lin_max")
LIMITS = (0.12, 0.06, 0.04, 0.03)
KAPPA_REL = 1e-7            # the finalize stage's acceptance of |k_ref + E alpha| <= kb (status 4 beyond it)
CERT_STAT_TOL = 8e-6        # tests/test_gpu_edges.py: the KKT certificate of a device solution
CERT_COMP_TOL = 4e-9
CERT_FEAS_TOL = 1e-9


def _golden_batch(golden, copies=1):
    """The GOLDEN tracks (and copies - 1 width-jitter variants of each, sharing its centre line), with normals, h, n_pts,
    the fixtures' w_veh and the centre ids of the shared centre lines."""
    gs = [golden(nm) for nm in GOLDEN]
    n = [g["reftrack"].shape[0] for g in gs]
    rt = np.zeros((len(gs), max(n), 4))
    for b, g in enumerate(gs):
        rt[b, :n[b]] = g["reftrack"]
    rt = torch.tensor(rt, device=DEV).repeat(copies, 1, 1)
    npts = torch.tensor(n, dtype=torch.int32, device=DEV).repeat(copies)
    wv = torch.tensor([float(g["w_veh"]) for g in gs], dtype=torch.float64, device=DEV).repeat(copies)
    B = rt.shape[0]
    cid = (torch.arange(B, device=DEV) % len(gs)).to(torch.int32)
    if copies > 1:
        seeds = torch.arange(B, dtype=torch.int64, device=DEV) + 17
        jit, _ = B_.jitter_widths_batch(rt, seeds, rel=0.05, centre_id=torch.arange(B, device=DEV), n_pts_base=npts)
        rt = torch.where((torch.arange(B, device=DEV) < len(gs))[:, None, None], rt, jit)
    _, _, nv, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    return rt, nv, h, npts, wv, cid


def _c1_batch(B=2112, n=1000, n_base=32):
    """A c1-sized batch: n_base synthetic centre lines and width-jitter variants of them (variant b of line b % n_base)."""
    base = torch.tensor(synth.make_batch(4242, n_base, n), device=DEV)
    rt, _ = B_.jitter_widths_batch(base, torch.arange(B, dtype=torch.int64, device=DEV) + 1)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    return rt, nv, h, (torch.arange(B, device=DEV) % n_base).to(torch.int32)


def _rows_equal(a, b, m, npts=None):
    """a[m] == b[m] bit for bit; with npts only the first npts[b] entries of each row of a [B, n_max] tensor."""
    if npts is not None and a.ndim == 2:
        valid = torch.arange(a.shape[1], device=a.device)[None, :] < npts[:, None].to(a.device)
        a, b = torch.where(valid, a, 0.0), torch.where(valid, b, 0.0)
    return torch.equal(a[m], b[m])


def _per_value(run, kb, keys, npts=None):
    """run(kappa_bound) -> dict: the call with the [B] tensor kb against the scalar calls, one per distinct value."""
    kb = torch.as_tensor(kb, dtype=torch.float64, device=DEV)
    got = run(kb)
    for v in torch.unique(kb).tolist():
        ref = run(v)
        m = kb == v
        for k in keys:
            assert _rows_equal(got[k], ref[k], m, npts), (k, v)
    return got


def _mixed(B):
    return torch.tensor([LIMITS[(3 * b + b // 7) % len(LIMITS)] for b in range(B)], dtype=torch.float64, device=DEV)


# ---- the QP with a constant tensor is the float call ------------------------------------------------------------------
def test_constant_tensor_is_the_float_call_on_the_golden_tracks(golden):
    rt, nv, h, npts, wv, cid = _golden_batch(golden, copies=3)
    B = rt.shape[0]
    for kb in (0.12, 0.04):
        for centre_id in (None, cid):
            for chunk in (B, 5):
                ref = B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts, centre_id=centre_id, max_chunk=chunk)
                got = B_.opt_min_curv_batch(rt, nv, h, torch.full((B,), kb, dtype=torch.float64, device=DEV), wv,
                                            n_pts=npts, centre_id=centre_id, max_chunk=chunk)
                for k in QP_KEYS:
                    assert _rows_equal(got[k], ref[k], slice(None), npts), (k, kb, centre_id is None, chunk)


def test_constant_tensor_is_the_float_call_on_a_c1_batch():
    rt, nv, h, cid = _c1_batch()
    B = rt.shape[0]
    for centre_id in (None, cid):
        ref = B_.opt_min_curv_batch(rt, nv, h, 0.12, 3.4, centre_id=centre_id, max_chunk=B // 2)
        got = B_.opt_min_curv_batch(rt, nv, h, torch.full((B,), 0.12, dtype=torch.float64, device=DEV), 3.4,
                                    centre_id=centre_id, max_chunk=B // 2)
        for k in QP_KEYS:
            assert torch.equal(got[k], ref[k]), k
        assert bool((ref["status"] == 0).all())


def test_a_few_tight_limits_in_a_c1_batch():
    rt, nv, h, cid = _c1_batch()
    B = rt.shape[0]
    kb = torch.full((B,), 0.12, dtype=torch.float64, device=DEV)
    kb[::97] = 0.03
    run = lambda k: B_.opt_min_curv_batch(rt, nv, h, k, 3.4, centre_id=cid, max_chunk=B // 2)      # noqa: E731
    got = _per_value(run, kb, QP_KEYS)
    assert bool((got["status"] == 0).all())
    assert bool((got["kappa_lin_max"] <= kb * (1.0 + KAPPA_REL)).all())


# ---- a mixed batch of limits -------------------------------------------------------------------------------------------
def test_mixed_limits_are_the_scalar_calls_and_certified(golden):
    rt, nv, h, npts, wv, cid = _golden_batch(golden, copies=4)
    B = rt.shape[0]
    kb = _mixed(B)
    for centre_id in (None, cid):
        run = lambda k: B_.opt_min_curv_batch(rt, nv, h, k, wv, n_pts=npts, centre_id=centre_id, max_chunk=11)  # noqa
        got = _per_value(run, kb, QP_KEYS, npts)
    # the curvature-row phase really runs: instances the box phase left at status 4 end at status 0
    d = B_.opt_min_curv_diff(rt[:, :, :2], rt[:, :, 2:], nv, h, kb, wv, n_pts=npts, max_chunk=11)
    rows = (d["grad_status"] == 4) & (d["status"] == 0)
    print(f"VEHFLOW mixed: {int(rows.sum())} of {B} instances solved by the curvature-row phase")
    assert int(rows.sum()) >= 4
    # the tightest limits are not reachable on every track: those instances keep a failure status (tph would raise)
    ok = got["status"] == 0
    print(f"VEHFLOW mixed: statuses {got['status'].tolist()}")
    assert int(ok.sum()) >= B // 2
    assert bool((got["kappa_lin_max"][ok] <= kb[ok] * (1.0 + KAPPA_REL)).all())
    # the KKT certificate of the full QP at each instance's own limit (the oracle's dense QP; tracks up to 520 points)
    worst = [0.0, 0.0]
    for b in range(B):
        n = int(npts[b])
        if n > 520 or not bool(ok[b]):
            continue
        r = rt[b, :n].cpu().numpy()
        _, _, A, nvo = T.calc_splines(np.vstack((r[:, :2], r[0, :2])))
        qp = T.assemble_min_curv(r, nvo, A, float(kb[b]), float(wv[b]))
        lb, ub, _ = Q.bounds(r, float(wv[b]))
        c = R.kkt_certificate(qp["H"], qp["f"], qp["E_kappa"], qp["k_kappa_ref"], lb, ub, float(kb[b]),
                              got["alpha"][b, :n].cpu().numpy(), act_box=1e-5, act_row=1e-4)
        assert c["box_viol"] <= CERT_FEAS_TOL and c["row_viol"] <= CERT_FEAS_TOL, (b, c)
        assert c["stat"] <= CERT_STAT_TOL and c["comp"] <= CERT_COMP_TOL, (b, c)
        worst = [max(worst[0], c["stat"]), max(worst[1], c["comp"])]
    print(f"VEHFLOW certificate: stationarity {worst[0]:.2e}, complementarity {worst[1]:.2e}")


def test_width_gradients_with_curvature_rows_per_value(golden):
    rt, nv, h, npts, wv, cid = _golden_batch(golden, copies=2)
    B, n_max = rt.shape[:2]
    kb = _mixed(B)
    w = torch.randn((B, n_max), dtype=torch.float64, device=DEV, generator=torch.Generator(DEV).manual_seed(5))

    def run(k):
        widths = rt[:, :, 2:].clone().requires_grad_()
        wvt = wv.clone().requires_grad_()
        res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, k, wvt, n_pts=npts, centre_id=cid, max_chunk=7,
                                   strict=False, curvature_rows=True)
        valid = torch.arange(n_max, device=DEV)[None, :] < npts[:, None]
        (torch.where(valid, res["alpha"], 0.0) * w).sum().backward()
        res = {k_: v.detach() for k_, v in res.items()}
        res.update(grad_widths=widths.grad.reshape(B, -1), grad_w_veh=wvt.grad)
        return res
    got = _per_value(run, kb, QP_KEYS + ("grad_status", "grad_w_veh"), npts)
    assert bool((got["grad_status"] == 0).any())
    ref_rows = {v: run(v)["grad_widths"] for v in torch.unique(kb).tolist()}
    for v, g in ref_rows.items():
        assert torch.equal(got["grad_widths"][kb == v], g[kb == v]), v


def test_iqp_and_refinement_per_value(golden):
    rt, nv, h, npts, wv, _ = _golden_batch(golden)
    B = rt.shape[0]
    kb = torch.tensor([0.12, 0.05] * (B // 2), dtype=torch.float64, device=DEV)
    iqp = lambda k: B_.iqp_batch(rt, nv, h, k, wv, 2.0, n_pts=npts)      # noqa: E731
    got = _per_value(iqp, kb, ("status", "n_pts", "outer_iters", "curv_error_max"))
    for v in torch.unique(kb).tolist():
        ref, m = iqp(v), kb == v
        L = min(got["alpha"].shape[1], ref["alpha"].shape[1])
        assert torch.equal(got["alpha"][m, :L], ref["alpha"][m, :L]) and torch.equal(got["reftrack"][m, :L], ref["reftrack"][m, :L])
    v = golden("velprofile")
    veh = dict(ggv=v["ggv"], ax_max_machines=v["ax_max_machines"], v_max=float(v["v_max"]), drag_coeff=float(v["dragcoeff"]),
               m_veh=float(v["mass"]))
    a0 = B_.opt_min_curv_batch(rt, nv, h, 0.12, wv, n_pts=npts)["alpha"]
    refine = lambda k: RR.refine_raceline_batch(rt, nv, a0, wv, n_pts=npts, metric_length=10.0, kappa_bound=k,  # noqa
                                                relinearise=2, max_iters=4, **veh)
    _per_value(refine, kb, ("alpha", "laptime", "status", "iters", "evals", "rounds", "kappa_lin_max", "curv_error_max"),
               npts)


# ---- refused limits on the device --------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", [float("nan"), 0.0, -0.1, float("inf")])
def test_a_refused_device_limit_touches_its_track_alone(golden, bad):
    rt, nv, h, npts, wv, cid = _golden_batch(golden, copies=2)
    B = rt.shape[0]
    kb = _mixed(B)
    ref = B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts, centre_id=cid, max_chunk=6)
    kb_bad = kb.clone()
    kb_bad[3] = bad
    got = B_.opt_min_curv_batch(rt, nv, h, kb_bad, wv, n_pts=npts, centre_id=cid, max_chunk=6)
    assert int(got["status"][3]) == -1
    others = torch.arange(B, device=DEV) != 3
    for k in QP_KEYS:
        assert _rows_equal(got[k], ref[k], others, npts), k
    d = B_.opt_min_curv_diff(rt[:, :, :2], rt[:, :, 2:], nv, h, kb_bad, wv, n_pts=npts, strict=False, curvature_rows=True)
    assert int(d["status"][3]) == -1 and int(d["grad_status"][3]) == -1


# ---- check_traj with a vehicle per trajectory --------------------------------------------------------------------------
def _cars(golden):
    v = golden("velprofile")
    ggv, mach = np.asarray(v["ggv"], float), np.asarray(v["ax_max_machines"], float)
    slow, weak = ggv.copy(), mach.copy()
    slow[:, 1:] *= 0.9
    weak[:, 1] *= 0.8
    return [dict(ggv=ggv, mach=mach, v_max=float(v["v_max"]), drag=float(v["dragcoeff"]), mass=float(v["mass"]),
                 curvlim=0.12, width_opt=3.4, length=4.7, width=2.0),
            dict(ggv=slow, mach=mach, v_max=float(v["v_max"]) - 10.0, drag=0.9, mass=1350.0, curvlim=0.05, width_opt=2.6,
                 length=4.2, width=1.8),
            dict(ggv=ggv, mach=weak, v_max=float(v["v_max"]), drag=0.7, mass=1100.0, curvlim=0.08, width_opt=3.0,
                 length=5.0, width=2.2)]


def _vehicles(cars, **kw):
    fields = {k: [c[k] for c in cars] for k in ("curvlim", "width_opt", "length", "width")}
    fields.update(kw)
    return B_.Vehicles([c["ggv"] for c in cars], [c["mach"] for c in cars], [c["v_max"] for c in cars],
                       [c["drag"] for c in cars], [c["mass"] for c in cars], **fields)


def _pars(car):
    p = globaltraj.default_pars()
    p["veh_params"].update(v_max=car["v_max"], length=car["length"], width=car["width"], mass=car["mass"],
                           dragcoeff=car["drag"], curvlim=car["curvlim"])
    p["optim_opts"]["width_opt"] = car["width_opt"]
    return p


def test_check_traj_per_trajectory_and_flags_per_vehicle(golden):
    rt, nv, h, npts, wv, _ = _golden_batch(golden)
    B = rt.shape[0]
    cars = _cars(golden)
    ids = torch.tensor([b % 3 for b in range(B)], dtype=torch.int32, device=DEV)
    out = globaltraj.globaltraj_batch(rt, "mincurv", _pars(cars[0]), cars[0]["ggv"], cars[0]["mach"], n_pts=npts,
                                      check=False)
    args = (rt, nv, out["raceline_interp"], out["psi"], out["kappa"], out["vx"], out["ax"])
    per = {k: torch.tensor([cars[int(i)][k] for i in ids.tolist()], dtype=torch.float64, device=DEV)
           for k in ("length", "width", "drag", "mass")}
    got = B_.check_traj_batch(*args, per["length"], per["width"], per["drag"], per["mass"], n_pts=npts, n_traj=out["n_out"])
    veh = _vehicles(cars)
    flags = B_.check_traj_flags(got, vehicles=veh, veh_id=ids)
    for k, c in enumerate(cars):
        ref = B_.check_traj_batch(*args, c["length"], c["width"], c["drag"], c["mass"], n_pts=npts, n_traj=out["n_out"])
        m = ids == k
        for key in ("min_dists",) + B_.EXTREMA:
            assert torch.equal(got[key][m], ref[key][m]), (key, k)
        rf = B_.check_traj_flags(ref, c["ggv"], c["mach"], c["v_max"], c["curvlim"])
        for key, f in rf.items():
            assert torch.equal(flags[key][m], f[m]), (key, k)
    # a trajectory whose device mass is not > 0 is refused alone
    bad = per["mass"].clone()
    bad[1] = 0.0
    ext = B_.traj_extrema_batch(out["kappa"], out["vx"], out["ax"], per["drag"], bad, n_traj=out["n_out"])
    ok = B_.traj_extrema_batch(out["kappa"], out["vx"], out["ax"], per["drag"], per["mass"], n_traj=out["n_out"])
    assert bool(torch.isnan(ext[1, :7]).all()) and float(ext[1, 7]) == float(out["n_out"][1])
    assert torch.equal(torch.cat((ext[:1], ext[2:])), torch.cat((ok[:1], ok[2:])))


# ---- globaltraj_batch with a car per track -----------------------------------------------------------------------------
@pytest.mark.parametrize("opt_type,refine", [("mincurv", None), ("mincurv_iqp", None), ("shortest_path", None),
                                             ("mincurv", {"metric_length": 10.0, "max_iters": 6}),
                                             ("mincurv", {"metric_length": 10.0, "max_iters": 4, "kappa_bound": "curvlim"})])
def test_globaltraj_with_a_car_per_track_is_each_cars_call(golden, opt_type, refine):
    """refine with kappa_bound "curvlim" (a marker of this test): the refinement under each car's limit, a [B] tensor
    gathered from the Vehicles against each car's scalar curvlim."""
    rt, nv, h, npts, wv, _ = _golden_batch(golden)
    B = rt.shape[0]
    cars = _cars(golden)
    ids = torch.tensor([(b * 2) % 3 for b in range(B)], dtype=torch.int32, device=DEV)
    veh = _vehicles(cars)
    limit = refine is not None and refine.get("kappa_bound") == "curvlim"
    ref_of = lambda c: dict(refine, kappa_bound=c["curvlim"]) if limit else refine       # noqa: E731
    got = globaltraj.globaltraj_batch(rt, opt_type, _pars(cars[0]), n_pts=npts, vehicles=veh, veh_id=ids,
                                      refine=dict(refine, kappa_bound=veh.per_track("curvlim", ids)) if limit else refine)
    if limit:
        assert int((got["refine_status"] == 0).sum() + (got["refine_status"] == 1).sum()) >= 2
    for k, c in enumerate(cars):
        ref = globaltraj.globaltraj_batch(rt, opt_type, _pars(c), c["ggv"], c["mach"], n_pts=npts, refine=ref_of(c))
        m = ids == k
        assert set(got) == set(ref)
        for key, r in ref.items():
            g = got[key]
            if not isinstance(r, torch.Tensor):
                continue
            if key in ("alpha", "qp_alpha") and opt_type != "mincurv_iqp":
                assert _rows_equal(g, r, m, npts), (key, k)
                continue
            if g.ndim > 1 and g.shape[1] != r.shape[1]:      # (capacities derived from the whole batch)
                L = min(g.shape[1], r.shape[1])
                g, r = g[:, :L], r[:, :L]
            assert torch.equal(torch.nan_to_num(g[m], nan=7.25), torch.nan_to_num(r[m], nan=7.25)), (key, k)
    if limit:
        return
    # a field the Vehicles leave unset comes from pars for every track
    part = globaltraj.globaltraj_batch(rt, opt_type, _pars(cars[1]), n_pts=npts, refine=refine,
                                       vehicles=_vehicles(cars, curvlim=None, width_opt=None), veh_id=ids)
    mixed = [dict(c, curvlim=cars[1]["curvlim"], width_opt=cars[1]["width_opt"]) for c in cars]
    ref = globaltraj.globaltraj_batch(rt, opt_type, _pars(mixed[0]), n_pts=npts, refine=refine, vehicles=_vehicles(mixed),
                                      veh_id=ids)
    for key in ("status", "laptime", "vx"):
        assert torch.equal(part[key], ref[key]), key


# ---- an id out of range on the device: NaN fields, refused tracks ---------------------------------------------------------
def test_a_non_finite_vehicle_width_stays_in_its_instance(golden):
    rt, nv, h, npts, wv, cid = _golden_batch(golden, copies=2)
    B = rt.shape[0]
    bad = wv.clone()
    bad[2] = float("nan")
    bad[B - 1] = float("inf")
    others = torch.ones(B, dtype=torch.bool, device=DEV)
    others[[2, B - 1]] = False
    for centre_id in (None, cid):
        ref = B_.opt_min_curv_batch(rt, nv, h, 0.12, wv, n_pts=npts, centre_id=centre_id, max_chunk=5)
        got = B_.opt_min_curv_batch(rt, nv, h, 0.12, bad, n_pts=npts, centre_id=centre_id, max_chunk=5)
        assert got["status"][~others].tolist() == [-1, -1]
        for k in QP_KEYS:
            assert _rows_equal(got[k], ref[k], others, npts), (k, centre_id is None)
    sp_ref = B_.opt_shortest_path_batch(rt, nv, wv, n_pts=npts)
    sp = B_.opt_shortest_path_batch(rt, nv, bad, n_pts=npts)
    # the shortest path ends the NaN instance with status 3; an infinite width is clamped to tph's 0.001 m bounds there
    assert int(sp["status"][2]) == 3
    for k in ("alpha", "status", "iters"):
        assert torch.equal(sp[k][others], sp_ref[k][others]), k
    # globaltraj_batch with a device veh_id out of range: that track's fields are NaN, its QP and profile are refused
    cars = _cars(golden)
    ids = torch.tensor([b % 3 for b in range(B)], dtype=torch.int32, device=DEV)
    ids_bad = ids.clone()
    ids_bad[2] = 7
    veh = _vehicles(cars)
    for opt_type in ("mincurv",):           # (a shortest-path alpha of status 3 is not finite: the raceline stage raises)
        ok = globaltraj.globaltraj_batch(rt, opt_type, _pars(cars[0]), n_pts=npts, vehicles=veh, veh_id=ids, check=False)
        out = globaltraj.globaltraj_batch(rt, opt_type, _pars(cars[0]), n_pts=npts, vehicles=veh, veh_id=ids_bad,
                                          check=False)
        assert int(out["status"][2]) == -1 and int(out["vel_status"][2]) == 5, opt_type
        keep = torch.arange(B, device=DEV) != 2
        assert torch.equal(out["status"][keep], ok["status"][keep]) and torch.equal(out["laptime"][keep], ok["laptime"][keep])
