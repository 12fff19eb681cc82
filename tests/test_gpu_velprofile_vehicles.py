"""GPU tests (-m gpu) of the velocity profile with a vehicle per track (batch.Vehicles, vehicles= / veh_id=;
csrc/vel_profile.cu: vel_profile_veh_kernel, vel_profile_adjoint_veh_kernel).  The contract: a track's profile, lap
time, status and gradient in vehicle mode are bit for bit those of the single-vehicle call for that track with its
vehicle's tables and scalars, however the vehicles are mixed in the batch.

1. K = 1 with veh_id all zero is the existing call, on the golden racelines and every lap of tests/vp_cases.py, both
   readings of decel_slice_upper, dyn_model_exp 1 / 1.5 / 2, mu and filter windows.
2. A mixed batch (every vp_cases lap x vehicles of 1, 2, 18 and 256 rows, top speeds on an interior and on the last
   knot, different drag and mass, veh_id interleaved so that every CTA holds several vehicles) is the per-vehicle calls
   track by track, and the host build of the same statements; at dyn_model_exp 1 its vx is the oracle's.
3. The lap-time matrix with vehicles is lap_time_matrix_batch per vehicle.
4. vel_profile_diff / lap_time_matrix_diff gradients are the per-vehicle calls', whatever max_chunk and batch order.
5. refine_raceline_batch with vehicles: each golden track's result is that track refined alone with its vehicle, and the
   objective does not synchronise the stream.
6. An out-of-range device veh_id refuses its track alone (status 5); inactive slots behave as without vehicles."""
import numpy as np
import pytest

import vp_cases as C
from oracle import tph_velprofile as VP
from vp_adj_ref import Harness

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine as R  # noqa: E402

DEV = "cuda"
CASES = C.cases()
BAD_VEHICLE = 5
GOLDEN = ["berlin", "handling", "modena", "synth333", "synth1000"]
# The oracle squares speeds with libm's pow, the kernel multiplies; pow(v, 2) is not always v * v, so on some (lap,
# vehicle) pairs vx differs from the oracle's in its last bits.  The host build of the kernel's statements differs in
# the same places; this bound on |vx - vx_oracle| was measured there at 7.1e-15 m/s (7 of 52 pairs, both readings)
ORACLE_VX_ATOL = 1e-14


def t_(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def ragged(tracks, n_max=None):
    n_max = n_max or max(k.size for k, _ in tracks)
    kap = np.full((len(tracks), n_max), np.nan)
    el = np.full((len(tracks), n_max), np.nan)
    for b, (k, e) in enumerate(tracks):
        kap[b, :k.size], el[b, :e.size] = k, e
    return t_(kap), t_(el), t_([k.size for k, _ in tracks], torch.int32)


def same(a: dict, b: dict, keys=("laptime", "status", "vx", "ax", "t")):
    for k in keys:
        assert torch.equal(a[k], b[k]), k


def golden_racelines(golden):
    return [(golden(nm)["rl_kappa"], golden(nm)["rl_el_lengths"]) for nm in GOLDEN]


def stock(golden):
    v = golden("velprofile")
    return dict(ggv=v["ggv"], ax_max_machines=v["ax_max_machines"], v_max=float(v["v_max"]),
                drag_coeff=float(v["dragcoeff"]), m_veh=float(v["mass"]))


def vehicles_of(vehs):
    """Vehicles from a list of dict(ggv, ax_max_machines, v_max, drag_coeff, m_veh)."""
    return B_.Vehicles([v["ggv"] for v in vehs], [v["ax_max_machines"] for v in vehs], [v["v_max"] for v in vehs],
                       [v["drag_coeff"] for v in vehs], [v["m_veh"] for v in vehs])


# ---- 1. K = 1 is the existing call -------------------------------------------------------------------------------------
def test_one_vehicle_is_the_existing_call_on_the_golden_racelines(golden):
    veh = stock(golden)
    kap, el, npts = ragged(golden_racelines(golden))
    one = vehicles_of([veh])
    zeros = torch.zeros(len(GOLDEN), dtype=torch.int32, device=DEV)
    for kw in (dict(), dict(decel_slice_upper=0), dict(dyn_model_exp=1.5), dict(filt_window=9)):
        ref = B_.vel_profile_batch(kap, el, n_pts=npts, **veh, **kw)
        got = B_.vel_profile_batch(kap, el, n_pts=npts, vehicles=one, veh_id=zeros, **kw)
        same(got, ref)
        assert bool((ref["status"] == 0).all())


@pytest.mark.parametrize("upper", [1, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_one_vehicle_is_the_existing_call_on_every_case(name, upper):
    c = CASES[name]
    rng = np.random.default_rng(len(name))
    mu = t_(0.75 + 0.4 * rng.random(c["kappa"].size))[None]
    veh = dict(ggv=c["ggv"], ax_max_machines=c["mach"], v_max=c["v_max"], **C.VEH)
    one = vehicles_of([veh])
    kap, el = t_(c["kappa"])[None], t_(c["el"])[None]
    for kw in (dict(), dict(dyn_model_exp=1.5), dict(dyn_model_exp=2.0), dict(mu=mu), dict(filt_window=9),
               dict(dyn_model_exp=1.5, mu=mu, filt_window=3)):
        ref = B_.vel_profile_batch(kap, el, decel_slice_upper=upper, **veh, **kw)
        got = B_.vel_profile_batch(kap, el, decel_slice_upper=upper, vehicles=one, veh_id=[0], **kw)
        same(got, ref)


# ---- 2. a mixed batch ------------------------------------------------------------------------------------------------
def mixed_vehicles():
    g18, m18 = C.ggv_table(18), C.mach_table(18)
    g256, m256 = C.ggv_table(256), C.mach_table(256)
    return [dict(ggv=C.ggv_table(1, v1=80.0), ax_max_machines=C.mach_table(1, v1=80.0), v_max=50.0, drag_coeff=0.75,
                 m_veh=1200.0),
            dict(ggv=C.ggv_table(2), ax_max_machines=C.mach_table(2), v_max=72.0, drag_coeff=0.9, m_veh=900.0),  # last knot
            dict(ggv=g18, ax_max_machines=m18, v_max=float(g18[11, 0]), drag_coeff=0.6, m_veh=1400.0),       # interior
            dict(ggv=g256, ax_max_machines=m256, v_max=float(g256[200, 0]), drag_coeff=1.1, m_veh=750.0)]


def mixed_batch():
    """(tracks, veh_id): every case's lap with every vehicle, the vehicles cycling from track to track."""
    names = sorted(CASES)
    K = len(mixed_vehicles())
    tracks, ids = [], []
    for r in range(K):
        for i, nm in enumerate(names):
            tracks.append((CASES[nm]["kappa"], CASES[nm]["el"]))
            ids.append((i + r) % K)
    return tracks, ids


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return Harness(tmp_path_factory.mktemp("vp_veh_gpu"))


@pytest.mark.parametrize("upper", [1, 0])
def test_a_mixed_batch_is_the_per_vehicle_calls(harness, upper):
    vehs = mixed_vehicles()
    tracks, ids = mixed_batch()
    kap, el, npts = ragged(tracks)
    got = B_.vel_profile_batch(kap, el, n_pts=npts, vehicles=vehicles_of(vehs), veh_id=ids, decel_slice_upper=upper)
    assert len(set(ids[:128])) == len(vehs)
    worst = 0.0
    for k, veh in enumerate(vehs):
        sel = [b for b in range(len(ids)) if ids[b] == k]
        alone = B_.vel_profile_batch(kap[sel], el[sel], n_pts=npts[sel], decel_slice_upper=upper, **veh)
        same({key: v[sel] for key, v in got.items()}, alone)
        for j, b in enumerate(sel):
            kk, ee = tracks[b]
            n = kk.size
            vx = got["vx"][b, 0, :n].cpu().numpy()
            h = harness.profile(kk, ee, veh["ggv"], veh["ax_max_machines"], veh["v_max"], upper=upper,
                                drag_coeff=veh["drag_coeff"], m_veh=veh["m_veh"])
            assert int(got["status"][b, 0]) == 0 and h["status"] == 0
            assert np.array_equal(vx, h["vx"]) and float(got["laptime"][b, 0]) == h["laptime"]
            saved = VP.DECEL_LAP_SLICE_UPPER
            VP.DECEL_LAP_SLICE_UPPER = bool(upper)
            try:
                ovx = VP.calc_vel_profile(ggv=veh["ggv"], ax_max_machines=veh["ax_max_machines"], v_max=veh["v_max"],
                                          kappa=kk, el_lengths=ee, closed=True, dyn_model_exp=1.0, filt_window=None,
                                          drag_coeff=veh["drag_coeff"], m_veh=veh["m_veh"])
            finally:
                VP.DECEL_LAP_SLICE_UPPER = saved
            if np.array_equal(h["vx"], ovx):
                assert np.array_equal(vx, ovx)
            worst = max(worst, float(np.abs(vx - ovx).max()))
    print(f"  mixed batch: max |vx - vx_oracle| {worst:.2e} m/s, bound {ORACLE_VX_ATOL:.0e}")
    assert worst <= ORACLE_VX_ATOL


def test_a_mixed_batch_with_per_variant_scales_and_top_speeds():
    vehs = mixed_vehicles()
    tracks, ids = mixed_batch()
    kap, el, npts = ragged(tracks)
    veh = vehicles_of(vehs)
    for v_max in (None, [45.0, 50.0, 40.0]):
        got = B_.vel_profile_batch(kap, el, n_pts=npts, vehicles=veh, veh_id=t_(ids, torch.int32), ggv_scales=[0.8, 1.0, 1.2],
                                   v_max=v_max)
        for k, vk in enumerate(vehs):
            sel = [b for b in range(len(ids)) if ids[b] == k]
            vm = [vk["v_max"]] * 3 if v_max is None else v_max
            alone = B_.vel_profile_batch(kap[sel], el[sel], vk["ggv"], vk["ax_max_machines"], vm, vk["drag_coeff"],
                                         vk["m_veh"], n_pts=npts[sel], ggv_scales=[0.8, 1.0, 1.2])
            same({key: v[sel] for key, v in got.items()}, alone)


# ---- 3. the lap-time matrix -----------------------------------------------------------------------------------------
def golden_vehicles(golden):
    s = stock(golden)
    return [s, dict(s, v_max=60.0, drag_coeff=0.9, m_veh=1000.0),
            dict(s, ggv=C.ggv_table(18), ax_max_machines=C.mach_table(18), v_max=68.0, m_veh=1350.0)]


def test_lap_time_matrix_with_vehicles_is_the_per_vehicle_matrix(golden):
    vehs = golden_vehicles(golden)
    kap, el, npts = ragged(golden_racelines(golden))
    ids = [2, 0, 1, 1, 0]
    scales, speeds = np.linspace(0.6, 1.3, 14), np.linspace(30.0, 70.0, 11)               # 154 cells
    got = B_.lap_time_matrix_batch(kap, el, ggv_scales=scales, top_speeds=speeds, n_pts=npts, vehicles=vehicles_of(vehs),
                                   veh_id=ids)
    own = B_.lap_time_matrix_batch(kap, el, ggv_scales=scales, n_pts=npts, vehicles=vehicles_of(vehs), veh_id=ids)
    for k, v in enumerate(vehs):
        sel = [b for b in range(len(ids)) if ids[b] == k]
        ref = B_.lap_time_matrix_batch(kap[sel], el[sel], v["ggv"], v["ax_max_machines"], scales, speeds, v["drag_coeff"],
                                       v["m_veh"], n_pts=npts[sel])
        assert torch.equal(got[sel], ref)
        ref1 = B_.lap_time_matrix_batch(kap[sel], el[sel], v["ggv"], v["ax_max_machines"], scales, [v["v_max"]],
                                        v["drag_coeff"], v["m_veh"], n_pts=npts[sel])
        assert torch.equal(own[sel], ref1)


# ---- 4. gradients ----------------------------------------------------------------------------------------------------
def _grads(fn, kap, el, w, **kw):
    """(fn's result, dL/dkappa, dL/del) for L = sum(w * laptime): w holds each track's (or cell's) upstream gradient."""
    k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
    out = fn(k, e, **kw)
    (out["laptime"] * w).sum().backward()
    return out, k.grad, e.grad


def weights(*shape):
    return torch.linspace(0.5, 1.5, int(np.prod(shape)), dtype=torch.float64, device=DEV).reshape(shape)


def test_vel_profile_diff_with_vehicles_is_the_per_vehicle_gradient(golden):
    vehs = golden_vehicles(golden)
    kap, el, npts = ragged(golden_racelines(golden))
    ids = [1, 2, 0, 2, 1]
    veh = vehicles_of(vehs)
    W = weights(len(ids))
    base = None
    for chunk, order in ((None, [0, 1, 2, 3, 4]), (1, [0, 1, 2, 3, 4]), (2, [4, 2, 0, 3, 1])):
        o = torch.tensor(order, device=DEV)
        out, gk, ge = _grads(B_.vel_profile_diff, kap[o], el[o], W[o], n_pts=npts[o], vehicles=veh,
                             veh_id=[ids[i] for i in order], max_chunk=chunk)
        inv = torch.argsort(o)
        res = (out["laptime"].detach()[inv], out["grad_status"][inv], gk[inv], ge[inv])
        if base is None:
            base = res
            assert bool((out["grad_status"] == 0).all())
        for a, b in zip(res, base):
            assert torch.equal(a, b)
    for b in range(len(ids)):
        v = vehs[ids[b]]
        out, gk, ge = _grads(B_.vel_profile_diff, kap[b:b + 1], el[b:b + 1], W[b:b + 1], n_pts=npts[b:b + 1], **v)
        assert torch.equal(out["laptime"].detach()[0], base[0][b])
        assert torch.equal(gk[0], base[2][b]) and torch.equal(ge[0], base[3][b])


def test_lap_time_matrix_diff_with_vehicles_is_the_per_vehicle_gradient(golden):
    vehs = golden_vehicles(golden)
    kap, el, npts = ragged(golden_racelines(golden))
    ids = [0, 2, 2, 1, 0]
    veh = vehicles_of(vehs)
    scales, speeds = [0.7, 1.0, 1.2], [40.0, 55.0]
    W = weights(len(ids), 2, 3)
    base = None
    for chunk, order in ((None, [0, 1, 2, 3, 4]), (2, [3, 1, 4, 0, 2])):
        o = torch.tensor(order, device=DEV)
        out, gk, ge = _grads(B_.lap_time_matrix_diff, kap[o], el[o], W[o], ggv_scales=scales, top_speeds=speeds,
                             n_pts=npts[o], vehicles=veh, veh_id=[ids[i] for i in order], max_chunk=chunk)
        inv = torch.argsort(o)
        res = (out["laptime"].detach()[inv], gk[inv], ge[inv])
        if base is None:
            base = res
            assert bool((out["grad_status"] == 0).all())
        for a, b in zip(res, base):
            assert torch.equal(a, b)
    for k, v in enumerate(vehs):
        sel = [b for b in range(len(ids)) if ids[b] == k]
        s = torch.tensor(sel, device=DEV)
        out, gk, ge = _grads(B_.lap_time_matrix_diff, kap[s], el[s], W[s], ggv=v["ggv"], ax_max_machines=v["ax_max_machines"],
                             ggv_scales=scales, top_speeds=speeds, drag_coeff=v["drag_coeff"], m_veh=v["m_veh"],
                             n_pts=npts[s])
        assert torch.equal(out["laptime"].detach(), base[0][s])
        assert torch.equal(gk, base[1][s]) and torch.equal(ge, base[2][s])


# ---- 5. the refinement -----------------------------------------------------------------------------------------------
REFINE = ["berlin", "handling", "modena", "synth1000"]


def _refine_batch(golden, names):
    gs = [golden(nm) for nm in names]
    n = [g["reftrack"].shape[0] for g in gs]
    rt = np.zeros((len(gs), max(n), 4))
    al = np.zeros((len(gs), max(n)))
    for b, g in enumerate(gs):
        rt[b, :n[b]], al[b, :n[b]] = g["reftrack"], g["alpha_mincurv"]
    rt, al = t_(rt), t_(al)
    npts = t_(n, torch.int32)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    wv = t_([float(g["w_veh"]) for g in gs])
    return rt, nv, al, npts, wv, n


def test_refinement_with_vehicles_is_each_track_refined_alone(golden):
    vehs = golden_vehicles(golden)
    ids = [1, 0, 2, 1]
    rt, nv, al, npts, wv, n = _refine_batch(golden, REFINE)
    res = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=2.0, max_iters=8, vehicles=vehicles_of(vehs),
                                  veh_id=ids)
    assert bool((res["status"] >= 0).all())
    for b in range(len(REFINE)):
        m = n[b]
        alone = R.refine_raceline_batch(rt[b:b + 1, :m], nv[b:b + 1, :m], al[b:b + 1, :m], wv[b:b + 1], n_pts=npts[b:b + 1],
                                        stepsize_interp=2.0, max_iters=8, **vehs[ids[b]])
        assert torch.equal(res["alpha"][b, :m], alone["alpha"][0]), REFINE[b]
        for k in ("laptime", "laptime_start", "iters", "evals", "status"):
            assert torch.equal(res[k][b], alone[k][0]), (REFINE[b], k)


def test_the_objective_with_vehicles_does_not_synchronise_the_stream(golden):
    vehs = golden_vehicles(golden)
    rt, nv, al, npts, wv, _ = _refine_batch(golden, ["handling", "modena"])
    obj = R.LapTime(rt, nv, npts, 2.0, dict(vehicles=vehicles_of(vehs), veh_id=[2, 1], dyn_model_exp=1.0, filt_window=None))
    mask = torch.ones(2, dtype=torch.bool, device=DEV)
    obj.start(al, mask)
    obj(al, mask, False), obj(al, mask, True)                 # (warm: workspaces allocated)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        f, _, redo = obj(al, mask, False)
        f2, g, _ = obj(al, mask, True)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(f, f2) and not redo.any() and bool(torch.isfinite(g).all())


# ---- 6. refused tracks and inactive slots ------------------------------------------------------------------------------
def test_an_out_of_range_device_veh_id_refuses_its_track_alone(golden):
    vehs = golden_vehicles(golden)
    veh = vehicles_of(vehs)
    kap, el, npts = ragged(golden_racelines(golden) * 2)                 # 10 tracks
    npts[7] = 0                                                           # an inactive slot, with a bad id too
    ids = t_([0, -1, 1, 2, 3, 1, 2, 99, 0, 1], torch.int32)
    bad = [1, 4]
    got = B_.vel_profile_batch(kap, el, n_pts=npts, vehicles=veh, veh_id=ids)
    for b in range(10):
        if b in bad:
            assert int(got["status"][b, 0]) == BAD_VEHICLE and float(got["laptime"][b, 0]) == 0.0
            assert not bool(got["vx"][b].any())
        elif b == 7:
            assert int(got["status"][b, 0]) == 0 and float(got["laptime"][b, 0]) == 0.0
        else:
            v = vehs[int(ids[b])]
            alone = B_.vel_profile_batch(kap[b:b + 1], el[b:b + 1], n_pts=npts[b:b + 1], **v)
            same({k: x[b:b + 1] for k, x in got.items()}, alone)
    ref_inactive = B_.vel_profile_batch(kap[7:8], el[7:8], n_pts=npts[7:8], **vehs[0])
    same({k: x[7:8] for k, x in got.items()}, ref_inactive)
    # the adjoint: the refused tracks get zero gradients and grad_status 5; strict=True refuses the backward
    W = weights(10)
    out, gk, ge = _grads(B_.vel_profile_diff, kap, el, W, n_pts=npts, vehicles=veh, veh_id=ids, strict=False)
    assert out["grad_status"].tolist() == [0, 5, 0, 0, 5, 0, 0, 0, 0, 0]
    assert not bool(gk[bad].any()) and not bool(ge[bad].any()) and not bool(gk[7].any())
    for b in (0, 2, 9):
        v = vehs[int(ids[b])]
        _, gk1, ge1 = _grads(B_.vel_profile_diff, kap[b:b + 1], el[b:b + 1], W[b:b + 1], n_pts=npts[b:b + 1], **v)
        assert torch.equal(gk[b], gk1[0]) and torch.equal(ge[b], ge1[0])
    with pytest.raises(RuntimeError, match="no gradient"):
        _grads(B_.vel_profile_diff, kap, el, W, n_pts=npts, vehicles=veh, veh_id=ids)
    with pytest.raises(RuntimeError, match="lap_time_matrix_batch"):
        B_.lap_time_matrix_batch(kap, el, ggv_scales=[1.0], top_speeds=[50.0], n_pts=npts, vehicles=veh, veh_id=ids)
