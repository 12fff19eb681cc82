"""GPU tests (-m gpu) of the iterative minimum-curvature path (batch.iqp_batch, tph.iqp_handler) and of create_raceline
where their kernels change code path, against the float64 reference of tests/iqp_ref.py and the dense oracle:

A  one re-linearisation step (mc_iqp_relinearise_batch: create_raceline_kernel, iqp_new_reftrack_kernel, then
   calc_splines_kernel at n_max_new) on a ragged batch whose tracks span PCR with 4 and 8 points per thread and the
   chunked recurrences, whose widths jump at the wrap from the last row to row 0, with an inactive slot, at a new capacity
   in shared memory (stepsize 3 m) and in global scratch (1 m), and one point short of a track's count;
B  create_raceline's stations, heading and curvature (and calc_head_curv's dkappa) on the same tracks with shared and
   global scratch, its capacity protocol (explicit n_out_max, the derived bound and its re-run) and a step longer than the
   lap;
C  per-track termination of iqp_batch (iqp_finish_kernel) in a batch whose tracks finish at different outer iterations,
   one at the iteration cap, one infeasible and one empty, against tph_dense.iqp_handler per track; then every track
   alone in the same batch, bit for bit.
Every measured error is printed next to its tolerance (pytest -s)."""
import math

import numpy as np
import pytest

import iqp_ref as I
import mincurv_ref as R
from conftest import rel_max

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import batch as B_, synth  # noqa: E402
from oracle import tph_dense as T  # noqa: E402

SPL_SMEM_MAX_N = 3488      # the largest n_max whose eight spline vectors fit in shared memory (splines.cu, SPL_SMEM_LIMIT)
# A: the device and the reference share every formula; what differs is the moment solve (PCR / chunked recurrences
# against a sparse LU) and the order of the length sums (chunked scan against np.cumsum): rounding at coordinates of
# ~1.2 km.  x, y and widths in metres, normals absolute.  Measured on an H100 80GB HBM3 (700 W power limit): xy 7.9e-12
# (n = 2048), widths 3.8e-13 (n = 2049), normals 5.7e-13 (n = 3000); the tolerances leave 10-20x.
RELIN_TOL = dict(xy=1e-10, w=1e-11, nv=1e-11)
# B: spline lengths relative to the longest; s, el and the arc length a t error moves a station by (dt * its spline's
# length) relative to the lap; x, y in metres; psi absolute [rad]; kappa and dkappa relative to their largest magnitude
# on the track.  Measured on an H100 80GB HBM3 (700 W): spline lengths 7.4e-14, s 1.3e-15, el 1.1e-15, t 1.4e-15
# (|dt| 2.9e-12), xy 7.9e-12, psi 3.7e-13, kappa 1.1e-12, dkappa 8.5e-12 (n 1025 .. 3000); the tolerances leave 10-20x.
RL_TOL = dict(sl=1e-12, s=2e-14, el=2e-14, t=2e-14, xy=1e-10, psi=1e-11, kappa=2e-11, dkappa=2e-10)
PER_SPLINE = ("coeffs_x", "coeffs_y", "spline_lengths")
KNOT_TIE = 1e-12           # a station this close (relative to the lap) to a knot may fall on either of its two splines


def _closed(p):
    return np.vstack((p[:, :2], p[0, :2]))


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


# ---------------------------------------------------------------------------------------------------------------------
# the tracks of A and B
# ---------------------------------------------------------------------------------------------------------------------
EDGE_N = [80, 97, 1024, 1025, 2048, 2049, 3000]     # PCR 4 / 8 points per thread, chunked recurrences (256 threads)


def _edge_cases():
    """dict(rt [n, 4], nv [n, 2], alpha [n]) per n of EDGE_N: a synthetic track whose right width grows by 1.2 m and left
    width shrinks by 0.9 m along the lap (so both jump at the wrap), its normals, and a smooth alpha inside the box of a
    2 m vehicle."""
    cases = []
    for n in EDGE_N:
        rt = synth.make_track(900 + n, n, step=2.5)
        u = np.arange(n) / n
        rt[:, 2] += 1.2 * u
        rt[:, 3] += 0.9 * (1.0 - u)
        assert abs(rt[-1, 2] - rt[0, 2]) >= 0.5 and abs(rt[-1, 3] - rt[0, 3]) >= 0.5
        _, _, nv = R.periodic_spline(_closed(rt))
        alpha = 1.2 * np.sin(2.0 * np.pi * (3.0 * u + 0.05))
        assert np.all(alpha < rt[:, 3] - 1.0) and np.all(-alpha < rt[:, 2] - 1.0)
        cases.append(dict(rt=rt, nv=nv, alpha=alpha))
    return cases


def _pack(cases, n_max=None):
    dev = torch.device("cuda")
    n = [c["rt"].shape[0] for c in cases]
    n_max = n_max or max(n)
    rt, nv, al = np.zeros((len(cases), n_max, 4)), np.zeros((len(cases), n_max, 2)), np.zeros((len(cases), n_max))
    for b, c in enumerate(cases):
        rt[b, :n[b]], nv[b, :n[b]], al[b, :n[b]] = c["rt"], c["nv"], c["alpha"]
    f64 = dict(dtype=torch.float64, device=dev)
    return (torch.tensor(rt, **f64), torch.tensor(nv, **f64), torch.tensor(al, **f64),
            torch.tensor(n, dtype=torch.int32, device=dev))


def _np(t):
    return t.detach().cpu().numpy()


def _report(tag, errs, tol):
    print(f"{tag}: " + ", ".join(f"{k} {errs[k][0]:.1e} (n={errs[k][1]}) / tol {tol[k]:.0e}" for k in errs))
    for k, (e, n) in errs.items():
        assert e <= tol[k], (tag, k, n, e)


def _worst(errs, key, e, n):
    if e >= errs.get(key, (-1.0, 0))[0]:
        errs[key] = (float(e), n)


# ---------------------------------------------------------------------------------------------------------------------
# A. the re-linearisation step
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("step", [3.0, 1.0])
def test_relinearise_against_the_reference(step):
    cases = _edge_cases()
    refs = [I.relinearise(c["rt"], c["nv"], c["alpha"], step) for c in cases]
    for c, r in zip(cases, refs):
        q = r["raceline"]["total"] / step             # the new point count is ceil(q): no rounding tie may decide it
        assert abs(q - round(q)) >= 1e-9, (c["rt"].shape[0], q)
    counts = [r["n"] for r in refs]
    n_max_new = max(counts) + 5
    assert (n_max_new > SPL_SMEM_MAX_N) == (step == 1.0) and max(EDGE_N) <= SPL_SMEM_MAX_N
    slots = cases + [cases[1]]                        # the last slot is inactive
    rt, nv, al, npts = _pack(slots)
    active = torch.ones(len(slots), dtype=torch.int32, device="cuda")
    active[-1] = 0
    rn, nn, npn = B_.iqp_relinearise_batch(rt, nv, al, step, n_pts=npts, active=active, n_max_new=n_max_new)
    rn_, nn_, npn_ = _np(rn), _np(nn), _np(npn)
    assert npn_.tolist() == counts + [0]
    errs = {}
    for b, r in enumerate(refs):
        m, n = counts[b], EDGE_N[b]
        _worst(errs, "xy", np.abs(rn_[b, :m, :2] - r["reftrack"][:, :2]).max(), n)
        _worst(errs, "w", np.abs(rn_[b, :m, 2:] - r["reftrack"][:, 2:]).max(), n)
        _worst(errs, "nv", np.abs(nn_[b, :m] - r["normvec"]).max(), n)
        assert not rn_[b, m:].any() and not nn_[b, m:].any(), n
    assert not rn_[-1].any() and not nn_[-1].any()
    _report(f"relinearise, step {step} m, n_max_new {n_max_new}", errs, RELIN_TOL)
    # one point short of the largest track: it reports -(points needed), every other track is bit for bit the same
    big = int(np.argmax(counts))
    m = counts[big] - 1
    assert sorted(counts)[-2] <= m
    rn2, nn2, npn2 = (_np(x) for x in B_.iqp_relinearise_batch(rt, nv, al, step, n_pts=npts, active=active, n_max_new=m))
    assert npn2.tolist() == [-counts[big] if b == big else npn_[b] for b in range(len(slots))]
    for b in range(len(slots)):
        if b == big:
            assert not rn2[b].any() and not nn2[b].any()
        else:
            assert np.array_equal(rn2[b], rn_[b, :m]) and np.array_equal(nn2[b], nn_[b, :m]), b


# ---------------------------------------------------------------------------------------------------------------------
# B. create_raceline: stations, heading, curvature, capacity
# ---------------------------------------------------------------------------------------------------------------------
def _check_raceline(tag, ref, out, b, n, errs):
    """Station-by-station comparison of track b of a create_raceline_batch result with the reference; returns the
    number of stations that sit on a knot within KNOT_TIE of the lap (and were assigned to the other spline)."""
    no = ref["no"]
    assert int(out["n_out"][b]) == no, (tag, n)
    total = ref["total"]
    sl = out["spline_lengths"][b, :n]
    si, tv = out["spline_inds"][b, :no], out["t_values"][b, :no]
    tie = si != ref["spline_inds"]
    for i in np.flatnonzero(tie):
        lo = min(si[i], ref["spline_inds"][i])
        assert abs(int(si[i]) - int(ref["spline_inds"][i])) == 1, (tag, n, i)
        assert abs(ref["s"][i] - ref["cum"][lo]) <= KNOT_TIE * total, (tag, n, i)
        t_lo, t_hi = (tv[i], ref["t"][i]) if si[i] == lo else (ref["t"][i], tv[i])
        assert t_lo >= 1.0 - 1e-9 and t_hi <= 1e-9, (tag, n, i)
    ok = ~tie
    _worst(errs, "sl", rel_max(sl, ref["spline_lengths"]), n)
    _worst(errs, "s", np.abs(out["s_interp"][b, :no] - ref["s"]).max() / total, n)
    _worst(errs, "el", np.abs(out["el_lengths_interp"][b, :no] - ref["el"]).max() / total, n)
    _worst(errs, "t", (np.abs(tv[ok] - ref["t"][ok]) * ref["spline_lengths"][si[ok]]).max() / total, n)
    _worst(errs, "xy", np.abs(out["raceline_interp"][b, :no] - ref["raceline"]).max(), n)
    # heading and curvature of the reference at its stations; at a knot tie, at the device's side of the knot
    ind, t = ref["spline_inds"].copy(), ref["t"].copy()
    ind[tie], t[tie] = si[tie], tv[tie]
    psi, kappa, dkappa = T.calc_head_curv_an(ref["coeffs_x"], ref["coeffs_y"], ind, t, calc_curv=True, calc_dcurv=True)
    p = out["psi"][b, :no]
    assert np.all(p >= -np.pi) and np.all(p < np.pi), (tag, n)
    assert p.min() < -3.0 and p.max() > 3.0, (tag, n)                  # the loop crosses the +-pi seam
    dp = np.abs(p - psi)
    _worst(errs, "psi", np.minimum(dp, 2.0 * np.pi - dp).max(), n)
    _worst(errs, "kappa", rel_max(out["kappa"][b, :no], kappa), n)
    _worst(errs, "dkappa", rel_max(out["dkappa"][b, :no], dkappa), n)
    assert not out["raceline_interp"][b, no:].any() and not out["spline_inds"][b, no:].any() and \
        not out["kappa"][b, no:].any() and not out["psi"][b, no:].any(), (tag, n)
    return int(tie.sum())


def _raceline_run(cases, step, n_max, n_out_max=None):
    rt, nv, al, npts = _pack(cases, n_max)
    out = B_.create_raceline_batch(rt, nv, al, step, n_pts=npts, n_out_max=n_out_max)
    psi, kappa, dkappa = B_.calc_head_curv_batch(out["coeffs_x"], out["coeffs_y"], out["spline_inds"], out["t_values"],
                                                 n_eval=out["n_out"].clamp(min=0), calc_dcurv=True)
    assert torch.equal(psi, out["psi"]) and torch.equal(kappa, out["kappa"])
    out = {k: _np(v) for k, v in out.items()}
    out["dkappa"] = _np(dkappa)
    return out


@pytest.mark.parametrize("step", [1.0, 3.0])
def test_create_raceline_stations_heading_and_curvature(step):
    cases = _edge_cases()
    refs = [I.create_raceline(c["rt"][:, :2], c["nv"], c["alpha"], step) for c in cases]
    runs = [_raceline_run(cases, step, n_max) for n_max in (3100, 3600)]     # shared-memory / global-memory scratch
    errs, ties = {}, 0
    for b, (n, ref) in enumerate(zip(EDGE_N, refs)):
        for k in runs[0]:
            x0, x1 = runs[0][k][b], runs[1][k][b]
            if k in PER_SPLINE:
                assert not x1[3100:].any()
                x1 = x1[:3100]
            assert np.array_equal(x0, x1), (n, k)
        ties += _check_raceline(f"step {step}", ref, runs[0], b, n, errs)
    print(f"create_raceline, step {step} m: {ties} station(s) on a knot tie")
    _report(f"create_raceline, step {step} m", errs, RL_TOL)


def test_create_raceline_capacity_protocol():
    cases = _edge_cases()
    step = 1.0
    out = _raceline_run(cases, step, 3100)
    no = out["n_out"]
    big = int(np.argmax(no))
    nmx = int(no[big])
    assert sorted(no.tolist())[-2] < nmx
    # an explicit capacity of exactly the largest count fits; one less: that track reports -(points needed)
    fit = _raceline_run(cases, step, 3100, n_out_max=nmx)
    short = _raceline_run(cases, step, 3100, n_out_max=nmx - 1)
    assert np.array_equal(fit["n_out"], no)
    assert short["n_out"].tolist() == [-nmx if b == big else int(no[b]) for b in range(len(cases))]
    for k, v in out.items():
        if k == "n_out":
            continue
        if k in PER_SPLINE:                           # (computed before the capacity is checked)
            assert np.array_equal(fit[k], v) and np.array_equal(short[k], v), k
            continue
        assert np.array_equal(fit[k], v[:, :nmx]), k
        for b in range(len(cases)):
            if b == big:
                assert not short[k][b].any(), k
            else:
                assert np.array_equal(short[k][b], v[b, :nmx - 1]), (k, b)
    # three- and four-point loops: the spline is >= 1.13 x the polygon, the derived bound (1.1 x polygon + 16) is too
    # small and the call is repeated with what the kernel asked for; the result is that of an explicit roomy capacity
    for th in (np.array([0.0, 2.0, 4.0]) * np.pi / 3.0, np.array([0.0, 0.6, np.pi, np.pi + 0.6])):
        p = 200.0 * np.column_stack((np.cos(th), np.sin(th)))
        _, _, nv = R.periodic_spline(_closed(p), False)
        c = dict(rt=np.column_stack((p, np.full((p.shape[0], 2), 5.0))), nv=nv, alpha=np.zeros(p.shape[0]))
        ref = I.create_raceline(p, nv, c["alpha"], step)
        poly = float(np.linalg.norm(np.roll(p, -1, axis=0) - p, axis=1).sum())
        assert math.ceil(poly * 1.1 / step) + 16 < ref["no"], p.shape[0]
        derived = _raceline_run([c], step, p.shape[0])
        roomy = _raceline_run([c], step, p.shape[0], n_out_max=2 * ref["no"])
        assert int(derived["n_out"][0]) == ref["no"] and derived["raceline_interp"].shape[1] == ref["no"] + 16
        for k, v in derived.items():
            w = roomy[k]
            assert np.array_equal(v, w if k == "n_out" or k in PER_SPLINE else w[:, :v.shape[1]]), (p.shape[0], k)
        errs = {}
        _check_raceline("tiny loop", ref, derived, 0, p.shape[0], errs)
        _report(f"create_raceline, {p.shape[0]}-point loop", errs, RL_TOL)
    # a step longer than the lap: one station at s = 0 whose element closes the loop
    c = cases[0]
    ref = I.create_raceline(c["rt"][:, :2], c["nv"], c["alpha"], 1e4)
    o = _raceline_run([c], 1e4, c["rt"].shape[0])
    assert ref["no"] == 1 and o["n_out"].tolist() == [1]
    assert o["s_interp"][0, 0] == 0.0 and o["spline_inds"][0, 0] == 0 and o["t_values"][0, 0] == 0.0
    assert abs(o["el_lengths_interp"][0, 0] - ref["total"]) <= RL_TOL["el"] * ref["total"]
    assert np.abs(o["raceline_interp"][0, 0] - ref["raceline"][0]).max() <= RL_TOL["xy"]


# ---------------------------------------------------------------------------------------------------------------------
# C. per-track termination of iqp_batch
# ---------------------------------------------------------------------------------------------------------------------
# (seed, n, amp) of synth.make_track and the outer iterations tph_dense.iqp_handler takes on each at CURV_ERROR_ALLOWED
# (iters_min 3, kappa_bound 0.12, a 2 m vehicle, stepsize 3 m; every curv_error_max of every iteration is >= 10 % away
# from the threshold).  The last track would need 5: MAX_ITERS stops it one iteration earlier (status 2).
IQP_TRACKS = [(2, 140, 0.6), (1, 96, 0.6), (3, 200, 0.6), (6, 216, 1.2)]
IQP_ITERS = [3, 4, 4, 5]
CURV_ERROR_ALLOWED = 0.0015
MAX_ITERS = 4
IQP_KB, IQP_W_VEH, IQP_STEP = 0.12, 2.0, 3.0
# alpha as max|diff| / max|oracle|, reftrack [m] and normvec absolute, curv_error_max relative.  The device stops its
# interior-point iterations at a tolerance (mincurv_ipm.cu), the oracle solves the QP exactly; four chained QPs and three
# re-samplings carry the difference.  Measured on an H100 80GB HBM3 (700 W): alpha 1.9e-7 (n = 96), reftrack 6.3e-8 m,
# normvec 5.5e-9, curv_error_max 1.9e-8 (the golden test of tph.iqp_handler allows 1e-3, 1e-3 m and 1e-4).
IQP_TOL = dict(alpha=2e-6, reftrack=1e-6, normvec=1e-7, cerr=1e-6)


def _iqp_oracle(rt):
    _, _, A, nv = T.calc_splines(_closed(rt))
    hist = []
    alpha, rt_new, nv_new = T.iqp_handler(rt, nv, A, IQP_KB, IQP_W_VEH, False, False, IQP_STEP, 3, CURV_ERROR_ALLOWED,
                                          max_iters=MAX_ITERS, history=hist)
    return dict(alpha=alpha, reftrack=rt_new, normvec=nv_new, hist=hist)


def _iqp_run(rts, n_pts, n_cap_min=0):
    dev = torch.device("cuda")
    n_max = max(r.shape[0] for r in rts)
    rt = np.zeros((len(rts), n_max, 4))
    for b, r in enumerate(rts):
        rt[b, :r.shape[0]] = r
    rt = torch.tensor(rt, device=dev)
    npts = torch.tensor(n_pts, dtype=torch.int32, device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, n_pts=npts)
    res = B_.iqp_batch(rt, nv, h, IQP_KB, IQP_W_VEH, IQP_STEP, iters_min=3, curv_error_allowed=CURV_ERROR_ALLOWED,
                       n_pts=npts, max_iters=MAX_ITERS, _n_cap_min=n_cap_min)
    return {k: (_np(v) if isinstance(v, torch.Tensor) else v) for k, v in res.items()}


def test_iqp_batch_per_track_termination_against_the_oracle():
    rts = [synth.make_track(s, n, amp=a) for s, n, a in IQP_TRACKS]
    narrow = rts[0].copy()
    narrow[50:54, 2:] = 0.5                                   # 1 m wide for a 2 m vehicle: infeasible in iteration 1
    ref = [_iqp_oracle(r) for r in rts]
    # the premise: the tracks finish at different iterations, the last one at the cap, and no curv_error_max is near
    # the threshold
    for r, want in zip(ref, IQP_ITERS):
        e = np.array([h["curv_error_max"] for h in r["hist"]])
        assert len(e) == min(want, MAX_ITERS) and np.all(np.abs(e / CURV_ERROR_ALLOWED - 1.0) >= 0.1), e
        assert (e[-1] <= CURV_ERROR_ALLOWED) == (want <= MAX_ITERS)
        for h in r["hist"][:-1]:
            q = h["s_total"] / IQP_STEP                       # no re-sampled count near a rounding tie
            assert abs(q - round(q)) >= 1e-3, q
    with pytest.raises(RuntimeError, match="Problem not solvable"):
        _iqp_oracle(narrow)
    slots = rts + [narrow, np.zeros((0, 4))]
    n_pts = [r.shape[0] for r in slots]
    res = _iqp_run(slots, n_pts)
    n_cap = res["alpha"].shape[1]
    assert res["outer_iters"].tolist() == [min(k, MAX_ITERS) for k in IQP_ITERS] + [1, 1]
    assert res["status"].tolist() == [0 if k <= MAX_ITERS else 2 for k in IQP_ITERS] + [1, -1]
    assert res["qp_solves"] == int(res["outer_iters"].sum())
    errs = {}
    for b, (r, (_, n0, _)) in enumerate(zip(ref, IQP_TRACKS)):
        n = r["reftrack"].shape[0]
        assert res["n_pts"][b] == n, (n0, res["n_pts"][b], n)
        _worst(errs, "alpha", rel_max(res["alpha"][b, :n], r["alpha"]), n0)
        _worst(errs, "reftrack", np.abs(res["reftrack"][b, :n] - r["reftrack"]).max(), n0)
        _worst(errs, "normvec", np.abs(res["normvec"][b, :n] - r["normvec"]).max(), n0)
        c = r["hist"][-1]["curv_error_max"]
        _worst(errs, "cerr", abs(res["curv_error_max"][b] - c) / c, n0)
        for k in ("alpha", "reftrack", "normvec"):
            assert not res[k][b, n:].any(), (n0, k)
    _report(f"iqp_batch at curv_error_allowed {CURV_ERROR_ALLOWED}, max_iters {MAX_ITERS}", errs, IQP_TOL)
    # the infeasible track keeps its input and a zero alpha; the empty slot stays empty
    b = len(rts)
    assert res["n_pts"][b] == narrow.shape[0] and not res["alpha"][b].any()
    assert np.array_equal(res["reftrack"][b, :narrow.shape[0]], narrow) and not res["reftrack"][b, narrow.shape[0]:].any()
    assert res["n_pts"][-1] == 0 and not res["alpha"][-1].any() and not res["reftrack"][-1].any()
    # every track alone in the same batch (every other slot empty) at the same capacity: the same bits -- a finished
    # track's result is not overwritten by the later iterations of the others, and nothing crosses between tracks
    for b in range(len(slots) - 1):
        alone = _iqp_run(slots, [n if i == b else 0 for i, n in enumerate(n_pts)], n_cap_min=n_cap)
        assert alone["alpha"].shape[1] == n_cap
        for k in ("alpha", "reftrack", "normvec", "n_pts", "outer_iters", "status", "curv_error_max"):
            assert np.array_equal(alone[k][b], res[k][b]), (b, k)
        assert alone["qp_solves"] == int(alone["outer_iters"].sum())
