"""GPU tests (-m gpu) of the velocity-profile kernels (csrc/vel_profile.cu: vel_profile_kernel, ax_t_profile_kernel,
vel_profile_adjoint_kernel; arithmetic in csrc/vel_profile_core.cuh) where they change code path, on the constructed laps
of tests/vp_cases.py: every branch of the forward / backward passes and the vehicle tables, tracks of 2 to 9, 127 to 129
and 20 188 points, the interleaved [vector][i][p] layout, every per-profile status, the stand-alone
calc_ax_t_profile_batch, and the adjoint in the same regimes.

References: the host build of the same statements (tests/vp_adj_ref.py), which the device must equal bit for bit at
dyn_model_exp 1; the oracle (oracle/tph_velprofile.py), which squares with libm's pow where the kernel multiplies, so
its step times can differ in the last bits (tests/test_vp_cases_host.py); and the exact step times of tests/vp_cases.py.
Every bound was measured on an H100 80GB HBM3 and is printed next to the value measured (pytest -s)."""
import numpy as np
import pytest

import vp_cases as C
from oracle import tph_velprofile as VP
from vp_adj_ref import Harness

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_  # noqa: E402

DEV = "cuda"
VEH = C.VEH
CASES = C.cases()
MC_STATUS_BREAKDOWN = 3
HOST_TOL = 2e-11                 # test_gpu_lap_time_grad.HOST_TOL: device adjoint against the host adjoint
# device against the oracle, max |dev - oracle| / max |oracle| -> the bound (measured on an H100 80GB HBM3)
T_TOL = 4e-12                    # step times at dyn_model_exp 1, libm pow(v, 2) != v * v: 8.1e-13 (the clamp case)
POW_TOL = {"vx": 2e-15, "t": 5e-15}                # dyn_model_exp 1.5 / 2 (device pow): vx 3.4e-16, t 9.3e-16
MU_TOL = {"vx": 5e-16, "t": 5e-16}                 # per-point mu (np.mean sums pairwise): vx 6.1e-17, t 9.2e-17
FILT_TOL = {"vx": 5e-15, "t": 1e-15}               # moving average (np.convolve sums in another order): vx 8.4e-16
#                                                    (windows 3 .. 139), t 1.9e-16 (window 9)
FILT_T_TOL = 1e-12               # t of windows of half-width <= n / 4: 1.1e-13
# On laps where consecutive speeds differ by a few ulps (the car creeping towards its drag-limited terminal speed, or a
# window that averages most of the lap) ax is rounding noise and tph's step time (-v + sqrt(v^2 + 2 a e)) / a loses most
# of its digits: a one-ulp difference of v^2 (libm pow against v * v) moves the lap time far more than rounding
LONG_VX_TOL = 1e-15              # the lap with two 20 km straights: vx 2.3e-16 (260 of 20 188 speeds differ)
LONG_LAP_TOL = 1e-5              # its lap time: 1.8e-6 relative
# that lap: the device's lap time minus the exact sum of 2 e / (v + v') on the device's vx (the oracle's own: 0.16718 s)
CREEP_GAP = 0.16599221565002154  # s
CREEP_STEP = 0.9628411287700409  # the worst relative error of a single step time


def report(what, measured, bound):
    print(f"  {what}: measured {measured:.3e}, bound {bound:.0e}")
    assert measured <= bound, what


def rel(a, b):
    a, b = np.asarray(a, dtype=float), np.asarray(b, dtype=float)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return Harness(tmp_path_factory.mktemp("vp_edges_gpu"))


def t_(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def ragged(tracks, n_max=None, pad=float("nan")):
    """kappa, el [B, n_max] padded with pad, n_pts [B] on the device."""
    n_max = n_max or max(k.size for k, _ in tracks)
    kap = np.full((len(tracks), n_max), pad)
    el = np.full((len(tracks), n_max), pad)
    for b, (k, e) in enumerate(tracks):
        kap[b, :k.size], el[b, :e.size] = k, e
    return t_(kap), t_(el), t_([k.size for k, _ in tracks], torch.int32)


def device(c, **kw):
    """One profile of case c on the device: dict of numpy vx, ax, t, laptime, status."""
    mu = kw.pop("mu", None)
    res = B_.vel_profile_batch(t_(c["kappa"][None]), t_(c["el"][None]), c["ggv"], c["mach"], kw.pop("v_max", c["v_max"]),
                               mu=None if mu is None else t_(mu[None]), **kw, **VEH)
    return {k: v[0, 0].cpu().numpy() for k, v in res.items()}


# ---- A. branches -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("upper", [1, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_branch_cases_bit_for_bit(harness, name, upper):
    c = CASES[name]
    d = device(c, decel_slice_upper=upper)
    h = harness.profile(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], upper=upper)
    assert int(d["status"]) == 0
    for k in ("vx", "ax", "t"):
        assert np.array_equal(d[k], h[k]), k                     # the same statements on the host
    assert float(d["laptime"]) == d["t"][-1] == h["laptime"]
    vx, ax, t = C.oracle(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], upper=upper)
    assert np.array_equal(d["vx"], vx) and np.array_equal(d["ax"], ax)
    report(f"{name} t vs oracle", rel(d["t"], t), T_TOL)


@pytest.mark.parametrize("name", sorted(CASES))
def test_branch_cases_with_exponent_mu_and_filter(name):
    c = CASES[name]
    rng = np.random.default_rng(len(name))
    mu = 0.75 + 0.4 * rng.random(c["kappa"].size)
    for label, kw, tol in (("exp 1.5", dict(dyn_model_exp=1.5), POW_TOL), ("exp 2", dict(dyn_model_exp=2.0), POW_TOL),
                           ("mu", dict(mu=mu), MU_TOL), ("filter 9", dict(filt_window=9), FILT_TOL),
                           ("exp 1.5, mu, scale 0.6", dict(dyn_model_exp=1.5, mu=mu, ggv_scales=[0.6]), POW_TOL)):
        d = device(c, **kw)
        scale = kw.get("ggv_scales", [1.0])[0]
        vx, ax, t = C.oracle(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], scale=scale,
                             exp=kw.get("dyn_model_exp", 1.0), filt=kw.get("filt_window"), mu=kw.get("mu"))
        assert int(d["status"]) == 0
        report(f"{name} {label} vx", rel(d["vx"], vx), tol["vx"])
        report(f"{name} {label} t", rel(d["t"], t), tol["t"])


# ---- B. sizes --------------------------------------------------------------------------------------------------------
SIZES = list(range(2, 10)) + [127, 128, 129]


def _size_tracks():
    out = []
    for n in SIZES:
        if n < 10:
            out.append(C.tiny_lap(n))
        else:
            i = np.arange(n)
            out.append((np.where(i % 40 < 12, 0.0, 1.0 / (25.0 + 10.0 * np.sin(i / 7.0))), 2.0 + 0.01 * (i % 5)))
    return out


def test_sizes_in_one_ragged_batch_and_alone(harness):
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    tracks = _size_tracks()
    kap, el, npts = ragged(tracks, n_max=140)
    res = B_.vel_profile_batch(kap, el, ggv, mach, [60.0, 38.0, 60.0], n_pts=npts, ggv_scales=[1.0, 1.0, 0.7], **VEH)
    assert not res["status"].any()
    for b, (k, e) in enumerate(tracks):
        n = k.size
        alone = B_.vel_profile_batch(t_(k[None]), t_(e[None]), ggv, mach, [60.0, 38.0, 60.0], ggv_scales=[1.0, 1.0, 0.7],
                                     **VEH)
        for v, (vm, sc) in enumerate(((60.0, 1.0), (38.0, 1.0), (60.0, 0.7))):
            for key in ("vx", "ax", "t"):
                got = res[key][b, v].cpu().numpy()
                assert np.array_equal(got[:n + (key == "t")], alone[key][0, v].cpu().numpy()), (n, v, key)
                assert not got[n + (key == "t"):].any()                      # the padding stays zero
            assert float(res["laptime"][b, v]) == float(alone["laptime"][0, v])
            h = harness.profile(k, e, ggv, mach, vm, scale=sc)
            assert np.array_equal(res["vx"][b, v, :n].cpu().numpy(), h["vx"]) and float(res["laptime"][b, v]) == h["laptime"]
            vx, _, t = C.oracle(k, e, ggv, mach, vm, scale=sc)
            assert np.array_equal(h["vx"], vx) and abs(h["laptime"] - t[-1]) <= T_TOL * t[-1]


def _creep_variants():
    speeds = np.linspace(40.0, 72.0, 14)
    scales = np.linspace(0.5, 1.0, 11)
    return np.repeat(speeds, 11), np.tile(scales, 14)


def test_a_track_of_20188_points_with_154_variants():
    """The lap of two 20 km straights, V = 154 (the reference's lap-time matrix), with a short track beside it: each
    equals itself alone, bit for bit, and cells against the oracle."""
    g, m = C.stock_tables()
    k, e = C.two_long_straights(20.0)
    vm, sc = _creep_variants()
    short = C.hairpin_lap(60, 20.0)
    kap, el, npts = ragged([short, (k, e)])
    both = B_.vel_profile_batch(kap, el, g, m, vm, ggv_scales=sc, n_pts=npts, want_profiles=False, **VEH)
    alone = B_.vel_profile_batch(t_(k[None]), t_(e[None]), g, m, vm, ggv_scales=sc, **VEH)
    assert not both["status"].any() and not alone["status"].any()
    assert torch.equal(both["laptime"][1], alone["laptime"][0])
    for v in (0, 77, 153):
        vx, _, t = C.oracle(k, e, g, m, vm[v], scale=sc[v])
        report(f"n 20188 cell {v} vx vs oracle", rel(alone["vx"][0, v].cpu().numpy(), vx), LONG_VX_TOL)
        report(f"n 20188 cell {v} lap time vs oracle", abs(float(alone["laptime"][0, v]) - t[-1]) / t[-1], LONG_LAP_TOL)


def test_the_step_time_gap_on_a_creeping_lap(harness):
    """tph's step time (-v + sqrt(v^2 + 2 a e)) / a cancels as the car creeps towards its drag-limited terminal speed;
    the kernel copies it for parity (DESIGN.md section 6).  Pinned: the device equals the host build bit for bit and the
    oracle to the bounds above, and the gap to the exact 2 e / (v + v') on its own profile is the value measured."""
    g, m = C.stock_tables()
    k, e = C.two_long_straights(20.0)
    d = device(dict(kappa=k, el=e, ggv=g, mach=m, v_max=70.0))
    h = harness.profile(k, e, g, m, 70.0)
    assert all(np.array_equal(d[key], h[key]) for key in ("vx", "ax", "t")) and float(d["laptime"]) == h["laptime"]
    vx, ax, t = C.oracle(k, e, g, m, 70.0)
    report("creeping lap vx vs oracle", rel(d["vx"], vx), LONG_VX_TOL)
    report("creeping lap lap time vs oracle", abs(float(d["laptime"]) - t[-1]) / t[-1], LONG_LAP_TOL)
    gap = float(d["laptime"]) - C.exact_lap_time(d["vx"], e)
    steps = C.exact_step_times(d["vx"], e)
    worst = float(np.max(np.abs(np.diff(d["t"]) - steps) / steps))
    print(f"  creeping lap: gap {gap:.17g} s (pinned {CREEP_GAP}), worst step {worst:.4f}")
    assert abs(gap - CREEP_GAP) <= 1e-9 and abs(worst - CREEP_STEP) <= 1e-6


# ---- item: filter windows against the track's own length ---------------------------------------------------------------
def test_filter_windows_up_to_n_max(harness):
    """Odd windows 3 .. n_max - 1 on the ragged batch of 2 to 9 and 127 to 129 points: a track whose half-width
    (w - 1) / 2 is at most n gets tph's cyclic average (to rounding: np.convolve sums in another order); a longer window
    is refused for that track alone (status 3, lap time 0.0, zeros), in the forward and in the adjoint."""
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    tracks = _size_tracks()
    n_max = 140
    kap, el, npts = ragged(tracks, n_max=n_max)
    worst = {"vx": 0.0, "t": 0.0}
    for w in range(3, n_max, 2):
        res = B_.vel_profile_batch(kap, el, ggv, mach, 60.0, filt_window=w, n_pts=npts, **VEH)
        for b, (k, e) in enumerate(tracks):
            n = k.size
            if (w - 1) // 2 > n:
                assert int(res["status"][b, 0]) == MC_STATUS_BREAKDOWN and float(res["laptime"][b, 0]) == 0.0, (n, w)
                assert not res["vx"][b].any() and not res["t"][b].any()
                continue
            assert int(res["status"][b, 0]) == 0, (n, w)
            h = harness.profile(k, e, ggv, mach, 60.0, filt=w)
            assert np.array_equal(res["vx"][b, 0, :n].cpu().numpy(), h["vx"]), (n, w)
            assert np.array_equal(res["t"][b, 0, :n + 1].cpu().numpy(), h["t"]), (n, w)
            narrow = 4 * ((w - 1) // 2) <= n
            if narrow or w in (3, 5) or w % 16 == 1:                # the oracle on a subset (it is slow)
                vx, _, t = C.oracle(k, e, ggv, mach, 60.0, filt=w)
                worst["vx"] = max(worst["vx"], rel(h["vx"], vx))
                key = "t" if narrow else "t_wide"
                worst[key] = max(worst.get(key, 0.0), rel(h["t"], t))
        if w in (5, 21, 139):
            kk, ee = kap.clone().nan_to_num_(0.0).requires_grad_(), el.clone().nan_to_num_(1.0).requires_grad_()
            r = B_.vel_profile_diff(kk, ee, ggv, mach, 60.0, filt_window=w, n_pts=npts, strict=False, **VEH)
            r["laptime"].sum().backward()
            refused = torch.tensor([(w - 1) // 2 > k.size for k, _ in tracks], device=DEV)
            assert torch.equal(r["grad_status"] == MC_STATUS_BREAKDOWN, refused)
            assert not kk.grad[refused].any() and not ee.grad[refused].any()
    report("filter windows vx vs oracle", worst["vx"], FILT_TOL["vx"])
    report("filter windows of half-width <= n / 4, t vs oracle", worst["t"], FILT_T_TOL)
    # a window over most of the lap leaves consecutive speeds a few ulps apart: the step times cancel (see above)
    print(f"  wider windows, t vs oracle: {worst['t_wide']:.3e} (not bounded: the device equals the host build)")


# ---- C. layout -------------------------------------------------------------------------------------------------------
def _layout_batch():
    names = [n for n, c in CASES.items() if c["ggv"].shape == (18, 3) and c["ggv"][0, 0] == 0.0 and c["ggv"][-1, 0] == 72.0
             and c["ggv"][0, 2] == 13.1]
    tracks = [(CASES[n]["kappa"], CASES[n]["el"]) for n in names] * 7 + _size_tracks()[:4]
    return tracks, C.ggv_table(18), C.mach_table(18)


def test_layout_matrix_cells_chunks_and_profiles():
    tracks, ggv, mach = _layout_batch()
    kap, el, npts = ragged(tracks)
    scales, speeds = [1.0, 0.83, 0.61], [40.0, 52.0, 63.0, 70.0, 45.5]
    B, V = len(tracks), len(scales) * len(speeds)
    assert (B * V) % 128 != 0 and B * V > 4 * 128
    ltm = B_.lap_time_matrix_batch(kap, el, ggv, mach, scales, speeds, n_pts=npts, **VEH)
    vm, sc, _, _ = B_._lap_time_variants(scales, speeds)
    full = B_.vel_profile_batch(kap, el, ggv, mach, vm, ggv_scales=sc, n_pts=npts, **VEH)
    lap_only = B_.vel_profile_batch(kap, el, ggv, mach, vm, ggv_scales=sc, n_pts=npts, want_profiles=False, **VEH)
    assert torch.equal(full["laptime"], lap_only["laptime"]) and torch.equal(ltm.reshape(B, V), full["laptime"])
    for chunk in (1, 7, 40):
        r = B_.vel_profile_batch(kap, el, ggv, mach, vm, ggv_scales=sc, n_pts=npts, max_chunk=chunk, **VEH)
        for key in ("vx", "ax", "t", "laptime", "status"):
            assert torch.equal(r[key], full[key]), (chunk, key)
    for i, top in enumerate(speeds):                      # each cell is the single-variant profile of that cell
        for j, s in enumerate(scales):
            one = B_.vel_profile_batch(kap, el, ggv, mach, [top], ggv_scales=[s], n_pts=npts, **VEH)
            assert torch.equal(ltm[:, i, j], one["laptime"][:, 0])
            assert torch.equal(one["vx"][:, 0], full["vx"][:, i * len(scales) + j])


def test_rotating_a_lap_rotates_its_profile():
    """Under decel_slice_upper = 0 the profile of a rotated lap is the rotated profile, bit for bit (measured), except
    where tph's phases depend on the seam: on the spiral lap the car never reaches v_max, so its acceleration phase wraps
    round the lap and where it first starts depends on the seam; there the device follows the oracle."""
    for name, c in CASES.items():
        k, e = c["kappa"], c["el"]
        base = device(c, decel_slice_upper=0)["vx"]
        for s in (1, 37, k.size // 2):
            rc = dict(c, kappa=np.roll(k, s), el=np.roll(e, s))
            got = device(rc, decel_slice_upper=0)["vx"]
            if name == "spiral":
                vx, _, _ = C.oracle(rc["kappa"], rc["el"], c["ggv"], c["mach"], c["v_max"], upper=0)
                assert np.array_equal(got, vx)
            else:
                assert np.array_equal(got, np.roll(base, s)), (name, s)


# ---- D. statuses -----------------------------------------------------------------------------------------------------
def test_statuses_in_the_middle_of_a_batch():
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    good = [(CASES[n]["kappa"], CASES[n]["el"]) for n in ("straights", "spiral", "phase_at_j0")]
    n_max = max(k.size for k, _ in good) + 3
    kap, el, npts = ragged(good + good[:1] * 6 + good, n_max=n_max, pad=0.0)
    npts = npts.clone()
    # slots 3..8: n_pts 0, 1, -5, n_max + 1; NaN kappa; el = 0
    npts[3], npts[4], npts[5], npts[6] = 0, 1, -5, n_max + 1
    kap[7, 10] = float("nan")
    el[8, 20] = 0.0
    res = B_.vel_profile_batch(kap, el, ggv, mach, [40.0, 70.0], ggv_scales=[1.0, 0.8], n_pts=npts, **VEH)
    rk, re_, rn = ragged(good, n_max=n_max, pad=0.0)
    ref = B_.vel_profile_batch(rk, re_, ggv, mach, [40.0, 70.0], ggv_scales=[1.0, 0.8], n_pts=rn, **VEH)
    for b_res, b_ref in ((0, 0), (1, 1), (2, 2), (9, 0), (10, 1), (11, 2)):    # the other tracks are unchanged
        for key in ("vx", "ax", "t", "laptime", "status"):
            assert torch.equal(res[key][b_res], ref[key][b_ref]), (b_res, key)
    st, lap = res["status"].cpu().numpy(), res["laptime"].cpu().numpy()
    assert (st[3] == 0).all() and (lap[3] == 0.0).all() and not res["vx"][3].any()                  # inactive slot
    for b in (4, 5, 6):                                                                             # refused: 3, 0.0
        assert (st[b] == MC_STATUS_BREAKDOWN).all() and (lap[b] == 0.0).all() and not res["vx"][b].any()
    for b in (7, 8):                                                                                # non-finite: 3
        assert (st[b] == MC_STATUS_BREAKDOWN).all() and not np.isfinite(lap[b]).any()
    assert not (np.isfinite(lap) & (lap != 0.0) & (st != 0)).any()     # no non-OK profile with a finite nonzero lap time
    assert (st[[0, 1, 2, 9, 10, 11]] == 0).all()
    # refused calls: a table of 257 rows, an even window, a window >= n_max
    with pytest.raises(ValueError, match="256 rows"):
        B_.vel_profile_batch(kap, el, C.ggv_table(257), mach, 40.0, n_pts=npts, **VEH)
    with pytest.raises(ValueError, match="256 rows"):
        B_.vel_profile_batch(kap, el, ggv, C.mach_table(257), 40.0, n_pts=npts, **VEH)
    kap2, el2, p = B_._vp_inputs(kap, el, ggv, mach, 40.0, None, VEH["drag_coeff"], VEH["m_veh"], 1.0, None, npts, None)
    g257 = t_(C.ggv_table(257))
    p.common = (257, g257) + p.common[2:]
    with pytest.raises(_lib.MinCurvLibError, match="256 rows"):
        B_._vel_profile_launch(kap2, el2, p, True)
    with pytest.raises(RuntimeError, match="must be odd"):
        B_.vel_profile_batch(kap, el, ggv, mach, 40.0, filt_window=4, n_pts=npts, **VEH)
    for w in (n_max, n_max + 1):
        with pytest.raises(_lib.MinCurvLibError, match="filt_window"):
            B_.vel_profile_batch(kap, el, ggv, mach, 40.0, filt_window=w | 1, n_pts=npts, **VEH)


# ---- E. calc_ax_t_profile_batch ----------------------------------------------------------------------------------------
def test_calc_ax_t_profile_batch_ragged_pitch_ax_in_and_t_start():
    rng = np.random.default_rng(9)
    P, n_max, pitch = 37, 50, 61
    npts = rng.integers(1, n_max + 1, P)
    npts[:3] = (1, n_max, 2)
    vx = 15.0 + 40.0 * rng.random((P, pitch))
    vx[:, 5] = vx[:, 6]                                   # ax == 0 exactly: the e / v branch
    vx[:, 20] = vx[:, 21]
    el = 0.5 + 3.0 * rng.random((P, n_max))
    worst = 0.0
    for t_start in (0.0, 12.375):
        ax, t = B_.calc_ax_t_profile_batch(t_(vx), t_(el), t_start=t_start, n_pts=t_(npts, torch.int32))
        ax, t = ax.cpu().numpy(), t.cpu().numpy()
        ax_in = np.zeros((P, n_max))
        for p in range(P):
            n = int(npts[p])
            ao = VP.calc_ax_profile(vx[p, :n + 1], el[p, :n])
            to = VP.calc_t_profile(vx[p, :n], el[p, :n], t_start=t_start, ax_profile=ao)
            assert np.array_equal(ax[p, :n], ao) and not ax[p, n:].any()
            worst = max(worst, rel(t[p, :n + 1], to))
            assert t[p, 0] == t_start and not t[p, n + 1:].any()
            if n > 21:
                assert ax[p, 5] == 0.0 and ax[p, 20] == 0.0
            ax_in[p, :n] = ao
        # with ax_in: vx needs only n entries per row
        ax2, t2 = B_.calc_ax_t_profile_batch(t_(vx[:, :n_max]), t_(el), ax_in=t_(ax_in), t_start=t_start,
                                             n_pts=t_(npts, torch.int32))
        assert np.array_equal(ax2.cpu().numpy(), ax_in) and np.array_equal(t2.cpu().numpy(), t)
    report("calc_ax_t_profile_batch t vs oracle", worst, T_TOL)


# ---- F. the adjoint in the same regimes --------------------------------------------------------------------------------
@pytest.mark.parametrize("upper", [1, 0])
def test_adjoint_on_the_branch_cases(harness, upper):
    worst = 0.0
    for name, c in CASES.items():
        k = t_(c["kappa"][None]).requires_grad_()
        e = t_(c["el"][None]).requires_grad_()
        r = B_.vel_profile_diff(k, e, c["ggv"], c["mach"], c["v_max"], decel_slice_upper=upper, **VEH)
        r["laptime"].sum().backward()
        h = harness.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, upper=upper)
        assert h["status"] == 0 and int(r["grad_status"][0]) == 0
        for got, want in ((k.grad[0], h["g_kappa"]), (e.grad[0], h["g_el"])):
            worst = max(worst, rel(got.cpu().numpy(), want))
    report(f"adjoint on the branch cases (upper {upper}) vs host", worst, HOST_TOL)


def test_adjoint_on_the_sizes_and_non_finite_forwards(harness):
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    tracks = _size_tracks()
    kap, el, npts = ragged(tracks, n_max=140, pad=0.0)
    kap[2, 1] = float("nan")                     # n = 4: a non-finite forward
    el[9, 3] = 0.0                               # n = 128
    k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
    r = B_.vel_profile_diff(k, e, ggv, mach, 60.0, n_pts=npts, strict=False, **VEH)
    r["laptime"].sum().backward()
    gs = r["grad_status"].cpu().numpy()
    assert gs[2] == MC_STATUS_BREAKDOWN and gs[9] == MC_STATUS_BREAKDOWN and r["status"][2] == MC_STATUS_BREAKDOWN
    assert not k.grad[[2, 9]].any() and not e.grad[[2, 9]].any()
    worst = 0.0
    for b, (kk, ee) in enumerate(tracks):
        if b in (2, 9):
            continue
        n = kk.size
        h = harness.adjoint(kk, ee, ggv, mach, 60.0, 1.0)
        assert gs[b] == 0 and h["status"] == 0
        for got, want in ((k.grad[b, :n], h["g_kappa"]), (e.grad[b, :n], h["g_el"])):
            worst = max(worst, rel(got.cpu().numpy(), want))
        assert not k.grad[b, n:].any() and not e.grad[b, n:].any()
    report("adjoint on n 2..9, 127..129 vs host", worst, HOST_TOL)
    with pytest.raises(_lib.MinCurvLibError, match="vel_profile_diff"):
        k2 = kap.clone().requires_grad_()
        B_.vel_profile_diff(k2, el, ggv, mach, 60.0, n_pts=npts, **VEH)["laptime"].sum().backward()
