"""GPU tests (-m gpu) of the velocity-profile adjoint (csrc/vel_profile.cu: vel_profile_adjoint_kernel,
vel_profile_adjoint_veh_kernel, vel_profile_adjoint_sum_kernel; arithmetic in csrc/vel_profile_core.cuh,
profile_adjoint_thread) against the extended-precision replay of tph's solver (tests/vp_grad_ref.py), per entry, where
the adjoint changes code path: every constructed lap of tests/vp_cases.py, dyn_model_exp 1.5 and 2, filter windows,
the lap-time matrix, a vehicle per track, the sizes of the unrolled loops, and the fixed point of the initial profile.

Per entry: |dev - ref| <= TOL * max |ref| + COND * cond (cond: vp_grad_ref._conditioning, 0 at dyn_model_exp 1; see
test_vp_grad_ref_host.py), and |dev - ref| / |ref| <= REL on entries >= 1e-3 max |ref| whose conditioning is below the
floor.  Every bound was measured on an H100 80GB HBM3 and is printed next to the value measured (pytest -s)."""
import numpy as np
import pytest

import vp_cases as C
import vp_grad_ref as G

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import batch as B_  # noqa: E402

DEV = "cuda"
VEH = C.VEH
CASES = C.cases()
NAMES = sorted(CASES)
PIN = 2.0 ** -40                 # test_vp_grad_ref_host.PIN: radicands at the rounding level of 1 - q^p
MC_STATUS_BREAKDOWN = 3
# measured on an H100 80GB HBM3 (max-normalised; relative on the large entries):
TOL = {1.0: 1e-14, 1.5: 1e-12, 2.0: 1e-12}       # 1.2e-15 at dyn_model_exp 1 (A with g_vx); 8.0e-14 at 1.5, 5.8e-14 at 2
REL = {1.0: 3e-12, 1.5: 1e-10, 2.0: 1e-10}       # 2.9e-13 (A with g_vx); 1.1e-11 (B, 1.5)
WIDE_TOL = 5e-14                                 # a window past n / 2: 2.2e-15 (6.2e-15 on the host's laps)
COND = 40.0                                      # test_vp_grad_ref_host.COND (<= 3.5 times the conditioning there)


def report(what, measured, bound):
    print(f"  {what}: measured {measured:.3e}, bound {bound:.0e}")
    assert measured <= bound, what


def t_(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def ragged(tracks, n_max=None, pad=float("nan")):
    n_max = n_max or max(k.size for k, _ in tracks)
    kap, el = np.full((len(tracks), n_max), pad), np.full((len(tracks), n_max), pad)
    for b, (k, e) in enumerate(tracks):
        kap[b, :k.size], el[b, :e.size] = k, e
    return t_(kap), t_(el), t_([k.size for k, _ in tracks], torch.int32)


def reference(c, upper=1, exp=1.0, g_lap=1.0, g_vx=None, filt=None, scale=1.0, v_max=None, **veh):
    lg = G.decide(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"] if v_max is None else v_max, scale=scale,
                  exp=exp, filt=filt, upper=upper, **veh)
    return G.replay(c["kappa"], c["el"], lg, g_lap=g_lap, g_vx=g_vx, pin=PIN)


class Worst:
    """The largest errors of a section: max-normalised (with and without the conditioned entries) and relative."""

    def __init__(self):
        self.ab, self.rel, self.cond = 0.0, 0.0, 0.0

    def check(self, label, got, ref, key, p, tol=None):
        tol = TOL[p] if tol is None else tol
        want = np.asarray(ref[key], dtype=float)
        got = np.asarray(got, dtype=float)
        s = max(float(np.abs(want).max()), 1e-300)
        d = np.abs(got - want)
        cond = ref["cond_kappa"] if key == "g_kappa" else np.zeros(want.size)
        excess = d - tol * s - COND * cond
        assert (excess <= 0).all(), (label, key, int(np.argmax(excess)), float(d.max() / s))
        plain = COND * cond <= tol * s
        big = plain & (np.abs(want) >= 1e-3 * s)
        if big.any():
            rel = float((d[big] / np.abs(want[big])).max())
            assert rel <= REL[p], (label, key, rel)
            self.rel = max(self.rel, rel)
        self.ab = max(self.ab, float(d[plain].max() / s) if plain.any() else 0.0)
        self.cond = max(self.cond, float(d.max() / s))

    def report(self, what, p, tol=None):
        report(f"{what}: max-normalised", self.ab, TOL[p] if tol is None else tol)
        report(f"{what}: relative on entries >= 1e-3 max", self.rel, REL[p])
        if self.cond > self.ab:
            print(f"  {what}: max-normalised with the lateral-limit points {self.cond:.3e} (bounded by the conditioning)")


def diff(tracks, ggv, mach, v_max, g_vx=None, **kw):
    """vel_profile_diff of a ragged batch, backward of sum(laptime) (+ sum(g_vx * vx)): (grad kappa, grad el,
    grad_status) as numpy."""
    kap, el, npts = ragged(tracks)
    k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
    r = B_.vel_profile_diff(k, e, ggv, mach, v_max, n_pts=npts, **kw, **VEH)
    loss = r["laptime"].sum()
    if g_vx is not None:
        loss = loss + (r["vx"] * t_(np.nan_to_num(g_vx))).sum()
    loss.backward()
    return k.grad.cpu().numpy(), e.grad.cpu().numpy(), r["grad_status"].cpu().numpy()


def _by_tables():
    """The laps grouped by their tables and top speed (one vel_profile_diff call shares them)."""
    groups = {}
    for name in NAMES:
        c = CASES[name]
        key = (c["ggv"].tobytes(), c["mach"].tobytes(), c["v_max"])
        groups.setdefault(key, []).append(name)
    return list(groups.values())


def _g_vx(names):
    n_max = max(CASES[n]["kappa"].size for n in names)
    g = np.zeros((len(names), n_max))
    for b, n in enumerate(names):
        g[b, :CASES[n]["kappa"].size] = 0.05 * np.random.default_rng(b + 7).standard_normal(CASES[n]["kappa"].size)
    return g


# ---- A. every constructed lap ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_vx", [False, True])
@pytest.mark.parametrize("upper", [1, 0])
def test_a_every_lap_against_the_reference(upper, with_vx):
    """Every lap of vp_cases through vel_profile_diff, in one ragged batch (NaN padding) per set of tables: g_lap
    alone, and with a g_vx upstream."""
    w = Worst()
    for names in _by_tables():
        c0 = CASES[names[0]]
        g_vx = _g_vx(names) if with_vx else None
        gk, ge, gs = diff([(CASES[n]["kappa"], CASES[n]["el"]) for n in names], c0["ggv"], c0["mach"], c0["v_max"],
                          g_vx=g_vx, decel_slice_upper=upper)
        assert not gs.any()
        for b, name in enumerate(names):
            c = CASES[name]
            n = c["kappa"].size
            r = reference(c, upper=upper, g_vx=None if g_vx is None else g_vx[b, :n])
            w.check(name, gk[b, :n], r, "g_kappa", 1.0)
            w.check(name, ge[b, :n], r, "g_el", 1.0)
            assert not gk[b, n:].any() and not ge[b, n:].any()
    w.report(f"A upper {upper}{' with g_vx' if with_vx else ''}", 1.0)


# ---- B. dyn_model_exp 1.5 and 2 ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("exp", [1.5, 2.0])
def test_b_exponents_against_the_reference(exp):
    """The device's pow at dyn_model_exp 1.5 / 2; at the lateral-limit steps (spiral, vmax_interior_knot) the bound is
    the conditioning of those steps (test_vp_grad_ref_host.py, section 3)."""
    w = Worst()
    for names in _by_tables():
        c0 = CASES[names[0]]
        gk, ge, gs = diff([(CASES[n]["kappa"], CASES[n]["el"]) for n in names], c0["ggv"], c0["mach"], c0["v_max"],
                          dyn_model_exp=exp)
        assert not gs.any()
        for b, name in enumerate(names):
            n = CASES[name]["kappa"].size
            r = reference(CASES[name], exp=exp)
            w.check(name, gk[b, :n], r, "g_kappa", exp)
            w.check(name, ge[b, :n], r, "g_el", exp)
    w.report(f"B p {exp}", exp)


# ---- C. filter windows -------------------------------------------------------------------------------------------------
def test_c_filter_windows_and_a_refused_window():
    """Windows 3, 5 and 195 (half-width 97, past half of the 176-point lap) on a ragged batch, with a g_vx; a window
    whose half-width exceeds a track's n is refused for that track alone (grad_status 3, zero gradients)."""
    names = ["phase_at_j0", "seam_braking", "spiral"]          # the same tables; n = 176, 208, 220
    c0 = CASES[names[0]]
    short = C.tiny_lap(7)
    tracks = [(CASES[n]["kappa"], CASES[n]["el"]) for n in names] + [short]
    n_max = max(k.size for k, _ in tracks)
    g_vx = np.zeros((len(tracks), n_max))
    g_vx[:3, :_g_vx(names).shape[1]] = _g_vx(names)
    for window, tol in ((3, TOL[1.0]), (5, TOL[1.0]), (2 * 97 + 1, WIDE_TOL)):
        w = Worst()
        gk, ge, gs = diff(tracks, c0["ggv"], c0["mach"], c0["v_max"], g_vx=g_vx, filt_window=window, strict=False)
        for b, name in enumerate(names):
            c = CASES[name]
            n = c["kappa"].size
            assert gs[b] == 0
            r = reference(c, g_vx=g_vx[b, :n], filt=window)
            w.check(name, gk[b, :n], r, "g_kappa", 1.0, tol)
            w.check(name, ge[b, :n], r, "g_el", 1.0, tol)
        refused = (window - 1) // 2 > short[0].size
        assert (gs[3] == MC_STATUS_BREAKDOWN) == refused
        if refused:
            assert not gk[3].any() and not ge[3].any()
        w.report(f"C window {window}", 1.0, tol)
    assert 97 > CASES["phase_at_j0"]["kappa"].size / 2          # the wide window wraps past half of that lap


# ---- D. the lap-time matrix --------------------------------------------------------------------------------------------
def test_d_lap_time_matrix_cells_against_the_reference_sum():
    """A 3 x 3 matrix: top speeds on an interior knot of the tables, on their last knot and one that binds in the
    passes, ggv scales 0.6 / 1.0 / 1.3, a weight per cell.  A track's gradient is the reference summed over its
    cells."""
    names = ["vmax_interior_knot", "seam_accel", "spiral"]
    g18, m18 = C.ggv_table(18), C.mach_table(18)
    speeds, scales = [float(g18[11, 0]), 72.0, 30.0], [0.6, 1.0, 1.3]
    wgt = np.array([[1.0, -0.5, 0.25], [2.0, 0.75, -1.0], [0.5, 1.5, 1.25]])
    kap, el, npts = ragged([(CASES[n]["kappa"], CASES[n]["el"]) for n in names])
    k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
    res = B_.lap_time_matrix_diff(k, e, g18, m18, scales, speeds, n_pts=npts, **VEH)
    assert not res["status"].any()
    (res["laptime"] * t_(wgt)[None]).sum().backward()
    w = Worst()
    for b, name in enumerate(names):
        c = dict(CASES[name], ggv=g18, mach=m18)
        n = c["kappa"].size
        tot = {"g_kappa": np.zeros(n, dtype=G.LD), "g_el": np.zeros(n, dtype=G.LD), "cond_kappa": np.zeros(n)}
        for t, vm in enumerate(speeds):
            for s, sc in enumerate(scales):
                r = reference(c, g_lap=wgt[t, s], scale=sc, v_max=vm)
                for key in tot:
                    tot[key] = tot[key] + r[key]
        w.check(name, k.grad[b, :n].cpu().numpy(), tot, "g_kappa", 1.0)
        w.check(name, e.grad[b, :n].cpu().numpy(), tot, "g_el", 1.0)
    w.report("D 3 x 3 matrix", 1.0)


# ---- E. a vehicle per track --------------------------------------------------------------------------------------------
def test_e_mixed_vehicles_against_the_reference():
    """Tables of 1, 2, 18 and 256 rows, one whose first knot is above 0, other top speeds, drag and mass per vehicle;
    each track against the reference for its vehicle."""
    g18, m18 = C.ggv_table(18), C.mach_table(18)
    vehs = [dict(ggv=C.ggv_table(1, v1=80.0), mach=C.mach_table(1, v1=80.0), v_max=50.0, drag_coeff=0.75, m_veh=1200.0),
            dict(ggv=C.ggv_table(2), mach=C.mach_table(2), v_max=72.0, drag_coeff=0.9, m_veh=900.0),
            dict(ggv=g18, mach=m18, v_max=float(g18[11, 0]), drag_coeff=0.6, m_veh=1400.0),
            dict(ggv=C.ggv_table(256), mach=C.mach_table(256), v_max=60.0, drag_coeff=1.1, m_veh=750.0),
            dict(ggv=C.ggv_table(18, 20.0), mach=C.mach_table(18, 20.0), v_max=60.0, drag_coeff=0.75, m_veh=1200.0)]
    veh = B_.Vehicles([v["ggv"] for v in vehs], [v["mach"] for v in vehs], [v["v_max"] for v in vehs],
                      [v["drag_coeff"] for v in vehs], [v["m_veh"] for v in vehs])
    names = ["one_row", "two_rows", "vmax_interior_knot", "rows256", "below_first_knot", "seam_braking", "spiral"]
    ids = [0, 1, 2, 3, 4, 2, 3]
    kap, el, npts = ragged([(CASES[n]["kappa"], CASES[n]["el"]) for n in names])
    for exp in (1.0, 2.0):
        k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
        r = B_.vel_profile_diff(k, e, n_pts=npts, vehicles=veh, veh_id=t_(ids, torch.int32), dyn_model_exp=exp)
        r["laptime"].sum().backward()
        assert not r["grad_status"].any()
        w = Worst()
        for b, (name, i) in enumerate(zip(names, ids)):
            v = vehs[i]
            c = dict(CASES[name], ggv=v["ggv"], mach=v["mach"], v_max=v["v_max"])
            n = c["kappa"].size
            ref = reference(c, exp=exp, drag_coeff=v["drag_coeff"], m_veh=v["m_veh"])
            w.check(name, k.grad[b, :n].cpu().numpy(), ref, "g_kappa", exp)
            w.check(name, e.grad[b, :n].cpu().numpy(), ref, "g_el", exp)
        w.report(f"E vehicles p {exp}", exp)


# ---- F. sizes ----------------------------------------------------------------------------------------------------------
def test_f_sizes_and_a_long_lap():
    """n = 2..9 and 127..129 (partial VP_UNROLL blocks, the wrap of the prefetch) and a lap of 2294 points, in one
    ragged batch."""
    from test_gpu_velprofile_edges import _size_tracks
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    tracks = _size_tracks() + [C.hairpin_lap(1100, 30.0)]
    assert tracks[-1][0].size > 2000
    gk, ge, gs = diff(tracks, ggv, mach, 60.0)
    assert not gs.any()
    w = Worst()
    for b, (k, e) in enumerate(tracks):
        n = k.size
        r = reference(dict(kappa=k, el=e, ggv=ggv, mach=mach, v_max=60.0))
        w.check(f"n {n}", gk[b, :n], r, "g_kappa", 1.0)
        w.check(f"n {n}", ge[b, :n], r, "g_el", 1.0)
    w.report("F sizes", 1.0)


# ---- G. the fixed point of the initial profile -------------------------------------------------------------------------
def test_g_fixed_point_derivative():
    """A speed-dependent ggv on laps without a straight: the initial profile converges in 1 to 20 iterations and its
    derivative D is carried through each; `straights` (kappa = 0: inf / inf) runs all 100."""
    ggv = np.array([[0.0, 14.0, 15.0], [20.0, 13.0, 14.0], [40.0, 12.5, 13.0], [60.0, 11.0, 12.0], [90.0, 10.0, 11.0]])
    mach = C.mach_table(18, v1=90.0)
    laps = [C.lap([(60, 1 / 200.0), (30, 1 / 15.0), (60, 1 / 300.0), (30, 1 / 20.0)]),
            C.lap([(40, 1 / 90.0), (50, C.spiral(50, 90.0, 12.0)), (40, 1 / 12.0), (50, C.spiral(50, 12.0, 400.0))])]
    iters = []
    for k, e in laps:
        iters.append(G.decide(k, e, ggv, mach, 70.0)["iters"])
    assert all(1 <= i < 20 for i in iters), iters
    c = CASES["straights"]
    assert G.decide(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"])["iters"] == 99
    w = Worst()
    for exp in (1.0, 2.0):
        gk, ge, gs = diff(laps, ggv, mach, 70.0, dyn_model_exp=exp)
        assert not gs.any()
        for b, (k, e) in enumerate(laps):
            n = k.size
            r = reference(dict(kappa=k, el=e, ggv=ggv, mach=mach, v_max=70.0), exp=exp)
            w.check(f"lap {b}", gk[b, :n], r, "g_kappa", exp)
            w.check(f"lap {b}", ge[b, :n], r, "g_el", exp)
    print(f"  G iterations {iters}")
    w.report("G fixed point", 2.0)
