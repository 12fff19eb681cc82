"""CPU tests (-m "not gpu") of the velocity-profile adjoint (csrc/vel_profile_core.cuh: profile_adjoint_thread, K5d)
against an extended-precision replay of tph's solver with the forward's decisions held (tests/vp_grad_ref.py), on the
constructed laps of tests/vp_cases.py, where the adjoint changes code path.

* The reference can be trusted: its decision run is the oracle bit for bit, its decisions are the host tape's branch
  codes, and its reverse tape agrees with long-double central differences of its own replay.
* The host build of K5d (tests/vp_adj_ref.py, vp_matrix_ref.py, the in-place vehicle tables of vp_veh_host.cpp)
  against the reference, entry by entry, for both decel_slice_upper readings, dyn_model_exp 1, 1.5 and 2, filter
  windows, an upstream gradient of vx, ggv scales and binding top speeds.
* dyn_model_exp != 1 at the lateral limit: conditioning, not a wrong derivative (DESIGN.md sections 3.12 and 6).

Every bound is printed next to the value measured (pytest -s)."""
import numpy as np
import pytest

import vp_cases as C
import vp_grad_ref as G
from vp_matrix_ref import MatrixHarness

CASES = C.cases()
NAMES = sorted(CASES)
PIN = 2.0 ** -40          # a radicand the forward evaluated in (0, 2^-40) is at the rounding level of 1 - q^p: pinned
# host against the reference, per entry: |dev - ref| <= TOL * max |ref| + COND * cond (the conditioning of
# vp_grad_ref._conditioning), and |dev - ref| / |ref| <= REL on entries >= 1e-3 max |ref|.  Measured on these laps:
TOL = {1.0: 1e-14, 1.5: 1e-12, 2.0: 1e-12}        # 1.2e-15 at p = 1; 8.0e-14 outside the lateral limit at p = 1.5 / 2
REL = {1.0: 3e-12, 1.5: 1e-10, 2.0: 1e-10}        # the H100's bounds (test_gpu_vp_adjoint_edges.py): the host equals it
WIDE_TOL = 5e-14                                  # a window of half-width > n / 2: 6.2e-15
COND = 40.0                                       # <= 3.5 times the conditioning at the lateral-limit steps
FD_TOL = 1e-10                                    # the tape against long-double central differences of the replay


def report(what, measured, bound):
    print(f"  {what}: measured {measured:.3e}, bound {bound:.0e}")
    assert measured <= bound, what


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    try:
        return MatrixHarness(tmp_path_factory.mktemp("vp_grad_ref"))
    except RuntimeError as e:
        pytest.skip(str(e))


def errors(got, ref):
    """(max |got - ref| / max |ref|, |got - ref|, max |ref|)."""
    ref = np.asarray(ref, dtype=float)
    d = np.abs(np.asarray(got, dtype=float) - ref)
    s = max(float(np.abs(ref).max()), 1e-300)
    return float(d.max() / s), d, s


def check(label, host, ref, p, tol=None):
    """host (dict g_kappa, g_el) against the reference per entry, with the bounds above.  Returns per key
    (max-normalised error, relative error on the large entries, max-normalised error where the conditioning is below
    the floor)."""
    worst = {}
    for key in ("g_kappa", "g_el"):
        want = np.asarray(ref[key], dtype=float)
        ab, d, s = errors(host[key], want)
        cond = ref["cond_kappa"] if key == "g_kappa" else np.zeros(want.size)
        tol = TOL[p] if tol is None else tol
        excess = d - tol * s - COND * cond
        assert (excess <= 0).all(), (label, key, int(np.argmax(excess)), float(excess.max() / s))
        plain = COND * cond <= tol * s
        big = plain & (np.abs(want) >= 1e-3 * s)
        rel = float((d[big] / np.abs(want[big])).max()) if big.any() else 0.0
        assert rel <= REL[p], (label, key, rel)
        worst[key] = (ab, rel, float(d[plain].max() / s) if plain.any() else 0.0)
    return worst


def reference(c, upper=1, exp=1.0, g_lap=1.0, g_vx=None, filt=None, scale=1.0, v_max=None, host=None, **veh):
    """(log, replay) of case c; host: the host adjoint, whose codes the replay takes where they differ (listed)."""
    lg = G.decide(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"] if v_max is None else v_max, scale=scale,
                  exp=exp, filt=filt, upper=upper, **veh)
    codes = None
    if host is not None:
        diffs = G.code_diffs(lg["codes"], host["codes"], c["kappa"].size, upper)
        assert host["iters"] == lg["iters"]
        assert not diffs, diffs                # no tie on these laps: the host decides as the reference
        codes = host["codes"]
    return lg, G.replay(c["kappa"], c["el"], lg, g_lap=g_lap, g_vx=g_vx, codes=codes, pin=PIN)


# ---- 1. the reference --------------------------------------------------------------------------------------------------
def _golden_laps(golden):
    v = golden("velprofile")
    out = {}
    for name in ("handling", "synth333"):
        g = golden(name)
        out[name] = dict(kappa=g["rl_kappa"], el=g["rl_el_lengths"], ggv=v["ggv"], mach=v["ax_max_machines"], v_max=70.0)
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    for n in range(2, 10):
        k, e = C.tiny_lap(n)
        out[f"tiny_lap({n})"] = dict(kappa=k, el=e, ggv=ggv, mach=mach, v_max=60.0)
    return out


@pytest.mark.parametrize("upper", [1, 0])
def test_decisions_are_the_oracle_and_the_host_codes(golden, harness, upper):
    """At p = 1 the decision run's vx is the oracle's bit for bit; its codes (with the table segments of every taken
    step) and its iteration count are the host tape's, on every constructed lap, tiny_lap(2..9) and two golden
    racelines; at p = 1.5 and 2 on the constructed laps too."""
    laps = dict(CASES, **_golden_laps(golden))
    for name, c in laps.items():
        for exp in ((1.0, 1.5, 2.0) if name in CASES else (1.0,)):
            lg = G.decide(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], exp=exp, upper=upper)
            vx, _, _ = C.oracle(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], exp=exp, upper=upper)
            assert np.array_equal(lg["vx"], vx), (name, exp)
            h = harness.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, exp=exp, upper=upper)
            assert h["status"] == 0 and h["iters"] == lg["iters"], (name, exp)
            diffs = G.code_diffs(lg["codes"], h["codes"], c["kappa"].size, upper)
            assert not diffs, (name, exp, diffs[:5])
    print(f"  upper {upper}: {len(laps)} laps, every decision equal (0 ties)")


def test_every_case_reaches_its_branches():
    """The codes show the branches the laps are built for: the clamp, vtmp won, the machine limit and the table
    clamped below the first knot at taken steps, leaving at v_max, a phase at j = 0 in both passes, and the clip."""
    seen = set()
    for name, c in CASES.items():
        lg = G.decide(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"])
        k, n = lg["codes"], c["kappa"].size
        taken = (k & G.TAKEN) != 0
        seen |= {b for b, m in (("clamp", G.CLAMP), ("vtmp", G.VTMP), ("mach", G.MACH)) if (k[taken] & m).any()}
        seen |= {"leave"} if (k & G.LEAVE).any() else set()
        seen |= {"clip"} if lg["clip"].any() else set()
        seen |= {"start_j0"} if (k[0] & G.TAKEN and k[2 * n] & G.TAKEN) else set()
        seen |= {"below_first"} if ((k[taken] >> 8 & 0xff) == 0).any() and c["ggv"][0, 0] > 0 else set()
    assert {"clamp", "vtmp", "mach", "leave", "clip", "start_j0", "below_first"} <= seen, seen


FD_CASES = [(name, 1.0) for name in NAMES] + [(name, 2.0) for name in ("clamp", "phase_at_j0", "seam_braking")]


@pytest.mark.parametrize("name,exp", FD_CASES)
def test_tape_matches_long_double_central_differences(name, exp):
    """The reverse tape against central differences of the same replay in long double (the decisions are held by
    construction), along random relative directions of kappa and el, one at a time."""
    c = CASES[name]
    lg = G.decide(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], exp=exp)
    rng = np.random.default_rng(len(name))
    g_vx = 0.01 * rng.standard_normal(c["kappa"].size)
    r = G.replay(c["kappa"], c["el"], lg, g_vx=g_vx)
    if exp != 1.0:                                   # nothing at the rounding level of 1 - q^p (see section 3)
        assert not any(0.0 < x < PIN for v in lg["rads"].values() for x in v if x is not None)
    k, e = c["kappa"].astype(G.LD), c["el"].astype(G.LD)
    worst = 0.0
    for which in ("kappa", "el"):
        u = rng.uniform(-1.0, 1.0, k.size).astype(G.LD)
        dk, de = (k * u, 0 * e) if which == "kappa" else (0 * k, e * u)

        def cd(d):
            lp = G.replay(k + d * dk, e + d * de, lg, g_vx=g_vx, tape=False)["loss"]
            return (lp - G.replay(k - d * dk, e - d * de, lg, g_vx=g_vx, tape=False)["loss"]) / (2 * d)

        d = G.LD(1e-5 if exp == 1.0 else 5e-7)     # (1 - q^2)^(1/2) curves hard near q = 1: a smaller step at p = 2
        fd = (4 * cd(d) - cd(2 * d)) / 3          # Richardson: the delta^2 term cancels
        an = (r["g_kappa"] * dk).sum() + (r["g_el"] * de).sum()
        worst = max(worst, float(abs(fd - an) / abs(an)))
    report(f"{name} p {exp}: tape vs central differences", worst, FD_TOL)


# ---- 2. the host build against the reference ---------------------------------------------------------------------------
@pytest.mark.parametrize("exp", [1.0, 1.5, 2.0])
@pytest.mark.parametrize("upper", [1, 0])
@pytest.mark.parametrize("name", NAMES)
def test_host_adjoint_against_the_reference(harness, name, upper, exp):
    c = CASES[name]
    h = harness.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, exp=exp, upper=upper)
    assert h["status"] == 0
    _, r = reference(c, upper=upper, exp=exp, host=h)
    w = check(name, h, r, exp)
    report(f"{name} upper {upper} p {exp}: g_kappa max-normalised", w["g_kappa"][2], TOL[exp])
    report(f"{name} upper {upper} p {exp}: g_el max-normalised", w["g_el"][0], TOL[exp])
    print(f"  (g_kappa max-normalised with the lateral-limit points: {w['g_kappa'][0]:.3e}, "
          f"conditioning {float(r['cond_kappa'].max()) / max(np.abs(r['g_kappa']).max(), 1e-300):.3e})")


@pytest.mark.parametrize("window", [3, 5, "wide"])
def test_host_adjoint_with_filter_windows_and_an_upstream_vx_gradient(harness, window):
    """Windows 3, 5 and one whose half-width is more than half the lap (it wraps), with g_lap and a random g_vx,
    the host's vectors at stride 3.  The wide window sums ~200 terms per entry in another order than the reference:
    its bound is WIDE_TOL."""
    tol = WIDE_TOL if window == "wide" else TOL[1.0]
    worst = {"g_kappa": 0.0, "g_el": 0.0}
    for name in ("phase_at_j0", "spiral", "seam_braking", "one_row"):
        c = CASES[name]
        n = c["kappa"].size
        w = (2 * (n // 2 + 7) + 1) if window == "wide" else window
        assert (w - 1) // 2 <= n and (window != "wide" or (w - 1) // 2 > n / 2)
        g_vx = 0.05 * np.random.default_rng(n).standard_normal(n)
        for upper in (1, 0):
            h = harness.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 0.5, g_vx=g_vx, filt=w,
                                upper=upper, stride=3)
            assert h["status"] == 0
            _, r = reference(c, upper=upper, g_lap=0.5, g_vx=g_vx, filt=w, host=h)
            for key, v in check(name, h, r, 1.0, tol).items():
                worst[key] = max(worst[key], v[0])
    for key, v in worst.items():
        report(f"window {window}: {key}", v, tol)


def test_host_matrix_cells_against_the_reference(harness):
    """Cells of the lap-time matrix: ggv scales 0.6 and 1.3, the case's top speed and one that binds in the passes;
    a track's matrix gradient against the reference sum over its cells."""
    worst = {"g_kappa": 0.0, "g_el": 0.0}
    for name in ("vmax_interior_knot", "vmax_last_knot", "stock_long_straights", "seam_accel"):
        c = CASES[name]
        speeds = [c["v_max"], 30.0]
        scales = [0.6, 1.3]
        g_lap = np.array([[1.0, -0.5], [0.25, 2.0]])
        m = harness.matrix_adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], scales, speeds, g_lap)
        assert not m["status"].any()
        tot = {"g_kappa": 0.0, "g_el": 0.0}
        for t, vm in enumerate(speeds):
            for s, sc in enumerate(scales):
                cell = m["cells"][t * len(scales) + s]
                lg, r = reference(c, g_lap=g_lap[t, s], scale=sc, v_max=vm, host=cell)
                if vm == 30.0:
                    assert (lg["codes"] & G.LEAVE).any()           # the top speed binds in the passes
                for key, v in check(f"{name} {vm} {sc}", cell, r, 1.0).items():
                    worst[key] = max(worst[key], v[0])
                    tot[key] = tot[key] + r[key]
        for key in tot:
            worst[key] = max(worst[key], errors(m[key], tot[key])[0])
    for key, v in worst.items():
        report(f"matrix cells and sums: {key}", v, TOL[1.0])


def test_host_vehicle_tables_against_the_reference(tmp_path_factory):
    """The in-place tables of the vehicle kernels (vp_veh_host.cpp), with other drag and mass."""
    from test_velprofile_vehicles_host import VehHarness
    veh = VehHarness(tmp_path_factory.mktemp("vp_grad_ref_veh"))
    worst = {"g_kappa": 0.0, "g_el": 0.0}
    for name in ("one_row", "two_rows", "rows256", "below_first_knot", "straights"):
        c = CASES[name]
        for exp in (1.0, 2.0):
            h = veh.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, exp=exp, drag_coeff=1.1,
                            m_veh=800.0)
            assert h["status"] == 0
            _, r = reference(c, exp=exp, host=h, drag_coeff=1.1, m_veh=800.0)
            for key, v in check(name, h, r, exp).items():
                worst[key] = max(worst[key], v[0])
    for key, v in worst.items():
        report(f"vehicle tables: {key}", v, TOL[2.0])


# ---- 3. dyn_model_exp != 1 at the lateral limit --------------------------------------------------------------------------
@pytest.mark.parametrize("exp", [1.5, 2.0])
@pytest.mark.parametrize("name", ["spiral", "vmax_interior_knot"])
def test_lateral_limit_at_exponents_other_than_one_is_conditioning(harness, name, exp):
    """Where a phase starts on an arc at the initial profile's lateral-limit speed, q = v^2 / (r ay_max) is 1 in exact
    arithmetic.  float64 gives 1 - q^p a few ulps above 0 (so the forward does not clamp it) and the frozen function
    takes (1 - q^p)^(1/p) there, whose derivative (1 - q^p)^(1/p - 1) is 1e5 (p = 1.5) to 4e7 (p = 2): set by
    rounding, not by the track.  In long double the same radicand is within 1e-18 of 0 (or below it: the replay's own
    point gives NaN).  With the forward's radicand pinned the reference agrees with the host to the conditioning of
    those steps (vp_grad_ref._conditioning), and everywhere else to the bound of p = 1."""
    c = CASES[name]
    h = harness.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, exp=exp)
    lg, r = reference(c, exp=exp, host=h)
    with np.errstate(invalid="ignore"):                                 # at the replay's own points: NaN
        free = G.replay(c["kappa"], c["el"], lg, codes=h["codes"])
    at_limit = [(key, k, x) for key, v in lg["rads"].items() for k, x in enumerate(v) if x is not None and 0 < x < PIN]
    assert at_limit
    for key, k, x in at_limit:
        assert x <= 8 * 2.0 ** -53 and abs(float(free["rads"][key][k])) <= 1e-18, (key, x)
    # every other unclamped radicand is far from the rounding level
    rest = [x for v in lg["rads"].values() for x in v if x is not None and x >= PIN]
    assert min(rest) > 1e-6
    ab_free = errors(h["g_kappa"], free["g_kappa"])[0]
    w = check(name, h, r, exp)
    s = float(np.abs(r["g_kappa"]).max())
    print(f"  {name} p {exp}: {len(at_limit)} steps at the lateral limit, radicands {min(x for *_, x in at_limit):.1e}"
          f"..{max(x for *_, x in at_limit):.1e} (long double: <= 1e-18); unpinned replay vs host {ab_free:.3e}")
    report(f"{name} p {exp}: pinned, g_kappa max-normalised", w["g_kappa"][0],
           TOL[exp] + COND * float(r["cond_kappa"].max()) / s)
    report(f"{name} p {exp}: pinned, g_el max-normalised", w["g_el"][0], TOL[exp])
    report(f"{name} p {exp}: pinned, g_kappa away from the lateral-limit points", w["g_kappa"][2], TOL[exp])


def test_host_fixed_point_derivative_of_a_converging_initial_profile(harness):
    """A speed-dependent ggv on laps without a straight: the initial profile settles after a few sweeps, so the
    derivative D it carries still depends on its first estimate (on the constructed laps, which all have a straight,
    the 100 sweeps of a contracting map forget it)."""
    ggv = np.array([[0.0, 14.0, 15.0], [20.0, 13.0, 14.0], [40.0, 12.5, 13.0], [60.0, 11.0, 12.0], [90.0, 10.0, 11.0]])
    mach = C.mach_table(18, v1=90.0)
    laps = [C.lap([(60, 1 / 200.0), (30, 1 / 15.0), (60, 1 / 300.0), (30, 1 / 20.0)]),
            C.lap([(40, 1 / 90.0), (50, C.spiral(50, 90.0, 12.0)), (40, 1 / 12.0), (50, C.spiral(50, 12.0, 400.0))])]
    worst = {"g_kappa": 0.0, "g_el": 0.0}
    for k, e in laps:
        c = dict(kappa=k, el=e, ggv=ggv, mach=mach, v_max=70.0)
        for exp in (1.0, 2.0):
            h = harness.adjoint(k, e, ggv, mach, 70.0, 1.0, exp=exp)
            assert h["status"] == 0 and 1 <= h["iters"] < 20
            _, r = reference(c, exp=exp, host=h)
            for key, v in check("fixed point", h, r, exp).items():
                worst[key] = max(worst[key], v[0])
    for key, v in worst.items():
        report(f"converging fixed point: {key}", v, TOL[2.0])
