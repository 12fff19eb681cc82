"""CPU tests of the constructed velocity-profile cases (tests/vp_cases.py): each case reaches the branch of
csrc/vel_profile_core.cuh it is named for, shown by the branch codes and the fixed-point iteration count that the host
build of the adjoint records (tests/vp_adj_ref.py), and the host build of the kernel's statements matches the oracle on
every case for both readings of decel_slice_upper.  The device runs the same cases in tests/test_gpu_velprofile_edges.py.

Where the host build and the oracle differ at all it is in the step times: tph squares v with math.pow, the kernel
multiplies, and libm's pow is not always correctly rounded (one ulp on some speeds), which the cancelling step-time
formula amplifies when the acceleration of a step is tiny."""
import math

import numpy as np
import pytest

import vp_cases as C
from oracle import tph_velprofile as VP
from vp_adj_ref import Harness

ACTIVE, TAKEN, LEAVE, VTMP, CLAMP, MACH, CLAMP2 = 1, 2, 4, 8, 16, 32, 64
CASES = C.cases()
# max |t - t_oracle| / t_lap of the host build over every case, both readings, dyn_model_exp 1 / 1.5 / 2 and filter
# windows 3 / 7 (vx and ax are bit for bit the oracle's): measured 8.2e-13 (the clamp case, pow(v, 2) != v * v)
T_TOL = 4e-12


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return Harness(tmp_path_factory.mktemp("vp_cases_host"))


def reached(harness, c, upper=1):
    """The set of branch names the case reaches on the host build (the names of vp_cases.cases()'s `reaches`)."""
    k, e = c["kappa"], c["el"]
    n = k.size
    h = harness.adjoint(k, e, c["ggv"], c["mach"], c["v_max"], 1.0, upper=upper)
    vx = harness.profile(k, e, c["ggv"], c["mach"], c["v_max"], upper=upper)["vx"]
    cf, cb = h["codes"][:2 * n - 1], h["codes"][2 * n:2 * n + (n - 1 if upper else 2 * n - 1)]
    every = np.concatenate((cf, cb))
    fwd_taken = ((cf & ACTIVE) > 0) & ((cf & TAKEN) > 0)
    out = {
        "taken": bool((every & TAKEN).any()),
        "leave": bool((every & LEAVE).any()),
        "vtmp": bool(((cb & ACTIVE) > 0).any() and (cb & VTMP).any()),
        "novtmp": bool((((cb & ACTIVE) > 0) & ((cb & VTMP) == 0)).any()),
        "clamp": bool((every & (CLAMP | CLAMP2)).any()),
        "mach": bool((cf & MACH).any()),
        "tyre": bool((fwd_taken & ((cf & MACH) == 0)).any()),
        "kappa0": bool((k == 0.0).any()),
        "iters100": h["iters"] == 99,
        "clip": vx.max() == c["v_max"],
        "below_first": vx.min() < c["ggv"][0, 0] and vx.min() < c["mach"][0, 0],
        "on_knot": bool(np.isin(vx, c["ggv"][1:-1, 0]).any() and np.isin(vx, c["mach"][1:-1, 0]).any()),
        "last_knot": bool((vx == c["ggv"][-1, 0]).any() and (vx == c["mach"][-1, 0]).any()),
        "start_j0": bool(cf[0] & ACTIVE and cb[0] & ACTIVE),
    }
    return {name for name, hit in out.items() if hit}, h


def test_the_stock_tables_are_the_golden_ones(golden):
    v = golden("velprofile")
    g, m = C.stock_tables()
    assert np.array_equal(g, v["ggv"]) and np.array_equal(m, v["ax_max_machines"])


@pytest.mark.parametrize("name", sorted(CASES))
def test_each_case_reaches_the_branches_it_is_named_for(harness, name):
    c = CASES[name]
    got, h = reached(harness, c)
    assert h["status"] == 0
    assert c["reaches"] <= got, c["reaches"] - got


def test_the_cases_together_reach_every_branch(harness):
    every = set().union(*(reached(harness, c)[0] for c in CASES.values()))
    assert every == {"taken", "leave", "vtmp", "novtmp", "clamp", "mach", "tyre", "kappa0", "iters100", "clip",
                     "below_first", "on_knot", "last_knot", "start_j0"}
    sizes = {c["ggv"].shape[0] for c in CASES.values()} | {c["mach"].shape[0] for c in CASES.values()}
    assert {1, 2, 18, 256} <= sizes
    assert any(c["ggv"][0, 0] > 0.0 for c in CASES.values())


@pytest.mark.parametrize("upper", [1, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_host_build_matches_the_oracle_on_every_case(harness, name, upper):
    c = CASES[name]
    for exp, filt in ((1.0, None), (1.5, None), (2.0, 3), (1.0, 7)):
        vx, ax, t = C.oracle(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], exp=exp, filt=filt, upper=upper)
        h = harness.profile(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], exp=exp, filt=filt or 0, upper=upper,
                            stride=3)
        assert h["status"] == 0
        assert np.array_equal(h["vx"], vx) and np.array_equal(h["ax"], ax), (exp, filt)
        assert np.abs(h["t"] - t).max() <= T_TOL * t[-1] and h["laptime"] == h["t"][-1], (exp, filt)


def test_host_build_matches_the_oracle_with_mu_and_a_ggv_scale(harness):
    rng = np.random.default_rng(11)
    for name in ("straights", "spiral", "phase_at_j0"):
        c = CASES[name]
        mu = 0.75 + 0.4 * rng.random(c["kappa"].size)
        for scale in (1.0, 0.55):
            vx, ax, t = C.oracle(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], scale=scale, mu=mu)
            h = harness.profile(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], scale=scale, mu=mu, stride=2)
            # np.mean sums mu pairwise, the kernel in order: the global lateral limit may differ in its last bit
            assert np.abs(h["vx"] - vx).max() <= 1e-14 * vx.max()
            assert np.abs(h["t"] - t).max() <= T_TOL * t[-1]


@pytest.mark.parametrize("n", range(2, 10))
def test_host_build_matches_the_oracle_on_tiny_laps(harness, n):
    k, e = C.tiny_lap(n)
    ggv, mach = C.ggv_table(18), C.mach_table(18)
    for upper in (1, 0):
        vx, ax, t = C.oracle(k, e, ggv, mach, 60.0, upper=upper)
        h = harness.profile(k, e, ggv, mach, 60.0, upper=upper)
        assert h["status"] == 0 and np.array_equal(h["vx"], vx) and np.abs(h["t"] - t).max() <= T_TOL * t[-1]


def test_filter_windows_that_wrap_the_lap():
    """tph's conv_filt on a closed lap of n points is the cyclic average while the half-width (w - 1) / 2 <= n, and
    returns a profile of the wrong length beyond that (the kernel refuses such a track per profile)."""
    rng = np.random.default_rng(3)
    for n in (2, 3, 5, 9):
        sig = 10.0 + rng.random(n)
        for w in range(3, 2 * n + 2, 2):
            h = (w - 1) // 2
            cyc = np.array([sum(sig[(i + j) % n] for j in range(-h, h + 1)) / w for i in range(n)])
            assert np.abs(VP.conv_filt(sig, w, True) - cyc).max() <= 1e-14 * cyc.max()
        for w in (2 * n + 3, 2 * n + 5):
            assert VP.conv_filt(sig, w, True).size != n


def test_exact_lap_time_reference():
    rng = np.random.default_rng(4)
    vx = 30.0 + 20.0 * rng.random(500)
    el = 1.0 + rng.random(500)
    steps = C.exact_step_times(vx, el)
    assert C.exact_lap_time(vx, el) == math.fsum(steps) or abs(C.exact_lap_time(vx, el) - math.fsum(steps)) <= 1e-13
    assert np.abs(steps - 2.0 * el / (vx + np.roll(vx, -1))).max() <= 1e-15


def test_step_time_formula_cancels_on_long_straights():
    """tph's step time (-v + sqrt(v^2 + 2 a e)) / a against the exact 2 e / (v + v') on the oracle's own profile: on
    1.5 km straights the two agree to 1e-11 s; on 20 km straights, where the car creeps towards its drag-limited terminal
    speed, the formula loses most digits of single steps and the lap comes out longer.  The kernel copies the formula
    (tests/test_gpu_velprofile_edges.py pins it to the oracle there); the gap is a deliberate parity deviation."""
    g, m = C.stock_tables()
    k, e = C.two_long_straights(1.5)
    vx, ax, t = C.oracle(k, e, g, m, 70.0)
    assert abs(t[-1] - C.exact_lap_time(vx, e)) <= 1e-11
    k, e = C.two_long_straights(20.0)
    vx, ax, t = C.oracle(k, e, g, m, 70.0)
    gap = t[-1] - C.exact_lap_time(vx, e)
    steps = C.exact_step_times(vx, e)
    worst = np.max(np.abs(np.diff(t) - steps) / steps)
    assert 0.1 < gap < 0.25 and worst > 0.5, (gap, worst)
