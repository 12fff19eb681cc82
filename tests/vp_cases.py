"""Constructed laps and vehicle tables for the velocity-profile stage (csrc/vel_profile_core.cuh, K5) at the places where
its code changes path, the oracle on them, and an exact reference of the lap time on a given speed profile.  Test
infrastructure (CPU, float64), not product code.

A case is a closed lap given as kappa and el_lengths (n points), a ggv table [k, 3], a machine table [m, 2] and a top
speed; `reaches` names the branches the case is built to reach (tests/test_vp_cases_host.py shows that it does).
"""
from fractions import Fraction

import numpy as np

from oracle import tph_velprofile as VP

VEH = dict(drag_coeff=0.75, m_veh=1200.0)


# ---- tables ----------------------------------------------------------------------------------------------------------
def ggv_table(rows, v0=0.0, v1=72.0, ax=(12.7, 10.3), ay=(13.1, 11.3)):
    """rows knots from v0 to v1 (a one-row table has its knot at v1) with ax_max and ay_max falling linearly: a table
    whose segments have slopes, so that interpolation inside a segment differs from its end values."""
    v = np.array([float(v1)]) if rows == 1 else np.linspace(v0, v1, rows)
    f = np.linspace(0.0, 1.0, rows) if rows > 1 else np.zeros(1)
    return np.column_stack((v, ax[0] + (ax[1] - ax[0]) * f, ay[0] + (ay[1] - ay[0]) * f))


def mach_table(rows, v0=0.0, v1=72.0, a=(5.3, 1.7)):
    v = np.array([float(v1)]) if rows == 1 else np.linspace(v0, v1, rows)
    f = np.linspace(0.0, 1.0, rows) if rows > 1 else np.zeros(1)
    return np.column_stack((v, a[0] + (a[1] - a[0]) * f))


def stock_tables():
    """The racecar's tables (tests/golden/velprofile.npz): 18 rows, ay_max flat at 12 m/s^2."""
    v = np.linspace(0.0, 60.0, 16)
    v = np.append(v, [66.0, 72.0])
    mach = np.array([5.3] * 10 + [5.1, 5.0, 4.6, 4.1, 3.7, 2.7, 2.2, 1.5])
    return np.column_stack((v, np.full(18, 12.0), np.full(18, 12.0))), np.column_stack((v, mach))


# ---- laps ------------------------------------------------------------------------------------------------------------
def lap(pieces, el=2.0):
    """A closed lap from pieces (points, kappa): kappa a number (a constant-radius arc, 0 for a straight) or a sequence
    of that many values.  el: one step length for all points, or a sequence."""
    k = np.concatenate([np.full(m, float(c)) if np.ndim(c) == 0 else np.asarray(c, dtype=float) for m, c in pieces])
    e = np.full(k.size, float(el)) if np.ndim(el) == 0 else np.asarray(el, dtype=float)
    assert e.size == k.size
    return k, e


def hairpin_lap(straight=60, r=15.0, el=2.0):
    """Two straights (kappa exactly 0) joined by two half circles of radius r."""
    m = int(round(np.pi * r / el))
    return lap([(straight, 0.0), (m, 1.0 / r), (straight, 0.0), (m, 1.0 / r)], el)


def spiral(m, r0, r1):
    """m points whose radius shrinks from r0 to r1: the braking zone where the backward pass's correction step wins."""
    return 1.0 / np.geomspace(r0, r1, m)


# ---- the cases -------------------------------------------------------------------------------------------------------
def cases():
    """{name: dict(kappa, el, ggv, mach, v_max, reaches)}."""
    g18, m18 = ggv_table(18), mach_table(18)
    gs, ms = stock_tables()
    out = {}

    def add(name, k_e, ggv, mach, v_max, reaches, mu=None):
        k, e = k_e
        out[name] = dict(kappa=k, el=e, ggv=ggv, mach=mach, v_max=float(v_max), reaches=set(reaches), mu=mu)

    # kappa == 0: R = inf, inf / inf = NaN in the fixed point (all 100 iterations), the v_max clip
    add("straights", hairpin_lap(150), g18, m18, 40.0, {"kappa0", "iters100", "clip", "taken", "leave", "mach", "tyre"})
    # ay_max r a perfect square on a flat ay column: v^2 / r / ay_max == 1 exactly, the radicand is clamped to 0
    add("clamp", lap([(40, 0.0), (19, 1 / 12.0), (40, 0.0), (42, 1 / 27.0), (30, 0.0), (118, 1 / 75.0)]), gs, ms, 70.0,
        {"clamp", "taken", "kappa0"})
    # a braking zone into a tightening spiral: the correction step wins at some steps and loses at others
    add("spiral", lap([(80, 0.0), (60, spiral(60, 400.0, 14.0)), (30, 1 / 14.0), (50, spiral(50, 14.0, 300.0))]), g18, m18,
        70.0, {"vtmp", "novtmp", "taken"})
    # a hairpin slower than the first ggv / machine knot (x < xp[0])
    add("below_first_knot", hairpin_lap(40, 6.0, 1.0), ggv_table(18, 20.0), mach_table(18, 20.0), 60.0,
        {"below_first", "taken"})
    # top speed on an interior knot of both tables (x == xp[lo])
    add("vmax_interior_knot", hairpin_lap(250, 25.0), g18, m18, float(g18[11, 0]), {"on_knot", "clip", "taken"})
    # top speed on the last knot of both tables (x >= xp[n - 1]); on the arc of radius 128 m the fixed point
    # sqrt(ay_max(v) r) lands exactly on that knot (12.5 * 128 = 40^2).  The steep last segment of ay_max makes the
    # interpolation formula evaluated at the knot round away from 12.5 (to 12.5 - 3.6e-15): only the branch taken for
    # x >= xp[n - 1] gives the table's value there
    g_last, m_last = ggv_table(18, v1=40.0, ay=(14.3, 12.5)), mach_table(18, v1=40.0, a=(5.3, 3.1))
    g_last[16, 2] = 32.44
    add("vmax_last_knot", lap([(150, 0.0), (60, 1.0 / 128.0), (150, 0.0), (40, 1 / 30.0)]), g_last, m_last, 40.0,
        {"last_knot", "clip", "taken"})
    # table sizes: one row (every speed below the only knot), two rows, 256 rows
    add("one_row", hairpin_lap(50, 20.0), ggv_table(1, v1=80.0), mach_table(1, v1=80.0), 50.0, {"below_first", "taken"})
    add("two_rows", hairpin_lap(50, 20.0), ggv_table(2), mach_table(2), 50.0, {"taken"})
    add("rows256", hairpin_lap(50, 20.0), ggv_table(256), mach_table(256), 50.0, {"taken"})
    # a phase that starts at j = 0 in both passes: the slowest point of a corner sits on the seam
    k, e = hairpin_lap(60, 18.0)
    m = int(round(np.pi * 18.0 / 2.0))
    k = np.roll(k, -(60 + m // 2))
    e = np.roll(e, -(60 + m // 2))
    k[0] *= 1.3
    k[-1] *= 1.3
    add("phase_at_j0", (k, e), g18, m18, 70.0, {"start_j0", "taken"})
    # the seam inside a braking zone and inside an accelerating run
    k, e = hairpin_lap(80, 15.0)
    add("seam_braking", (np.roll(k, 8), np.roll(e, 8)), g18, m18, 70.0, {"taken"})
    add("seam_accel", (np.roll(k, -(24 + 10)), np.roll(e, -(24 + 10))), g18, m18, 70.0, {"taken"})
    # the stock tables, a lap whose straights are long enough for drag to hold the car below v_max
    add("stock_long_straights", hairpin_lap(400, 30.0), gs, ms, 70.0, {"taken", "mach"})
    return out


def tiny_lap(n):
    """A lap of n points (2 <= n <= 9 covers every partial VP_UNROLL block and the wrap of the prefetch)."""
    i = np.arange(n)
    k = 1.0 / (20.0 + 15.0 * np.cos(2.0 * np.pi * i / n + 0.3))
    k[n // 2] = 0.0
    return k, np.full(n, 3.0 + 0.1 * (n % 3))


def two_long_straights(km=20.0, el=2.0, r=60.0):
    """Two straights of km kilometres joined by half circles: on the stock tables the car creeps towards its drag-limited
    terminal speed, where tph's step-time formula cancels."""
    return hairpin_lap(int(round(km * 1000.0 / el)), r, el)


# ---- the oracle ------------------------------------------------------------------------------------------------------
def oracle(kappa, el, ggv, mach, v_max, scale=1.0, exp=1.0, filt=None, mu=None, upper=None):
    """(vx [n], ax [n], t [n + 1]) of oracle/tph_velprofile.py: calc_vel_profile -> calc_ax_profile -> calc_t_profile, the
    call sequence of main_globaltraj.py.  upper: DECEL_LAP_SLICE_UPPER for this call (None: the module's)."""
    g = np.array(ggv, dtype=float)
    g[:, 1:] *= scale
    saved = VP.DECEL_LAP_SLICE_UPPER
    if upper is not None:
        VP.DECEL_LAP_SLICE_UPPER = bool(upper)
    try:
        vx = VP.calc_vel_profile(ggv=g, ax_max_machines=mach, v_max=v_max, kappa=kappa, el_lengths=el, closed=True,
                                 dyn_model_exp=exp, filt_window=filt, mu=mu, **VEH)
    finally:
        VP.DECEL_LAP_SLICE_UPPER = saved
    ax = VP.calc_ax_profile(vx_profile=np.append(vx, vx[0]), el_lengths=el, eq_length_output=False)
    t = VP.calc_t_profile(vx_profile=vx, ax_profile=ax, el_lengths=el)
    return vx, ax, t


# ---- the exact step times --------------------------------------------------------------------------------------------
def exact_step_times(vx, el):
    """2 e_i / (v_i + v_i+1) of the closed profile vx, each in exact rational arithmetic and rounded once to a double:
    the time of a step of constant acceleration, in the form that does not cancel."""
    vn = np.roll(vx, -1)
    return np.array([float(2 * Fraction(e) / (Fraction(a) + Fraction(b))) for a, b, e in zip(vx, vn, el)])


def exact_lap_time(vx, el):
    """Sum over the closed profile of 2 e_i / (v_i + v_i+1), exact: each term in rational arithmetic, rounded to a
    multiple of 2^-90 s (far below any double's resolution of a lap time), and summed as integers."""
    vn = np.roll(vx, -1)
    acc = 0
    for a, b, e in zip(vx, vn, el):
        acc += round(2 * Fraction(e) / (Fraction(a) + Fraction(b)) * 2 ** 90)
    return float(Fraction(acc, 2 ** 90))
