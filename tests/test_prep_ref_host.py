"""CPU tests of tests/prep_ref.py, the converged reference of the prep_track kernel: against the dense restatement
oracle/tph_prep.py on small tracks (n = 5, where the wrap couplings of the cyclic pentadiagonal system fall on
neighbouring nodes, up to ~300), against the committed fixtures, the monotone residual F(lam), the closest-point
residual, and the n_out encoding the wrapper mirrors from include/mincurv_b200.h."""
import os
import re
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import prep_ref as R  # noqa: E402
from oracle import tph_prep as P  # noqa: E402


def ngon(k, perim, seed, jit=0.05):
    rng = np.random.default_rng(seed)
    a = np.linspace(0.0, 2.0 * np.pi, k, endpoint=False) + rng.uniform(-jit, jit, k) * 2.0 * np.pi / k
    r = 1.0 + rng.uniform(-jit, jit, k)
    p = np.column_stack((r * np.cos(a), r * np.sin(a)))
    p *= perim / np.sum(np.linalg.norm(np.roll(p, -1, axis=0) - p, axis=1))
    return np.column_stack((p, np.full(k, 3.0), 2.0 + rng.uniform(0.0, 1.0, k)))


SMALL = [(5, 4.6, 0.1), (5, 5.6, 0.1), (6, 6.6, 0.3), (7, 8.6, 0.1), (8, 11.6, 0.05), (12, 40.5, 0.2), (30, 120.5, 0.01),
         (60, 299.5, 10.0)]          # (raw points, perimeter [m], s as a fraction of F(inf); the last: s = 10 m^2)


@pytest.mark.parametrize("k,perim,sf", SMALL)
def test_fit_and_root_match_the_dense_oracle(k, perim, sf):
    tr = ngon(k, perim, k)
    sys_ = R.system(tr)
    s = sf * sys_.F_inf if sf < 1.0 else sf
    f_o, gam_o, lam_o = P.reinsch_periodic(sys_.u, 1.0, sys_.pts, s)
    f, gam, Fv = R.fit(sys_, lam_o)                    # the same lam: the sparse and the dense solve agree to rounding
    scale = np.abs(sys_.pts).max()
    assert np.abs(f - f_o).max() <= 1e-12 * scale and np.abs(gam - gam_o).max() <= 1e-9 * np.abs(gam_o).max()
    lam = R.root(sys_, s)
    assert abs(lam - lam_o) <= 1e-9 * lam_o           # the oracle stops its bisection at a 1e-14 bracket
    assert abs(R.F(sys_, lam) - s) <= 1e-11 * s          # (measured <= 1.7e-12: lam is exact to one ulp)
    got = R.outputs(sys_, lam, 1.0 if perim < 50 else 3.0)
    ref = P.spline_approximation_reinsch(tr, s_reg=s, stepsize_reg=1.0 if perim < 50 else 3.0)
    assert got.out.shape == ref.shape
    assert np.abs(got.out[:, :2] - ref[:, :2]).max() <= 1e-9 * scale
    assert np.abs(got.out[:, 2:] - ref[:, 2:]).max() <= 1e-5        # (the oracle's bounded scalar search: xatol 1e-13 in t)
    assert got.resid.max() <= 1e-12 * scale


@pytest.mark.parametrize("name", ["rounded_rectangle", "handling_track", "berlin_2018", "modena_2019"])
def test_reference_reproduces_the_fixtures(name):
    import pin_against_tph as kit
    raw = kit.raw_tracks()[name]
    gold = np.load(os.path.join(HERE, "golden", "prep_track.npz"))
    got, lam, sys_ = R.spline_approximation(raw, s_reg=10.0)
    ref = gold[name + "_reinsch"]
    assert got.out.shape == ref.shape
    assert np.abs(got.out[:, :2] - ref[:, :2]).max() <= 1e-11      # measured 1.0e-13 .. 5.7e-13 m
    assert np.abs(got.out[:, 2:] - ref[:, 2:]).max() <= 1e-5       # measured 6.3e-8 .. 3.5e-6 m (the oracle's search)
    assert got.resid.max() <= 1e-11 and abs(got.F - 10.0) <= 1e-12 * 10.0
    if name == "rounded_rectangle":
        mw = R.outputs(sys_, lam, 3.0, min_width=6.0).out
        assert np.abs(mw - gold[name + "_minwidth6"]).max() <= 1e-5


def test_residual_is_monotone_and_tends_to_the_constant_fit():
    sys_ = R.system(ngon(40, 255.5, 40))
    lams = np.logspace(-14, 14, 57)
    Fs = np.array([R.F(sys_, lam) for lam in lams])
    assert np.all(np.diff(Fs) >= -1e-8 * sys_.F_inf)        # (rounding of F near F(inf): 2.5e-9 relative)
    assert Fs[0] <= 1e-16 * sys_.F_inf and abs(Fs[-1] - sys_.F_inf) <= 1e-6 * sys_.F_inf
    with pytest.raises(ValueError, match="not below F"):
        R.root(sys_, sys_.F_inf)


def test_closest_point_residual_is_zero_at_the_solution_and_not_a_micrometre_away():
    tr = ngon(40, 255.5, 40)
    got, lam, sys_ = R.spline_approximation(tr, s_reg=10.0)
    assert got.resid.max() <= 1e-12
    for i in (0, 7, 40):
        t = got.t_close[i]
        x, dx, _ = (v[0] for v in R.eval3(sys_.u, got.f, got.gam, [t]))
        tm = t + 1e-6 / np.linalg.norm(dx)             # the curve point moved 1 um along the curve
        xm, dxm, _ = (v[0] for v in R.eval3(sys_.u, got.f, got.gam, [tm]))
        q = np.append(tr, tr[:1], axis=0)[i, :2]
        res = abs(float((xm - q) @ dxm)) / np.linalg.norm(dxm)
        assert 0.5e-6 <= res <= 2e-6


def test_wrapper_mirrors_the_n_out_encoding_of_the_header():
    torch = pytest.importorskip("torch")  # noqa: F841
    from global_racetrajectory_optimization_b200 import batch as B_
    h = open(os.path.join(ROOT, "include", "mincurv_b200.h")).read()
    assert re.search(r"#define MC_PREP_REFUSED \(1 << 30\)", h) and B_.PREP_REFUSED == 1 << 30
    codes = {int(v): k for k, v in re.findall(r"#define (MC_PREP_R_\w+) (\d+)", h)}
    assert sorted(codes) == sorted(B_.PREP_REASONS) == list(range(1, 7))
