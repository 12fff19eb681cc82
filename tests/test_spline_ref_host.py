"""CPU tests of the long-double spline reference (tests/spline_ref.py) that the GPU tests of csrc/splines.cu measure
against: exact rational arithmetic on small tracks, the dense float64 oracle (oracle/tph_dense.py) on the golden tracks,
and the residual of the moment system."""
import math
from fractions import Fraction

import numpy as np
import pytest

import spline_ref as S
from global_racetrajectory_optimization_b200 import synth
from oracle import tph_dense as T

GOLDEN = ("handling", "synth333", "berlin")


def _small_track(n, seed):
    rng = np.random.default_rng(seed)
    th = np.sort(rng.uniform(0.0, 2.0 * np.pi, n))
    r = 50.0 * (1.0 + 0.2 * rng.standard_normal(n))
    return np.column_stack((r * np.cos(th), r * np.sin(th)))


def _exact_coeffs(p, h):
    """Coefficients [n, 4] per coordinate of the closed spline, by Gauss-Jordan elimination in Fractions."""
    n = p.shape[0]
    P = [[Fraction(float(v)) for v in row] for row in p]
    H = [Fraction(float(v)) for v in h]
    out = []
    for k in range(2):
        A = [[Fraction(0)] * (n + 1) for _ in range(n)]
        for i in range(n):
            im, ip = (i - 1) % n, (i + 1) % n
            A[i][im] += H[im]
            A[i][i] += 2 * (H[im] + H[i])
            A[i][ip] += H[i]
            A[i][n] = 6 * ((P[ip][k] - P[i][k]) / H[i] - (P[i][k] - P[im][k]) / H[im])
        for c in range(n):
            piv = next(r for r in range(c, n) if A[r][c] != 0)
            A[c], A[piv] = A[piv], A[c]
            for r in range(n):
                if r != c and A[r][c] != 0:
                    f = A[r][c] / A[c][c]
                    A[r] = [a - f * b for a, b in zip(A[r], A[c])]
        m = [A[i][n] / A[i][i] for i in range(n)]
        rows = []
        for i in range(n):
            ip, h2 = (i + 1) % n, H[i] * H[i]
            rows.append([P[i][k], P[ip][k] - P[i][k] - h2 * (2 * m[i] + m[ip]) / 6, h2 * m[i] / 2, h2 * (m[ip] - m[i]) / 6])
        out.append(rows)
    return out


@pytest.mark.parametrize("scaled", [False, True])
@pytest.mark.parametrize("n", range(3, 13))
def test_reference_against_exact_rational_arithmetic(n, scaled):
    p = _small_track(n, n)
    h = np.random.default_rng(100 + n).uniform(0.05, 20.0, n) if scaled else np.ones(n)
    cx, cy, _, _ = S.closed_spline(p, S.ld(h))
    for got, exact in zip((cx, cy), _exact_coeffs(p, h)):
        for k in range(4):
            col = [r[k] for r in exact]
            scale = max(abs(v) for v in col)
            err = max(abs(Fraction(*g.as_integer_ratio()) - e) for g, e in zip(got[:, k], col))
            assert err / scale <= Fraction(1, 10 ** 17), (n, scaled, k, float(err / scale))


def _closed(xy):
    return np.vstack((xy[:, :2], xy[:1, :2]))


def _rel(a, b, scale):
    return float(np.abs(np.asarray(a, dtype=float) - np.asarray(b, dtype=float)).max() / scale)


@pytest.mark.parametrize("name", GOLDEN)
def test_reference_against_the_dense_oracle(golden, name):
    g = golden(name)
    rt = g["reftrack"]
    scale = np.abs(rt[:, :2]).max()
    for ds in (False, True):
        ox, oy, _, onv = T.calc_splines(_closed(rt), use_dist_scaling=ds)
        cx, cy, nv, _ = S.calc_splines(rt, use_dist_scaling=ds)
        assert _rel(cx, ox, scale) <= 1e-13 and _rel(cy, oy, scale) <= 1e-13, (name, ds)
        assert np.abs(np.asarray(nv, dtype=float) - onv).max() <= 1e-13
    nvec = g["normvec"]
    o = T.create_raceline(rt[:, :2], nvec, g["alpha_mincurv"], 2.0)
    r = S.create_raceline(rt[:, :2], nvec, g["alpha_mincurv"], 2.0)
    assert r["no"] == o[0].shape[0]
    assert np.array_equal(r["spline_inds"], o[4])
    for k, ov in (("coeffs_x", o[2]), ("coeffs_y", o[3]), ("raceline_interp", o[0]), ("s_interp", o[6]),
                  ("spline_lengths", o[7]), ("el_lengths_interp", o[8])):
        assert _rel(r[k], ov, scale) <= 1e-13, (name, k)
    assert _rel(r["t_values"], o[5], 1.0) <= 1e-12
    psi, kappa = T.calc_head_curv_an(o[2], o[3], o[4], o[5])
    assert _rel(r["kappa"], kappa, np.abs(kappa).max()) <= 1e-12
    assert np.abs(S.angle_diff(r["psi"], psi)).max() <= 1e-12


@pytest.mark.parametrize("n,ratio", [(5, 1.0), (400, 1.0), (400, 20.0), (4097, 1000.0)])
def test_moment_system_residual_in_long_double(n, ratio):
    rng = np.random.default_rng(n)
    p = _small_track(n, n) if n < 100 else synth.make_track(n, n)[:, :2]
    h = np.where(rng.random(n) < 0.5, 1.0, ratio) * rng.uniform(0.5, 2.0, n)
    a, b, c, r = S.moment_system(p, S.ld(h))
    m = S.moments(p, S.ld(h))
    assert m.dtype == S.LD
    res = a[:, None] * np.roll(m, 1, axis=0) + b[:, None] * m + c[:, None] * np.roll(m, -1, axis=0) - r
    assert np.abs(res).max() <= 16 * np.finfo(S.LD).eps * np.abs(r).max(), float(np.abs(res).max() / np.abs(r).max())


def test_normalize_psi_and_head_curv_at_the_wrap():
    # tangents along -y and just beside it: atan2 - pi/2 is -pi exactly, which normalize_psi keeps, or just above -pi,
    # or just below -pi, which it wraps to just below +pi
    xd = np.array([0.0, -0.0, 1e-3, -1e-3])
    cx = np.column_stack((np.zeros(4), xd, np.full(4, 0.5), np.full(4, 0.1)))
    cy = np.tile([0.0, -1.0, 0.0, 0.2], (4, 1))
    psi, kappa, dkappa = S.head_curv(cx, cy, np.zeros(4))
    assert psi[0] == -S.PI and psi[1] == -S.PI
    assert -S.PI < psi[2] < -S.PI + S.LD(2e-3) and S.PI - S.LD(2e-3) < psi[3] < S.PI
    assert abs(float(S.angle_diff(psi[3], -S.PI)) + 1e-3) < 1e-9
    assert np.array_equal(np.asarray(psi[:2], dtype=float), T.calc_head_curv_an(cx, cy, np.arange(2), np.zeros(2))[0])
    assert float(kappa[0]) == 1.0 and np.isfinite(np.asarray(dkappa, dtype=float)).all()
