"""The long-double reference of the minimum-curvature post-solve kernel (tests/finalize_ref.py) against tph's dense
restatement (oracle/tph_dense.py), against itself (slab replay against definition) and on its edges: the error about
the line alpha = a, lin_alpha = 0, NaN and inf in alpha, and the status rules on every (status, limit) pair."""
import itertools

import numpy as np
import pytest

import finalize_ref as F
import mincurv_ref as R
from oracle import tph_dense as T

# from_inputs against the oracle (k_kappa_ref + E_kappa alpha per point, curv_error_max_from), max |diff| / max |ref|
# for kappa and |diff| / max(curv_error_max, 1e-3 kappa_lin_max) for the error.  The oracle inverts the dense 4N spline
# system in float64: measured 4.9e-13 / 7.8e-14 on the golden tracks; 1:20 spacing (cond 7e4 of that system) 3.4e-11 /
# 1.6e-12.
ORACLE_TOL = dict(kappa=5e-12, err=1e-12)
ORACLE_TOL_1_20 = dict(kappa=3e-10, err=2e-11)
# from_slab on from_inputs' own vectors, max |diff| / max |ref| (Z) and / max |kappa_lin| (the curvatures): the slab
# splits the moments of P + alpha n into those of P and of alpha n, which long double rounds at 5e-20 of the
# coordinates; the curvature carries that as |P| / (h^2 kappa).  Measured: Z 0 (the same solve), curvatures 2.0e-16 on
# the golden tracks (|P| 200 m, h 3 m) and 2.9e-14 at 1:20 spacing (|P| 1.5e3 m, h 2.9 m, kappa 10x smaller).
LD_TOL = dict(z=1e-17, kappa=2e-15)
LD_TOL_1_20 = dict(z=1e-17, kappa=3e-13)
GOLDEN = ["handling", "synth128", "synth160_kappa", "synth200", "synth333", "synth333_kappa"]       # up to 350 points


def _closed(rt):
    return np.vstack((rt[:, :2], rt[:1, :2]))


def _h(rt):
    return np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1)


def _cases(golden):
    out = []
    for name in GOLDEN:
        g = golden(name)
        out.append((name, g["reftrack"], g["alpha_mincurv"], float(g["w_veh"])))
    rt = R.uneven_track(300, 20.0, 2)
    _, _, A, nv = T.calc_splines(_closed(rt))
    out.append(("spacing 1:20", rt, T.opt_min_curv(rt, nv, A, 10.0, 2.0)[0], 2.0))
    return out


@pytest.fixture(scope="module")
def cases(golden):
    return _cases(golden)


def _rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def test_from_inputs_matches_the_dense_oracle(cases):
    for name, rt, alpha, wv in cases:
        _, _, A, nv = T.calc_splines(_closed(rt))
        qp = T.assemble_min_curv(rt, nv, A, 10.0, wv)
        ref_k = qp["k_kappa_ref"] + qp["E_kappa"] @ alpha
        ref_e = T.curv_error_max_from(qp, alpha)
        r = F.from_inputs(rt, nv, _h(rt), alpha)
        ek = _rel(r["klin"], ref_k)
        ee = abs(float(r["emax"]) - ref_e) / max(ref_e, 1e-3 * float(r["kmax"]))
        tol = ORACLE_TOL_1_20 if "1:20" in name else ORACLE_TOL
        print(f"{name}: kappa_lin {ek:.1e} (bound {tol['kappa']:.0e}), curv_error_max {ee:.1e} (bound {tol['err']:.0e}), "
              f"curv_error_max {ref_e:.3e}")
        assert ek <= tol["kappa"] and ee <= tol["err"], name


@pytest.mark.parametrize("lin", [False, True])
def test_slab_replay_of_the_definition(cases, lin):
    """from_slab fed from_inputs' own slab vectors gives from_inputs' quantities to long-double rounding; the LIN
    branch recomputes the centre line's first derivatives from PX / MX."""
    for name, rt, alpha, _ in cases:
        _, _, _, nv = T.calc_splines(_closed(rt))
        la = 0.5 * alpha if lin else None
        d = F.from_inputs(rt, nv, _h(rt), alpha, lin_alpha=la)
        s = F.from_slab(d["slab"], alpha, lin=lin)
        scale = np.abs(d["klin"]).max()
        tol = LD_TOL_1_20 if "1:20" in name else LD_TOL
        ez = max(float(np.abs(s[k] - d[k]).max() / np.abs(d[k]).max()) for k in ("zx", "zy"))
        ek = max(float(np.abs(s[k] - d[k]).max() / scale) for k in ("klin", "c0", "c1", "err"))
        print(f"LIN {lin} {name}: Z {ez:.1e} (bound {tol['z']:.0e}), curvatures {ek:.1e} (bound {tol['kappa']:.0e})")
        assert ez <= tol["z"] and ek <= tol["kappa"], name


def test_error_vanishes_about_the_line_and_zero_lin_is_the_centre_line(cases):
    for name, rt, alpha, _ in cases[:3] + cases[-1:]:
        _, _, _, nv = T.calc_splines(_closed(rt))
        h = _h(rt)
        about = F.from_inputs(rt, nv, h, alpha, lin_alpha=alpha)
        e = float(about["emax"]) / float(about["kmax"])
        print(f"{name}: about the line, curv_error_max / kappa_lin_max {e:.1e}")
        assert e <= 1e-16
        s = F.from_slab(about["slab"], alpha, lin=True)
        assert float(s["emax"]) <= 1e-16 * float(s["kmax"])
        centre, zero = F.from_inputs(rt, nv, h, alpha), F.from_inputs(rt, nv, h, alpha, lin_alpha=np.zeros_like(alpha))
        for k in ("zx", "zy", "klin", "c1", "err"):
            assert np.array_equal(centre[k], zero[k]), (name, k)
        for k in F.SLAB_KEYS:
            assert np.array_equal(centre["slab"][k], zero["slab"][k]), (name, k)
        a, b = F.from_slab(zero["slab"], alpha, lin=True), F.from_slab(zero["slab"], alpha, lin=False)
        for k in ("klin", "c0", "c1", "err"):
            assert np.allclose(a[k], b[k], rtol=0, atol=1e-17 * float(b["kmax"])), (name, k)


@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", [0, 57, -1])
def test_non_finite_alpha_propagates_to_both_maxima(cases, bad, where):
    name, rt, alpha, _ = cases[-1]
    _, _, _, nv = T.calc_splines(_closed(rt))
    a = np.array(alpha)
    a[where] = bad
    d = F.from_inputs(rt, nv, _h(rt), a)
    s = F.from_slab(d["slab"], a)
    for r in (d, s):
        assert np.isnan(r["kmax"]) and np.isnan(r["emax"]), (name, bad, where)


KB = [0.1, 0.0, -0.0, -1.0, np.nan, np.inf, -np.inf, 5e-324, 1e300]
STATUSES = [0, 1, 2, 3, 4, -1]


def test_status_rules_on_every_pair():
    """The rules, pair by pair: 1 and negative statuses are skipped with zeros; with the per-instance limit one that is
    not finite or not > 0 turns a status >= 0 into -1 (1 included); 4 only from 0, by kmax > kb (1 + 1e-7) in float64;
    2, 3 and 4 keep their status and get values.  The scalar form never refuses a limit."""
    kmax = 0.05
    for st, kb, kbb in itertools.product(STATUSES, KB, (False, True)):
        got = F.status_after(st, kmax, kb, kbb)
        bad = not (kb > 0.0 and kb < np.inf)
        if kbb and bad and st >= 0:
            want = (-1, True)
        elif st == 1 or st < 0:
            want = (st, True)
        elif st == 0:
            want = (4 if kmax > kb * (1.0 + 1e-7) else 0, False)
        else:
            want = (st, False)
        assert got == want, (st, kb, kbb, got)
    # the threshold itself, in float64 and ulp by ulp
    kb = 0.1
    t = kb * (1.0 + 1e-7)
    assert F.status_after(0, t, kb) == (0, False)
    assert F.status_after(0, np.nextafter(t, 1.0), kb) == (4, False)
    assert F.status_after(0, np.nan, kb) == (0, False)
    assert F.status_after(0, np.inf, kb) == (4, False)
    for st in (2, 3, 4):
        assert F.status_after(st, 1.0, kb) == (st, False)
