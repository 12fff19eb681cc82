"""CPU tests (-m "not gpu") of the exact shortest-path reference (tests/sp_ref.py) that the device edge tests rely on: its
assembly against the dense oracle, its solutions against the oracle's Goldfarb-Idnani solves, and its certificate on
exact and on perturbed solutions."""
import numpy as np
import pytest

import sp_ref as R
import sp_sens as S
from oracle import tph_dense as T
from global_racetrajectory_optimization_b200 import synth

FIXTURES = ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth1000", "synth128",
            "synth160_kappa", "synth200", "synth2000", "synth333", "synth333_kappa", "synth500", "synth500_narrow"]
SMALL = (3, 4, 5)
H_TOL = 2e-15           # |H - H_tph|: tph squares with **, one ulp of 4 (4.4e-16) measured on two points of synth1000
F_TOL = 4e-15           # f summed in another order than tph's, relative to max|x, y| (it cancels): 9.0e-16 measured
SOLVE_TOL = 5e-11       # max|alpha - alpha_GI| [m]: 5.0e-12 measured (synth2000), 2.5e-12 in the interior regime
CERT_TOL = dict(pg=2e-13, stat=3e-13)      # at the exact solutions: pg 1.4e-14 m, stat 2.7e-14 measured
DELTA = 1e-6


def _normals(rt):
    return T.calc_splines(np.vstack((rt[:, :2], rt[:1, :2])))[3]


def _tracks(golden):
    """name -> (reftrack, normvec, w_veh): the fixtures, perturbed polygons of 3, 4 and 5 points and the box regimes."""
    out = {nm: (golden(nm)["reftrack"], golden(nm)["normvec"], float(golden(nm)["w_veh"])) for nm in FIXTURES}
    for n in SMALL:
        rt = R.polygon_track(n, 100 + n)
        out[f"polygon{n}"] = (rt, _normals(rt), 2.0)
    rt = synth.make_track(7, 400)
    nv = _normals(rt)
    for name, r, wv in R.box_variants(rt):
        out[name] = (r, nv, wv)
    return out


def _dense(diag, off):
    return R.matrix(diag, off).toarray()


def test_assemble_matches_the_dense_oracle_in_one_ragged_batch(golden):
    tr = _tracks(golden)
    names = FIXTURES + [f"polygon{n}" for n in SMALL]
    n = [tr[nm][0].shape[0] for nm in names]
    rt, nv = np.full((len(names), max(n) + 3, 4), np.nan), np.full((len(names), max(n) + 3, 2), np.nan)
    for b, nm in enumerate(names):
        rt[b, :n[b]], nv[b, :n[b]] = tr[nm][0], tr[nm][1]
    wv = np.array([tr[nm][2] for nm in names])
    diag, off, f, lb, ub = R.assemble(rt, nv, wv, n_pts=n)
    for b, nm in enumerate(names):
        m = n[b]
        qp = T.assemble_shortest_path(*tr[nm])
        assert np.abs(_dense(diag[b, :m], off[b, :m]) - qp["H"]).max() <= H_TOL, nm
        assert np.abs(f[b, :m] - qp["f"]).max() <= F_TOL * np.abs(tr[nm][0][:, :2]).max(), nm
        assert np.array_equal(ub[b, :m], qp["h"][:m]) and np.array_equal(-lb[b, :m], qp["h"][m:]), nm
        pad = slice(m, None)
        assert (diag[b, pad] == 1).all() and not off[b, pad].any() and not f[b, pad].any(), nm
        assert not lb[b, pad].any() and not ub[b, pad].any(), nm
    # a single track gives the same arrays without the batch axis
    one = R.assemble(*tr["synth128"])
    for x, y in zip(one, (diag, off, f, lb, ub)):
        assert np.array_equal(x, y[names.index("synth128"), :128])


def test_rows_the_kernel_does_not_solve_assemble_as_padding():
    rt = np.stack([R.polygon_track(5, 1)] * 4)
    nv = np.stack([_normals(rt[0])] * 4)
    diag, off, f, lb, ub = R.assemble(rt, nv, 2.0, n_pts=[5, 2, 6, -1])
    assert (diag[1:] == 1).all() and not f[1:].any() and not off[1:].any() and not ub[1:].any() and not lb[1:].any()
    assert np.array_equal(f[0], R.assemble(rt[0], nv[0], 2.0)[2])


def test_solve_exact_matches_goldfarb_idnani_on_every_regime(golden):
    worst = {}
    for nm, (rt, nv, wv) in _tracks(golden).items():
        a = R.solve_exact(*R.assemble(rt, nv, wv))
        worst[nm] = float(np.abs(a - S.solve(rt, nv, wv)).max())
    assert max(worst.values()) <= SOLVE_TOL, worst


def test_the_box_regimes_are_what_their_names_say(golden):
    tr = _tracks(golden)
    n = 400
    act = {}
    for nm in ("both_clamped", "right_clamped", "interior", "tight", "w_veh_2.6"):
        q = R.assemble(*tr[nm])
        a = R.solve_exact(*q)
        act[nm] = R.certificate(*q, a)["active"]
        if nm == "both_clamped":
            assert (q[4] == R.CLAMP).all() and (q[3] == -R.CLAMP).all() and np.abs(a).max() <= R.CLAMP
        if nm == "right_clamped":
            assert (q[4] == R.CLAMP).all() and (q[3] < -0.5).all()
        if nm == "interior":
            H = _dense(q[0], q[1])
            assert np.abs(a - np.linalg.solve(H, -q[2])).max() <= 1e-10 * np.abs(a).max()
    assert act["interior"] == 0 and act["tight"] > n // 2 and act["both_clamped"] > n // 2, act
    assert 0 < act["right_clamped"] < n and 0 < act["w_veh_2.6"] < n, act


def test_small_tracks_without_an_m_matrix_are_solved():
    # consecutive normals of a triangle point more than 90 degrees apart: H has positive off-diagonal entries
    rt = R.polygon_track(3, 103)
    nv = _normals(rt)
    q = R.assemble(rt, nv, 2.0)
    assert (q[1] > 0).any()
    assert np.abs(R.solve_exact(*q) - S.solve(rt, nv, 2.0)).max() <= SOLVE_TOL


def test_solve_exact_refuses_non_finite_input():
    q = list(R.assemble(R.polygon_track(8, 3), _normals(R.polygon_track(8, 3)), 2.0))
    q[2] = q[2].copy()
    q[2][4] = np.nan
    with pytest.raises(ValueError):
        R.solve_exact(*q)


def test_certificate_is_at_rounding_level_on_exact_solutions(golden):
    for nm, (rt, nv, wv) in _tracks(golden).items():
        q = R.assemble(rt, nv, wv)
        c = R.certificate(*q, R.solve_exact(*q))
        assert c["box"] == 0.0 and c["comp"] == 0.0, (nm, c)
        assert c["pg"] <= CERT_TOL["pg"] and c["stat"] <= CERT_TOL["stat"], (nm, c)


def test_certificate_of_a_ragged_batch_equals_that_of_each_instance(golden):
    names = ["synth128", "handling", "berlin"]
    n = [golden(nm)["reftrack"].shape[0] for nm in names]
    rt, nv, a = np.full((3, max(n) + 5, 4), np.nan), np.full((3, max(n) + 5, 2), np.nan), np.full((3, max(n) + 5), np.nan)
    ones = []
    for b, nm in enumerate(names):
        g = golden(nm)
        rt[b, :n[b]], nv[b, :n[b]], a[b, :n[b]] = g["reftrack"], g["normvec"], g["alpha_shpath"]
        ones.append(R.certificate(*R.assemble(g["reftrack"], g["normvec"], float(g["w_veh"])), g["alpha_shpath"]))
    wv = np.array([float(golden(nm)["w_veh"]) for nm in names])
    c = R.certificate(*R.assemble(rt, nv, wv, n_pts=n), a, n_pts=n)
    for b in range(3):
        for k in ones[b]:
            assert c[k][b] == ones[b][k], (names[b], k)


def test_certificate_sees_a_free_point_moved_by_a_micrometre(golden):
    q = R.assemble(*_tracks(golden)["synth500"])
    a = R.solve_exact(*q)
    free = np.flatnonzero((a > q[3] + 0.01) & (a < q[4] - 0.01))
    for j in free[:: max(1, free.size // 5)]:
        b = a.copy()
        b[j] += DELTA
        c = R.certificate(*q, b)
        assert 0.9 * DELTA <= c["pg"] <= 1.1 * DELTA and c["box"] == 0.0, (j, c)
        assert c["stat"] * np.abs(q[2]).max() >= 0.9 * q[0][j] * DELTA, (j, c)


def test_certificate_sees_a_micrometre_past_a_bound(golden):
    q = R.assemble(*_tracks(golden)["synth500"])
    a = R.solve_exact(*q)
    for j, sign in ((int(np.flatnonzero(a == q[4])[0]), 1.0), (int(np.flatnonzero(a == q[3])[0]), -1.0)):
        b = a.copy()
        b[j] += sign * DELTA
        c = R.certificate(*q, b)
        assert 0.99 * DELTA <= c["box"] <= 1.01 * DELTA and 0.99 * DELTA <= c["pg"] <= 1.01 * DELTA, (j, c)
