"""CPU tests (-m "not gpu") of tests/iqp_ref.py, the reference of the re-linearisation step and of create_raceline's
stations, heading and curvature in tests/test_gpu_iqp_edges.py: against oracle/tph_dense.py (create_raceline,
calc_head_curv_an, interp_track_widths, calc_splines without distance scaling) on the golden tracks the dense oracle can
afford, and against the rl_* golden keys on every golden track."""
import numpy as np
import pytest

import iqp_ref as I
from oracle import tph_dense as T

SMALL = ["synth128", "synth160_kappa", "synth200", "handling", "synth333", "synth333_kappa"]      # <= 350 points
RL_GOLDEN = SMALL + ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "modena", "synth500", "synth500_narrow",
                     "synth1000", "synth2000"]
ROUND = 1e-12           # max|diff| / max(max|ref|, 1): what two orders of the same float64 sums leave


def _close(got, want, tol=ROUND):
    want = np.asarray(want, float)
    return float(np.abs(np.asarray(got, float) - want).max() / max(np.abs(want).max(), 1.0)) <= tol


@pytest.mark.parametrize("name", SMALL)
def test_create_raceline_and_head_curv_equal_the_dense_oracle(golden, name):
    g = golden(name)
    rt, nv, al = g["reftrack"], g["normvec"], g["alpha_mincurv"]
    for step in (1.0, 2.0, 3.0):
        r = I.create_raceline(rt[:, :2], nv, al, step)
        o = T.create_raceline(rt[:, :2], nv, al, step)
        assert r["no"] == o[4].size and np.array_equal(r["spline_inds"], o[4]), (name, step)
        for got, want in ((r["raceline"], o[0]), (r["coeffs_x"], o[2]), (r["coeffs_y"], o[3]), (r["t"], o[5]),
                          (r["s"], o[6]), (r["spline_lengths"], o[7]), (r["el"], o[8])):
            assert _close(got, want), (name, step)
        assert np.array_equal(r["spline_lengths"], T.calc_spline_lengths(r["coeffs_x"], r["coeffs_y"]))
        psi, kappa, dkappa = T.calc_head_curv_an(o[2], o[3], o[4], o[5], calc_curv=True, calc_dcurv=True)
        dpsi = np.abs(r["psi"] - psi)
        assert np.minimum(dpsi, 2.0 * np.pi - dpsi).max() <= ROUND
        assert _close(r["kappa"], kappa) and _close(r["dkappa"], dkappa)


@pytest.mark.parametrize("name", SMALL)
def test_relinearise_equals_the_oracle_widths_and_splines(golden, name):
    g = golden(name)
    rt, nv, al = g["reftrack"], g["normvec"], g["alpha_mincurv"]
    for step in (1.0, 3.0):
        r = I.relinearise(rt, nv, al, step)
        o = T.create_raceline(rt[:, :2], nv, al, step)
        w = rt[:, 2:] + np.column_stack((-al, al))
        w_o = T.interp_track_widths(w, o[4], o[5], incl_last_point=False)
        assert r["n"] == o[0].shape[0] == r["normvec"].shape[0]
        assert _close(r["reftrack"][:, :2], o[0]) and _close(r["reftrack"][:, 2:], w_o)
        _, _, _, nv_o = T.calc_splines(np.vstack((o[0], o[0][0])), use_dist_scaling=False)
        assert _close(r["normvec"], nv_o)
        # the last spline interpolates toward row 0: its stations carry widths between rows n - 1 and 0
        last = r["raceline"]["spline_inds"] == rt.shape[0] - 1
        if step == 1.0:
            t = r["raceline"]["t"][last]
            assert _close(r["reftrack"][last, 2:], w[-1] + (w[0] - w[-1]) * t[:, None])


@pytest.mark.parametrize("name", RL_GOLDEN)
def test_reference_reproduces_the_golden_raceline_keys(golden, name):
    g = golden(name)
    r = I.create_raceline(g["reftrack"][:, :2], g["normvec"], g["alpha_mincurv"], 2.0)
    assert np.array_equal(r["spline_inds"], g["rl_spline_inds"])
    for key, got in (("rl_raceline_interp", r["raceline"]), ("rl_coeffs_x", r["coeffs_x"]), ("rl_coeffs_y", r["coeffs_y"]),
                     ("rl_t_values", r["t"]), ("rl_s", r["s"]), ("rl_spline_lengths", r["spline_lengths"]),
                     ("rl_el_lengths", r["el"]), ("rl_kappa", r["kappa"])):
        assert _close(got, g[key]), (name, key)
    dpsi = np.abs(r["psi"] - g["rl_psi"])
    assert np.minimum(dpsi, 2.0 * np.pi - dpsi).max() <= ROUND
