"""CPU tests of tests/linalg_ref.py, the extended-precision reference that tests/test_gpu_linalg_edges.py holds the
device's factorisations and adjoint solves to: its refined solutions agree with mpmath, its backward error flags the
solutions of deliberately broken solvers, and a numpy model of the device's elimination order stays inside the GPU
bounds on the fixtures' H at the diagonals of a final interior-point iterate (this is where the bounds come from)."""
import numpy as np
import pytest
import scipy.linalg as sla

import linalg_ref as R
import qp_sens as Q

BROKEN_MIN = 100.0 * R.ETA_MAX       # a broken solver is flagged by orders of magnitude, not by a factor


def _band_spd(n, rng):
    """Cyclic H = R^T R, R cyclic banded (half-bandwidth 16): positive semidefinite, cyclic half-bandwidth 32."""
    Rm = np.zeros((n, n))
    for d in range(-16, 17):
        Rm[np.arange(n), (np.arange(n) + d) % n] = rng.standard_normal(n) * (0.6 ** abs(d))
    return Rm.T @ Rm


def _extreme_d(n, rng, frac=0.4):
    """D of a final iterate: about frac of the points active (1e12 .. 1e10), the rest 1e-12 .. 1e-10."""
    act = rng.random(n) < frac
    return np.where(act, 10.0 ** rng.uniform(10, 12, n), 10.0 ** rng.uniform(-12, -10, n)), act


def _band(M):
    """The device band rows of a cyclic M: hb[i][d] = M[i][(i + d) % n]."""
    n = M.shape[0]
    i = np.arange(n)
    return np.stack([M[i, (i + d) % n] for d in range(R.HBW + 1)], axis=1)


def cyc_solve(dg, off, dd, rhs, corner=True):
    """Python restatement of cyc_solve (csrc/shortest_path.cu): Thomas on T = M - u v^T, u = (gamma, 0, .., cN),
    v = (1, 0, .., cN / gamma), gamma = -M_00, then Sherman-Morrison; corner=False drops the corner term of v."""
    n = dg.size
    d0 = dg[0] + dd[0]
    gamma, cN = -d0, off[n - 1]
    c = cN / gamma if corner else 0.0
    cp, x, q = np.zeros(n), np.zeros(n), np.zeros(n)
    cpp = xp = qp = 0.0
    for i in range(n):
        offm = off[i - 1] if i > 0 else 0.0
        dgi = dg[i] + dd[i] - (gamma if i == 0 else 0.0) - (cN * cN / gamma if i == n - 1 else 0.0)
        mi = 1.0 / (dgi - offm * cpp)
        cp[i] = (off[i] if i < n - 1 else 0.0) * mi
        ui = gamma if i == 0 else (cN if i == n - 1 else 0.0)
        q[i] = qp = (ui - offm * qp) * mi
        x[i] = xp = (rhs[i] - offm * xp) * mi
        cpp = cp[i]
    for i in range(n - 2, -1, -1):
        x[i] -= cp[i] * x[i + 1]
        q[i] -= cp[i] * q[i + 1]
    return x - q * (x[0] + c * x[n - 1]) / (1.0 + q[0] + c * q[n - 1])


def test_dense_from_device_band_round_trips():
    rng = np.random.default_rng(0)
    for n in (80, 97, 143):
        H = _band_spd(n, rng)
        D = rng.uniform(0.1, 1.0, n)
        hb = np.zeros((n + 64, 34))
        hb[:n, :33] = _band(H)
        assert np.array_equal(R.dense_from_device_band(hb, n, D), H + np.diag(D))


@pytest.mark.parametrize("n", [80, 101, 143])
def test_refinement_agrees_with_mpmath(n):
    rng = np.random.default_rng(n)
    H = _band_spd(n, rng)
    D, _ = _extreme_d(n, rng)
    M = H + np.diag(D)
    g = rng.standard_normal(n)
    x = R.solve_extended(M, g)
    xm = R.solve_mpmath(M, g)
    fe = R.forward_error(M, x, xm)
    print(f"n={n}: cond(M) {np.linalg.cond(M):.1e}, cond(SMS) {R.cond_scaled(M):.1e}, refinement vs mpmath {fe:.1e}")
    assert fe <= 1e-16
    assert R.backward_error(M, np.asarray(x, dtype=np.float64), g) <= 2.0 * R.U


@pytest.mark.parametrize("n", [3, 4, 5, 9])
def test_refinement_agrees_with_mpmath_on_the_cyclic_tridiagonal(n):
    rng = np.random.default_rng(100 + n)
    nrm = rng.standard_normal((n, 2))
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    dg = 4.0 * np.ones(n)
    off = -2.0 * np.sum(nrm * np.roll(nrm, -1, axis=0), axis=1)
    dd, _ = _extreme_d(n, rng, 0.5)
    M = R.cyclic_tridiag(dg, off, dd)
    g = rng.standard_normal(n)
    assert R.forward_error(M, R.solve_extended(M, g), R.solve_mpmath(M, g)) <= 1e-16


def test_backward_error_flags_broken_band_solvers():
    """A dropped band entry and a diagonal shifted by one row, against the same solve done right."""
    rng = np.random.default_rng(7)
    n = 120
    H = _band_spd(n, rng)
    D, _ = _extreme_d(n, rng)
    M = H + np.diag(D)
    g = rng.standard_normal(n)
    assert R.backward_error(M, np.linalg.solve(M, g), g) <= R.ETA_MAX
    dropped = M.copy()
    dropped[40, 40 + 17] = dropped[40 + 17, 40] = 0.0
    shifted = H + np.diag(np.roll(D, 1))
    for what, Mb in (("dropped band entry", dropped), ("D shifted by one row", shifted)):
        eta = R.backward_error(M, np.linalg.solve(Mb, g), g)
        print(f"{what}: eta {eta:.1e}")
        assert eta >= BROKEN_MIN, what


def test_backward_error_flags_a_woodbury_correction_without_one_strong_row():
    """M = K + E_S^T W_S E_S solved by Woodbury with all strong rows and with one left out."""
    rng = np.random.default_rng(8)
    n, m = 150, 6
    K = _band_spd(n, rng) + np.diag(_extreme_d(n, rng)[0])
    E = np.zeros((m, n))
    for j, c in enumerate(rng.choice(n - 4, m, replace=False)):
        E[j, c:c + 3] = (1.0, -2.0, 1.0)                        # curvature-like rows
    W = 10.0 ** rng.uniform(0.5, 12, m)
    W[0] = 20.0                                                 # a row just above the split at W = 1
    M = R.with_strong_rows(K, E, W)
    g = rng.standard_normal(n)

    def woodbury(keep):
        Es, Ws = E[keep], W[keep]
        Kg, KE = np.linalg.solve(K, g), np.linalg.solve(K, Es.T)
        return Kg - KE @ np.linalg.solve(np.diag(1.0 / Ws) + Es @ KE, Es @ Kg)
    assert R.backward_error(M, woodbury(np.arange(m)), g) <= R.ETA_MAX
    eta = R.backward_error(M, woodbury(np.arange(1, m)), g)
    print(f"Woodbury without the row of weight {W[0]:.0f}: eta {eta:.1e}")
    assert eta >= BROKEN_MIN


@pytest.mark.parametrize("wmax", [1e3, 1e9, 1e15])
def test_rows_reference_agrees_with_mpmath_and_bounds_an_fp64_woodbury(wmax):
    """solve_extended_rows against mpmath on M = K + E_S^T W_S E_S with strong weights from just above 1 to wmax (the
    curvature-row phase ends with weights up to 1e15, where M is singular to fp64), and an fp64 Woodbury solve in the
    order of mincurv_adjoint_rows_kernel within fe_bound(cond(SMS) of K) / 8 of it, in the scaling of K."""
    rng = np.random.default_rng(int(np.log10(wmax)))
    n, m = 140, 8
    K = _band_spd(n, rng) + np.diag(_extreme_d(n, rng)[0])
    E = np.zeros((m, n))
    for j, c in enumerate(np.sort(rng.choice(n - 4, m, replace=False))):
        E[j, c:c + 3] = rng.uniform(0.5, 2.0) * np.array([1.0, -2.0, 1.0])
    W = 10.0 ** rng.uniform(0.0, np.log10(wmax), m)
    W[0] = 1.0 + 1e-9
    g = rng.standard_normal(n)
    x = R.solve_extended_rows(K, E, W, g)
    xm = R.solve_mpmath(K, g, rows=(E, W))
    c = R.cond_scaled(K)
    Kg, KE = np.linalg.solve(K, g), np.linalg.solve(K, E.T)
    Sg = np.diag(1.0 / W) + E @ KE
    v = Kg - KE @ sla.cho_solve(sla.cho_factor(Sg, lower=True), E @ Kg)
    fe = R.forward_error(K, v, x)
    print(f"W up to {wmax:.0e}: cond(SMS) of the dense M {R.cond_scaled(R.with_strong_rows(K, E, W)):.1e}, "
          f"cond(SMS) of K {c:.1e}, fp64 Woodbury forward {fe:.1e} = {fe / (R.U * c):.2f} u cond, "
          f"reference vs mpmath {R.forward_error(K, x, xm):.1e}")
    assert R.forward_error(K, x, xm) <= 1e-16
    assert fe <= R.fe_bound(c) / 8


@pytest.mark.parametrize("n", [3, 4, 5, 64])
def test_backward_error_flags_sherman_morrison_without_its_corner_term(n):
    """The restated cyc_solve is backward stable with point 0 active (gamma = -1e12) or not; without the corner term of
    v it is flagged wherever point n-1 is inactive.  Where it is active the corner's share of the scaled system,
    |cN| / sqrt(M_00 M_n-1n-1), is 1e-6 or less, and leaving it out costs no more than that."""
    rng = np.random.default_rng(9 + n)
    nrm = rng.standard_normal((n, 2))
    nrm /= np.linalg.norm(nrm, axis=1)[:, None]
    dg, off = 4.0 * np.ones(n), -2.0 * np.sum(nrm * np.roll(nrm, -1, axis=0), axis=1)
    g = rng.standard_normal(n)
    for d0, dn in ((1e12, 1e-12), (1e-12, 1e12), (1e-12, 1e-12), (1e12, 1e12)):
        dd = 10.0 ** rng.uniform(-12, 12, n)
        dd[0], dd[n - 1] = d0, dn
        M = R.cyclic_tridiag(dg, off, dd)
        assert R.backward_error(M, cyc_solve(dg, off, dd, g), g) <= R.ETA_MAX, (d0, dn)
        eta = R.backward_error(M, cyc_solve(dg, off, dd, g, corner=False), g)
        assert eta >= BROKEN_MIN or dn > 1.0, (d0, dn, eta)


MODEL_FIXTURES = ["synth128", "synth200", "synth333", "handling", "berlin500_jitter_a"]


@pytest.mark.parametrize("name", MODEL_FIXTURES)
def test_device_elimination_model_stays_inside_the_gpu_bounds(golden, name):
    """The fixture's H with D = 1e+-12, 1e+-10, 1e+-6 on the oracle's active set, and log-uniform 1e-12 .. 1e12, solved
    in the device's order: eta <= ETA_MAX / 8 and the scaled forward error against the refined solution
    <= FE_C u cond(SMS) / 8, so the GPU bounds leave a margin of eight over the model."""
    g = golden(name)
    H = Q.dense_from_band(g["H_band"])
    lb, ub, _ = Q.bounds(g["reftrack"], float(g["w_veh"]))
    au, al, _, _ = Q.active_set(H, g["f"], g["alpha_mincurv_boxonly"], lb, ub)
    n = H.shape[0]
    rng = np.random.default_rng(1)
    pats = {f"1e+-{e}": np.where(au | al, 10.0 ** e, 10.0 ** -e) for e in (12, 10, 6)}
    pats["log-uniform"] = 10.0 ** rng.uniform(-12, 12, n)
    for what, D in pats.items():
        M = H + np.diag(D)
        rhs = rng.standard_normal(n)
        x = R.device_model_solve(M, rhs)
        eta = R.backward_error(M, x, rhs)
        c = R.cond_scaled(M)
        fe = R.forward_error(M, x, R.solve_extended(M, rhs))
        print(f"{name} {what}: eta {eta:.1e}, cond(SMS) {c:.1e}, forward {fe:.1e} = {fe / (R.U * c):.2f} u cond")
        assert eta <= R.ETA_MAX / 8, (what, eta)
        assert fe <= R.fe_bound(c) / 8, (what, fe, c)
