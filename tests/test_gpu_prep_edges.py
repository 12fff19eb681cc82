"""GPU tests (-m gpu) of the prep_track kernel (csrc/prep_track.cu, DESIGN.md section 3.9) where it changes code path,
against the converged float64 reference tests/prep_ref.py:

A. the smoothing parameter: F(lam_kernel) from the reference equals s_reg (brackets that grow from lam = 1 and that
   shrink, s_reg from 1e-6 to just below F(inf));
B. the curve at the kernel's lam (not at the reference's root, so an error in the root cannot hide one in the fit):
   pre-interpolated n = 5..12 (the wrap terms of penta_cyclic_solve2), n across 256, n in the thousands; raw counts 5..300;
C. widths against converged closest points: the seam, duplicate raw points, a collinear run, a sharp asymmetric corner
   whose closest points lie up to 3.5 pre-interpolation steps from the chord-length guess, min_width below / at / above;
D. layout: ragged batches with NaN beyond n_raw[b]; one track alone, among others, with larger capacities and repeated
   more times than there are resident CTAs, bit for bit;
E. capacities (-needed, the wrapper's retry) and every refusal of the kernel, alone and in the middle of a batch whose
   other tracks come out bit for bit as without it, and the wrapper's messages.
Each bound is stated next to the H100 value it was set from (margin <= 10x)."""
import ctypes
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import prep_ref as R  # noqa: E402
from global_racetrajectory_optimization_b200 import _lib, batch as B_  # noqa: E402

REFUSED = B_.PREP_REFUSED
R_N_RAW, R_TOO_FEW, R_NONFINITE, R_COUNT, R_BUDGET, R_FEW_OUT = 1, 2, 3, 4, 5, 6


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def ngon(k, perim, seed, jit=0.05, w=(3.0, 3.0)):
    """A jittered k-gon of the given perimeter [m] with constant widths (unclosed raw track [k, 4])."""
    rng = np.random.default_rng(seed)
    a = np.linspace(0.0, 2.0 * np.pi, k, endpoint=False) + rng.uniform(-jit, jit, k) * 2.0 * np.pi / k
    r = 1.0 + rng.uniform(-jit, jit, k)
    p = np.column_stack((r * np.cos(a), r * np.sin(a)))
    p *= perim / np.sum(np.linalg.norm(np.roll(p, -1, axis=0) - p, axis=1))
    return np.column_stack((p, np.full(k, w[0]), np.full(k, w[1])))


def special_track():
    """Raw points for section C: a 12 m straight of collinear points along y = 0 (side 0), a duplicated point, a sharp
    asymmetric spike (out along a long edge, back along a short one) and varying widths; point 0 sits just after a
    corner so its closest curve point lies across the seam."""
    pts = [(0.0, 0.0), (4.0, 0.0), (8.0, 0.0), (8.0, 0.0), (12.0, 0.0), (20.0, 0.0), (30.0, 2.0), (40.0, 0.0),
           (50.0, 0.0), (52.0, 14.0), (56.0, 0.0), (70.0, 0.0), (75.0, 20.0), (60.0, 40.0), (30.0, 42.0), (5.0, 35.0),
           (-5.0, 18.0), (-3.0, 4.0)]
    p = np.asarray(pts)
    k = p.shape[0]
    w = 2.5 + 0.8 * np.sin(np.arange(k) * 1.7)
    return np.column_stack((p, w, 5.5 - w))


# Heavy smoothing (s_reg a large fraction of F(inf), lam >= 0.4): (R + lam Q^T Q) has a condition number of order
# lam / h^5, and the kernel's unpivoted bordered LDL^T and the reference's sparse LU part by ~1e-10 relative there.
HEAVY = ("n258_raw257_half", "n301_raw40_near_Finf")
# name -> (raw track, s_reg or ("f", fraction of F(inf)), stepsize_reg)
CASES = {
    "n5_raw5": (ngon(5, 4.6, 5), ("f", 0.1), 1.0),
    "n6_raw5": (ngon(5, 5.6, 5), ("f", 0.1), 1.0),
    "n7_raw6": (ngon(6, 6.6, 6), ("f", 0.1), 1.0),
    "n9_raw7": (ngon(7, 8.6, 7), ("f", 0.1), 1.0),
    "n12_raw8": (ngon(8, 11.6, 8), ("f", 0.1), 1.0),
    "n256_raw40": (ngon(40, 255.5, 40), 10.0, 3.0),
    "n257_raw256": (ngon(256, 256.5, 256), 1e-6, 3.0),
    "n258_raw257_half": (ngon(257, 257.5, 257), ("f", 0.5), 3.0),
    "n301_raw40_tiny_s": (ngon(40, 300.0, 41), 1e-6, 3.0),
    "n3001_raw300": (ngon(300, 3000.5, 300), 10.0, 3.0),
    "n301_raw40_near_Finf": (ngon(40, 300.0, 40), ("f", 0.999), 0.01),
    "special": (special_track(), 10.0, 1.0),
}


def s_of(case):
    tr, s, _ = CASES[case]
    return s[1] * R.system(tr).F_inf if isinstance(s, tuple) else float(s)


def capi(tracks, s_reg=10.0, stepsize_prep=1.0, stepsize_reg=3.0, min_width=0.0, n_raw=None, n_raw_max=None,
         n_int_max=4000, n_out_max=1500, fill=np.nan):
    """One direct mc_prep_track_batch call; rows beyond n_raw[b] hold `fill`.  Returns (out, n_out, lam) on the host."""
    lib = _lib.load()
    B = len(tracks)
    counts = [t.shape[0] for t in tracks] if n_raw is None else list(n_raw)
    n_raw_max = n_raw_max or max(t.shape[0] for t in tracks)
    arr = np.full((B, n_raw_max, 4), fill)
    for b, t in enumerate(tracks):
        arr[b, :min(t.shape[0], n_raw_max)] = t[:n_raw_max]
    track = torch.tensor(arr, device="cuda")
    nr = torch.tensor(counts, dtype=torch.int32, device="cuda")
    out = torch.full((B, n_out_max, 4), -7.0, dtype=torch.float64, device="cuda")
    n_out = torch.zeros((B,), dtype=torch.int32, device="cuda")
    lam = torch.full((B,), -1.0, dtype=torch.float64, device="cuda")
    nb = lib.mc_prep_track_workspace_bytes(B, n_raw_max, n_int_max)
    ws = torch.empty((nb,), dtype=torch.uint8, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    rc = lib.mc_prep_track_batch(B, n_raw_max, p(nr), p(track), 3, float(s_reg), float(stepsize_prep), float(stepsize_reg),
                                 float(min_width), int(n_int_max), int(n_out_max), p(out), p(n_out), p(lam), p(ws), nb, None)
    assert rc == 0
    torch.cuda.synchronize()
    return out.cpu().numpy(), n_out.cpu().numpy(), lam.cpu().numpy()


_RUNS = {}


def run(case, min_width=None):
    """The wrapper on one case, and the reference evaluated at the kernel's lam (cached)."""
    key = (case, min_width)
    if key not in _RUNS:
        tr, _, sr = CASES[case]
        s = s_of(case)
        out, n_out, lam = B_.spline_approximation_batch(torch.tensor(tr[None], device="cuda"), s_reg=s, stepsize_reg=sr,
                                                        min_width=min_width)
        sys_ = R.system(tr)
        ref = R.outputs(sys_, float(lam[0]), sr, min_width)
        _RUNS[key] = (out[0, :int(n_out[0])].cpu().numpy(), int(n_out[0]), float(lam[0]), ref, sys_, s)
    return _RUNS[key]


# ---------------------------------------------------------------------------------------------------------------------
# A. the smoothing parameter
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_A_residual_at_the_kernels_lambda_is_the_budget(case):
    got, n, lam, ref, sys_, s = run(case)
    rel = abs(ref.F - s) / s
    print(f"A {case}: n = {sys_.n}, s = {s:.4g}, F(inf) = {sys_.F_inf:.4g}, lam = {lam:.6g}, F(1) = {R.F(sys_, 1.0):.4g}, "
          f"|F(lam_kernel) - s| / s = {rel:.2e}")
    assert rel <= (1e-8 if case in HEAVY else 3e-13)  # H100: <= 3.4e-14 (n3001_raw300); heavy smoothing <= 1.8e-9


def test_A_brackets_grow_and_shrink_from_one():
    """F(1) < s (the bracket grows) and F(1) > s (it shrinks) both occur among the cases."""
    above = [c for c in CASES if R.F(R.system(CASES[c][0]), 1.0) > s_of(c)]
    below = [c for c in CASES if R.F(R.system(CASES[c][0]), 1.0) < s_of(c)]
    assert above and below


# ---------------------------------------------------------------------------------------------------------------------
# B. the curve at the kernel's lam
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_B_resampled_curve_at_the_kernels_lambda(case):
    got, n, lam, ref, sys_, s = run(case)
    assert n == ref.n_reg
    scale = float(np.abs(sys_.pts).max())
    err = float(np.abs(got[:, :2] - ref.out[:, :2]).max()) / scale
    print(f"B {case}: n_pre = {sys_.n}, n_raw = {sys_.track.shape[0]}, n_out = {n}, max |xy - ref| / max |p| = {err:.2e}")
    assert err <= (1e-8 if case in HEAVY else 1e-13)  # H100: <= 1.2e-14 (n3001_raw300); heavy smoothing <= 2.0e-9


# ---------------------------------------------------------------------------------------------------------------------
# C. widths against converged closest points
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(CASES))
def test_C_widths_against_converged_closest_points(case):
    got, n, lam, ref, sys_, s = run(case)
    if ref.resid.max() > 1e-9:          # (a closest point at the window's edge: the kernel's search is local, like tph's)
        pytest.skip(f"closest point outside the +-4 step window (residual {ref.resid.max():.1e} m)")
    err = float(np.abs(got[:, 2:] - ref.out[:, 2:]).max())
    print(f"C {case}: max |w - ref| = {err:.2e} m, max stationarity residual of the reference {ref.resid.max():.1e} m")
    assert err <= (2e-4 if case in HEAVY else 7e-12)   # [m] H100: <= 7.5e-13 (n3001_raw300); heavy smoothing <= 4.0e-5


def test_C_special_track_reaches_the_edges_it_is_for():
    got, n, lam, ref, sys_, s = run("special")
    assert ref.t_close[0] < 0.0 or ref.t_close[-1] > 1.0              # across the seam
    assert np.any(ref.sides == 0.0)                                  # on the collinear run
    assert ref.resid.max() <= 1e-9
    far = run("n258_raw257_half")
    steps = (far[3].t_close - far[4].dists_cl / far[4].L_raw) * far[4].L_raw
    assert np.abs(steps).max() > 1.5 and far[3].resid.max() <= 1e-9  # beyond +-1 pre-interpolation step, inside +-4


@pytest.mark.parametrize("where", ["below", "at", "between", "above"])
def test_C_min_width(where):
    got, n, lam, ref, sys_, s = run("special")
    sums = got[:, 2] + got[:, 3]
    mw = {"below": 0.5 * sums.min(), "at": float(sums.min()), "between": 0.5 * (sums.min() + sums.max()),
          "above": 2.0 * sums.max()}[where]
    g2, n2, lam2, ref2, _, _ = run("special", min_width=mw)
    assert n2 == n and lam2 == lam
    err = float(np.abs(g2[:, 2:] - ref2.out[:, 2:]).max())
    print(f"C min_width {where} ({mw:.6g} m): max |w - ref| = {err:.2e} m")
    assert err <= 4e-13 and (g2[:, 2] + g2[:, 3]).min() >= mw - 1e-12   # [m] H100: 4.1e-14
    if where in ("below", "at"):
        assert np.array_equal(g2, got)


# ---------------------------------------------------------------------------------------------------------------------
# D. layout
# ---------------------------------------------------------------------------------------------------------------------
LAYOUT = ["n12_raw8", "special", "n257_raw256", "n256_raw40", "n3001_raw300"]


def test_D_ragged_batch_with_nan_beyond_each_track_is_bitwise_its_single_runs():
    trs = [CASES[c][0] for c in LAYOUT]
    kw = dict(stepsize_reg=1.0, n_out_max=4000)                     # (n12_raw8 keeps 3 points or more at 1 m)
    single = [capi([t], **kw) for t in trs]
    out, n_out, lam = capi(trs, **kw)
    for b, (o1, n1, l1) in enumerate(single):
        assert n_out[b] == n1[0] > 0 and lam[b] == l1[0]
        assert np.array_equal(out[b, :n1[0]], o1[0, :n1[0]])
        assert np.all(out[b, n1[0]:] == 0.0)


def test_D_one_track_repeated_beyond_the_resident_ctas_with_larger_capacities():
    tr = CASES["special"][0]
    o1, n1, l1 = capi([tr])
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    reps = 2 * sms + 3                                               # one 256-thread CTA of 244 registers per SM
    others = [CASES[c][0] for c in LAYOUT]
    batch = [tr if b % 3 == 0 else others[b % len(others)] for b in range(reps)]
    out, n_out, lam = capi(batch, n_raw_max=700, n_int_max=5000, n_out_max=2000)
    for b in range(0, reps, 3):
        assert n_out[b] == n1[0] and lam[b] == l1[0] and np.array_equal(out[b, :n1[0]], o1[0, :n1[0]])


# ---------------------------------------------------------------------------------------------------------------------
# E. capacities and refusals
# ---------------------------------------------------------------------------------------------------------------------
def test_E_capacity_codes_are_the_counts_needed():
    tr = CASES["n256_raw40"][0]
    sys_ = R.system(tr)
    ref = run("n256_raw40")[3]
    _, n_out, _ = capi([tr], n_int_max=sys_.n)                       # one short of n + 1 (the closed point set)
    assert n_out[0] == -(sys_.n + 1)
    _, n_out, _ = capi([tr], n_out_max=ref.n_reg - 1)
    assert n_out[0] == -ref.n_reg
    _, n_out, _ = capi([tr], n_int_max=sys_.n + 1, n_out_max=ref.n_reg)
    assert n_out[0] == ref.n_reg


def test_E_wrapper_retries_a_capacity_to_the_same_result(monkeypatch):
    tr = CASES["n3001_raw300"][0]
    want = run("n3001_raw300")
    real = B_._closed_polygon_length
    monkeypatch.setattr(B_, "_closed_polygon_length", lambda *a, **k: real(*a, **k) * 0.25)   # both capacities too small
    out, n_out, lam = B_.spline_approximation_batch(torch.tensor(tr[None], device="cuda"), s_reg=10.0, stepsize_reg=3.0)
    assert int(n_out[0]) == want[1] and float(lam[0]) == want[2]
    assert np.array_equal(out[0, :want[1]].cpu().numpy(), want[0])


def _bad_cases():
    """name -> (tracks list for capi with the bad one in the middle, n_raw override, s_reg, stepsize_reg, reason)."""
    good = ngon(40, 255.5, 40)
    hexa = ngon(6, 5.5, 6)                                      # n = 6, a curve shorter than 6 m
    tiny = ngon(6, 6.0, 11, w=(1.0, 1.0)) * np.array([1.0 / 6.0, 1.0 / 6.0, 1.0, 1.0])   # 1 m: n < 5
    inf_pt, nan_pt, nan_w, huge, far = good.copy(), good.copy(), good.copy(), good.copy(), good.copy()
    inf_pt[7, 0] = np.inf
    nan_pt[3, 1] = np.nan
    nan_w[12, 3] = np.nan
    huge[:, :2] *= 1e306                                        # finite points, infinite length
    far[:, :2] *= 1e12                                          # finite length, count above 2^30
    small = ngon(6, 6.0 * 2 * np.pi / 6 * 1.05, 3)             # F(inf) ~ 6: s_reg = 10 cannot be reached
    return {
        "n_raw_above_max": (good, {"n_raw": 41}, 10.0, 3.0, R_N_RAW),
        "n_raw_negative": (good, {"n_raw": -3}, 10.0, 3.0, R_N_RAW),
        "n_raw_4": (good, {"n_raw": 4}, 10.0, 3.0, R_TOO_FEW),
        "n_pre_below_5": (tiny, {}, 1e-6, 0.1, R_TOO_FEW),
        "inf_coordinate": (inf_pt, {}, 10.0, 3.0, R_NONFINITE),
        "nan_coordinate": (nan_pt, {}, 10.0, 3.0, R_NONFINITE),
        "nan_width": (nan_w, {}, 10.0, 3.0, R_NONFINITE),
        "length_overflow": (huge, {}, 10.0, 3.0, R_NONFINITE),
        "count_above_2_30": (far, {}, 10.0, 3.0, R_COUNT),
        "budget_above_F_inf": (small, {}, 10.0, 3.0, R_BUDGET),
        "resampled_below_3": (hexa, {}, 1e-3, 3.0, R_FEW_OUT),
    }


@pytest.mark.parametrize("name", list(_bad_cases()))
def test_E_refusal_alone_and_in_the_middle_of_a_batch(name):
    bad, over, s_reg, sr, reason = _bad_cases()[name]
    cap = dict(n_int_max=4000, n_out_max=4000)
    left, right = ngon(40, 255.5, 40), ngon(257, 257.5, 257)
    n_raw_max = 300
    nr_bad = over.get("n_raw", bad.shape[0])
    if nr_bad > bad.shape[0]:
        n_raw_max = bad.shape[0]                                # the row holds bad.shape[0] points, n_raw asks for more
        left, right = left[:n_raw_max], right[:n_raw_max]
    _, n_alone, _ = capi([bad], s_reg=s_reg, stepsize_reg=sr, n_raw=[nr_bad], n_raw_max=n_raw_max, **cap)
    assert n_alone[0] == -REFUSED - reason
    out, n_out, lam = capi([left, bad, right], s_reg=s_reg, stepsize_reg=sr,
                           n_raw=[left.shape[0], nr_bad, right.shape[0]], n_raw_max=n_raw_max, **cap)
    assert n_out[1] == -REFUSED - reason
    assert np.all(out[1] == -7.0)                               # nothing written to the refused row
    for b, t in ((0, left), (2, right)):
        o1, n1, l1 = capi([t], s_reg=s_reg, stepsize_reg=sr, n_raw_max=n_raw_max, **cap)
        assert n_out[b] == n1[0] > 0 and lam[b] == l1[0] and np.array_equal(out[b], o1[0])


def test_E_inactive_slot_stays_silent():
    good = ngon(40, 255.5, 40)
    out, n_out, lam = capi([good, good], n_raw=[40, 0])
    assert n_out[1] == 0 and lam[1] == 0.0 and n_out[0] > 0


@pytest.mark.parametrize("name,match", [
    ("n_raw_above_max", r"track 1 is refused: n_raw = 41 is outside \[0, 40\]"),
    ("n_raw_negative", r"track 1 is refused: n_raw = -3 is outside"),
    ("n_raw_4", r"track 1 is refused: 4 raw points, fewer than 5"),
    ("n_pre_below_5", r"track 1 is refused: fewer than 5 points"),
    ("inf_coordinate", r"track 1 is refused: a non-finite coordinate"),
    ("nan_width", r"track 1 is refused: a non-finite coordinate"),
    ("length_overflow", r"track 1 is refused: a non-finite coordinate"),
    ("count_above_2_30", r"track 1 is refused: a point count"),
    ("budget_above_F_inf", r"track 1 is refused: the residual budget s_reg is not reached"),
    ("resampled_below_3", r"track 1 is refused: fewer than 3 re-sampled points"),
])
def test_E_wrapper_messages(name, match):
    bad, over, s_reg, sr, reason = _bad_cases()[name]
    good = ngon(40, 255.5, 40)
    nr = over.get("n_raw", bad.shape[0])
    arr = np.full((2, max(40, bad.shape[0]), 4), np.nan)
    arr[0, :40], arr[1, :bad.shape[0]] = good, bad
    with pytest.raises(ValueError, match=match):
        B_.spline_approximation_batch(torch.tensor(arr, device="cuda"), s_reg=s_reg, stepsize_reg=sr,
                                      n_raw=torch.tensor([40, nr], dtype=torch.int32))
