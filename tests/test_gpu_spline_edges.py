"""GPU tests (-m gpu) of the closed-spline kernels (csrc/splines.cu: calc_splines_kernel, create_raceline_kernel,
head_curv_kernel, create_raceline_adjoint_kernel) where they change code path, against the long-double reference
tests/spline_ref.py:

A  the three moment solves of closed_spline: PCR with four and eight points per thread (n <= 1024, n <= 2048) and the
   chunked recurrences above (TRI_CHUNK 8, TRI_WARM 56) at their boundaries, a partial last chunk (2056, 2057) and
   thread 0 running two or three chunks (4096, 4097); unit scales (five PCR steps) and distance scales (six), given and
   computed; xy strides 2 and 4; normals only; h_out;
B  tiny tracks where the PCR stride wraps (s % n == 0 for n = 4, 8, 16 and, on the scaled path, 32; i - s == i + s
   mod n where 2 s == 0 mod n): n = 3 .. 9, 15 .. 17, 31 .. 33;
C  scratch placement: n_max 3488 (shared memory) against 3489 (global memory), bit for bit, for calc_splines,
   create_raceline and the adjoint;
D  adversarial spacing on the scaled path: 1:20, 1:1000 and runs of geometrically shrinking segments (a_i -> 1/2);
E  create_raceline's stations: the segment search against numpy on the device's own lengths, the station count,
   stations on knots, segments without stations, stations on segment 0, the overflow code and the zero padding;
F  head_curv: psi at the wrap of normalize_psi (tangent along -y), kappa and dkappa, padding;
G  the create_raceline adjoint against autograd of tests/raceline_ref.py (float64 dense) on tracks of A - E;
H  batch independence: a ragged batch padded with NaN gives each track's bits when it runs alone.

Coefficient errors are max |device - reference| relative to the track's scale: max |P| for the coefficients of order 0
and 1 (both are differences of points), the largest reference coefficient of that order for orders 2 and 3.  Every
bound was measured on an H100 80GB HBM3, set at about ten times the measurement, and is printed next to the value
measured (pytest -s)."""
import math

import numpy as np
import pytest

import mincurv_ref as MR
import raceline_ref as RR
import spline_ref as S

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402

DEV = "cuda"
THREADS = 256                       # the CTA size of every spline kernel
SMEM_LIMIT = 220 * 1024             # SPL_SMEM_LIMIT
# Bounds on the errors of the module docstring, about ten times the largest value measured on an H100 80GB HBM3.
# Coefficients: unit scales 7.5e-15 (A), tiny tracks 7.6e-15 (B), scratch placement 3.0e-14 (C), el_lengths given
# 4.5e-13 (A), chords 1.2e-10 (A), adversarial spacing 9.5e-13 (D).  The scaled bounds above 1e-12 are the conditioning
# of the inputs, not the solve: on uneven_track(4097, 1:20) the coordinates reach 2.1e4 m (ulp 3.6e-12 m) while the
# largest cubic coefficient is ~1e-2 m, so the second differences of the right-hand side round at ~1e-10 of it; a
# float64 sparse LU solve of the same system is 1.2e-10 from the long-double reference there, and rounding the chords to
# float64 (h_out) alone moves the long-double result by 8.6e-11.
COEF_TOL = dict(unit=1e-13, tiny=1e-13, scratch=3e-13, el=5e-12, chords=1e-9, spacing=1e-11)
NORMVEC_TOL = 5e-15                 # unit normals, absolute: 5.0e-16
H_TOL = 2e-15                       # computed chords relative to themselves (one sqrt): 1.7e-16
# Stations: points 1.2e-14, s 6.7e-15, el 1.2e-15, spline lengths 9.3e-14 of the track's scale; u = j + t 5.5e-12,
# kappa 3.2e-11 relative, psi 7.0e-12 rad.  u, kappa and psi are those of the 700-point 1:20 lap (22 km, 0.3 m
# segments): the station distances and CUM are float64 sums of 22 km (ulp 3.6e-12 m), and t = (dist - CUM[j-1]) / sl[j]
# turns that into 1.2e-11 on a 0.3 m segment; every other lap is below 1e-12.
STATION_TOL = dict(points=1e-13, s=1e-13, el=1e-14, lengths=1e-12, u=6e-11, kappa=3e-10, psi=7e-11)
HEAD_TOL = dict(psi=7e-15, kappa=4e-16, dkappa=3e-15)      # measured 7.1e-16 rad, 4.1e-17, 3.1e-16
# the adjoint: 9.4e-12 (n = 2049), the sum over thousands of stations of terms that hold t, n_out and the segments fixed
ADJ_TOL = 1e-10                     # |device - autograd| / max |autograd| per gradient


def report(what, measured, bound):
    print(f"  {what}: measured {measured:.3e}, bound {bound:.0e}")
    assert measured <= bound, what


def t_(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def pack(arrs, n_max, pad=0.0):
    """[B, n_max, ...] of the arrays arrs (first axis n_b), padded with pad."""
    out = np.full((len(arrs), n_max) + np.shape(arrs[0])[1:], pad)
    for b, a in enumerate(arrs):
        out[b, :len(a)] = a
    return out


def smem_bytes(n_max):
    """spline_smem_bytes: eight vectors of ceil32(n_max) + 32 doubles."""
    return 8 * ((n_max + 31) // 32 * 32 + 32) * 8


# ---- tracks ------------------------------------------------------------------------------------------------------------
def with_widths(xy):
    return np.column_stack((xy[:, :2], np.full(len(xy), 3.0), np.full(len(xy), 3.0)))


def blob(n, seed, R=50.0):
    """A star-shaped closed track of n points at jittered angles."""
    rng = np.random.default_rng(seed)
    th = 2.0 * np.pi * (np.arange(n) + 0.4 * rng.uniform(-1.0, 1.0, n)) / n
    r = R * (1.0 + 0.15 * np.cos(2.0 * th + rng.uniform(0.0, 2.0 * np.pi)))
    return with_widths(np.column_stack((r * np.cos(th), r * np.sin(th))))


def geometric_track(n, q, run, R=200.0):
    """Points on a smooth closed curve whose steps shrink geometrically by q over runs of `run` steps: spacing ratio
    q^-(run - 1) inside a run, and the same jump back to the longest step after it."""
    d = q ** (np.arange(n) % run)
    th = np.concatenate(([0.0], np.cumsum(d)[:-1])) / d.sum() * 2.0 * np.pi
    r = R * (1.0 + 0.05 * np.cos(3.0 * th))
    return with_widths(np.column_stack((r * np.cos(th), r * np.sin(th))))


def polygon(n, R):
    th = 2.0 * np.pi * np.arange(n) / n
    return with_widths(np.column_stack((R * np.cos(th), R * np.sin(th))))


def alpha_of(n, seed):
    rng = np.random.default_rng(seed)
    return 0.3 * np.sin(np.linspace(0.0, 6.0 * np.pi, n, endpoint=False)) + 0.05 * rng.standard_normal(n)


# ---- runs ----------------------------------------------------------------------------------------------------------------
def splines(tracks, n_max, ds, el=None, stride=4, want_coeffs=True, pad=0.0):
    """calc_splines_batch on a ragged batch: per track dict(cx, cy, nv, h) as numpy [:n]."""
    n = [len(t) for t in tracks]
    xy = t_(pack([t[:, :stride] for t in tracks], n_max, pad))
    elt = None if el is None else t_(pack(el, n_max, pad))
    cx, cy, nv, h = B_.calc_splines_batch(xy, n_pts=t_(n, torch.int32), el_lengths=elt, use_dist_scaling=ds,
                                          want_coeffs=want_coeffs)
    out = []
    for b, m in enumerate(n):
        out.append(dict(nv=nv[b, :m].cpu().numpy(), h=h[b, :m].cpu().numpy(),
                        cx=None if cx is None else cx[b, :m].cpu().numpy(),
                        cy=None if cy is None else cy[b, :m].cpu().numpy()))
    return out


def coef_err(cx, cy, rcx, rcy):
    """max over orders of the coefficient error relative to the track's scale (module docstring)."""
    e = []
    for k in range(4):
        d = max(np.abs(np.asarray(cx[:, k], dtype=S.LD) - rcx[:, k]).max(),
                np.abs(np.asarray(cy[:, k], dtype=S.LD) - rcy[:, k]).max())
        k_ = 0 if k < 2 else k
        scale = max(np.abs(rcx[:, k_]).max(), np.abs(rcy[:, k_]).max())
        e.append(float(d / scale))
    return max(e)


def spline_errors(got, track, ds, el=None):
    rcx, rcy, rnv, rh = S.calc_splines(track, el, ds)
    return coef_err(got["cx"], got["cy"], rcx, rcy), float(np.abs(np.asarray(got["nv"], dtype=S.LD) - rnv).max()), rh


def raceline(tracks, nvs, alphas, step, n_max, n_out_max=None, pad=0.0):
    n = [len(t) for t in tracks]
    rl = B_.create_raceline_batch(t_(pack(tracks, n_max, pad)), t_(pack(nvs, n_max, pad)), t_(pack(alphas, n_max, pad)),
                                  step, n_pts=t_(n, torch.int32), n_out_max=n_out_max)
    return rl, n


def normals(tracks):
    """Device normals with distance scaling (the pipeline's) of each track, run alone."""
    return [splines([t], len(t), True, want_coeffs=False)[0]["nv"] for t in tracks]


def device_cum(sl):
    """create_raceline_kernel's inclusive sum of the spline lengths in its order: a chunk of ceil(n / 256) per thread,
    an exclusive scan of the chunk sums, the running sum inside each chunk."""
    n = len(sl)
    chunk = -(-n // THREADS)
    parts = []
    for t in range(THREADS):
        p = 0.0
        for i in range(t * chunk, min(t * chunk + chunk, n)):
            p += float(sl[i])
        parts.append(p)
    cum, run = np.empty(n), 0.0
    for t in range(THREADS):
        r = run
        for i in range(t * chunk, min(t * chunk + chunk, n)):
            r += float(sl[i])
            cum[i] = r
        run += parts[t]
    return cum


def station_errors(rl, b, n, track, nv, alpha, step, tag):
    """Checks the stations of track b of a create_raceline_batch result against the device's own lengths and the
    reference; returns the errors and the device arrays."""
    no = int(rl["n_out"][b])
    d = {k: v[b].cpu().numpy() for k, v in rl.items() if k != "n_out"}
    sl = d["spline_lengths"][:n]
    cum = device_cum(sl)
    total = cum[-1]
    assert no == math.ceil(total / step), tag
    dist = np.arange(no) * (total / no)
    si = d["spline_inds"][:no]
    assert np.array_equal(d["s_interp"][:no], dist), tag
    assert np.array_equal(si, np.searchsorted(cum, dist, side="right")), tag
    r = S.create_raceline(track[:, :2], nv, alpha, step)
    assert r["no"] == no, tag
    scale = float(np.abs(np.column_stack((r["coeffs_x"][:, 0], r["coeffs_y"][:, 0]))).max())
    L = lambda a: np.asarray(a, dtype=S.LD)      # noqa: E731
    e = dict(points=float(np.abs(L(d["raceline_interp"][:no]) - r["raceline_interp"]).max() / scale),
             s=float(np.abs(L(d["s_interp"][:no]) - r["s_interp"]).max() / scale),
             el=float(np.abs(L(d["el_lengths_interp"][:no]) - r["el_lengths_interp"]).max() / scale),
             u=float(np.abs(L(si) + L(d["t_values"][:no]) - (r["spline_inds"] + r["t_values"])).max()),
             kappa=float(np.abs(L(d["kappa"][:no]) - r["kappa"]).max() / np.abs(r["kappa"]).max()),
             psi=float(np.abs(S.angle_diff(d["psi"][:no], r["psi"])).max()),
             lengths=float(np.abs(L(sl) - r["spline_lengths"]).max() / r["spline_lengths"].max()))
    tv = d["t_values"][:no]
    assert np.all((tv >= 0.0) & (tv < 1.0 + 1e-12)), tag
    return e, d, cum, dist


# ---- A. moment-solve algorithms --------------------------------------------------------------------------------------
N_A = [1023, 1024, 1025, 2047, 2048, 2049, 2056, 2057, 4096, 4097]


def _el_given(track):
    """Scales that are not the chords: the chords times a smooth factor in [0.7, 1.3]."""
    d = np.linalg.norm(np.roll(track[:, :2], -1, axis=0) - track[:, :2], axis=1)
    return d * (1.0 + 0.3 * np.sin(np.linspace(0.0, 10.0 * np.pi, len(d), endpoint=False)))


@pytest.mark.parametrize("group", ["shared", "global"])
def test_moment_solves_at_their_boundaries(group):
    ns = [n for n in N_A if (n <= 2057) == (group == "shared")]
    n_max = max(ns)
    assert (smem_bytes(n_max) <= SMEM_LIMIT) == (group == "shared")
    uni = [synth.make_track(n, n) for n in ns]
    une = [MR.uneven_track(n, 20.0, n) for n in ns]
    els = [_el_given(t) for t in une]
    runs = {"unit scales, stride 4": (uni, False, None, 4, "unit"), "unit scales, stride 2": (uni, False, None, 2, "unit"),
            "chords, stride 2": (une, True, None, 2, "chords"), "chords, stride 4": (une, True, None, 4, "chords"),
            "el_lengths given": (une, True, els, 4, "el")}
    for label, (tracks, ds, el, stride, tol) in runs.items():
        got = splines(tracks, n_max, ds, el, stride)
        only = splines(tracks, n_max, ds, el, stride, want_coeffs=False)
        for b, n in enumerate(ns):
            ce, ne, rh = spline_errors(got[b], tracks[b], ds, None if el is None else el[b])
            report(f"A {group} n={n} {label}: coefficients", ce, COEF_TOL[tol])
            report(f"A {group} n={n} {label}: normals", ne, NORMVEC_TOL)
            assert np.array_equal(only[b]["nv"], got[b]["nv"]) and np.array_equal(only[b]["h"], got[b]["h"])
            if not ds:
                assert np.all(got[b]["h"] == 1.0)
            elif el is not None:
                assert np.array_equal(got[b]["h"], el[b])
            else:
                report(f"A {group} n={n} {label}: h_out", float((np.abs(got[b]["h"] - rh) / rh).max()), H_TOL)


# ---- B. tiny tracks ------------------------------------------------------------------------------------------------------
N_B = list(range(3, 10)) + [15, 16, 17, 31, 32, 33]


def test_tiny_tracks_where_the_stride_wraps():
    tracks = [blob(n, n) for n in N_B]
    for ds in (False, True):
        got = splines(tracks, max(N_B), ds)
        for b, n in enumerate(N_B):
            ce, ne, _ = spline_errors(got[b], tracks[b], ds)
            report(f"B n={n} {'chords' if ds else 'unit scales'}: coefficients", ce, COEF_TOL["tiny"])
            report(f"B n={n} {'chords' if ds else 'unit scales'}: normals", ne, NORMVEC_TOL)


# ---- C. scratch placement ------------------------------------------------------------------------------------------------
N_C = [3, 700, 1500, 3000, 3488]


def _adjoint(tracks, nvs, alphas, n_max, n_out_max, step=2.0, seed=5, pad=0.0):
    """Gradients (refline, normvec, alpha) of a fixed random weighting of raceline_interp, kappa and el_lengths_interp,
    as numpy [:n] per track; the weights beyond a track's n_out are pad."""
    n = [len(t) for t in tracks]
    ref = t_(pack([t[:, :2] for t in tracks], n_max, pad)).requires_grad_()
    nv = t_(pack(nvs, n_max, pad)).requires_grad_()
    al = t_(pack(alphas, n_max, pad)).requires_grad_()
    rl = B_.create_raceline_diff(ref, nv, al, step, n_pts=t_(n, torch.int32), n_out_max=n_out_max)
    no = rl["n_out"].cpu().numpy()
    gs = []
    for b in range(len(n)):
        rng = np.random.default_rng(seed + n[b])
        gs.append((rng.standard_normal((no[b], 2)), 100.0 * rng.standard_normal(no[b]), rng.standard_normal(no[b])))
    g_ri = t_(pack([g[0] for g in gs], n_out_max, pad))
    g_k = t_(pack([g[1] for g in gs], n_out_max, pad))
    g_el = t_(pack([g[2] for g in gs], n_out_max, pad))
    grads = torch.autograd.grad((rl["raceline_interp"], rl["kappa"], rl["el_lengths_interp"]), (ref, nv, al),
                                (g_ri, g_k, g_el))
    return [tuple(g[b, :n[b]].cpu().numpy() for g in grads) for b in range(len(n))], rl, gs


def test_scratch_placement_is_bit_for_bit():
    assert smem_bytes(3488) <= SMEM_LIMIT < smem_bytes(3489)
    tracks = [blob(3, 3)] + [synth.make_track(n, n) for n in N_C[1:]]
    els = [_el_given(t) for t in tracks]
    nvs = normals(tracks)
    alphas = [alpha_of(len(t), len(t)) for t in tracks]
    res = {}
    for n_max in (3488, 3489):
        sp = {ds: splines(tracks, n_max, ds) for ds in (False, True)}
        sp["el"] = splines(tracks, n_max, True, els)
        rl, n = raceline(tracks, nvs, alphas, 2.0, n_max, n_out_max=6400)
        rl = {k: v.cpu().numpy() for k, v in rl.items()}
        grads, _, _ = _adjoint(tracks, nvs, alphas, n_max, 6400)
        res[n_max] = (sp, rl, grads)
    (sp0, rl0, g0), (sp1, rl1, g1) = res[3488], res[3489]
    for key in sp0:
        for b in range(len(tracks)):
            for k in ("cx", "cy", "nv", "h"):
                assert np.array_equal(sp0[key][b][k], sp1[key][b][k]), (key, N_C[b], k)
    assert np.array_equal(rl0["n_out"], rl1["n_out"]) and (rl0["n_out"] > 0).all()
    for b, m in enumerate(N_C):
        no = rl0["n_out"][b]
        for k in rl0:
            if k != "n_out":
                lim = m if k in ("coeffs_x", "coeffs_y", "spline_lengths") else no
                assert np.array_equal(rl0[k][b, :lim], rl1[k][b, :lim]), (m, k)
        for x0, x1 in zip(g0[b], g1[b]):
            assert np.array_equal(x0, x1), m
        ce, ne, _ = spline_errors(sp0[True][b], tracks[b], True)
        report(f"C n={m} chords: coefficients", ce, COEF_TOL["scratch"])


# ---- D. adversarial spacing -------------------------------------------------------------------------------------------
SPACINGS = {"1:20": MR.uneven_track(400, 20.0, 7), "1:1000": MR.uneven_track(400, 1000.0, 8),
            "geometric 0.3 x 10 (ratio 5e4)": geometric_track(400, 0.3, 10),
            "geometric 0.1 x 11 (ratio 1e10)": geometric_track(440, 0.1, 11),
            "geometric 0.5 x 40 (ratio 5e11), n 2100": geometric_track(2100, 0.5, 40)}


def test_adversarial_spacing_on_the_scaled_path():
    names = list(SPACINGS)
    tracks = [SPACINGS[k] for k in names]
    got = splines(tracks, max(len(t) for t in tracks), True)
    for b, name in enumerate(names):
        h = got[b]["h"]
        ce, ne, _ = spline_errors(got[b], tracks[b], True)
        print(f"  D {name}: spacing ratio {h.max() / h.min():.1e}")
        report(f"D {name}: coefficients", ce, COEF_TOL["spacing"])
        report(f"D {name}: normals", ne, NORMVEC_TOL)


# ---- E. create_raceline stations ---------------------------------------------------------------------------------------
def test_stations_against_the_reference_and_the_devices_own_lengths():
    tracks = [synth.make_track(200, 200), synth.make_track(333, 333), MR.uneven_track(700, 20.0, 9, step=0.3),
              synth.make_track(3000, 3000), blob(5, 11)]
    nvs = normals(tracks)
    alphas = [alpha_of(len(t), len(t)) for t in tracks]
    rl, n = raceline(tracks, nvs, alphas, 2.0, 3000)
    for b, t in enumerate(tracks):
        e, d, _, _ = station_errors(rl, b, n[b], t, nvs[b], alphas[b], 2.0, n[b])
        for k, v in e.items():
            report(f"E n={n[b]} {k}", v, STATION_TOL[k])


def test_stations_on_knots_and_segments_without_stations():
    # a regular polygon: equal spline lengths up to rounding, and with 2 n stations every other one falls on a knot
    cases = []
    for n, R in ((4, 64.0), (16, 40.0), (64, 100.0)):
        t = polygon(n, R)
        nv = normals([t])[0]
        rl, _ = raceline([t], [nv], [np.zeros(n)], 1.0, n)      # (for the lap's length)
        total = device_cum(rl["spline_lengths"][0, :n].cpu().numpy())[-1]
        cases.append(("knots", t, nv, np.zeros(n), total / (2 * n) * (1.0 + 1e-9)))
    # steps of about 3.7 segments: most segments hold no station; then steps shorter than a segment on segment 0
    t = blob(40, 4, R=20.0)
    nv = normals([t])[0]
    cases.append(("sparse", t, nv, np.zeros(40), 11.7))
    cases.append(("dense", t, nv, alpha_of(40, 2), 0.37))
    ties = near = 0
    for kind, t, nv, al, step in cases:
        n = len(t)
        rl, _ = raceline([t], [nv], [al], step, n)
        e, d, cum, dist = station_errors(rl, 0, n, t, nv, al, step, (kind, n))
        si = d["spline_inds"][:len(dist)]
        for k, v in e.items():
            report(f"E {kind} n={n} {k}", v, STATION_TOL[k])
        if kind == "knots":
            assert len(dist) == 2 * n
            gap = np.abs(dist[2::2] - cum[:n - 1][:len(dist[2::2])])
            ties += int((gap == 0.0).sum())
            near += int((gap <= 4.0 * np.spacing(cum[:len(gap)])).sum())
            onknot = np.flatnonzero(np.isin(dist, cum))
            assert np.all(d["t_values"][onknot] == 0.0) and np.all(cum[si[onknot] - 1] == dist[onknot])
        elif kind == "sparse":
            assert len(np.unique(si)) < n // 2                 # segments without stations
        else:
            assert (si == 0).sum() >= 3 and d["t_values"][0] == 0.0 and si[0] == 0
    print(f"  E stations on knots: {ties} exact ties of dist and CUM[j], {near} within 4 ulps")
    assert near > 0


def _raw_raceline(track, nv, al, step, n_out_max):
    """mc_create_raceline_batch on buffers prefilled with NaN (-7 for the ints)."""
    n = len(track)
    f = lambda *s: torch.full(s, float("nan"), dtype=torch.float64, device=DEV)      # noqa: E731
    out = dict(coeffs_x=f(1, n, 4), coeffs_y=f(1, n, 4), spline_lengths=f(1, n),
               n_out=torch.full((1,), -7, dtype=torch.int32, device=DEV), raceline_interp=f(1, n_out_max, 2),
               spline_inds=torch.full((1, n_out_max), -7, dtype=torch.int32, device=DEV), t_values=f(1, n_out_max),
               s_interp=f(1, n_out_max), el_lengths_interp=f(1, n_out_max), psi=f(1, n_out_max), kappa=f(1, n_out_max))
    ws = B_._workspace("splines", _lib.load().mc_create_raceline_workspace_bytes(1, n), DEV)
    B_._call("mc_create_raceline_batch", 1, n, None, t_(track[None]), 4, t_(nv[None]), t_(al[None]), float(step), n_out_max,
             *out.values(), ws=ws)
    return {k: v[0].cpu().numpy() for k, v in out.items()}


def test_station_overflow_and_zero_padding():
    t = synth.make_track(150, 150)
    nv, al = normals([t])[0], alpha_of(150, 1)
    full = _raw_raceline(t, nv, al, 2.0, 2000)
    no = int(full["n_out"])
    assert 0 < no < 2000
    for k, v in full.items():
        if k not in ("n_out", "coeffs_x", "coeffs_y", "spline_lengths"):
            assert np.all(v[no:] == 0) and not np.isnan(v[:no]).any(), k
    over = _raw_raceline(t, nv, al, 2.0, no - 1)
    assert int(over["n_out"]) == -no
    assert np.array_equal(over["spline_lengths"], full["spline_lengths"])
    assert np.isnan(over["raceline_interp"]).all()                  # nothing written at stations
    exact = _raw_raceline(t, nv, al, 2.0, no)
    assert int(exact["n_out"]) == no and np.array_equal(exact["raceline_interp"], full["raceline_interp"][:no])


# ---- F. head_curv ------------------------------------------------------------------------------------------------------------
def test_head_curv_at_the_wrap_with_dkappa():
    # tangents along -y (atan2 - pi/2 == -pi: normalize_psi keeps -pi) and beside it on both sides; then a real spline
    xd = np.array([0.0, -0.0, 1e-300, -1e-300, 1e-3, -1e-3, 1e-9, -1e-9])
    wrap_x = np.column_stack((np.zeros(8), xd, np.full(8, 0.5), np.full(8, 0.1)))
    wrap_y = np.tile([0.0, -1.0, 0.0, 0.2], (8, 1))
    tr = synth.make_track(300, 300)
    cx, cy, _, _ = B_.calc_splines_batch(t_(tr[None]))
    cx, cy = cx[0].cpu().numpy(), cy[0].cpu().numpy()
    rng = np.random.default_rng(0)
    m = 1000
    ind = np.concatenate((np.arange(8), 8 + rng.integers(0, 300, m)))
    t = np.concatenate((np.zeros(8), rng.random(m)))
    t[8:18] = 0.0
    t[18:28] = 1.0
    coeff_x, coeff_y = np.vstack((wrap_x, cx)), np.vstack((wrap_y, cy))
    ne = len(t)
    n_eval_max = ne + 40
    cxt, cyt = t_(coeff_x[None]), t_(coeff_y[None])
    psi, kappa, dkappa = B_.calc_head_curv_batch(cxt, cyt, t_(pack([ind], n_eval_max), torch.int32),
                                                 t_(pack([t], n_eval_max)), n_eval=t_([ne], torch.int32),
                                                 calc_curv=True, calc_dcurv=True)
    psi, kappa, dkappa = (x[0].cpu().numpy() for x in (psi, kappa, dkappa))
    assert np.all(psi[ne:] == 0.0) and np.all(kappa[ne:] == 0.0) and np.all(dkappa[ne:] == 0.0)
    psi, kappa, dkappa = psi[:ne], kappa[:ne], dkappa[:ne]
    assert np.all((psi >= -np.pi) & (psi < np.pi))
    assert np.all(psi[:4] == -np.pi)
    assert psi[4] < -3.0 and psi[6] < -3.0 and psi[5] > 3.0 and psi[7] > 3.0     # either side of the wrap
    rp, rk, rdk = S.head_curv(coeff_x[ind], coeff_y[ind], t)
    report("F psi (wrap-aware)", float(np.abs(S.angle_diff(psi, rp)).max()), HEAD_TOL["psi"])
    for name, got, ref in (("kappa", kappa, rk), ("dkappa", dkappa, rdk)):
        report(f"F {name}", float(np.abs(np.asarray(got, dtype=S.LD) - ref).max() / np.abs(ref).max()), HEAD_TOL[name])


# ---- G. adjoint ------------------------------------------------------------------------------------------------------------
def test_adjoint_against_autograd_of_the_dense_reference():
    tracks = [blob(n, n) for n in (3, 4, 8, 16, 17, 33)] + [blob(40, 4, R=20.0)] + \
             [synth.make_track(n, n) for n in (1023, 1025, 2049, 2057, 4097)]
    nvs = normals(tracks)
    alphas = [alpha_of(len(t), len(t)) for t in tracks]
    n_max = max(len(t) for t in tracks)
    for step in (2.0, 11.7):
        sub = [b for b, t in enumerate(tracks) if step == 2.0 or len(t) <= 40]
        grads, rl, gs = _adjoint([tracks[b] for b in sub], [nvs[b] for b in sub], [alphas[b] for b in sub], n_max, 7600,
                                 step, seed=int(step))
        for k, b in enumerate(sub):
            n, no = len(tracks[b]), int(rl["n_out"][k])
            seg = rl["spline_inds"][k, :no].cpu().long()
            xs = [torch.tensor(x).requires_grad_() for x in (tracks[b][:, :2], nvs[b], alphas[b])]
            rr = RR.create_raceline(*xs, step, no=no, seg=seg)
            gri, gk, gel = (torch.tensor(g) for g in gs[k])
            loss = (rr["raceline"] * gri).sum() + (rr["kappa"] * gk).sum() + (rr["el_lengths"] * gel).sum()
            want = torch.autograd.grad(loss, xs)
            e = max(float(np.abs(got - w.numpy()).max() / w.abs().max()) for got, w in zip(grads[k], want))
            report(f"G n={n} step {step}: adjoint", e, ADJ_TOL)


# ---- H. batch independence -------------------------------------------------------------------------------------------------
def test_a_ragged_nan_padded_batch_gives_each_tracks_bits_alone():
    tracks = [blob(3, 1), blob(17, 2), synth.make_track(1025, 1025), synth.make_track(2057, 2057),
              MR.uneven_track(3000, 20.0, 3, step=0.2)]
    els = [_el_given(t) for t in tracks]
    nvs = normals(tracks)
    alphas = [alpha_of(len(t), len(t) + 1) for t in tracks]
    n_max = 3100
    nan = float("nan")
    for ds, el in ((False, None), (True, None), (True, els)):
        many = splines(tracks, n_max, ds, el, pad=nan)
        for b, t in enumerate(tracks):
            one = splines([t], len(t), ds, None if el is None else [el[b]])[0]
            for k in ("cx", "cy", "nv", "h"):
                assert np.array_equal(many[b][k], one[k]), (len(t), ds, k)
    rl, n = raceline(tracks, nvs, alphas, 2.0, n_max, n_out_max=5000, pad=nan)
    g_many, _, _ = _adjoint(tracks, nvs, alphas, n_max, 5000, pad=nan)
    for b, t in enumerate(tracks):
        rl1, _ = raceline([t], [nvs[b]], [alphas[b]], 2.0, len(t))
        no = int(rl1["n_out"][0])
        assert int(rl["n_out"][b]) == no
        for k, v in rl1.items():
            if k != "n_out":
                lim = len(t) if k in ("coeffs_x", "coeffs_y", "spline_lengths") else no
                assert torch.equal(rl[k][b, :lim], v[0, :lim]), (len(t), k)
        g1, _, _ = _adjoint([t], [nvs[b]], [alphas[b]], len(t), no)
        for x0, x1 in zip(g_many[b], g1[0]):
            assert np.array_equal(x0, x1), len(t)
