"""Constructed cases of the normals-crossing check (tph.check_normals_crossing, oracle/tph_prep.py) where the 2 x 2 solve of
csrc/traj_check_core.cuh normals_cross changes path: the inclusive width comparisons, the 1e-8 collinearity threshold,
pivot ties and swaps; and tracks whose only crossing pair is across index 0 or needs a horizon of n - 1.  Shared by
tests/test_refback_edges_host.py and tests/test_gpu_refback_edges.py."""
import numpy as np

S = np.sqrt(0.5)


def _pair(tag, p, n1, q, n2, w1=(5.0, 5.0), w2=(5.0, 5.0), expect=None):
    return dict(tag=tag, p=np.array([p[0], p[1], w1[0], w1[1]]), n1=np.array(n1, dtype=float),
                q=np.array([q[0], q[1], w2[0], w2[1]]), n2=np.array(n2, dtype=float), expect=expect)


def normals_pairs():
    """One (point, neighbour) pair each: rows [x, y, w_tr_right, w_tr_left] and unit normals.  expect: the bits of
    tc_host_normals_cross_info (tests/host_harness/tc_host.cpp) the case is built to reach."""
    below = np.nextafter(2.0, 0.0)
    t_hi, t_lo = np.nextafter(1e-8, 1.0), 1e-8
    out = [
        # p + l1 (1, 0) meets q + l2 (0, 1) at l1 = 2, l2 = 1: l1 == w1r decides, then one ulp short of it
        _pair("l1_at_w1r", (0.0, 0.0), (1.0, 0.0), (2.0, -1.0), (0.0, 1.0), w1=(2.0, 5.0), expect=(1 << 3) | (1 << 6)),
        _pair("l1_ulp_beyond_w1r", (0.0, 0.0), (1.0, 0.0), (2.0, -1.0), (0.0, 1.0), w1=(below, 5.0), expect=0),
        # ... and at -w1l (l1 = -2), and at l2 == w2r / -w2l
        _pair("l1_at_minus_w1l", (0.0, 0.0), (1.0, 0.0), (-2.0, -1.0), (0.0, 1.0), w1=(5.0, 2.0), expect=(1 << 2) | (1 << 6)),
        _pair("l2_at_w2r", (0.0, 0.0), (1.0, 0.0), (2.0, -1.0), (0.0, 1.0), w2=(1.0, 5.0), expect=(1 << 5) | (1 << 6)),
        _pair("l2_at_minus_w2l", (0.0, 0.0), (1.0, 0.0), (2.0, 1.0), (0.0, 1.0), w2=(5.0, 1.0), expect=(1 << 4) | (1 << 6)),
        # |cross| one ulp above 1e-8 (solved: the lines meet at l1 = 0, l2 = 1) and exactly 1e-8 (collinear: skipped)
        _pair("cross_above_1e-8", (0.0, 0.0), (1.0, 0.0), (-np.sqrt(1.0 - t_hi * t_hi), -t_hi),
              (np.sqrt(1.0 - t_hi * t_hi), t_hi), expect=1 << 6),
        _pair("cross_at_1e-8", (0.0, 0.0), (1.0, 0.0), (-np.sqrt(1.0 - t_lo * t_lo), -t_lo),
              (np.sqrt(1.0 - t_lo * t_lo), t_lo), expect=1 << 1),
        # pivot search: a tie |a10| == |a00| keeps the first row (idamax), a larger |a10| swaps
        _pair("pivot_tie", (0.0, 0.0), (S, S), (1.0, -0.5), (0.0, 1.0), expect=1 << 6),
        _pair("pivot_tie_negative", (0.0, 0.0), (S, -S), (1.0, -3.0), (0.0, 1.0), expect=1 << 6),
        _pair("pivot_swap", (0.0, 0.0), (0.6, 0.8), (1.5, 0.5), (1.0, 0.0), expect=1 | (1 << 6)),
        _pair("pivot_swap_miss", (0.0, 0.0), (0.6, 0.8), (1.5, 0.5), (1.0, 0.0), w1=(0.5, 5.0), expect=1),
    ]
    return out


def pair_track(c):
    """A 3-point track holding the pair at indices 0 and 1 and a third point far away whose zero widths and distance keep
    it from crossing either (the oracle decides the whole track)."""
    track = np.array([c["p"], c["q"], [1.0e4, 1.0e4 + 7.25, 0.0, 0.0]])
    nv = np.array([c["n1"], c["n2"], [0.28, 0.96]])
    return track, nv


def ring_track(n, cross_at=None, radius=20.0):
    """n points around a circle, outward normals, widths 1 m (no crossing).  cross_at = (i, j): the normals of i and j are
    turned towards each other and widened until they cross (only that pair)."""
    ang = 2.0 * np.pi * np.arange(n) / n
    xy = radius * np.column_stack((np.cos(ang), np.sin(ang)))
    nv = np.column_stack((np.cos(ang), np.sin(ang)))
    track = np.column_stack((xy, np.ones(n), np.ones(n)))
    if cross_at is not None:
        i, j = cross_at
        mid = 0.5 * (xy[i] + xy[j]) + 3.0 * (nv[i] + nv[j])     # a point outside the ring between i and j
        for k in (i, j):
            d = mid - xy[k]
            nv[k] = d / np.sqrt(d @ d)
            track[k, 2] = 2.0 * np.sqrt(d @ d)
    return track, nv


def load_tc_host(so_dir):
    """tests/host_harness/tc_host.cpp (the statements of csrc/traj_check_core.cuh) built with g++ into so_dir, or None
    without g++."""
    import ctypes
    import os
    import shutil
    import subprocess
    cxx = shutil.which("g++")
    if cxx is None:
        return None
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = os.path.join(str(so_dir), "libtc_host.so")
    subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-std=c++17", "-o", so,
                           os.path.join(root, "tests", "host_harness", "tc_host.cpp")])
    lib = ctypes.CDLL(so)
    DP, I, D, IP = ctypes.POINTER(ctypes.c_double), ctypes.c_int, ctypes.c_double, ctypes.POINTER(ctypes.c_int)
    for name, res, args in (("tc_host_interp_track", I, [I, DP, I, DP, D, I, D, I, DP]),
                            ("tc_host_min_bound_dists", None, [I, DP, DP, I, DP, I, DP, I, D, D, DP, IP]),
                            ("tc_host_normals_crossing", I, [I, DP, DP, I]),
                            ("tc_host_extrema", None, [I, DP, DP, DP, DP, D, D, DP]),
                            ("tc_host_interp_exact_hits", I, [I, DP, I, D]),
                            ("tc_host_normals_cross_info", I, [DP, DP, DP, DP])):
        getattr(lib, name).restype = res
        getattr(lib, name).argtypes = args
    return lib


def ptr(a):
    """ctypes pointer of a C-contiguous numpy array (None: NULL)"""
    import ctypes
    if a is None:
        return None
    assert a.flags.c_contiguous
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_int if a.dtype == np.int32 else ctypes.c_double))


def reference_extrema(kappa, vx, ax, min_dists, dragcoeff, mass):
    """The 8 extrema of traj_extrema_kernel from the quantities check_traj.py:93-131 forms, with the reference's NaN
    semantics: min_dist and max |kappa| by np.amin / np.amax (NaN propagates), the rest as np.any(x > limit) sees them
    (NaN points skipped: np.fmax / np.fmin)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        radii = np.abs(np.divide(1.0, kappa, out=np.full(kappa.size, np.inf), where=kappa != 0))
        ay = np.divide(np.power(vx, 2), radii)
        ax_wo = ax - (-np.power(vx, 2) * dragcoeff / mass)
        a_tot = np.sqrt(np.power(ax_wo, 2) + np.power(ay, 2))
    return np.array([np.amin(min_dists) if min_dists is not None else np.inf, np.amax(np.abs(kappa)), np.fmax.reduce(ay),
                     np.fmax.reduce(ax_wo), np.fmin.reduce(ax_wo), np.fmax.reduce(a_tot), np.fmax.reduce(vx), kappa.size])


def same(a, b):
    """bit for bit, NaN equal to NaN (payloads aside)"""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a[~na].view(np.int64), b[~nb].view(np.int64)))
