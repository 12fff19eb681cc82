"""Extended-precision reference (np.longdouble) of the closed-spline kernels of csrc/splines.cu: the periodic moment
solve with its coefficients and normal vectors (calc_splines_kernel), create_raceline (create_raceline_kernel) and
head_curv (head_curv_kernel, with dkappa).  Written from the kernels' comments and oracle/tph_dense.py; where the kernel
rounds in float64 this module rounds 11 bits later, so its results are the exact values of the same formulas to about
1e-19 relative.  Test infrastructure, not product code."""
import math

import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "the spline reference needs an 80-bit or quad long double"
PI = np.arccos(LD(-1.0))
T15 = np.linspace(0.0, 1.0, 15).astype(LD)          # tph.calc_spline_lengths samples (no_interp_points=15)


def ld(a):
    return np.asarray(a, dtype=np.float64).astype(LD)


def scales(p, el_lengths=None, use_dist_scaling=True):
    """The parameter scales h [n] of calc_splines_kernel: 1 without distance scaling, el_lengths when given, else the
    chord |p_{i+1} - p_i| (cyclic)."""
    p = ld(p)
    if not use_dist_scaling:
        return np.ones(p.shape[0], dtype=LD)
    if el_lengths is not None:
        return ld(el_lengths)
    d = np.roll(p[:, :2], -1, axis=0) - p[:, :2]
    return np.sqrt((d * d).sum(axis=1))


def moment_system(p, h):
    """(sub, diag, sup, rhs [n, 2]) of the cyclic system of the moments m (second derivatives in arc parameter):
    h_{i-1} m_{i-1} + 2 (h_{i-1} + h_i) m_i + h_i m_{i+1} = 6 ((p_{i+1} - p_i) / h_i - (p_i - p_{i-1}) / h_{i-1})."""
    p, h = ld(p)[:, :2], np.asarray(h, dtype=LD)
    hm = np.roll(h, 1)
    dp = np.roll(p, -1, axis=0) - p
    rhs = 6.0 * (dp / h[:, None] - np.roll(dp, 1, axis=0) / hm[:, None])
    return hm, 2.0 * (hm + h), h.copy(), rhs


def _thomas(a, b, c, r):
    """Non-cyclic tridiagonal solve (a[0] and c[-1] ignored) of r [n, k]."""
    n = b.size
    cp = np.empty(n, dtype=LD)
    rp = np.empty_like(r)
    cp[0], rp[0] = c[0] / b[0], r[0] / b[0]
    for i in range(1, n):
        den = b[i] - a[i] * cp[i - 1]
        cp[i] = c[i] / den
        rp[i] = (r[i] - a[i] * rp[i - 1]) / den
    x = np.empty_like(r)
    x[-1] = rp[-1]
    for i in range(n - 2, -1, -1):
        x[i] = rp[i] - cp[i] * x[i + 1]
    return x


def cyclic_solve(a, b, c, r):
    """x with a_i x_{i-1} + b_i x_i + c_i x_{i+1} = r_i (indices mod n, n >= 3): the cyclic Thomas algorithm, the
    Thomas solve of the matrix with its corners moved onto the diagonal and a Sherman-Morrison correction."""
    n = b.size
    r = np.asarray(r, dtype=LD).reshape(n, -1)
    gamma = -b[0]
    bb = b.copy()
    bb[0] -= gamma
    bb[-1] -= c[-1] * a[0] / gamma
    u = np.zeros((n, 1), dtype=LD)
    u[0, 0], u[-1, 0] = gamma, c[-1]
    x = _thomas(a, bb, c, r)
    z = _thomas(a, bb, c, u)
    fact = (x[0] + a[0] * x[-1] / gamma) / (1.0 + z[0, 0] + a[0] * z[-1, 0] / gamma)
    return x - z * fact[None, :]


def moments(p, h):
    a, b, c, r = moment_system(p, h)
    return cyclic_solve(a, b, c, r)


def closed_spline(p, h):
    """(cx [n, 4], cy [n, 4], normvec [n, 2], m [n, 2]) in long double, formed as closed_spline forms them:
    [p_i, dp_i - h_i^2 (2 m_i + m_{i+1}) / 6, h_i^2 m_i / 2, h_i^2 (m_{i+1} - m_i) / 6] and (c1y, -c1x) / |c1|."""
    p, h = ld(p)[:, :2], np.asarray(h, dtype=LD)
    m = moments(p, h)
    mp = np.roll(m, -1, axis=0)
    h2 = (h * h)[:, None]
    a1 = (np.roll(p, -1, axis=0) - p) - h2 * (2.0 * m + mp) / 6.0
    c = [np.column_stack((p[:, k], a1[:, k], 0.5 * h2[:, 0] * m[:, k], h2[:, 0] * (mp[:, k] - m[:, k]) / 6.0))
         for k in range(2)]
    nv = np.column_stack((a1[:, 1], -a1[:, 0]))
    return c[0], c[1], nv / np.sqrt((nv * nv).sum(axis=1))[:, None], m


def calc_splines(xy, el_lengths=None, use_dist_scaling=True):
    """calc_splines_kernel for one closed track xy [n, >=2] (no repeated last point): (cx, cy, normvec, h)."""
    h = scales(xy, el_lengths, use_dist_scaling)
    cx, cy, nv, _ = closed_spline(xy, h)
    return cx, cy, nv, h


def poly(c, t):
    return c[..., 0] + c[..., 1] * t + c[..., 2] * t * t + c[..., 3] * t * t * t


def spline_lengths(cx, cy):
    """15-sample polyline length of every segment (tph.calc_spline_lengths)."""
    x, y = poly(cx[:, None, :], T15[None, :]), poly(cy[:, None, :], T15[None, :])
    return np.sqrt(np.diff(x, axis=1) ** 2 + np.diff(y, axis=1) ** 2).sum(axis=1)


def normalize_psi(psi):
    """tph.normalize_psi: sign(psi) * mod(|psi|, 2 pi), then into [-pi, pi)."""
    psi = np.asarray(psi, dtype=LD)
    out = np.sign(psi) * np.mod(np.abs(psi), 2.0 * PI)
    out = np.where(out >= PI, out - 2.0 * PI, out)
    return np.where(out < -PI, out + 2.0 * PI, out)


def angle_diff(a, b):
    """a - b wrapped into [-pi, pi) (headings on either side of the wrap of normalize_psi)."""
    d = np.asarray(a, dtype=LD) - np.asarray(b, dtype=LD)
    return np.mod(d + PI, 2.0 * PI) - PI


def head_curv(cx, cy, t):
    """(psi, kappa, dkappa) at parameter t of the segments with coefficients cx, cy [m, 4] (calc_head_curv_an)."""
    cx, cy, t = np.asarray(cx, dtype=LD), np.asarray(cy, dtype=LD), np.asarray(t, dtype=LD)
    xd = cx[:, 1] + 2.0 * cx[:, 2] * t + 3.0 * cx[:, 3] * t * t
    yd = cy[:, 1] + 2.0 * cy[:, 2] * t + 3.0 * cy[:, 3] * t * t
    xdd, ydd = 2.0 * cx[:, 2] + 6.0 * cx[:, 3] * t, 2.0 * cy[:, 2] + 6.0 * cy[:, 3] * t
    xddd, yddd = 6.0 * cx[:, 3], 6.0 * cy[:, 3]
    q = xd * xd + yd * yd
    cross = xd * ydd - yd * xdd
    psi = normalize_psi(np.arctan2(yd, xd) - PI / 2.0)
    return psi, cross / (q * np.sqrt(q)), (q * (xd * yddd - yd * xddd) - 3.0 * cross * (xd * xdd + yd * ydd)) / (q * q * q)


def create_raceline(refline, normvec, alpha, stepsize):
    """create_raceline_kernel for one closed track: the spline through P = refline + alpha normvec with unit scales,
    its 15-sample lengths, their cumulative sum CUM, n_interp = ceil(CUM[-1] / stepsize) + 1 linspace stations of which
    the last (the lap's end) is dropped, each on the first segment j with dist < CUM[j]; the points, t, s, el, psi and
    kappa there.  A dict of long double arrays (spline_inds int) and the station count no."""
    P = ld(refline)[:, :2] + ld(alpha)[:, None] * ld(normvec)
    cx, cy, _, _ = closed_spline(P, np.ones(P.shape[0], dtype=LD))
    sl = spline_lengths(cx, cy)
    cum = np.cumsum(sl)
    total = cum[-1]
    n_interp = int(math.ceil(total / LD(stepsize))) + 1
    no = n_interp - 1
    dist = np.arange(no, dtype=LD) * (total / LD(no))
    j = np.searchsorted(cum, dist, side="right")
    prev = np.concatenate(([LD(0.0)], cum))[j]
    t = (dist - prev) / sl[j]
    psi, kappa, _ = head_curv(cx[j], cy[j], t)
    el = np.append(np.diff(dist), total - dist[-1])
    return dict(coeffs_x=cx, coeffs_y=cy, spline_lengths=sl, cum=cum, no=no, spline_inds=j, t_values=t,
                raceline_interp=np.column_stack((poly(cx[j], t), poly(cy[j], t))), s_interp=dist, el_lengths_interp=el,
                psi=psi, kappa=kappa)
