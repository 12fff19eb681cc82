"""Extended-precision reference (np.longdouble) of the post-solve kernel of the minimum-curvature QP,
mincurv_finalize_kernel (K2c, csrc/mincurv_finalize.cu): kappa_lin_max = max |k_ref + E alpha|, the linearisation error
curv_error_max and the status rules; and the long-double quantities of its two neighbours there (the sensitivity
exports and the projection QP's Hessian and linear term).

from_slab   replays the kernel statement by statement from the vectors of an instance's slab (H, NX/NY, MX/MY, XP/YP,
            SX/SY, KREF, PX/PY): Z (n alpha) by the periodic moment solve, the linearised curvature, c0, c1 and the
            centre line's first derivatives of the LIN form.
from_inputs builds the same quantities from their definition: the moments of P and of P + alpha n, the first
            derivatives of the linearisation line P + a n, the knot curvature of the spline through P + alpha n.  It
            shares no statement with the kernel's assembly (mincurv_setup.cu) or its finalize, so a mismatch between the
            two would show.
status_after the status rules of the kernel.
Test infrastructure, not product code."""
import numpy as np

import spline_ref as S

LD = S.LD
SLAB_KEYS = ("H", "NX", "NY", "MX", "MY", "XP", "YP", "SX", "SY", "KREF", "PX", "PY")
KAPPA_TOL_REL = 1e-7            # status 4: kappa_lin_max > kappa_bound * (1 + 1e-7)


def _d2(h, v):
    """6 D2 v: 6 ((v_{i+1} - v_i) / h_i - (v_i - v_{i-1}) / h_{i-1}) (cyclic)."""
    return 6.0 * ((np.roll(v, -1) - v) / h - (v - np.roll(v, 1)) / np.roll(h, 1))


def _tri_solve(h, rx, ry):
    """Tri^{-1} [rx, ry] with Tri the cyclic tridiagonal spline matrix (diagonal 2 (h_{i-1} + h_i), off-diagonal h_i)."""
    hm = np.roll(h, 1)
    z = S.cyclic_solve(hm, 2.0 * (hm + h), h.copy(), np.column_stack((rx, ry)))
    return z[:, 0], z[:, 1]


def _moments(p, h):
    """moments [n, 2] of the closed h-spline through p [n, 2] (spline_ref.moments without its float64 round of p)"""
    return np.column_stack(_tri_solve(h, _d2(h, p[:, 0]), _d2(h, p[:, 1])))


def _first(p, m, h2):
    """first derivatives at the knots of the h-spline through p [n] with moments m: dp - h^2 (2 m + m_next) / 6"""
    return (np.roll(p, -1) - p) - h2 * (2.0 * m + np.roll(m, -1)) / 6.0


def _out(zx, zy, klin, c0, c1):
    err = np.abs(c1 - c0)
    return dict(zx=zx, zy=zy, klin=klin, c0=c0, c1=c1, err=err,
                kmax=np.amax(np.abs(klin)), emax=np.amax(err))           # (np.amax: a NaN propagates, as in tph)


def from_slab(v, alpha, lin=False):
    """K2c on the slab vectors v (dict of SLAB_KEYS -> [n]) at alpha [n], in long double: dict of per-point zx, zy
    (Z (n_x alpha), Z (n_y alpha)), klin = KREF + SY zy - SX zx, c0, c1, err = |c1 - c0| and the maxima kmax, emax."""
    g = {k: np.asarray(v[k], dtype=LD) for k in SLAB_KEYS}     # (float64 or long double: exact)
    al = S.ld(alpha)
    with np.errstate(all="ignore"):
        h = g["H"]
        h2 = h * h
        vx, vy = g["NX"] * al, g["NY"] * al
        zx, zy = _tri_solve(h, _d2(h, vx), _d2(h, vy))
        klin = g["KREF"] + g["SY"] * zy - g["SX"] * zx
        ddx, ddy = h2 * (g["MX"] + zx), h2 * (g["MY"] + zy)
        xp, yp = g["XP"], g["YP"]
        xc, yc = (_first(g["PX"], g["MX"], h2), _first(g["PY"], g["MY"], h2)) if lin else (xp, yp)
        xpt = xc + (np.roll(vx, -1) - vx) - h2 * (2.0 * zx + np.roll(zx, -1)) / 6.0
        ypt = yc + (np.roll(vy, -1) - vy) - h2 * (2.0 * zy + np.roll(zy, -1)) / 6.0
        q0, q1 = xp * xp + yp * yp, xpt * xpt + ypt * ypt
        c0 = (xp * ddy - yp * ddx) / (q0 * np.sqrt(q0))
        c1 = (xpt * ddy - ypt * ddx) / (q1 * np.sqrt(q1))
    return _out(zx, zy, klin, c0, c1)


def _curvature(dx, dy, ddx, ddy):
    q = dx * dx + dy * dy
    return (dx * ddy - dy * ddx) / (q * np.sqrt(q))


def from_inputs(reftrack, normvec, h, alpha, lin_alpha=None):
    """The quantities of from_slab from their definition, about the line P + a n (a = lin_alpha, None: the centre line):
    zx, zy the moments of n alpha; klin the curvature with the first derivatives of P + a n and the second derivatives
    of P + alpha n; c1 the knot curvature of the spline through P + alpha n; c0 = klin.  Also 'slab': the slab vectors
    of that linearisation (as mincurv_setup.cu defines them), for from_slab."""
    P, N, h, al = S.ld(reftrack)[:, :2], S.ld(normvec), S.ld(h), S.ld(alpha)
    a = np.zeros_like(al) if lin_alpha is None else S.ld(lin_alpha)
    with np.errstate(all="ignore"):
        h2 = h * h
        m = _moments(P, h)                                  # the centre line's
        Ps = P + a[:, None] * N
        ms = m if lin_alpha is None else _moments(Ps, h)
        Pa = P + al[:, None] * N
        ma = _moments(Pa, h)
        z = _moments(al[:, None] * N, h)
        xs, ys = _first(Ps[:, 0], ms[:, 0], h2), _first(Ps[:, 1], ms[:, 1], h2)
        xa, ya = _first(Pa[:, 0], ma[:, 0], h2), _first(Pa[:, 1], ma[:, 1], h2)
        klin = _curvature(xs, ys, h2 * ma[:, 0], h2 * ma[:, 1])
        c1 = _curvature(xa, ya, h2 * ma[:, 0], h2 * ma[:, 1])
        c = 1.0 / ((xs * xs + ys * ys) * np.sqrt(xs * xs + ys * ys))
        sx, sy = c * ys * h2, c * xs * h2
        slab = dict(H=h, NX=N[:, 0], NY=N[:, 1], MX=m[:, 0], MY=m[:, 1], XP=xs, YP=ys, SX=sx, SY=sy,
                    KREF=sy * m[:, 1] - sx * m[:, 0], PX=P[:, 0], PY=P[:, 1])
    return dict(_out(z[:, 0], z[:, 1], klin, klin, c1), slab=slab)


def status_after(st, kmax, kb, kbb=False):
    """(status, zeroed) after the kernel, for the incoming status st, the maximum kmax the kernel computes and the limit
    kb (kbb: the per-instance form, kappa_bound_batch).  zeroed: the kernel writes 0 for both maxima and skips the
    instance.  The comparison is the kernel's, in float64."""
    kb = float(kb)
    if kbb and st >= 0 and not (kb > 0.0 and kb < np.inf):
        st = -1                                                   # (so 1 -> -1 as well)
    if st == 1 or st < 0:
        return st, True
    if st == 0 and float(kmax) > kb * (1.0 + KAPPA_TOL_REL):
        return 4, False
    return st, False


def sens_ratios(LU, SU, LL, SL):
    """sens of the export kernels: lu / su, ll / sl (float64, as the kernel divides)."""
    return np.asarray(LU) / np.asarray(SU), np.asarray(LL) / np.asarray(SL)


def row_weights(L3, S3, L4, S4):
    """(w, n_rows) of mincurv_sens_rows_export_kernel: w = l3 / s3 + l4 / s4 and the count of strong rows, w > 1."""
    w = np.asarray(L3) / np.asarray(S3) + np.asarray(L4) / np.asarray(S4)
    return w, int((w > 1.0).sum())


def prox_linear_term(v, mu, x, q):
    """c = mu q - (E^T E x + mu x) of mincurv_prox_kernel in long double, with the full operator E of the slab vectors
    v (E u = S_y Z (n_y u) - S_x Z (n_x u), E^T w = N_y Z^T (S_y w) - N_x Z^T (S_x w), Z = Tri^{-1} 6 D2)."""
    g = {k: np.asarray(v[k], dtype=LD) for k in SLAB_KEYS}     # (float64 or long double: exact)
    x, q, mu = S.ld(x), S.ld(q), LD(mu)
    h = g["H"]
    zx, zy = _tri_solve(h, _d2(h, g["NX"] * x), _d2(h, g["NY"] * x))
    ex = g["SY"] * zy - g["SX"] * zx
    tx, ty = _tri_solve(h, g["SX"] * ex, g["SY"] * ex)
    hx = g["NY"] * _d2(h, ty) - g["NX"] * _d2(h, tx)
    return mu * q - (hx + mu * x)
