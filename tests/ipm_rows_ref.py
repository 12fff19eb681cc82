"""Replay (np.longdouble by default) of the curvature-row interior-point iteration that three kernels run on the
minimum-curvature QP with its curvature rows: the dense small-track kernel (mincurv_dense_kernel, csrc/mincurv_dense.cu),
the banded curvature-row phase (mincurv_pdip_kappa_kernel<false>, csrc/mincurv_ipm.cu) and its projection variant
(mincurv_pdip_kappa_kernel<true>).  The QP

    min 1/2 a^T (E^T E + mu_p I) a + f^T a,   lb <= a <= ub,   -kb <= k_ref + E a <= kb

(mu_p = 0 except for the projection QP) is built here in long double from the periodic moments of tests/spline_ref.py,
as csrc/mincurv_setup.cu P1-P5 builds it (FIX_EPS widening of collapsed boxes, f_scale, the LIN form about a given
line), and the iteration follows the kernels statement by statement: the start point, the predictor, the four c-sums
of the centring rule, the corrector with its second-order terms, the damped steps, the exact dual residual and the
three exits in the kernels' order, then the finalize quantities of csrc/mincurv_finalize.cu and the status-4 override.

Options that the tests use to tell which decisions rounding can move: dtype=np.float64 (the kernels' precision),
perm (a permutation: every sum reduction is taken in that order), band=32 (the normal matrix replaced by its cyclic band
of half-width 32 with the exact entries of E^T (I + W) E, what assemble_hband hands the banded factor).
Test infrastructure, not product code."""
import numpy as np

import spline_ref as S

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "the interior-point replay needs an 80-bit or quad long double"
FIX_EPS = 1e-8              # common.cuh: half-width given to a collapsed box
MAX_ITER = 40               # the curvature-row phase's PdipParams (mincurv_kappa_phase, mincurv_dense)
MU_REL = 1e-11
RD_REL = 1e-8
ETA = 0.995
LAM0_REL = 1e-2
HBW = 32                    # common.cuh: half-bandwidth of the banded normal matrix
DENSE_LD_MAX = 130          # above this a float64 replay factors with LAPACK (the long-double one always by hand)


def _d2(h):
    """6 D2 [n, n]: (6 D2 p)_i = 6 ((p_{i+1} - p_i) / h_i - (p_i - p_{i-1}) / h_{i-1})."""
    n = h.size
    D = np.zeros((n, n), dtype=LD)
    for i in range(n):
        D[i, (i + 1) % n] += 6.0 / h[i]
        D[i, i] -= 6.0 / h[i] + 6.0 / h[i - 1]
        D[i, i - 1] += 6.0 / h[i - 1]
    return D


def _tri_solve(h, r):
    """Tri^-1 r (Tri the cyclic moment matrix of scales h) for r [n, k]."""
    hm = np.roll(h, 1)
    return S.cyclic_solve(hm, 2.0 * (hm + h), h.copy(), r)


def qp_data(reftrack, normvec, h, w_veh, f_scale=2.0, lin_alpha=None):
    """The QP of one closed track in long double, as mincurv_setup.cu assembles it (dense E, no band truncation):
    dict(E, k_ref, f, lb, ub and the geometry the finalize needs) or None where some lb > ub (status 1)."""
    rt, nv, h = S.ld(reftrack), S.ld(normvec), S.ld(h)
    n = rt.shape[0]
    ub = rt[:, 2] - 0.5 * LD(w_veh)
    lb = -(rt[:, 3] - 0.5 * LD(w_veh))
    if (lb > ub).any():
        return None
    col = ub - lb < 2.0 * FIX_EPS
    mid = 0.5 * (lb + ub)
    lb, ub = np.where(col, mid - FIX_EPS, lb), np.where(col, mid + FIX_EPS, ub)
    P = rt[:, :2]
    M = S.moments(P, h)
    h2 = h * h

    def first(Q, MQ):
        return (np.roll(Q, -1, axis=0) - Q) - h2[:, None] * (2.0 * MQ + np.roll(MQ, -1, axis=0)) / 6.0

    d1c = first(P, M)
    if lin_alpha is None:
        d1 = d1c
    else:
        Ps = P + S.ld(lin_alpha)[:, None] * nv
        d1 = first(Ps, S.moments(Ps, h))
    q = (d1 * d1).sum(axis=1)
    c = 1.0 / (q * np.sqrt(q))
    sy, sx = c * d1[:, 0] * h2, c * d1[:, 1] * h2
    k_ref = sy * M[:, 1] - sx * M[:, 0]
    Z = _tri_solve(h, _d2(h))
    E = Z * (sy[:, None] * nv[None, :, 1] - sx[:, None] * nv[None, :, 0])
    return dict(n=n, E=E, k_ref=k_ref, f=LD(f_scale) * (E.T @ k_ref), lb=lb, ub=ub, h=h, nv=nv, M=M, d1=d1, d1c=d1c,
                sx=sx, sy=sy)


def finalize(d, alpha):
    """(kappa_lin_max, curv_error_max) at alpha, as mincurv_finalize.cu forms them: k_ref + S_y zy - S_x zx with
    z = Tri^-1 6 D2 (n alpha), and the linearised curvature error between the line's first derivatives and those of
    the centre line moved by alpha n (long double)."""
    a = S.ld(alpha)
    nv, h, M = d["nv"], d["h"], d["M"]
    h2 = h * h
    z = _tri_solve(h, _d2(h) @ (nv * a[:, None]))
    klin = d["k_ref"] + d["sy"] * z[:, 1] - d["sx"] * z[:, 0]
    dd = h2[:, None] * (M + z)
    xp, yp = d["d1"][:, 0], d["d1"][:, 1]
    na = nv * a[:, None]
    t = d["d1c"] + (np.roll(na, -1, axis=0) - na) - h2[:, None] * (2.0 * z + np.roll(z, -1, axis=0)) / 6.0
    q0, q1 = xp * xp + yp * yp, (t * t).sum(axis=1)
    c0 = (xp * dd[:, 1] - yp * dd[:, 0]) / (q0 * np.sqrt(q0))
    c1 = (t[:, 0] * dd[:, 1] - t[:, 1] * dd[:, 0]) / (q1 * np.sqrt(q1))
    return np.abs(klin).max(), np.abs(c1 - c0).max(), klin


def _band_mask(n, w):
    i = np.arange(n)
    dist = np.abs(i[:, None] - i[None, :])
    return np.minimum(dist, n - dist) <= w


def _chol(K):
    """Lower Cholesky factor of K, column by column (right-looking, as dense_factor); None on a non-positive pivot."""
    n = K.shape[0]
    L = np.tril(K).copy()
    for j in range(n):
        p = L[j, j]
        if not p > 0.0:
            return None
        l = np.sqrt(p)
        L[j, j] = l
        L[j + 1:, j] /= l
        L[j + 1:, j + 1:] -= np.tril(np.outer(L[j + 1:, j], L[j + 1:, j]))
    return L


def _chol_solve(L, r):
    n = L.shape[0]
    y = r.copy()
    for j in range(n):
        y[j] /= L[j, j]
        y[j + 1:] -= L[j + 1:, j] * y[j]
    for j in range(n - 1, -1, -1):
        y[j] /= L[j, j]
        y[:j] -= L[j, :j] * y[j]
    return y


class _Factor:
    """The factor of one iteration.  Long double: the hand-written Cholesky (any n).  float64 at more than DENSE_LD_MAX
    points: LAPACK, of K itself or, with order, of K with rows and columns in that order (another elimination order,
    so other rounding)."""

    def __init__(self, K, fast, order=None):
        self.fast, self.order = fast, order
        if fast:
            import scipy.linalg
            Kf = K.astype(np.float64)
            if order is not None:
                Kf = Kf[np.ix_(order, order)]
            try:
                self.c = scipy.linalg.cho_factor(Kf, lower=True)
                self.ok = bool(np.isfinite(self.c[0]).all())
            except np.linalg.LinAlgError:
                self.ok = False
        else:
            self.L = _chol(K)
            self.ok = self.L is not None

    def solve(self, r, dtype):
        if self.fast:
            import scipy.linalg
            rf = r.astype(np.float64)
            if self.order is None:
                return scipy.linalg.cho_solve(self.c, rf).astype(dtype)
            x = np.empty_like(rf)
            x[self.order] = scipy.linalg.cho_solve(self.c, rf[self.order])
            return x.astype(dtype)
        return _chol_solve(self.L, r)


def replay(d, kb, dtype=LD, perm=None, band=None, prox_mu=0.0, prox_x=None, prox_q=None, override="dense", mu_rel=MU_REL):
    """Run the iteration on the QP d (qp_data) with curvature limit kb.  Returns dict(status, iters, result, exit,
    alpha, kappa_lin_max, curv_error_max, trace).  exit: 'converged' (mu <= 1e-11 mu0, |r_d| <= rd_tol,
    |r_p| <= 1e-8 kb), 'mu_floor' (mu <= 1e-13 mu0: status 0 or 2), 'pivot' (non-positive pivot: late-accept 0 or 3),
    'cap' (max_iter + 20 iterations).  override 'dense': status 4 wherever the last iterate violates the rows by more than
    kb 1e-7 (or is not finite), however the iteration ended (mincurv_dense_kernel); 'banded': only a status-0 result
    becomes 4 (the finalize pass after the curvature-row phase).  prox_mu > 0: the projection QP, Hessian H + mu I and
    linear term c = mu q - (H + mu I) x (mincurv_prox_kernel).  trace: per iteration mu, rdmax, rpmax, the affine and
    damped ap / ad and whether each was a full step, the ratios of the three stopping tests to their thresholds, and
    the number of start slacks clamped at 1e-2 kb.  mu_rel: the first exit's threshold (the kernels' 1e-11; smaller
    values run the iteration closer to the optimum, for the checks of the replay itself)."""
    with np.errstate(all="ignore"):
        return _replay(d, kb, dtype, perm, band, prox_mu, prox_x, prox_q, override, mu_rel)


def _replay(d, kb, dtype, perm, band, prox_mu, prox_x, prox_q, override, mu_rel):
    n = d["n"]
    E = d["E"].astype(dtype)
    KR, LB, UB = d["k_ref"].astype(dtype), d["lb"].astype(dtype), d["ub"].astype(dtype)
    kb = dtype(kb)
    mu_p = dtype(prox_mu)
    if prox_mu > 0.0:
        x = S.ld(prox_x).astype(dtype)
        F = mu_p * S.ld(prox_q).astype(dtype) - (E.T @ (E @ x) + mu_p * x)
    else:
        F = d["f"].astype(dtype)
    fast = dtype == np.float64 and n > DENSE_LD_MAX
    mask = _band_mask(n, band) if band is not None else None
    order = np.arange(n) if perm is None else np.asarray(perm)

    def tot(v):                         # a sum reduction, in the order of perm
        return v[order].sum()

    def mx(*vs):                        # a max reduction from 0 that skips NaN (fmax)
        r = dtype(0.0)
        for v in vs:
            r = np.fmax(r, np.fmax.reduce(v))
        return r

    m4 = dtype(4.0 * n)
    AL = dtype(0.5) * (LB + UB)
    ED = E @ AL
    g = E.T @ ED + mu_p * AL + F
    gmax, fmaxv = mx(np.abs(g)), mx(np.abs(F))
    lam0 = dtype(LAM0_REL) * gmax + dtype(1e-300)
    LU, LL = np.fmax(-g, 0.0) + lam0, np.fmax(g, 0.0) + lam0
    SU, SL = UB - AL, AL - LB
    KL = KR + ED
    clamp = dtype(1e-2) * kb
    clamped = int((kb - KL < clamp).sum() + (kb + KL < clamp).sum())
    S3, S4 = np.fmax(kb - KL, clamp), np.fmax(kb + KL, clamp)
    L3, L4 = np.full(n, lam0, dtype=dtype), np.full(n, lam0, dtype=dtype)
    mu0 = tot(SU * LU + SL * LL + (S3 + S4) * lam0) / m4
    rd_tol = dtype(RD_REL) * (fmaxv + gmax) + dtype(1e-300)
    mu, rdmax, rpmax = mu0, dtype(1e300), dtype(1e300)
    result, ex, trace = 2, "cap", []
    it = 0
    while it < MAX_ITER + 20:
        rp3, rp4 = KL + S3 - kb, -KL + S4 - kb
        WK = L3 / S3 + L4 / S4
        DD = LU / SU + LL / SL + mu_p
        VV = (KL - KR) + L3 * rp3 / S3 - L4 * rp4 / S4
        RHS = -F - E.T @ VV - mu_p * AL
        K = E.T @ (E * (1.0 + WK)[:, None])
        if mask is not None:
            K = np.where(mask, K, 0.0)
        K[np.diag_indices(n)] += DD
        Kf = K.astype(np.float64)                       # lambda_min / lambda_max of the matrix factored (0: not finite)
        kcond = float(np.divide(*np.linalg.eigvalsh(Kf)[[0, -1]])) if np.isfinite(Kf).all() else 0.0
        fac = _Factor(K, fast, None if perm is None else order)
        if not fac.ok:
            late = bool(mu <= 1e-7 * mu0 and rdmax <= 1e3 * rd_tol and rpmax <= 1e-6 * kb)
            result, ex = (0 if late else 3), "pivot"
            break
        DX = fac.solve(RHS, dtype)
        ED = E @ DX
        p, mm = DX / SU, DX / SL
        ds3, ds4 = -(KL + S3 - kb) - ED, -(-KL + S4 - kb) + ED
        dlu, dll = LU * (p - 1.0), -LL * (1.0 + mm)
        dl3, dl4 = -L3 - L3 * ds3 / S3, -L4 - L4 * ds4 / S4
        rp = mx(p, -mm, -ds3 / S3, -ds4 / S4)
        rdl = mx(1.0 - p, 1.0 + mm, -dl3 / L3, -dl4 / L4)
        ap_a = 1.0 / rp if rp > 1.0 else dtype(1.0)
        ad_a = 1.0 / rdl if rdl > 1.0 else dtype(1.0)
        c00 = tot(SU * LU + SL * LL + S3 * L3 + S4 * L4)
        c01 = tot(SU * dlu + SL * dll + S3 * dl3 + S4 * dl4)
        c10 = tot(DX * (LL - LU) + ds3 * L3 + ds4 * L4)
        c11 = tot(DX * (dll - dlu) + ds3 * dl3 + ds4 * dl4)
        sigma = (c00 + ad_a * c01 + ap_a * c10 + ap_a * ad_a * c11) / m4 / mu
        smu = sigma * sigma * sigma * mu
        TU = smu - SU * LU + DX * dlu
        TL = smu - SL * LL - DX * dll
        T3 = smu - S3 * L3 - ds3 * dl3
        T4 = smu - S4 * L4 - ds4 * dl4
        VV = (KL - KR) + L3 - L4 + (T3 + L3 * rp3) / S3 - (T4 + L4 * rp4) / S4
        RHS = -(F + LU - LL) - TU / SU + TL / SL - E.T @ VV - mu_p * AL
        DX = fac.solve(RHS, dtype)
        ED = E @ DX
        ds3, ds4 = -(KL + S3 - kb) - ED, -(-KL + S4 - kb) + ED
        dlu, dll = (TU + LU * DX) / SU, (TL - LL * DX) / SL
        dl3, dl4 = (T3 - L3 * ds3) / S3, (T4 - L4 * ds4) / S4
        rp = mx(DX / SU, -DX / SL, -ds3 / S3, -ds4 / S4)
        rdl = mx(-dlu / LU, -dll / LL, -dl3 / L3, -dl4 / L4)
        ap = ETA / rp if ETA < rp else dtype(1.0)
        ad = ETA / rdl if ETA < rdl else dtype(1.0)
        AL = AL + ap * DX
        SU, SL, S3, S4 = SU - ap * DX, SL + ap * DX, S3 + ap * ds3, S4 + ap * ds4
        LU, LL, L3, L4 = LU + ad * dlu, LL + ad * dll, L3 + ad * dl3, L4 + ad * dl4
        KL = KL + ap * ED
        mu = tot(SU * LU + SL * LL + S3 * L3 + S4 * L4) / m4
        rpmax = mx(np.abs(KL + S3 - kb), np.abs(-KL + S4 - kb))
        rdmax = mx(np.abs(E.T @ ((KL - KR) + L3 - L4) + mu_p * AL + F + LU - LL))
        it += 1
        trace.append(dict(mu=float(mu / mu0), rdmax=float(rdmax), rpmax=float(rpmax), ap_aff=float(ap_a),
                          ad_aff=float(ad_a), ap=float(ap), ad=float(ad), aff_full=(ap_a == 1.0, ad_a == 1.0),
                          full=(ap == 1.0, ad == 1.0), sigma=float(sigma), kcond=kcond,
                          margin=dict(mu=float(mu / (mu_rel * mu0)), rd=float(rdmax / rd_tol),
                                      rp=float(rpmax / (1e-8 * kb)), floor=float(mu / (1e-2 * mu_rel * mu0)))))
        if mu <= mu_rel * mu0 and rdmax <= rd_tol and rpmax <= 1e-8 * kb:
            result, ex = 0, "converged"
            break
        if mu <= 1e-2 * mu_rel * mu0:
            result = 0 if (rdmax <= 1e3 * rd_tol and rpmax <= 1e-6 * kb) else 2
            ex = "mu_floor"
            break
    alpha = AL.astype(LD)
    klin_max, cerr, _ = finalize(d, alpha)
    viol = not (klin_max <= S.ld(kb) * (1.0 + 1e-7))
    if override == "dense":
        status = 4 if viol else result
    else:
        status = 4 if (result == 0 and klin_max > S.ld(kb) * (1.0 + 1e-7)) else result
    return dict(status=status, iters=it, result=result, exit=ex, alpha=alpha, kappa_lin_max=klin_max,
                curv_error_max=cerr, trace=trace, clamped=clamped, mu0=float(mu0), rd_tol=float(rd_tol),
                mult=dict(lu=LU, ll=LL, l3=L3, l4=L4))


def permutation(n, seed=0):
    return np.random.default_rng(seed).permutation(n)


EPS64 = float(np.finfo(np.float64).eps)


def stability(d, kb, **kw):
    """The long-double replay and the two float64 replays (plain, and permuted: reductions in another order and, above
    DENSE_LD_MAX points, the factorisation in another elimination order) of one case: (ld run, stable, runs) with stable
    True where all three give the same status and iteration count.  runs[0]['unresolved']: some normal matrix the
    long-double run factored has lambda_min / lambda_max below the float64 epsilon, so that a float64 factorisation does
    not determine the step along its near-null direction (see statuses)."""
    r = replay(d, kb, **kw)
    r64 = replay(d, kb, dtype=np.float64, **kw)
    rp = replay(d, kb, dtype=np.float64, perm=permutation(d["n"]), **kw)
    runs = (r, r64, rp)
    r["unresolved"] = any(t["kcond"] < EPS64 for t in r["trace"])
    return r, len({(x["status"], x["iters"]) for x in runs}) == 1, runs


def statuses(runs):
    """The statuses the kernels may end in on a case: those of the three runs and, where the long-double run's last
    step was taken on a normal matrix float64 cannot resolve (lambda_min / lambda_max < eps) and it ended at a
    converged or mu-floor exit, both outcomes of the mu-floor test (0 and 2).  That last step lands on the same mu (on
    the H100 mu and both step lengths agree with the replay's to six digits), but the dual residual it leaves depends on how the
    particular float64 factorisation rounds along that direction: on the 200-point projection QPs the kernel's
    bordered band factor leaves |r_d| at 5.5e3 rd_tol where LAPACK and long double leave 1.7e-2 rd_tol, with
    lambda_min / lambda_max = 4e-17 at that step."""
    out = {x["status"] for x in runs}
    r = runs[0]
    if r["trace"] and r["trace"][-1]["kcond"] < EPS64 and r["exit"] in ("converged", "mu_floor"):
        out |= {0, 2}
    return out


def kappa_min(d):
    """(kb_min, alpha): the smallest curvature limit the rows can meet inside the box, min t over lb <= a <= ub,
    -t <= k_ref + E a <= t, by LP (HiGHS), with max |k_ref + E a| at the LP's vertex re-evaluated in long double."""
    import scipy.optimize
    E, kr = d["E"].astype(np.float64), d["k_ref"].astype(np.float64)
    n = d["n"]
    c = np.zeros(n + 1)
    c[-1] = 1.0
    one = np.ones((n, 1))
    A = np.vstack((np.hstack((E, -one)), np.hstack((-E, -one))))
    b = np.concatenate((-kr, kr))
    bounds = [(float(l), float(u)) for l, u in zip(d["lb"], d["ub"])] + [(0.0, None)]
    res = scipy.optimize.linprog(c, A_ub=A, b_ub=b, bounds=bounds, method="highs")
    assert res.status == 0, res.message
    a = S.ld(res.x[:n])
    return np.abs(d["k_ref"] + d["E"] @ a).max(), a


# ---- the constructed cases of tests/test_ipm_rows_ref_host.py and tests/test_gpu_ipm_rows_edges.py ----

def _closed(rt):
    return np.vstack((rt[:, :2], rt[0, :2]))


def track(rt, w_veh=2.0, f_scale=2.0, lin_alpha=None):
    """dict(rt, nv, h, w_veh, f_scale, lin_alpha, d): a closed track with the dense oracle's normals, its chord lengths
    as the spline scales, and its QP in long double."""
    from oracle import tph_dense as T
    rt = np.asarray(rt, dtype=np.float64)
    _, _, _, nv = T.calc_splines(_closed(rt))
    h = np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1)
    return dict(rt=rt, nv=nv, h=h, w_veh=w_veh, f_scale=f_scale, lin_alpha=lin_alpha,
                d=qp_data(rt, nv, h, w_veh, f_scale=f_scale, lin_alpha=lin_alpha))


def regimes(d, **kw):
    """The curvature limits of the four regimes of a QP: 'box' (only the box binds: 3x the rows' largest |kappa| at the
    box-only optimum), 'rows' (half way between kb_min and that value: the rows bind), 'feasible' (kb_min (1 + 1e-3))
    and 'infeasible' (kb_min (1 - 1e-3)); kb_min by kappa_min.  kw: the projection QP's arguments."""
    kbox = replay(d, 1e3, override="banded", **kw)["kappa_lin_max"]
    kmin, _ = kappa_min(d)
    out = dict(box=float(3.0 * kbox), feasible=float(kmin * (1 + 1e-3)), infeasible=float(kmin * (1 - 1e-3)))
    if kbox > kmin * (1 + 1e-2):
        out["rows"] = float(0.5 * (kmin + kbox))
    return out


def collapsed(n, seed=3):
    from global_racetrajectory_optimization_b200 import synth
    rt = synth.make_track(seed, n).copy()
    rt[n // 3, 2:] = 1.0                        # w_r + w_l == w_veh: lb == ub == 0 there (FIX_EPS widening)
    rt[(2 * n) // 3, 2:] = 1.0 + 2e-9           # a box just narrower than 2 FIX_EPS
    return rt


def lin_line(n):
    return 0.3 * np.sin(np.arange(n) * 0.37)


DENSE_NS = (3, 4, 5, 6, 7, 8, 15, 16, 17, 31, 32, 33, 63, 64, 65, 79, 80, 97, 108)
BANDED_NS = (80, 81, 96, 108, 130, 200, 333)


def dense_cases():
    """[(name, track dict, kb)] of the dense kernel: every size of DENSE_NS in each regime, strongly uneven spacing,
    collapsed boxes, a narrower vehicle, f_scale 1 and the LIN form, and the named cases that reach the exits of the
    iteration (f_scale 1e-12 puts the dual residual test at the edge of rounding; kb relative to kb_min)."""
    from global_racetrajectory_optimization_b200 import synth
    import mincurv_ref as R
    out = []
    for i, n in enumerate(DENSE_NS):
        rt = synth.make_track(1 + i, n)
        t = track(rt, w_veh=min(2.0, 0.5 * float((rt[:, 2] + rt[:, 3]).min())))     # (the widths of tiny tracks are capped)
        for reg, kb in regimes(t["d"]).items():
            out.append((f"synth{n}_{reg}", t, kb))
    more = [("uneven40_r20", track(R.uneven_track(40, 20.0, seed=1))), ("uneven64_r50", track(R.uneven_track(64, 50.0, seed=2))),
            ("collapsed31", track(collapsed(31))), ("collapsed64", track(collapsed(64))),
            ("wveh1.5_n33", track(synth.make_track(40, 33), w_veh=1.5)),
            ("fscale1_n16", track(synth.make_track(41, 16), f_scale=1.0)),
            ("fscale1_n65", track(synth.make_track(42, 65), f_scale=1.0)),
            ("lin_n17", track(synth.make_track(43, 17), lin_alpha=lin_line(17))),
            ("lin_n64", track(synth.make_track(44, 64), lin_alpha=lin_line(64))),
            ("lin_n97", track(synth.make_track(45, 97), lin_alpha=lin_line(97)))]
    for name, t in more:
        for reg, kb in regimes(t["d"]).items():
            out.append((f"{name}_{reg}", t, kb))
    # the exits (found by a search with this replay over synth tracks, f_scale and kb / kb_min)
    for name, seed, n, fac in (("exit_mu_floor_0", 1, 4, 1 + 1e-9), ("exit_mu_floor_2", 3, 4, 1 + 1e-7),
                               ("exit_pivot_late0", 5, 6, 3.0), ("exit_pivot_3", 7, 4, 1 + 1e-3)):
        t = track(synth.make_track(seed, n), f_scale=1e-12)
        out.append((name, t, float(kappa_min(t["d"])[0] * fac)))
    return out


def banded_cases():
    """[(name, track dict, kb)] of the banded curvature-row phase: BANDED_NS at a limit where the box-only optimum
    violates the rows and at kb_min (1 + 1e-3)."""
    from global_racetrajectory_optimization_b200 import synth
    out = []
    for i, n in enumerate(BANDED_NS):
        t = track(synth.make_track(60 + i, n))
        reg = regimes(t["d"])
        if "rows" in reg:
            out.append((f"banded{n}_rows", t, reg["rows"]))
        out.append((f"banded{n}_feasible", t, reg["feasible"]))
    return out


def prox_cases():
    """[(name, track dict, kb, mu, x, q)] of the projection QP (mincurv_pdip_kappa_kernel<true>) at two mu = l^-4: x a
    line through the box whose projection violates the rows, q a smooth linear term."""
    from global_racetrajectory_optimization_b200 import synth
    out = []
    for n, seed in ((120, 70), (200, 71)):
        t = track(synth.make_track(seed, n))
        d = t["d"]
        lb, ub = d["lb"].astype(np.float64), d["ub"].astype(np.float64)
        x = 0.5 * (lb + ub) + 0.45 * (ub - lb) * np.sin(np.arange(n) * 0.9)
        q = 1e-3 * np.cos(np.arange(n) * 0.21)
        for length in (5.0, 12.0):
            mu = length ** -4
            kbox = replay(d, 1e3, prox_mu=mu, prox_x=x, prox_q=q, override="banded")["kappa_lin_max"]
            kmin, _ = kappa_min(d)
            out.append((f"prox{n}_l{length:g}", t, float(0.5 * (kmin + kbox)), mu, x, q))
    return out
