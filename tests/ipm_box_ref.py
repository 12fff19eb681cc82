"""Replay (np.longdouble by default) of the box phase of the minimum-curvature QP, the Mehrotra iteration that
mincurv_pdip_kernel (K2b, csrc/mincurv_ipm.cu) runs on

    min 1/2 a^T H a + f^T a,   lb <= a <= ub,      H the cyclic band of half-width 32 of E^T E

statement by statement: the start at the box centre with g0 = H a0 + f and lam0 = lam0_rel max|g0| + 1e-300, mu0 and
rd_tol, the affine direction with its step lengths from the max-ratios, the four c-sums of mu_aff and the cubic
centring, the corrector terms and the corrector's right-hand side, the damped steps, the update with the carried dual
residual rd + ap (rhs - D dx) + ad (dlu - dll) and the slacks carried as variables of their own, and the exits in the
kernel's order (converged: mu, r_d and the step test; the mu floor, status 0 or 2; the cap, status 2; a non-positive
pivot, status 3).

The factor is the kernel's elimination order: a chain band of half-width 32 over the first n - 32 points, bordered by
the 32 separator rows, factored column by column (LL^T, each column's update vectorised over the band), then the dense
separator.  rotate=k runs the same QP with its indices rotated cyclically by k (an exact symmetry: another elimination
order, the separator elsewhere, other summation orders) and rotates the result back.
Test infrastructure, not product code."""
import numpy as np

import ipm_rows_ref as IR

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "the interior-point replay needs an 80-bit or quad long double"
HBW = 32                    # common.cuh: half-bandwidth of H
N_MIN = 80                  # common.cuh: the band must not wrap onto itself
FIX_EPS = IR.FIX_EPS
# the PdipParams mc_mincurv_pdip_batch sets (the MC_DEBUG_PDIP_* knobs override them)
MAX_ITER = 40
MU_REL = 1e-10
RD_REL = 1e-8
ETA = 0.995
DX_REL = 1e-5
LAM0_REL = 1e-2
COND_N_MAX = 600            # lambda_min / lambda_max of the factored matrix is traced up to this n (a dense eigvalsh)


# ---- the QP of one instance: (hb [n, 33], f, lb, ub) ----

def box(reftrack, w_veh):
    """(lb, ub) in long double as mincurv_setup.cu forms them (FIX_EPS widening of collapsed boxes); None where some
    lb > ub (status 1)."""
    rt = np.asarray(reftrack, dtype=np.float64)
    ub = rt[:, 2].astype(LD) - 0.5 * LD(w_veh)
    lb = -(rt[:, 3].astype(LD) - 0.5 * LD(w_veh))
    if (lb > ub).any():
        return None
    col = ub - lb < 2.0 * FIX_EPS
    mid = 0.5 * (lb + ub)
    return np.where(col, mid - FIX_EPS, lb), np.where(col, mid + FIX_EPS, ub)


def band_of(K, w=HBW):
    """Cyclic band rows hb[i][d] = K[i][(i + d) % n], d = 0..w, of a symmetric K [n, n]."""
    n = K.shape[0]
    i = np.arange(n)
    return np.stack([K[i, (i + d) % n] for d in range(w + 1)], axis=1)


def qp(hb, f, lb, ub):
    return dict(n=len(f), hb=np.asarray(hb).astype(LD), f=np.asarray(f).astype(LD), lb=np.asarray(lb).astype(LD),
                ub=np.asarray(ub).astype(LD))


def qp_of_track(t):
    """The box-phase QP of an ipm_rows_ref.track: the long-double band of E^T E cut to half-width 32, f = f_scale
    E^T k_ref and the box of qp_data (None: status 1)."""
    d = t["d"]
    if d is None:
        return None
    E = d["E"]
    return qp(band_of(E.T @ E), d["f"], d["lb"], d["ub"])


def qp_of_fixture(g):
    """The box-phase QP of a golden fixture: its H_band and f (the oracle's float64 assembly) and the box of its
    reftrack and w_veh."""
    b = box(g["reftrack"], float(g["w_veh"]))
    return None if b is None else qp(g["H_band"], g["f"], *b)


def dense(hb, diag=None):
    """The symmetric cyclic matrix of band rows hb [n, 33] plus diag(diag), in the band's dtype."""
    n = hb.shape[0]
    M = np.zeros((n, n), dtype=hb.dtype)
    i = np.arange(n)
    for d in range(HBW, -1, -1):
        M[(i + d) % n, i] = hb[:, d]
        M[i, (i + d) % n] = hb[:, d]
    if diag is not None:
        M[i, i] += diag
    return M


def matvec(hb, v):
    """H v of the cyclic band (in the dtype of hb and v)."""
    n = hb.shape[0]
    out = hb[:, 0] * v
    for d in range(1, HBW + 1):
        out = out + hb[:, d] * np.roll(v, -d) + np.roll(hb[:, d] * v, d)
    return out


def rotate_qp(q, k):
    """The same QP with its indices rotated: point i of the result is point (i + k) % n of q."""
    return dict(n=q["n"], **{key: np.roll(q[key], -k, axis=0) for key in ("hb", "f", "lb", "ub")})


# ---- the bordered band factor of M = H + diag(D) ----

class BandFactor:
    """LL^T of the cyclic band M (rows hb [n, 33] plus diag D) in the order of the kernel's factor: the chain of the
    first NA = n - 32 points as a band of half-width 32, with the 32 separator rows as its border, then the dense
    32 x 32 Schur complement.  ok False: a non-positive pivot (chain or separator), as factor() reports it."""

    def __init__(self, hb, D):
        n = hb.shape[0]
        assert n >= N_MIN, n
        dt = hb.dtype
        NA = n - HBW
        self.n, self.NA = n, NA
        M = hb.copy()
        M[:, 0] = M[:, 0] + D
        # chain columns k: Lb[k, d] = M[k + d, k] for k + d < NA (32 zero rows of padding below)
        Lb = np.zeros((NA + HBW + 1, HBW + 1), dtype=dt)
        k = np.arange(NA)
        dd = np.arange(HBW + 1)
        inside = k[:, None] + dd[None, :] < NA
        Lb[:NA] = np.where(inside, M[:NA], 0.0)
        # border F[k, r] = M[NA + r, k]: directly (NA + r - k <= 32) or across the wrap (k <= r)
        F = np.zeros((NA + HBW + 1, HBW), dtype=dt)
        for r in range(HBW):
            lo = max(NA + r - HBW, 0)
            F[lo:NA, r] = M[lo:NA, :][np.arange(NA - lo), NA + r - np.arange(lo, NA)]
            F[:r + 1, r] = M[NA + r, HBW - r + np.arange(r + 1)]
        i = np.arange(HBW)
        lo, dist = np.minimum(i[:, None], i[None, :]), np.abs(i[:, None] - i[None, :])
        S = M[NA + lo, dist]
        # the column update of the band: column k + j (j = 1..32) loses c[j + d - 1] c[j - 1] at offset d
        J, Dd = np.nonzero(np.add.outer(np.arange(1, HBW + 1), np.arange(HBW + 1)) <= HBW)
        J = J + 1
        self.ok = True
        for c in range(NA):
            p = Lb[c, 0]
            if not p > 0.0:
                self.ok = False
                return
            l = np.sqrt(p)
            Lb[c, 0] = l
            Lb[c, 1:] /= l
            F[c] /= l
            col = Lb[c, 1:]
            Lb[c + J, Dd] -= col[J + Dd - 1] * col[J - 1]
            F[c + 1:c + HBW + 1] -= np.outer(col, F[c])
            S = S - np.outer(F[c], F[c])
        self.LS = IR._chol(S)
        if self.LS is None:
            self.ok = False
            return
        self.Lb, self.F = Lb, F

    def solve(self, g):
        NA, Lb, F = self.NA, self.Lb, self.F
        y = np.zeros(NA + HBW + 1, dtype=g.dtype)
        y[:NA] = g[:NA]
        for c in range(NA):
            y[c] /= Lb[c, 0]
            y[c + 1:c + HBW + 1] -= Lb[c, 1:] * y[c]
        gs = g[NA:] - F[:NA].T @ y[:NA]
        xs = IR._chol_solve(self.LS, gs)
        t = y[:NA] - F[:NA] @ xs
        x = np.zeros(NA + HBW + 1, dtype=g.dtype)
        for c in range(NA - 1, -1, -1):
            x[c] = (t[c] - Lb[c, 1:] @ x[c + 1:c + HBW + 1]) / Lb[c, 0]
        x[NA:NA + HBW] = xs
        return x[:NA + HBW]


# ---- the iteration ----

def replay(q, dtype=LD, rotate=0, max_iter=MAX_ITER, mu_rel=MU_REL, dx_rel=DX_REL, lam0_rel=LAM0_REL, eta=ETA,
           cond=None):
    """Run the box phase on the QP q (qp, qp_of_track, qp_of_fixture).  Returns dict(status, iters, exit, decided,
    alpha, su, sl, lu, ll, rd, D, mu, mu0, rd_tol, trace), the vectors in long double and in the order of q.
    exit: 'converged' / 'mu_floor' / 'cap' / 'pivot'.  decided (converged only): the tests among 'mu', 'rd', 'step' that
    failed one iteration earlier (None if the first iteration converged).  D: the barrier diagonal lu / su + ll / sl of
    the final state (what the update pass leaves in DD).  trace: per iteration mu / mu0, the carried and the exact
    |r_d| / rd_tol, the step-test ratio ap max|dx| / (dx_rel' max(max|a|, 0.01)) (dx_rel' = dx_rel, or the default
    where dx_rel = 0), whether the 1 cm floor is active, the affine and the damped ap / ad, and lambda_min / lambda_max
    of the matrix factored (cond: always / never / None: up to COND_N_MAX points)."""
    with np.errstate(all="ignore"):
        return _replay(q, dtype, rotate, max_iter, mu_rel, dx_rel, lam0_rel, eta, cond)


def _replay(q, dtype, rotate, max_iter, mu_rel, dx_rel, lam0_rel, eta, cond):
    n = q["n"]
    if rotate:
        q = rotate_qp(q, rotate)
    HB, F, LB, UB = (q[k].astype(dtype) for k in ("hb", "f", "lb", "ub"))
    HBL, FL = q["hb"].astype(LD), q["f"].astype(LD)
    want_cond = (n <= COND_N_MAX) if cond is None else cond
    one = dtype(1.0)
    m2 = dtype(2.0 * n)
    # initial point: box centre, multipliers from the gradient
    AL = dtype(0.5) * (LB + UB)
    G0 = matvec(HB, AL) + F
    gmax, fmaxv = np.abs(G0).max(), np.abs(F).max()
    lam0 = dtype(lam0_rel) * gmax + dtype(1e-300)
    LU, LL = np.fmax(-G0, 0.0) + lam0, np.fmax(G0, 0.0) + lam0
    RD = G0 + LU - LL
    SU, SL = UB - AL, AL - LB
    DD = LU / SU + LL / SL
    RHS = -RD + LU - LL
    mu0 = (SU * LU + SL * LL).sum() / m2
    rd_tol = dtype(RD_REL) * (fmaxv + gmax) + dtype(1e-300)
    mu = mu0
    status, ex, trace = None, "cap", []
    it = 0
    dxr = dtype(dx_rel if dx_rel > 0.0 else DX_REL)
    while it < max_iter:
        Kcond = None
        if want_cond:
            Mf = dense(HB.astype(np.float64), DD.astype(np.float64))
            Kcond = float(np.divide(*np.linalg.eigvalsh(Mf)[[0, -1]])) if np.isfinite(Mf).all() else 0.0
        fac = BandFactor(HB, DD)
        if not fac.ok:
            status, ex = 3, "pivot"
            break
        DXA = fac.solve(RHS)
        # affine direction: step lengths 1 / max-ratio, mu_aff as a polynomial in (ap, ad)
        p, m = DXA / SU, DXA / SL
        rp = max(dtype(0.0), np.fmax(p, -m).max())
        rdl = max(dtype(0.0), np.fmax(1.0 - p, 1.0 + m).max())
        dlu, dll = LU * (p - 1.0), -LL * (1.0 + m)
        c00 = (SU * LU + SL * LL).sum()
        c01 = (SU * dlu + SL * dll).sum()
        c10 = (DXA * (LL - LU)).sum()
        c11 = (DXA * (dll - dlu)).sum()
        ap_a = one / rp if rp > 1.0 else one
        ad_a = one / rdl if rdl > 1.0 else one
        sigma = (c00 + ad_a * c01 + ap_a * c10 + ap_a * ad_a * c11) / m2 / mu
        smu = sigma * sigma * sigma * mu
        # corrector
        TU = smu - SU * LU + DXA * dlu
        TL = smu - SL * LL - DXA * dll
        RHS = -RD - TU / SU + TL / SL
        DX = fac.solve(RHS)
        dlu, dll = (TU + LU * DX) / SU, (TL - LL * DX) / SL
        rp = max(dtype(0.0), np.fmax(DX / SU, -DX / SL).max())
        rdl = max(dtype(0.0), np.fmax(-dlu / LU, -dll / LL).max())
        ap = dtype(eta) / rp if eta < rp else one
        ad = dtype(eta) / rdl if eta < rdl else one
        # update: the state, the carried dual residual, the next D and right-hand side
        AL = AL + ap * DX
        LU, LL = LU + ad * dlu, LL + ad * dll
        RD = RD + ap * (RHS - DD * DX) + ad * (dlu - dll)
        SU, SL = SU - ap * DX, SL + ap * DX
        DD = LU / SU + LL / SL
        RHS = -RD + LU - LL
        mu = (SU * LU + SL * LL).sum() / m2
        rdmax = np.abs(RD).max()
        dxmax, amax = np.abs(DX).max(), np.abs(AL).max()
        it += 1
        exact = np.abs(matvec(HBL, AL.astype(LD)) + FL + LU.astype(LD) - LL.astype(LD)).max()
        step = float(ap * dxmax / (dxr * max(amax, dtype(0.01))))
        trace.append(dict(mu=float(mu / mu0), rd=float(rdmax / rd_tol), rd_exact=float(exact / LD(rd_tol)), step=step,
                          amax=float(amax), floor=bool(amax < 0.01), ap_aff=float(ap_a), ad_aff=float(ad_a), ap=float(ap), ad=float(ad),
                          sigma=float(sigma), kcond=Kcond,
                          ok=dict(mu=bool(mu <= mu_rel * mu0), rd=bool(rdmax <= rd_tol), step=step <= 1.0)))
        settled = True
        if dx_rel > 0.0 and mu <= mu_rel * mu0:
            settled = ap * dxmax <= dtype(dx_rel) * max(amax, dtype(0.01))
        if mu <= mu_rel * mu0 and rdmax <= rd_tol and settled:
            status, ex = 0, "converged"
            break
        if mu <= 1e-4 * mu_rel * mu0:
            status, ex = (0 if rdmax <= 1e3 * rd_tol else 2), "mu_floor"
            break
    if status is None:
        status = 2
    decided = None
    if ex == "converged" and len(trace) > 1:
        decided = tuple(k for k in ("mu", "rd", "step") if not trace[-2]["ok"][k])

    def back(v):
        v = v.astype(LD)
        return np.roll(v, rotate) if rotate else v
    return dict(status=status, iters=it, exit=ex, decided=decided, alpha=back(AL), su=back(SU), sl=back(SL),
                lu=back(LU), ll=back(LL), rd=back(RD), D=back(DD), mu=float(mu), mu0=float(mu0), rd_tol=float(rd_tol),
                trace=trace)


def stability(q, **kw):
    """The long-double replay, the float64 replay and the float64 replay rotated by n // 3: (ld run, stable, runs), stable
    True where all three end in the same (status, iters)."""
    r = replay(q, **kw)
    r64 = replay(q, dtype=np.float64, **kw)
    rr = replay(q, dtype=np.float64, rotate=q["n"] // 3, **kw)
    runs = (r, r64, rr)
    return r, len({(x["status"], x["iters"]) for x in runs}) == 1, runs


def outcomes(runs):
    return {(x["status"], x["iters"]) for x in runs}


# ---- constructed cases ----

def synth_track(n, seed=None, w_veh=2.0, f_scale=2.0):
    from global_racetrajectory_optimization_b200 import synth
    return IR.track(synth.make_track(n if seed is None else seed, n), w_veh=w_veh, f_scale=f_scale)


def narrow_track(n=120, seed=5, half=0.004):
    """A track whose boxes are |a| <= half (< 5 mm) everywhere: the 1 cm floor of the step test is active."""
    from global_racetrajectory_optimization_b200 import synth
    rt = synth.make_track(seed, n).copy()
    rt[:, 2] = 1.0 + half
    rt[:, 3] = 1.0 + half
    return IR.track(rt, w_veh=2.0)


def uneven(n, ratio, seed=1, w_veh=2.0):
    import mincurv_ref as R
    return IR.track(R.uneven_track(n, ratio, seed=seed), w_veh=w_veh)


KNOB_ENV = dict(lam0_rel="MC_DEBUG_PDIP_LAM0", eta="MC_DEBUG_PDIP_ETA", dx_rel="MC_DEBUG_PDIP_DX_REL",
                mu_rel="MC_DEBUG_PDIP_MU_REL")


def exit_cases():
    """name -> (track dict, knobs): constructed cases that reach the exits the fixtures do not (found by a search with
    this replay; knobs are replay arguments, set on the device through KNOB_ENV).
    floor_narrow   boxes |a| <= 2 mm: converged where the step test passes only through its 1 cm floor
    mu_floor_0     lam0 = 1e4 max|g0|: mu falls 1e4 below the stopping test while |r_d| is between 1 and 1e3 rd_tol
    mu_floor_2     lam0 = 1e6 max|g0|: likewise with |r_d| above 1e3 rd_tol
    cap            mu_rel = 1e-300: no test can pass, 40 iterations"""
    return dict(floor_narrow=(narrow_track(120, 6, 0.002), {}),
                mu_floor_0=(synth_track(96), dict(lam0_rel=1e4)),
                mu_floor_2=(synth_track(96), dict(lam0_rel=1e6)),
                cap=(synth_track(96), dict(mu_rel=1e-300)))
