"""Extended-precision reference of the linear algebra under the interior-point solvers and their adjoints (test
infrastructure, not product code): the dense matrices the device factorises, the normwise backward error of a computed
solution, and solutions exact to far below fp64 round-off.

The measure of a solve M v = g is the backward error of the diagonally scaled system (Rigal-Gaches, infinity norm)

    eta = |S (M v - g)| / (|S M S| |S^-1 v| + |S g|),    S = diag(M_ii)^-1/2,

with the residual in np.longdouble.  At the last iterate of an interior-point solve the diagonal D of M = H + D spans
1e-12 .. 1e12, cond(M) reaches 1e19 and any bound of the form u cond(M) is void; cond(S M S) stays near 1e5 .. 1e8, and
eta of a backward-stable solver is a small multiple of u = 1.1e-16 whatever D is.  The forward error in the scaled norm,
|S^-1 (v - x)| / |S^-1 x|, is then about eta cond(SMS) at most.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla

HBW = 32            # half-bandwidth of the minimum-curvature H (csrc/common.cuh)
U = np.finfo(np.float64).eps / 2
# The bounds of the device's solves (tests/test_gpu_linalg_edges.py).  device_model_solve on the fixtures' H at the
# diagonals of a final iterate reaches eta <= 6e-16 and a forward error <= 0.85 u cond(SMS)
# (tests/test_linalg_ref_host.py); the bounds are about 30 and 19 times that.  A wrong factor entry, a shifted diagonal or a
# missing strong row gives eta of 1e-11 and more.
ETA_MAX = 2e-14
FE_C = 16.0


def fe_bound(cond: float) -> float:
    """The bound of a scaled forward error (and of a gradient computed from the solution): FE_C u cond(SMS), with cond
    taken as at least 10 -- at cond(SMS) = 1 a few u remain, the rounding of the solution and of the gradient itself."""
    return FE_C * U * max(cond, 10.0)


def dense_from_device_band(hb, n: int, diag=None) -> np.ndarray:
    """Symmetric cyclic M from the device band rows hb[i][d] = M[i][(i + d) % n], d = 0..32 (HB_PITCH columns, any
    padding rows beyond n ignored), plus diag(diag)."""
    hb = np.asarray(hb, dtype=np.float64)
    M = np.zeros((n, n))
    i = np.arange(n)
    for d in range(HBW, -1, -1):             # (d = 0 last: the diagonal is its own mirror)
        M[(i + d) % n, i] = hb[:n, d]
        M[i, (i + d) % n] = hb[:n, d]
    if diag is not None:
        M[i, i] += np.asarray(diag, dtype=np.float64)[:n]
    return M


def with_strong_rows(K: np.ndarray, E_S: np.ndarray, W_S: np.ndarray) -> np.ndarray:
    """K + E_S^T diag(W_S) E_S: the rows carried by the Woodbury correction, added back densely."""
    E_S = np.asarray(E_S, dtype=np.float64)
    return K + E_S.T @ (np.asarray(W_S, dtype=np.float64)[:, None] * E_S)


def cyclic_tridiag(dg, off, dd) -> np.ndarray:
    """The shortest path's M: diagonal dg + dd, M[i][i+1] = M[i+1][i] = off[i], corner M[n-1][0] = M[0][n-1] = off[n-1]."""
    dg, off, dd = (np.asarray(a, dtype=np.float64) for a in (dg, off, dd))
    n = dg.size
    M = np.diag(dg + dd)
    i = np.arange(n - 1)
    M[i, i + 1] = M[i + 1, i] = off[:n - 1]
    M[n - 1, 0] = M[0, n - 1] = off[n - 1]
    return M


def _scaling(M):
    d = np.diag(M)
    if not np.all(d > 0.0):
        raise ValueError("the diagonal of M must be positive")
    return 1.0 / np.sqrt(np.asarray(d, dtype=np.longdouble))


def backward_error(M, v, g) -> float:
    """eta of the module docstring; the residual, the scaling and the norms in np.longdouble."""
    s = _scaling(M)
    Ml = np.asarray(M, dtype=np.longdouble)
    vl, gl = np.asarray(v, dtype=np.longdouble), np.asarray(g, dtype=np.longdouble)
    r = s * (Ml @ vl - gl)
    SMS = np.abs(Ml * s[:, None] * s[None, :]).sum(axis=1).max()
    den = SMS * np.abs(vl / s).max() + np.abs(s * gl).max()
    return float(np.abs(r).max() / den) if den > 0 else float(np.abs(r).max() > 0) * np.inf


def cond_scaled(M) -> float:
    """2-norm condition number of S M S (M symmetric positive definite)."""
    s = np.asarray(_scaling(M), dtype=np.float64)
    ev = np.linalg.eigvalsh(M * s[:, None] * s[None, :])
    return float(ev[-1] / ev[0]) if ev[0] > 0 else np.inf


def _refine(A, b, sweeps: int = 8):
    """y = A^-1 b (np.longdouble A, b): fp64 LU of A and iterative refinement with longdouble residuals and a
    longdouble iterate, which converges to about u_longdouble cond(A) relative when cond(A) << 1 / u."""
    lu = sla.lu_factor(np.asarray(A, dtype=np.float64))
    y = np.asarray(sla.lu_solve(lu, np.asarray(b, dtype=np.float64)), dtype=np.longdouble)
    for _ in range(sweeps):
        r = b - A @ y
        dy = sla.lu_solve(lu, np.asarray(r, dtype=np.float64))
        y = y + np.asarray(dy, dtype=np.longdouble)
        if np.abs(dy).max() <= 1e-3 * np.finfo(np.longdouble).eps * np.abs(y).max():
            break
    return y


def solve_extended(M, g, sweeps: int = 8) -> np.ndarray:
    """x = M^-1 g to well below fp64 round-off (np.longdouble): _refine on S M S, which has cond(SMS) << 1 / u."""
    s = _scaling(M)
    A = np.asarray(M, dtype=np.longdouble) * s[:, None] * s[None, :]
    return s * _refine(A, s * np.asarray(g, dtype=np.longdouble), sweeps)


def solve_extended_rows(K, E_S, W_S, g, sweeps: int = 12) -> np.ndarray:
    """x = (K + E_S^T diag(W_S) E_S)^-1 g to well below fp64 round-off (np.longdouble), K symmetric positive definite.
    With weights up to 1e15 the dense M is singular to fp64 and cannot even be stored without losing K to rounding, so
    the residual is formed as g - K x - E_S^T (W_S (E_S x)) in longdouble and the corrections come from an fp64 Woodbury
    solve (Cholesky of the scaled K and of the scaled Sigma = W_S^-1 + E_S K^-1 E_S^T)."""
    E = np.asarray(E_S, dtype=np.float64)
    W = np.asarray(W_S, dtype=np.float64)
    if W.size == 0:
        return solve_extended(K, g, sweeps)
    s = np.asarray(_scaling(K), dtype=np.float64)
    kc = sla.cho_factor(np.asarray(K, dtype=np.float64) * s[:, None] * s[None, :], lower=True)

    def ksolve(r):
        return (s * sla.cho_solve(kc, (s * r.T).T).T).T
    KE = ksolve(E.T)
    Sg = np.diag(1.0 / W) + E @ KE
    t = 1.0 / np.sqrt(np.diag(Sg))
    sc = sla.cho_factor(Sg * t[:, None] * t[None, :], lower=True)

    def wsolve(r):
        kr = ksolve(r)
        return kr - KE @ (t * sla.cho_solve(sc, t * (E @ kr)))
    Kl, El, Wl = (np.asarray(a, dtype=np.longdouble) for a in (K, E, W))
    gl = np.asarray(g, dtype=np.longdouble)
    x = np.asarray(wsolve(np.asarray(g, dtype=np.float64)), dtype=np.longdouble)
    for _ in range(sweeps):
        r = gl - Kl @ x - El.T @ (Wl * (El @ x))
        dx = wsolve(np.asarray(r, dtype=np.float64))
        x = x + np.asarray(dx, dtype=np.longdouble)
        if np.abs(dx).max() <= 1e-3 * np.finfo(np.longdouble).eps * np.abs(x).max():
            break
    return x


def solve_mpmath(M, g, dps: int = 50, rows=None) -> np.ndarray:
    """x = M^-1 g in mpmath at dps decimal digits (for n up to about 150), rounded to np.longdouble.  rows = (E_S, W_S):
    M + E_S^T diag(W_S) E_S, the sum formed in mpmath (in fp64 it would round K away next to weights of 1e15)."""
    import mpmath
    with mpmath.workdps(dps):
        A = mpmath.matrix(np.asarray(M, dtype=np.float64).tolist())
        if rows is not None:
            E = mpmath.matrix(np.asarray(rows[0], dtype=np.float64).tolist())
            A += E.T * mpmath.diag([mpmath.mpf(float(w)) for w in rows[1]]) * E
        x = mpmath.lu_solve(A, mpmath.matrix(np.asarray(g, dtype=np.float64).tolist()))
        return np.array([np.longdouble(mpmath.nstr(xi, dps)) for xi in x], dtype=np.longdouble)


def forward_error(M, v, x) -> float:
    """|S^-1 (v - x)| / |S^-1 x| (infinity norm, longdouble), x the exact solution, S = diag(M)^-1/2 (for a system with
    strong rows, M = K)."""
    s = _scaling(M)
    vl, xl = np.asarray(v, dtype=np.longdouble), np.asarray(x, dtype=np.longdouble)
    return float(np.abs((vl - xl) / s).max() / np.abs(xl / s).max())


def rel_err(got, ref) -> float:
    """max |got - ref| / max |ref| (longdouble)."""
    g, r = np.asarray(got, dtype=np.longdouble), np.asarray(ref, dtype=np.longdouble)
    return float(np.abs(g - r).max() / max(np.abs(r).max(), np.longdouble(1e-300)))


# ---- a model of the device's elimination order (csrc/mincurv_ipm.cu, factor / solve), to set the GPU bounds on CPU ----

def device_model_solve(M, g, panel: int = 8, sep: int = HBW) -> np.ndarray:
    """Solve M x = g in fp64 the way the interior-point kernel does: LDL^T in natural order with the last `sep` nodes
    as the separator; the chain's forward and backward sweeps one panel of eight at a time, each panel's triangular
    solve a mat-vec with the explicit inverse Q = L11^-1 of its unit-lower block; the separator's block by plain
    substitution."""
    n = M.shape[0]
    na = n - sep
    A = np.array(M, dtype=np.float64)
    L = np.eye(n)
    d = np.zeros(n)
    for k in range(n):
        d[k] = A[k, k]
        if not d[k] > 0.0:
            raise FloatingPointError(f"non-positive pivot at {k}")
        w = 1.0 / d[k]
        v = A[k + 1:, k].copy()
        L[k + 1:, k] = v * w
        A[k + 1:, k + 1:] -= np.outer(L[k + 1:, k], v)
    panels = [(k0, min(k0 + panel, na)) for k0 in range(0, na, panel)]
    Qs = [sla.solve_triangular(L[a:b, a:b], np.eye(b - a), lower=True, unit_diagonal=True) for a, b in panels]
    y = np.array(g, dtype=np.float64)
    for (a, b), Q in zip(panels, Qs):
        y[a:b] = Q @ y[a:b]
        y[b:] -= L[b:, a:b] @ y[a:b]
    y[na:] = sla.solve_triangular(L[na:, na:], y[na:], lower=True, unit_diagonal=True)
    z = y / d
    x = np.zeros(n)
    x[na:] = sla.solve_triangular(L[na:, na:].T, z[na:], lower=False, unit_diagonal=True)
    for (a, b), Q in reversed(list(zip(panels, Qs))):
        x[a:b] = Q.T @ (z[a:b] - L[b:, a:b].T @ x[b:])
    return x
