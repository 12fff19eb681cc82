"""Exact CPU reference of the shortest-path QP in float64 (test infrastructure, not product code), written from the QP's
definition (tests/sp_sens.py, oracle.tph_dense.assemble_shortest_path):

    min 1/2 a^T H a + f^T a   s.t.  lb <= a <= ub
    H_ii = 4 |n_i|^2,  H_i,i+1 = H_i+1,i = -2 n_i.n_{i+1},  f_i = 2 n_i.(2 p_i - p_{i+1} - p_{i-1})   (cyclic)
    ub = max(w_right - w_veh / 2, 0.001),  lb = -max(w_left - w_veh / 2, 0.001)

assemble() builds diag, off (off[i] couples i and i + 1 mod n), f, lb and ub of a whole ragged batch; solve_exact()
finds one instance's exact active set and proves it with the KKT sign conditions; certificate() measures how far the
alpha of every instance of a batch is from optimal.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

CLAMP = 0.001           # tph's lower limit of w - w_veh / 2
FREE_SLACK = 1e-3       # [m] a point this far inside both bounds counts as free in certificate()
GI_MAX_N = 200          # up to here the active set comes from Goldfarb-Idnani (H need not be an M-matrix on small tracks)
GI_FALLBACK_MAX_N = 3000    # dense Goldfarb-Idnani is O(N^3): no fallback above this
MAX_SWEEPS = 50         # sweeps before the Goldfarb-Idnani fallback; 4x that without one (measured: 18-21 at N = 500-2000, 75 at
                        # N = 10 000 on synthetic tracks)


def _rows(n_pts, B, N):
    """Points per row; rows the kernel does not solve (n < 3 or n > N) count as empty."""
    n = np.full(B, N) if n_pts is None else np.asarray(n_pts, dtype=np.int64).reshape(B)
    return np.where((n >= 3) & (n <= N), n, 0)


def _neighbours(n, N):
    """ip, im [B, N]: the cyclic next and previous point of every point; a padding point is its own neighbour."""
    i = np.arange(N)[None, :]
    m = n[:, None]
    ip = np.where(i < m, np.where(i + 1 < m, i + 1, 0), i)
    im = np.where(i < m, np.where(i > 0, i - 1, m - 1), i)
    return ip, im


def assemble(reftrack, normvec, w_veh, n_pts=None):
    """(diag, off, f, lb, ub), each [B, N] ([N] for a single track [N, 4]).  w_veh: a number or one per track.  The
    padding (i >= n_pts, and every point of a row with n_pts < 3 or > N) gets diag 1, off 0, f 0, lb = ub = 0, whatever
    the inputs hold there, so that its solution is 0."""
    rt = np.asarray(reftrack, dtype=float)
    nv = np.asarray(normvec, dtype=float)
    single = rt.ndim == 2
    if single:
        rt, nv = rt[None], nv[None]
    B, N = rt.shape[:2]
    n = _rows(n_pts, B, N)
    ip, im = _neighbours(n, N)
    r = np.arange(B)[:, None]
    p = rt[..., :2]
    pad = np.arange(N)[None, :] >= n[:, None]
    diag = 4.0 * (nv[..., 0] * nv[..., 0] + nv[..., 1] * nv[..., 1])
    off = -2.0 * (nv[..., 0] * nv[r, ip, 0] + nv[..., 1] * nv[r, ip, 1])
    c = 2.0 * p - p[r, ip] - p[r, im]
    f = 2.0 * (nv[..., 0] * c[..., 0] + nv[..., 1] * c[..., 1])
    wv = np.broadcast_to(np.asarray(w_veh, dtype=float).reshape(-1), (B,))[:, None]
    ub = np.maximum(rt[..., 2] - wv / 2, CLAMP)
    lb = -np.maximum(rt[..., 3] - wv / 2, CLAMP)
    out = tuple(np.where(pad, v, x) for x, v in ((diag, 1.0), (off, 0.0), (f, 0.0), (lb, 0.0), (ub, 0.0)))
    return tuple(x[0] for x in out) if single else out


def matrix(diag, off):
    """H of one instance as a sparse CSR matrix."""
    n = diag.size
    H = sp.diags([off[:-1], diag, off[:-1]], [-1, 0, 1], format="lil")
    H[n - 1, 0] = H[0, n - 1] = off[n - 1]
    return H.tocsr()


def _solve_on(H, f, lb, ub, upper, lower):
    """alpha with the points of upper / lower on their bound and H a + f = 0 on the rest; and g = H a + f."""
    a = np.where(upper, ub, np.where(lower, lb, 0.0))
    free = ~(upper | lower)
    if free.any():
        act = ~free
        rhs = -f[free] - H[free][:, act] @ a[act]
        a[free] = spla.spsolve(H[free][:, free].tocsc(), rhs) if free.sum() > 1 else rhs / H[free][:, free].toarray()[0]
    return a, H @ a + f


def _gi_active_set(H, f, lb, ub):
    """(upper, lower) of the Goldfarb-Idnani solution (the solver of sp_sens.solve): its bounds with a positive multiplier."""
    from oracle.quadprog_gi import solve_qp
    n = f.size
    C = np.hstack((-np.eye(n), np.eye(n)))                  # -a >= -ub, a >= lb
    lag = solve_qp(H.toarray(), -f, C, np.concatenate((-ub, lb)), 0)[4]
    return lag[:n] > 0, lag[n:] > 0


def solve_exact(diag, off, f, lb, ub):
    """The exact solution of one instance ([n] arrays).  A primal-dual active-set iteration with a sparse solve on the free
    points; it ends when the active set reproduces itself, which is when every free point lies in its box, every upper
    bound has a positive multiplier -g and every lower bound a positive multiplier g.  On an M-matrix H (consecutive
    normals with a positive dot product) it ends after finitely many sweeps.  Small tracks need not have one, so for
    n <= GI_MAX_N, or when the iteration does not settle, it starts from Goldfarb-Idnani's active set instead.  Raises
    unless the KKT conditions hold at the result."""
    diag, off, f, lb, ub = (np.asarray(x, dtype=float) for x in (diag, off, f, lb, ub))
    n = f.size
    if not all(np.isfinite(x).all() for x in (diag, off, f, lb, ub)) or (lb > ub).any():
        raise ValueError("solve_exact: non-finite or empty box")
    H = matrix(diag, off)
    starts = ["gi"] if n <= GI_MAX_N else ["cold", "gi"] if n <= GI_FALLBACK_MAX_N else ["cold"]
    sweeps = MAX_SWEEPS if n <= GI_FALLBACK_MAX_N else 4 * MAX_SWEEPS
    for start in starts:
        if start == "gi":
            upper, lower = _gi_active_set(H, f, lb, ub)
        else:
            upper = lower = np.zeros(n, dtype=bool)
        for _ in range(sweeps):
            a, g = _solve_on(H, f, lb, ub, upper, lower)
            lam = np.where(upper | lower, -g, 0.0)            # > 0 pushes against ub, < 0 against lb
            z = a + lam / diag
            nu = np.where(upper, lam > 0, z > ub)
            nl = np.where(lower, lam < 0, z < lb) & ~nu
            if np.array_equal(nu, upper) and np.array_equal(nl, lower):
                _check_kkt(a, g, f, lb, ub, upper, lower)
                return a
            upper, lower = nu, nl
    raise RuntimeError(f"solve_exact: the active set did not settle (n = {n})")


def _check_kkt(a, g, f, lb, ub, upper, lower):
    free = ~(upper | lower)
    scale = max(np.abs(f).max(), 1e-300)
    ok = (np.isfinite(a).all() and (a >= lb).all() and (a <= ub).all() and (a[upper] == ub[upper]).all()
          and (a[lower] == lb[lower]).all() and (g[upper] < 0).all() and (g[lower] > 0).all()
          and (np.abs(g[free]).max(initial=0.0) <= 1e-9 * scale))
    if not ok:
        raise RuntimeError("solve_exact: the KKT conditions do not hold at the settled active set")


def certificate(diag, off, f, lb, ub, alpha, n_pts=None) -> dict:
    """Optimality measures of every instance ([B] arrays; numbers for [N] inputs), over its n_pts points, with g = H a + f
    and a point counted at a bound when its projected step a - g / diag lands on that bound or beyond.  An interior-point
    iterate is never on a bound; a point of it within FREE_SLACK of one is measured by pg and comp, not by stat:
        box     max violation of lb <= a <= ub [m]
        pg      projected-gradient residual max |a - clip(a - g / diag, lb, ub)| [m]
        stat    max |g| over the free points (at least FREE_SLACK inside both bounds) / max |f|
        comp    complementarity max(mu_u (ub - a) + mu_l (a - lb)) / max |f| [m], mu_u = max(-g, 0) at the upper bounds,
                mu_l = max(g, 0) at the lower bounds
        active  the number of points at a bound
    It asserts nothing."""
    arrs = [np.asarray(x, dtype=float) for x in (diag, off, f, lb, ub, alpha)]
    single = arrs[0].ndim == 1
    if single:
        arrs = [x[None] for x in arrs]
    diag, off, f, lb, ub, a = arrs
    B, N = a.shape
    n = _rows(n_pts, B, N)
    ip, im = _neighbours(n, N)
    r = np.arange(B)[:, None]
    valid = np.arange(N)[None, :] < n[:, None]
    a = np.where(valid, a, 0.0)
    g = diag * a + off * a[r, ip] + off[r, im] * a[r, im] + f
    z = a - g / diag
    at_u, at_l = valid & (z >= ub), valid & (z <= lb) & ~(z >= ub)
    free = valid & (ub - a >= FREE_SLACK) & (a - lb >= FREE_SLACK)
    scale = np.maximum(np.abs(np.where(valid, f, 0.0)).max(axis=1), 1e-300)

    def vmax(x, where):
        return np.where(where, x, 0.0).max(axis=1)
    out = dict(box=vmax(np.maximum(a - ub, lb - a).clip(min=0.0), valid),
               pg=vmax(np.abs(a - np.clip(z, lb, ub)), valid),
               stat=vmax(np.abs(g), free) / scale,
               comp=np.maximum(vmax(np.maximum(-g, 0.0) * np.abs(ub - a), at_u),
                               vmax(np.maximum(g, 0.0) * np.abs(a - lb), at_l)) / scale,
               active=(at_u | at_l).sum(axis=1))
    return {k: v[0].item() for k, v in out.items()} if single else out


# ---- inputs shared by the host and the device tests ----
def polygon_track(n: int, seed: int) -> np.ndarray:
    """reftrack [n, 4] of a perturbed regular n-gon, counter-clockwise, about 3 m between points (at least 6 m radius),
    widths 1.2 ... 3.5 m."""
    rng = np.random.default_rng(seed)
    R = max(3.0 * n / (2.0 * np.pi), 6.0)
    th = 2.0 * np.pi * (np.arange(n) + rng.uniform(-0.2, 0.2, n)) / n
    r = R * (1.0 + rng.uniform(-0.05, 0.05, n))
    return np.column_stack((r * np.cos(th), r * np.sin(th), rng.uniform(1.2, 3.5, n), rng.uniform(1.2, 3.5, n)))


def box_variants(reftrack: np.ndarray):
    """[(name, reftrack, w_veh)]: one centre line in every box regime of the shortest path."""
    w = reftrack[:, 2:]
    right = reftrack.copy()
    right[:, 2] = 0.8                                       # < w_veh / 2: ub clamped to 0.001 everywhere
    wide, tight = reftrack.copy(), reftrack.copy()
    wide[:, 2:] *= 20.0                                     # no bound active
    tight[:, 2:] *= 0.3                                     # most bounds active, some clamped
    return [("both_clamped", reftrack, 2.0 * float(w.max()) + 1.0), ("right_clamped", right, 2.0),
            ("interior", wide, 2.0), ("tight", tight, 2.0), ("w_veh_2.6", reftrack, 2.6)]
