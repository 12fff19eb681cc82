"""A float64 torch restatement of create_raceline (tph.create_raceline + calc_head_curv_an's kappa), the reference of
its derivative: autograd of this function, at the station segments and the station count the forward chose, is what the
create_raceline adjoint (create_raceline_adjoint_kernel) must give.  Dense cyclic moment solve, 15-sample polyline
lengths, cumulative sum, linspace stations, searchsorted, head_curv.  Test infrastructure, not product code."""
import math

import torch

T15 = torch.linspace(0.0, 1.0, 15, dtype=torch.float64)


def coefficients(P):
    """Closed spline through P [n, 2] with unit parameter scales: coefficients cx, cy [n, 4] (tph.calc_splines,
    use_dist_scaling=False): m = A^-1 6 D2 p with A = circ(1, 4, 1)."""
    n = P.shape[0]
    idx = torch.arange(n)
    A = torch.zeros((n, n), dtype=torch.float64)
    A[idx, idx] = 4.0
    A[idx, (idx + 1) % n] += 1.0
    A[idx, (idx - 1) % n] += 1.0
    Pp, Pm = torch.roll(P, -1, 0), torch.roll(P, 1, 0)
    M = torch.linalg.solve(A, 6.0 * (Pp - 2.0 * P + Pm))
    Mp = torch.roll(M, -1, 0)
    c0, c1, c2, c3 = P, (Pp - P) - (2.0 * M + Mp) / 6.0, 0.5 * M, (Mp - M) / 6.0
    return torch.stack((c0[:, 0], c1[:, 0], c2[:, 0], c3[:, 0]), 1), torch.stack((c0[:, 1], c1[:, 1], c2[:, 1], c3[:, 1]), 1)


def spline_lengths(cx, cy):
    t = T15.to(cx.device)
    tp = torch.stack((torch.ones_like(t), t, t * t, t * t * t), 0)        # [4, 15]
    x, y = cx @ tp, cy @ tp
    return torch.sqrt(torch.diff(x, dim=1) ** 2 + torch.diff(y, dim=1) ** 2).sum(1)


def create_raceline(refline, normvec, alpha, stepsize, no=None, seg=None):
    """dict(raceline [no, 2], kappa [no], el_lengths [no], coeffs_x, coeffs_y, spline_lengths, spline_inds, t, no) of the
    closed raceline refline + alpha * normvec.  no / seg: the station count and the station segments to hold (None: the
    forward's own choice)."""
    P = refline + alpha[:, None] * normvec
    cx, cy = coefficients(P)
    sl = spline_lengths(cx, cy)
    cum = torch.cumsum(sl, 0)
    total = cum[-1]
    if no is None:
        no = int(math.ceil(float(total) / stepsize))
    dist = torch.arange(no, dtype=torch.float64) * (total / no)
    if seg is None:
        seg = torch.searchsorted(cum.detach(), dist.detach(), right=True)
    prev = torch.cat((torch.zeros(1, dtype=torch.float64), cum))[seg]
    t = (dist - prev) / sl[seg]
    a, c = cx[seg], cy[seg]
    tt = torch.stack((torch.ones_like(t), t, t * t, t * t * t), 1)
    pts = torch.stack(((a * tt).sum(1), (c * tt).sum(1)), 1)
    xd = a[:, 1] + 2.0 * a[:, 2] * t + 3.0 * a[:, 3] * t * t
    yd = c[:, 1] + 2.0 * c[:, 2] * t + 3.0 * c[:, 3] * t * t
    xdd, ydd = 2.0 * a[:, 2] + 6.0 * a[:, 3] * t, 2.0 * c[:, 2] + 6.0 * c[:, 3] * t
    q = xd * xd + yd * yd
    kappa = (xd * ydd - yd * xdd) / (q * torch.sqrt(q))
    el = torch.cat((torch.diff(dist), (total - dist[-1]).reshape(1)))
    return dict(raceline=pts, kappa=kappa, el_lengths=el, coeffs_x=cx, coeffs_y=cy, spline_lengths=sl, spline_inds=seg,
                t=t, no=no)
