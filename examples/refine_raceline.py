"""How much lap time does the minimum-curvature raceline leave on the table?  The minimum-curvature alpha of a synthetic
closed track and a few width variants of it, refined for the quasi-steady-state lap time inside the same box:

    widths -> opt_min_curv_batch -> alpha -> refine_raceline_batch -> alpha' (lower lap time, same box)

prints, per variant, the lap time of both lines, the iterations and the status: with steps in the identity metric (the
default), in the curvature metric I + l^4 H of the QP (metric_length, DESIGN.md section 3.13), and in that metric under
the QP's curvature limit (kappa_bound: every step stays inside opt_min_curv's feasible set), with the raceline's max
|kappa| of each.

    python examples/refine_raceline.py [--n 600] [--variants 4] [--max-iters 100] [--metric-length 10] [--kappa-bound 0.12]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine, synth  # noqa: E402

GGV = np.array([[0.0, 12.0, 12.0], [90.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.3], [40.0, 5.1], [60.0, 2.7], [90.0, 1.5]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=600)
    ap.add_argument("--variants", type=int, default=4)
    ap.add_argument("--max-iters", type=int, default=raceline_refine.MAX_ITERS)
    ap.add_argument("--metric-length", type=float, default=10.0)
    ap.add_argument("--kappa-bound", type=float, default=0.12)
    args = ap.parse_args()
    dev = torch.device("cuda")
    base = torch.tensor(synth.make_track(7, args.n), device=dev)
    rt = base[None].repeat(args.variants, 1, 1).contiguous()
    rt[:, :, 2:] *= torch.linspace(0.8, 1.2, args.variants, device=dev, dtype=torch.float64)[:, None, None]
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    alpha = B_.opt_min_curv_batch(rt, nv, h, args.kappa_bound, 2.0)["alpha"]
    for ell, kb in ((None, None), (args.metric_length, None), (args.metric_length, args.kappa_bound)):
        res = raceline_refine.refine_raceline_batch(rt, nv, alpha, 2.0, GGV, MACH, 70.0, drag_coeff=0.75, m_veh=1200.0,
                                                    stepsize_interp=2.0, max_iters=args.max_iters, metric_length=ell,
                                                    kappa_bound=kb)
        rl = B_.create_raceline_batch(rt, nv, res["alpha"], 2.0)
        k = torch.where(torch.arange(rl["kappa"].shape[1], device=dev)[None] < rl["n_out"][:, None], rl["kappa"].abs(), 0.0)
        print("identity metric" if ell is None else f"curvature metric, l = {ell:g} m" +
              ("" if kb is None else f", curvature limit {kb:g} 1/m"))
        for b in range(args.variants):
            t0, t1 = float(res["laptime_start"][b]), float(res["laptime"][b])
            st = int(res["status"][b])
            fb = f", {int(res['metric_fallbacks'][b])} identity steps" if "metric_fallbacks" in res else ""
            print(f"  variant {b}: width scale {float(rt[b, 0, 2] / base[0, 2]):.2f}, minimum curvature {t0:.3f} s, "
                  f"refined {t1:.3f} s ({100.0 * (t0 - t1) / t0:.2f} % faster), {int(res['iters'][b])} iterations, "
                  f"status {st} ({raceline_refine.STATUS_TEXT[st]}){fb}, "
                  f"largest move {1000.0 * float((res['alpha'][b] - alpha[b]).abs().max()):.1f} mm, "
                  f"max |kappa| {float(k[b].max()):.4f} 1/m")


if __name__ == "__main__":
    main()
