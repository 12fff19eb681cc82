"""Where would one more metre of track width save the most lap time?  One backward pass through the device chain

    widths -> opt_min_curv_diff -> alpha -> create_raceline_diff -> kappa, el_lengths -> vel_profile_diff -> lap time

on a synthetic closed track and a few width variants of it; prints, per variant, the lap time and the points where
widening the track (both sides) saves the most time.

    python examples/lap_time_gradient.py [--n 600] [--variants 4]
"""
import argparse
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from global_racetrajectory_optimization_b200 import batch as B_, synth  # noqa: E402

GGV = np.array([[0.0, 12.0, 12.0], [90.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.3], [40.0, 5.1], [60.0, 2.7], [90.0, 1.5]])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=600)
    ap.add_argument("--variants", type=int, default=4)
    args = ap.parse_args()
    dev = torch.device("cuda")
    base = torch.tensor(synth.make_track(7, args.n), device=dev)
    rt = base[None].repeat(args.variants, 1, 1).contiguous()
    rt[:, :, 2:] *= torch.linspace(0.8, 1.2, args.variants, device=dev, dtype=torch.float64)[:, None, None]
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    widths = rt[:, :, 2:].clone().requires_grad_()
    alpha = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, 2.0)["alpha"]
    rl = B_.create_raceline_diff(rt[:, :, :2], nv, alpha, 2.0)
    lap = B_.vel_profile_diff(rl["kappa"], rl["el_lengths_interp"], GGV, MACH, 70.0, drag_coeff=0.75, m_veh=1200.0,
                              n_pts=rl["n_out"])["laptime"]
    lap.sum().backward()
    per_metre = widths.grad.sum(dim=2)                       # d laptime / d (both widths at a point) [s/m]
    for b in range(args.variants):
        best = torch.argsort(per_metre[b])[:5].tolist()
        print(f"variant {b}: width scale {float(rt[b, 0, 2] / base[0, 2]):.2f}, lap time {float(lap[b].detach()):.3f} s; "
              "widening by 1 m saves most at points " +
              ", ".join(f"{i} ({-float(per_metre[b, i]):.4f} s)" for i in best))


if __name__ == "__main__":
    main()
