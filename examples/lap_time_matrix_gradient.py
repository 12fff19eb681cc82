"""Which widening saves time at every grip level?  One backward pass through the device chain

    widths -> opt_min_curv_diff -> alpha -> create_raceline_diff -> kappa, el_lengths -> lap_time_matrix_diff

for the reference's stock lap-time matrix (ggv scales 0.3 ... 1.0, top speeds 100 ... 150 km/h; main_globaltraj.py:77-82)
on a synthetic closed track: prints the gradient of the matrix's mean lap time with respect to the track widths, and
the points where widening helps at the lowest and at full grip.

    python examples/lap_time_matrix_gradient.py [--n 600]
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
SCALES = np.linspace(0.3, 1.0, int((1.0 - 0.3) / 0.05) + 1)
SPEEDS = np.linspace(100.0 / 3.6, 150.0 / 3.6, int((150.0 - 100.0) / 5.0) + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=600)
    args = ap.parse_args()
    dev = torch.device("cuda")
    rt = torch.tensor(synth.make_track(7, args.n), device=dev)[None].contiguous()
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)

    def chain(widths):
        alpha = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, 2.0)["alpha"]
        rl = B_.create_raceline_diff(rt[:, :, :2], nv, alpha, 2.0)
        return B_.lap_time_matrix_diff(rl["kappa"], rl["el_lengths_interp"], GGV, MACH, SCALES, SPEEDS, drag_coeff=0.75,
                                       m_veh=1200.0, n_pts=rl["n_out"])["laptime"][0]        # [top speeds, ggv scales]

    widths = rt[:, :, 2:].clone().requires_grad_()
    ltm = chain(widths)
    lt = ltm.detach()
    per_metre = torch.autograd.grad(ltm.mean(), widths, retain_graph=True)[0][0].sum(dim=1)   # [s/m] per point
    print(f"{SPEEDS.size} x {SCALES.size} lap-time matrix: {float(lt.min()):.2f} ... {float(lt.max()):.2f} s, "
          f"mean {float(lt.mean()):.3f} s")
    best = torch.argsort(per_metre)[:5].tolist()
    print("widening by 1 m (both sides) saves most of the mean lap time at points " +
          ", ".join(f"{i} ({-float(per_metre[i]):.4f} s)" for i in best))
    for s, label in ((0, "lowest grip"), (SCALES.size - 1, "full grip")):
        g = torch.autograd.grad(ltm[:, s].mean(), widths, retain_graph=True)[0][0].sum(dim=1)
        print(f"{label} (ggv scale {SCALES[s]:.2f}): best points " + ", ".join(str(i) for i in torch.argsort(g)[:5].tolist()))


if __name__ == "__main__":
    main()
