"""Cost of the width sensitivities of small closed tracks (opt_min_curv_diff(small_tracks=True, curvature_rows=True),
DESIGN.md section 3.14): 8192 synthetic closed tracks at n = 40 and n = 79, with the box alone binding (kappa_bound 0.12)
and with the curvature rows binding (0.03).  For each: the solve alone (opt_min_curv_batch(small_tracks=True)), the
differentiable forward (the same solve with the row export) and its backward (the dense adjoint K2e-d), one form after
the other in every round.  Medians over the rounds, with the card's name, power limit and clocks read in the same run.

    python tools/small_sens_time.py [--reps 5] [--batch 8192] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from sens_time import card  # noqa: E402
from small_time import timed  # noqa: E402
from global_racetrajectory_optimization_b200 import batch as B_, synth  # noqa: E402

W_VEH = 2.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/small_sens_time.py needs a CUDA device")
    dev = torch.device("cuda")
    cases = {}
    for n in (40, 79):
        base = synth.make_batch(1, 64, n)                           # 64 distinct tracks, repeated to the batch size
        rt = torch.tensor(np.resize(base, (args.batch, n, 4)), device=dev)
        _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
        for kb in (0.12, 0.03):
            cases[f"n{n}_kb{kb}"] = (rt, nv, h, kb)
    times = {f"{c}_{k}": [] for c in cases for k in ("solve", "forward", "backward")}
    info = {}
    for r in range(args.reps + 1):                  # round 0 warms every path up
        for name, (rt, nv, h, kb) in cases.items():
            ms, _ = timed(lambda: B_.opt_min_curv_batch(rt, nv, h, kb, W_VEH, small_tracks=True))
            widths = rt[:, :, 2:].clone().requires_grad_()
            ms_f, res = timed(lambda: B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, W_VEH, small_tracks=True,
                                                           curvature_rows=True, strict=False))
            gbar = torch.ones_like(res["alpha"])
            ms_b, _ = timed(lambda: torch.autograd.grad(res["alpha"], (widths,), gbar))
            if r:
                times[f"{name}_solve"].append(ms)
                times[f"{name}_forward"].append(ms_f)
                times[f"{name}_backward"].append(ms_b)
            info[name] = int((res["grad_status"] == 0).sum())
    med = {k: float(np.median(v)) for k, v in times.items()}
    out = dict(card=card(), batch=args.batch, reps=args.reps, median_ms=med, grad_status_0=info)
    txt = json.dumps(out, indent=1)
    print(txt)
    if args.out:
        with open(args.out, "w") as f:
            f.write(txt + "\n")


if __name__ == "__main__":
    main()
