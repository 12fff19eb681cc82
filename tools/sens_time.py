"""Cost of the width sensitivities on the headline workload (c1 of bench.py: 2112 tracks, N = 1000, 32 centre lines
shared through centre_id): CUDA-event times of opt_min_curv_batch, of the forward of opt_min_curv_diff and of its
backward (torch.autograd.grad of alpha with a seeded upstream gradient), after warm-up, the three alternated, with the
card's name and power limit read in the same run.

    python tools/sens_time.py [--reps 3] [--batch 2112] [--n 1000] [--kappa-bound KB] [--curvature-rows]

--kappa-bound sets the curvature limit (default: bench.py's); --curvature-rows differentiates the instances the
curvature-row phase solved too (opt_min_curv_diff(curvature_rows=True)) and reports how many there are and their strong
rows.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import KAPPA_BOUND, N_BASE_LINES, W_VEH, make_inputs  # noqa: E402
from global_racetrajectory_optimization_b200 import batch as B_  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.splitlines()[0].split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--batch", type=int, default=2112)
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--kappa-bound", type=float, default=KAPPA_BOUND)
    ap.add_argument("--curvature-rows", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/sens_time.py needs a CUDA device")
    dev = torch.device("cuda")
    rt = torch.tensor(make_inputs(args.batch, args.n, seed0=10_000), device=dev)
    cid = (torch.arange(args.batch, device=dev) % min(N_BASE_LINES, args.batch)).to(torch.int32)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    centre = rt[:, :, :2].contiguous()
    gbar = torch.tensor(np.random.default_rng(1).standard_normal((args.batch, args.n)), device=dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def solve():
        return B_.opt_min_curv_batch(rt, nv, h, args.kappa_bound, W_VEH, centre_id=cid)

    def forward():
        widths = rt[:, :, 2:].clone().requires_grad_()
        return widths, B_.opt_min_curv_diff(centre, widths, nv, h, args.kappa_bound, W_VEH, centre_id=cid, strict=False,
                                            curvature_rows=args.curvature_rows)

    times = dict(solve=[], forward=[], backward=[])
    for r in range(args.reps + 1):                  # round 0 warms every path up
        t_s, ref = timed(solve)
        t_f, (widths, res) = timed(forward)
        t_b, (gw,) = timed(lambda: torch.autograd.grad(res["alpha"], (widths,), gbar))
        if r:
            times["solve"].append(t_s)
            times["forward"].append(t_f)
            times["backward"].append(t_b)
    assert torch.equal(res["alpha"].detach(), ref["alpha"]) and torch.equal(res["status"], ref["status"])
    med = {k: float(np.median(v)) for k, v in times.items()}
    # the instances the curvature-row phase solved and their strong rows (weight l3/s3 + l4/s4 > 1), from the export
    rows = {}
    if args.curvature_rows:
        B, n = rt.shape[:2]
        sr = torch.empty((B, n), dtype=torch.float64, device=dev)
        nr = torch.empty((B,), dtype=torch.int32, device=dev)
        sens, gs = torch.empty((B, 2, n), dtype=torch.float64, device=dev), torch.empty((B,), dtype=torch.int32, device=dev)
        B_._mincurv_launch("mc_mincurv_solve_batch_sens", B, None, rt, nv, h, args.kappa_bound, W_VEH, None, B_.F_SCALE, cid,
                           *B_._mincurv_results(B, n, dev).values(), sens, gs, sr, nr)
        inst = (sr > 0).any(dim=1)
        rows = dict(row_instances=int(inst.sum()), strong_rows_total=int(nr.sum()), strong_rows_max=int(nr.max()),
                    weak_rows_total=int(((sr > 0) & (sr <= 1.0)).sum()))
    print(json.dumps(dict(card=card(), batch=args.batch, n=args.n, centre_lines=N_BASE_LINES, reps=args.reps,
                          kappa_bound=args.kappa_bound, curvature_rows=args.curvature_rows, **rows,
                          ms=times, median_ms=med, backward_over_forward=med["backward"] / med["forward"],
                          grad_status=torch.bincount(res["grad_status"].clamp(min=0).long(), minlength=5).tolist(),
                          grad_finite=bool(torch.isfinite(gw).all()))))


if __name__ == "__main__":
    main()
