"""Cost of the shortest-path sensitivities on the shortest-path workload of c5 in bench.py (32768 width variants of 32
centre lines, N = 500, the vehicle-width grid of the sweep): CUDA-event times of opt_shortest_path_batch, of the forward
of opt_shortest_path_diff and of its backward (torch.autograd.grad of alpha with a seeded upstream gradient, to the
reftrack, the normals and w_veh), after warm-up, the three alternated, with the card's name and power limit read in the
same run.

    python tools/sp_sens_time.py [--reps 5] [--batch 32768] [--n 500]
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
from global_racetrajectory_optimization_b200 import batch as B_, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--n", type=int, default=500)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/sp_sens_time.py needs a CUDA device")
    dev = torch.device("cuda")
    base = torch.tensor(synth.make_batch(20_000, 32, args.n), device=dev)               # bench.py c5, rank 0
    rt, _ = B_.jitter_widths_batch(base, torch.arange(args.batch, dtype=torch.int64, device=dev) + 1_000_003)
    _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
    grid = torch.linspace(1.6, 3.4, 7, dtype=torch.float64, device=dev)
    wv = grid[torch.arange(args.batch, device=dev) % 7].contiguous()
    gbar = torch.tensor(np.random.default_rng(1).standard_normal((args.batch, args.n)), device=dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def forward():
        r, v, w = rt.clone().requires_grad_(), nv.clone().requires_grad_(), wv.clone().requires_grad_()
        return (r, v, w), B_.opt_shortest_path_diff(r, v, w)

    times = dict(solve=[], forward=[], backward=[])
    for r in range(args.reps + 1):                  # round 0 warms every path up
        t_s, ref = timed(lambda: B_.opt_shortest_path_batch(rt, nv, wv))
        t_f, (inputs, res) = timed(forward)
        t_b, grads = timed(lambda: torch.autograd.grad(res["alpha"], inputs, gbar))
        if r:
            times["solve"].append(t_s)
            times["forward"].append(t_f)
            times["backward"].append(t_b)
    assert torch.equal(res["alpha"].detach(), ref["alpha"]) and torch.equal(res["status"], ref["status"])
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps(dict(card=card(), batch=args.batch, n=args.n, reps=args.reps, ms=times, median_ms=med,
                          backward_over_forward=med["backward"] / med["forward"],
                          forward_over_solve=med["forward"] / med["solve"],
                          grad_status={int(k): int(c) for k, c in zip(*torch.unique(res["grad_status"], return_counts=True))},
                          grad_finite=all(bool(torch.isfinite(g).all()) for g in grads))))


if __name__ == "__main__":
    main()
