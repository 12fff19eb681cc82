"""Cost of the dense small-track solver of the minimum-curvature QP (opt_min_curv_batch(small_tracks=True), DESIGN.md
section 3.14).

1. 8192 synthetic closed tracks at n = 40 and n = 79, with the box alone binding (kappa_bound 0.12 on tracks whose rows
   stay slack at 0.12) and with the curvature rows binding (0.03), one form after the other in every round.
2. The c1 workload of bench.py (2112 tracks x N = 1000) with small_tracks False and True: the same banded solve through
   mc_mincurv_solve_batch_shared against mc_mincurv_solve_batch_ex plus one dense launch whose CTAs all exit at once;
   the two are also checked bit for bit.

The FP64 operation count per instance is computed from the shapes (per iteration: K = E^T (I + W) E, n^3 multiply-adds
on its lower triangle counted as n^3 flops; Cholesky n^3 / 3; two solves 4 n^2; five products with E or E^T 10 n^2).
Medians over the rounds, with the card's name, power limit and clocks read in the same run.

    python tools/small_time.py [--reps 5] [--batch 8192]
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
from bench import BATCH_PER_GPU, KAPPA_BOUND, N_BASE_LINES, N_POINTS, W_VEH, make_inputs  # noqa: E402
from global_racetrajectory_optimization_b200 import batch as B_, synth  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def flops_per_iteration(n):
    return n ** 3 + n ** 3 / 3 + 4 * n ** 2 + 10 * n ** 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=8192)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/small_time.py needs a CUDA device")
    dev = torch.device("cuda")
    small = {}
    for n in (40, 79):
        base = synth.make_batch(1, 64, n)                           # 64 distinct tracks, repeated to the batch size
        rt = torch.tensor(np.resize(base, (args.batch, n, 4)), device=dev)
        _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
        for kb in (0.12, 0.03):
            small[f"n{n}_kb{kb}"] = (rt, nv, h, kb)
    rt1 = torch.tensor(make_inputs(BATCH_PER_GPU, N_POINTS, seed0=10_000), device=dev)
    _, _, nv1, h1 = B_.calc_splines_batch(rt1, want_coeffs=False)
    cid = (torch.arange(BATCH_PER_GPU, device=dev) % N_BASE_LINES).to(torch.int32)
    forms = {name: (lambda a=a: B_.opt_min_curv_batch(a[0], a[1], a[2], a[3], W_VEH, small_tracks=True))
             for name, a in small.items()}
    forms["c1_plain"] = lambda: B_.opt_min_curv_batch(rt1, nv1, h1, KAPPA_BOUND, W_VEH, centre_id=cid)
    forms["c1_small_tracks"] = lambda: B_.opt_min_curv_batch(rt1, nv1, h1, KAPPA_BOUND, W_VEH, centre_id=cid,
                                                             small_tracks=True)
    times = {f: [] for f in forms}
    out = {}
    for r in range(args.reps + 1):                  # round 0 warms every path up
        for name, fn in forms.items():
            ms, out[name] = timed(fn)
            if r:
                times[name].append(ms)
    med = {f: float(np.median(t)) for f, t in times.items()}
    per = {}
    for name, (rt, _, _, _) in small.items():
        n = rt.shape[1]
        st, it = out[name]["status"], out[name]["iters"].double()
        per[name] = dict(qp_per_s=args.batch / med[name] * 1e3, mean_iters=float(it.mean()),
                         status_counts={int(s): int((st == s).sum()) for s in st.unique()},
                         fp64_flop_per_instance=float(flops_per_iteration(n) * it.mean()),
                         fp64_tflops=float(flops_per_iteration(n) * it.sum()) / (med[name] * 1e-3) / 1e12,
                         smem_bytes=(2 * n * n + 38 * n) * 8)
    same = all(torch.equal(out["c1_plain"][k], out["c1_small_tracks"][k]) for k in out["c1_plain"])
    print(json.dumps(dict(card=card(), batch=args.batch, reps=args.reps, median_ms=med, ms=times, small=per,
                          c1_ratio=med["c1_small_tracks"] / med["c1_plain"], c1_bit_identical=same)))


if __name__ == "__main__":
    main()
