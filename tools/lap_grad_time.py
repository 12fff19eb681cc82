"""Cost of the lap-time sensitivities on the c1 workload of bench.py (2112 synthetic closed tracks, N = 1000, racelines
resampled every STEP m): CUDA-event times, after warm-up, alternated, with the card's name and power limit read in the
same run, of
  * vel_profile_batch, the forward of vel_profile_diff and its backward (to kappa and el_lengths);
  * create_raceline_batch, the forward of create_raceline_diff and its backward (to alpha, the line and the normals);
  * the chain widths -> opt_min_curv_diff -> create_raceline_diff -> vel_profile_diff: forward and backward.

    python tools/lap_grad_time.py [--reps 5] [--batch 2112] [--n 1000]
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

STEP = 2.0
GGV = np.array([[0.0, 12.0, 12.0], [90.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.3], [40.0, 5.1], [60.0, 2.7], [90.0, 1.5]])
VEH = dict(drag_coeff=0.75, m_veh=1200.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batch", type=int, default=2112)
    ap.add_argument("--n", type=int, default=1000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/lap_grad_time.py needs a CUDA device")
    dev = torch.device("cuda")
    rt = torch.tensor(synth.make_batch(10_000, args.batch, args.n), device=dev)
    _, _, nv, _ = B_.calc_splines_batch(rt, want_coeffs=False)
    rl = B_.create_raceline_batch(rt, nv, torch.zeros(rt.shape[:2], dtype=torch.float64, device=dev), STEP)
    kap, el, n_out = rl["kappa"].contiguous(), rl["el_lengths_interp"].contiguous(), rl["n_out"]
    gbar = torch.tensor(np.random.default_rng(1).uniform(0.5, 2.0, args.batch), device=dev)

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def forward():
        k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
        return (k, e), B_.vel_profile_diff(k, e, GGV, MACH, 70.0, n_pts=n_out, **VEH)

    _, _, nv1, h1 = B_.calc_splines_batch(rt, want_coeffs=False)
    alpha = B_.opt_min_curv_batch(rt, nv1, h1, 0.12, 2.0)["alpha"]
    no_max = int(B_.create_raceline_batch(rt, nv1, alpha, STEP)["kappa"].shape[1])
    gk = torch.tensor(np.random.default_rng(2).standard_normal((args.batch, no_max)), device=dev)

    def rl_forward():
        a, v = alpha.clone().requires_grad_(), nv1.clone().requires_grad_()
        return (a, v), B_.create_raceline_diff(rt, v, a, STEP, n_out_max=no_max)

    def chain_forward():
        w = rt[:, :, 2:].clone().requires_grad_()
        al = B_.opt_min_curv_diff(rt[:, :, :2], w, nv1, h1, 0.12, 2.0, strict=False)["alpha"]
        r = B_.create_raceline_diff(rt[:, :, :2], nv1, al, STEP, n_out_max=no_max, strict=False)
        return w, B_.vel_profile_diff(r["kappa"], r["el_lengths_interp"], GGV, MACH, 70.0, n_pts=r["n_out"], strict=False,
                                     **VEH)

    times = {k: [] for k in ("batch", "forward", "backward", "rl_batch", "rl_forward", "rl_backward", "chain_forward",
                             "chain_backward")}
    for r in range(args.reps + 1):                  # round 0 warms every path up
        t = {}
        t["batch"], ref = timed(lambda: B_.vel_profile_batch(kap, el, GGV, MACH, 70.0, n_pts=n_out, **VEH))
        t["forward"], (inputs, res) = timed(forward)
        t["backward"], grads = timed(lambda: torch.autograd.grad(res["laptime"], inputs, gbar))
        t["rl_batch"], rl_ref = timed(lambda: B_.create_raceline_batch(rt, nv1, alpha, STEP, n_out_max=no_max))
        t["rl_forward"], (rl_in, rl_res) = timed(rl_forward)
        t["rl_backward"], _ = timed(lambda: torch.autograd.grad(rl_res["kappa"], rl_in, gk))
        t["chain_forward"], (w, ch) = timed(chain_forward)
        t["chain_backward"], _ = timed(lambda: torch.autograd.grad(ch["laptime"].sum(), w))
        if r:
            for k, v in t.items():
                times[k].append(v)
    assert torch.equal(rl_res["kappa"].detach(), rl_ref["kappa"])
    assert torch.equal(res["laptime"].detach(), ref["laptime"][:, 0]) and torch.equal(res["vx"].detach(), ref["vx"][:, 0])
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps(dict(card=card(), batch=args.batch, n=args.n, n_out_max=int(kap.shape[1]), reps=args.reps, ms=times,
                          median_ms=med, backward_over_forward=med["backward"] / med["forward"],
                          forward_over_batch=med["forward"] / med["batch"],
                          rl_backward_over_forward=med["rl_backward"] / med["rl_forward"],
                          chain_backward_over_forward=med["chain_backward"] / med["chain_forward"],
                          grad_status={int(k): int(c) for k, c in zip(*torch.unique(res["grad_status"], return_counts=True))},
                          grad_finite=all(bool(torch.isfinite(g).all()) for g in grads))))


if __name__ == "__main__":
    main()
