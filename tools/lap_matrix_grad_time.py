"""Cost of the lap-time matrix's sensitivities on the racelines of bench.py's c1 workload: the stock matrix of the
reference (15 ggv scales x 11 top speeds, main_globaltraj.py:77-82; bench.py's next_stage) for the first 512 racelines,
with CUDA-event times after a warm-up and the card's name and power limit read in the same run, of
  * lap_time_matrix_batch (the forward alone);
  * the forward of lap_time_matrix_diff;
  * its backward from the mean of the matrix to kappa and el_lengths.

    python tools/lap_matrix_grad_time.py [--reps 3] [--racelines 512]
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
from bench import KAPPA_BOUND, N_POINTS, STEP_INTERP, W_VEH, make_inputs  # noqa: E402
from global_racetrajectory_optimization_b200 import _lib, batch as B_  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--racelines", type=int, default=512)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/lap_matrix_grad_time.py needs a CUDA device")
    dev = torch.device("cuda")
    n = N_POINTS
    rt = torch.tensor(make_inputs(args.racelines, n, seed0=10_000), device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    alpha = B_.opt_min_curv_batch(rt, nv, h, KAPPA_BOUND, W_VEH)["alpha"]
    rl = B_.create_raceline_batch(rt, nv, alpha, STEP_INTERP, n_out_max=int(np.ceil(1.25 * n * 3.0 / STEP_INTERP)) + 64)
    kap, el, n_out = rl["kappa"].contiguous(), rl["el_lengths_interp"].contiguous(), rl["n_out"]
    g = np.load(os.path.join(ROOT, "tests", "golden", "velprofile.npz"))
    scales = np.linspace(0.3, 1.0, int((1.0 - 0.3) / 0.05) + 1)
    speeds = np.linspace(100.0 / 3.6, 150.0 / 3.6, int((150.0 - 100.0) / 5.0) + 1)
    mat = (g["ggv"], g["ax_max_machines"], scales, speeds, float(g["dragcoeff"]), float(g["mass"]))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def forward():
        k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
        return (k, e), B_.lap_time_matrix_diff(k, e, *mat, n_pts=n_out)

    times = {k: [] for k in ("batch", "forward", "backward")}
    for r in range(args.reps + 1):                  # round 0 warms every path up
        t = {}
        t["batch"], ref = timed(lambda: B_.lap_time_matrix_batch(kap, el, *mat, n_pts=n_out))
        t["forward"], (inputs, res) = timed(forward)
        t["backward"], grads = timed(lambda: torch.autograd.grad(res["laptime"].mean(), inputs))
        if r:
            for k, v in t.items():
                times[k].append(v)
    assert torch.equal(res["laptime"].detach(), ref)
    V = scales.size * speeds.size
    B, n_max = kap.shape
    tape = _lib.load().mc_vel_profile_adjoint_workspace_bytes(B * V, n_max)
    med = {k: float(np.median(v)) for k, v in times.items()}
    print(json.dumps(dict(card=card(), racelines=B, variants=V, profiles=B * V, n_out_max=n_max,
                          n_out_mean=float(n_out.double().mean()), tape_bytes_all_profiles=tape,
                          reps=args.reps, ms=times, median_ms=med, backward_over_forward=med["backward"] / med["forward"],
                          lap_time_s_stock_car_mean=float(ref[:, -1, -1].mean()),
                          grad_status={int(k): int(c) for k, c in zip(*torch.unique(res["grad_status"], return_counts=True))},
                          grad_finite=all(bool(torch.isfinite(x).all()) for x in grads))))


if __name__ == "__main__":
    main()
