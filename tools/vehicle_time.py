"""Cost of a vehicle per track on the lap-time matrix: the stock matrix of the reference (14 ggv scales x 11 top speeds,
154 cells; as tools/lap_matrix_grad_time.py) over the first 512 racelines of bench.py's c1 workload, forward
(lap_time_matrix_batch) and backward (the backward of lap_time_matrix_diff from the mean of the matrix), in four forms:
  * single: the existing path (one vehicle for the call, its tables staged in shared memory once per CTA);
  * K1:     vehicle mode with one vehicle (the stock car), veh_id all zero;
  * K8:     eight vehicles (the stock car's tables, mass and drag varied), veh_id = track mod 8;
  * K512:   one vehicle per track (mass and drag varied per track).
Vehicle mode reads each vehicle's table rows in place from global memory (L1 / read-only path) instead of the staged
shared-memory copy.  The forms run alternately in every round; the medians over the rounds are reported with the card's
name and power limit, read in the same run.  K1 is also checked bit for bit against single.

    python tools/vehicle_time.py [--reps 7] [--racelines 512]
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
from global_racetrajectory_optimization_b200 import batch as B_  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--racelines", type=int, default=512)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/vehicle_time.py needs a CUDA device")
    dev = torch.device("cuda")
    n = N_POINTS
    rt = torch.tensor(make_inputs(args.racelines, n, seed0=10_000), device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    alpha = B_.opt_min_curv_batch(rt, nv, h, KAPPA_BOUND, W_VEH)["alpha"]
    rl = B_.create_raceline_batch(rt, nv, alpha, STEP_INTERP, n_out_max=int(np.ceil(1.25 * n * 3.0 / STEP_INTERP)) + 64)
    kap, el, n_out = rl["kappa"].contiguous(), rl["el_lengths_interp"].contiguous(), rl["n_out"]
    B = kap.shape[0]
    g = np.load(os.path.join(ROOT, "tests", "golden", "velprofile.npz"))
    ggv, mach, drag, mass = g["ggv"], g["ax_max_machines"], float(g["dragcoeff"]), float(g["mass"])
    scales = np.linspace(0.3, 1.0, int((1.0 - 0.3) / 0.05) + 1)
    speeds = np.linspace(100.0 / 3.6, 150.0 / 3.6, int((150.0 - 100.0) / 5.0) + 1)

    def fleet(K):
        f = np.linspace(0.85, 1.15, K) if K > 1 else np.ones(1)
        return B_.Vehicles([ggv] * K, [mach] * K, [float(g["v_max"])] * K, list(drag * f), list(mass * f[::-1]))
    forms = {
        "single": dict(ggv=ggv, ax_max_machines=mach, drag_coeff=drag, m_veh=mass),
        "K1": dict(vehicles=fleet(1), veh_id=torch.zeros(B, dtype=torch.int32, device=dev)),
        "K8": dict(vehicles=fleet(8), veh_id=torch.arange(B, dtype=torch.int32, device=dev) % 8),
        "K512": dict(vehicles=fleet(B), veh_id=torch.arange(B, dtype=torch.int32, device=dev)),
    }

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1), out

    def backward(kw):
        k, e = kap.clone().requires_grad_(), el.clone().requires_grad_()
        res = B_.lap_time_matrix_diff(k, e, ggv_scales=scales, top_speeds=speeds, n_pts=n_out, **kw)
        torch.cuda.synchronize()
        ms, grads = timed(lambda: torch.autograd.grad(res["laptime"].mean(), (k, e)))
        return ms, grads

    times = {f: {"forward": [], "backward": []} for f in forms}
    out = {}
    for r in range(args.reps + 1):                  # round 0 warms every path up
        for name, kw in forms.items():
            ms_f, ltm = timed(lambda: B_.lap_time_matrix_batch(kap, el, ggv_scales=scales, top_speeds=speeds, n_pts=n_out,
                                                               **kw))
            ms_b, grads = backward(kw)
            out[name] = (ltm, grads)
            if r:
                times[name]["forward"].append(ms_f)
                times[name]["backward"].append(ms_b)
    same = torch.equal(out["K1"][0], out["single"][0]) and all(torch.equal(a, b) for a, b in zip(out["K1"][1],
                                                                                                  out["single"][1]))
    med = {f: {k: float(np.median(v)) for k, v in t.items()} for f, t in times.items()}
    print(json.dumps(dict(card=card(), racelines=B, cells=scales.size * speeds.size, n_out_max=kap.shape[1], reps=args.reps,
                          median_ms=med, ms=times, k1_bit_identical_to_single=bool(same),
                          ratio_to_single={f: {k: med[f][k] / med["single"][k] for k in ("forward", "backward")}
                                           for f in forms})))


if __name__ == "__main__":
    main()
