"""Cost of a vehicle per track in the minimum-curvature QP and in globaltraj_batch.

1. The c1 workload of bench.py (2112 tracks x N = 1000, 32 centre lines shared by their width-jitter variants) through
   opt_min_curv_batch in three forms, alternating in every round:
     * scalar:  kappa_bound = 0.12 (mc_mincurv_solve_batch_shared);
     * tensor:  a [B] tensor of 0.12 (the same stages launched one by one, with kappa_bound_batch);
     * tight:   the tensor with every 97th track at 0.03 (those tracks go through the curvature-row phase).
2. globaltraj_batch('mincurv', check=True) over the first --flow tracks of the same inputs with pars against
   vehicles= at K = 1, 8 and --flow vehicles (identical copies of the stock car, so that every form does the same work).

The medians over the rounds are reported with the card's name, power limit and clocks, read in the same run; the tensor
and K forms are also checked bit for bit against the scalar ones.

    python tools/vehicle_flow_time.py [--reps 7] [--flow 2112]
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
from global_racetrajectory_optimization_b200 import batch as B_, globaltraj  # noqa: E402


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--flow", type=int, default=BATCH_PER_GPU, help="tracks of the globaltraj_batch part")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/vehicle_flow_time.py needs a CUDA device")
    dev = torch.device("cuda")
    B = BATCH_PER_GPU
    rt = torch.tensor(make_inputs(B, N_POINTS, seed0=10_000), device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    cid = (torch.arange(B, device=dev) % N_BASE_LINES).to(torch.int32)
    tight = torch.full((B,), KAPPA_BOUND, dtype=torch.float64, device=dev)
    tight[::97] = 0.03
    qp_forms = {"scalar": KAPPA_BOUND, "tensor": torch.full((B,), KAPPA_BOUND, dtype=torch.float64, device=dev),
                "tight": tight}

    g = np.load(os.path.join(ROOT, "tests", "golden", "velprofile.npz"))
    ggv, mach = g["ggv"], g["ax_max_machines"]
    pars = globaltraj.default_pars()
    pars["veh_params"].update(v_max=float(g["v_max"]), dragcoeff=float(g["dragcoeff"]), mass=float(g["mass"]))
    pars["optim_opts"]["width_opt"] = W_VEH
    veh, F = pars["veh_params"], args.flow

    def fleet(K):
        return B_.Vehicles([ggv] * K, [mach] * K, veh["v_max"], veh["dragcoeff"], veh["mass"], curvlim=veh["curvlim"],
                           width_opt=W_VEH, length=veh["length"], width=veh["width"])
    flow_forms = {"pars": dict(ggv=ggv, ax_max_machines=mach)}
    for K in (1, 8, F):
        flow_forms[f"K{K}"] = dict(vehicles=fleet(K), veh_id=torch.arange(F, dtype=torch.int32, device=dev) % K)

    times = {f: [] for f in list(qp_forms) + list(flow_forms)}
    out = {}
    for r in range(args.reps + 1):                  # round 0 warms every path up
        for name, kb in qp_forms.items():
            ms, out[name] = timed(lambda: B_.opt_min_curv_batch(rt, nv, h, kb, W_VEH, centre_id=cid))
            if r:
                times[name].append(ms)
        for name, kw in flow_forms.items():
            ms, out[name] = timed(lambda: globaltraj.globaltraj_batch(rt[:F], "mincurv", pars, **kw))
            if r:
                times[name].append(ms)
    same_qp = all(torch.equal(out["tensor"][k], out["scalar"][k]) for k in out["scalar"])
    keep = tight == KAPPA_BOUND
    same_tight = all(torch.equal(out["tight"][k][keep], out["scalar"][k][keep]) for k in out["scalar"])
    same_flow = {f: all(torch.equal(torch.nan_to_num(out[f][k]), torch.nan_to_num(v)) for k, v in out["pars"].items()
                        if isinstance(v, torch.Tensor)) for f in flow_forms if f != "pars"}
    med = {f: float(np.median(t)) for f, t in times.items()}
    print(json.dumps(dict(card=card(), batch=B, n=N_POINTS, flow_tracks=F, reps=args.reps, median_ms=med, ms=times,
                          ratio={"tensor": med["tensor"] / med["scalar"], "tight": med["tight"] / med["scalar"],
                                 **{f: med[f] / med["pars"] for f in flow_forms if f != "pars"}},
                          tight_rows_status=out["tight"]["status"][~keep].tolist()[:8],
                          tensor_bit_identical=same_qp, tight_others_bit_identical=same_tight,
                          flow_bit_identical=same_flow)))


if __name__ == "__main__":
    main()
