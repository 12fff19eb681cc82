"""The metric length of the lap-time refinement (raceline_refine.refine_raceline_batch(metric_length=l)) swept on the
golden tracks of tests/golden/ from their minimum-curvature alpha, with the fixtures' ggv and machine tables, against the
identity metric.  Per run and track: lap time, status, ||P(alpha - g) - alpha||_inf, the largest move from the
minimum-curvature alpha, the identity fallbacks, and max |kappa| of the raceline against curvlim.  Every metric length runs
without the curvature limit (kappa_bound None: a violation shows in max |kappa|) and with each --kappa-bounds kb, where
the steps stay inside the QP's curvature-limited set (kappa_lin_max: the QP's linearised max |kappa| at the result).
Prints one JSON line with the card's name and power limit read in the same run.

    python tools/refine_sweep.py [--lengths 5 10 20 40 80] [--kappa-bounds 0.12] [--max-iters 100] [--out FILE]
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
from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine as R  # noqa: E402

NAMES = ["berlin", "handling", "modena", "synth1000"]
STEP = 2.0
CURVLIM = 0.12


def _golden(name):
    return dict(np.load(os.path.join(ROOT, "tests", "golden", name + ".npz"), allow_pickle=False))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lengths", type=float, nargs="+", default=[5.0, 10.0, 20.0, 40.0, 80.0])
    ap.add_argument("--kappa-bounds", type=float, nargs="*", default=[CURVLIM])
    ap.add_argument("--max-iters", type=int, default=R.MAX_ITERS)
    ap.add_argument("--relinearise", type=int, default=0, help="outer rounds that re-linearise the curvature rows")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/refine_sweep.py needs a CUDA device")
    dev = torch.device("cuda")
    gs = [_golden(nm) for nm in NAMES]
    v = _golden("velprofile")
    veh = dict(ggv=v["ggv"], ax_max_machines=v["ax_max_machines"], v_max=float(v["v_max"]),
               drag_coeff=float(v["dragcoeff"]), m_veh=float(v["mass"]))
    n = [g["reftrack"].shape[0] for g in gs]
    rt = np.zeros((len(gs), max(n), 4))
    al = np.zeros((len(gs), max(n)))
    for b, g in enumerate(gs):
        rt[b, :n[b]], al[b, :n[b]] = g["reftrack"], g["alpha_mincurv"]
    rt, al = torch.tensor(rt, device=dev), torch.tensor(al, device=dev)
    npts = torch.tensor(n, dtype=torch.int32, device=dev)
    wv = torch.tensor([float(g["w_veh"]) for g in gs], device=dev)
    _, _, nv, _ = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    runs = []
    for ell, kb in [(None, None)] + [(ell, kb) for ell in args.lengths for kb in [None] + list(args.kappa_bounds)]:
        res = R.refine_raceline_batch(rt, nv, al, wv, n_pts=npts, stepsize_interp=STEP, max_iters=args.max_iters,
                                      metric_length=ell, kappa_bound=kb,
                                      relinearise=args.relinearise if kb is not None else 0, **veh)
        rl = B_.create_raceline_batch(rt, nv, res["alpha"], STEP, n_pts=npts)
        tracks = {}
        for b, nm in enumerate(NAMES):
            no = int(rl["n_out"][b])
            tracks[nm] = dict(laptime_start=float(res["laptime_start"][b]), laptime=float(res["laptime"][b]),
                              status=int(res["status"][b]), iters=int(res["iters"][b]),
                              pg_norm=float(res["pg_norm"][b]),
                              max_move_m=float((res["alpha"][b, :n[b]] - al[b, :n[b]]).abs().max()),
                              metric_fallbacks=(int(res["metric_fallbacks"][b]) if "metric_fallbacks" in res
                                                else None),
                              kappa_lin_max=float(res["kappa_lin_max"][b]) if kb is not None else None,
                              max_abs_kappa=float(rl["kappa"][b, :no].abs().max()))
        runs.append(dict(metric_length=ell, kappa_bound=kb, tracks=tracks))
    line = json.dumps(dict(card=card(), max_iters=args.max_iters, curvlim=CURVLIM, runs=runs))
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
