"""Cost of the lap-time refinement on small closed tracks (refine_raceline_batch(small_tracks=True), DESIGN.md sections
3.13 and 3.14): 8192 synthetic closed tracks at n = 40 and n = 79, started from their minimum-curvature alpha
(opt_min_curv_batch(small_tracks=True)) at kappa_bound 0.12 and at a binding limit per track (0.97 of the largest
|k_ref + E alpha| at the box-only optimum), in four forms: the identity refinement, metric_length 10 m, the same with
the kappa_bound, and that with relinearise 2.  CUDA events bracket the objective's parts per iteration ('trial',
'forward', 'backward', 'metric', 'projection'; tools/refine_time.py's Recorder).  Prints one JSON line with the card's
name and power limit read in the same run, the per-iteration split and the mean lap-time gain of every case.

    python tools/small_refine_time.py [--batch 8192] [--max-iters 30] [--out FILE]
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
from refine_time import GGV, MACH, PARTS, STEP, VEH, Recorder  # noqa: E402
from sens_time import card  # noqa: E402
from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine as R, synth  # noqa: E402

ELL = 10.0
W_VEH = 2.0
FORMS = dict(identity={}, metric=dict(metric_length=ELL), kappa=dict(metric_length=ELL, kappa_bound=True),
             relinearise=dict(metric_length=ELL, kappa_bound=True, relinearise=2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8192)
    ap.add_argument("--max-iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/small_refine_time.py needs a CUDA device")
    dev = torch.device("cuda")
    vp = dict(ggv=GGV, ax_max_machines=MACH, dyn_model_exp=1.0, filt_window=None, **VEH)
    cases = {}
    for n in (40, 79):
        base = synth.make_batch(1, 64, n)                           # 64 distinct tracks, repeated to the batch size
        rt = torch.tensor(np.resize(base, (args.batch, n, 4)), device=dev)
        rt[:, :, 2:] = rt[:, :, 2:].clamp(min=2.0)                  # (room for the car beside the centre line)
        _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
        a_box = B_.opt_min_curv_batch(rt, nv, h, 1e3, W_VEH, small_tracks=True)["alpha"]
        k_box = R.CurvatureProjection(rt, nv, None, W_VEH, 1e3, ELL, small_tracks=True).kappa_lin(
            a_box, torch.ones(args.batch, dtype=torch.bool, device=dev))
        for kb_name, kb in (("0.12", 0.12), ("binding", 0.97 * k_box)):
            qp = B_.opt_min_curv_batch(rt, nv, h, kb, W_VEH, small_tracks=True)
            cases[f"n{n}_kb{kb_name}"] = (rt, nv, qp["alpha"], kb, int((qp["status"] == 0).sum()))

    def run(rt, nv, alpha, kb, form, max_iters, rec=None):
        obj = R.LapTime(rt, nv, None, STEP, vp)
        if rec is not None:
            obj.timer = rec
        kw = dict(FORMS[form])
        if kw.get("kappa_bound"):
            kw["kappa_bound"] = kb
        return R.refine_raceline_batch(rt, nv, alpha, W_VEH, GGV, MACH, stepsize_interp=STEP, max_iters=max_iters,
                                       objective=obj, callback=None if rec is None else rec.callback, small_tracks=True,
                                       **kw, **VEH)

    out = dict(card=card(), batch=args.batch, max_iters=args.max_iters, metric_length=ELL, cases={})
    for name, (rt, nv, alpha, kb, qp_ok) in cases.items():
        for form in FORMS:
            run(rt, nv, alpha, kb, form, 2)                 # warm-up: every launch and allocation size once
            torch.cuda.synchronize()
            rec = Recorder()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            res = run(rt, nv, alpha, kb, form, args.max_iters, rec)
            e1.record()
            rows = rec.iterations()
            sums = {p: float(sum(r[p] for r in rows)) for p in PARTS + ("step", "ms")}
            kept = torch.isfinite(res["laptime"])
            gain = 1.0 - res["laptime"][kept] / res["laptime_start"][kept]
            out["cases"][f"{name}_{form}"] = dict(
                qp_status_0=qp_ok, total_ms=e0.elapsed_time(e1), iterations=len(rows),
                per_iteration_ms={k: v / max(len(rows), 1) for k, v in sums.items()},
                status={int(k): int(c) for k, c in zip(*torch.unique(res["status"], return_counts=True))},
                iters_median=float(res["iters"].double().median()),
                metric_fallbacks_max=(int(res["metric_fallbacks"].max()) if "metric_fallbacks" in res else None),
                rounds_max=(int(res["rounds"].max()) if "rounds" in res else None),
                gain_pct_mean=100.0 * float(gain.mean()) if bool(kept.any()) else None, refined=int(kept.sum()))
            print(name, form, json.dumps(out["cases"][f"{name}_{form}"]), file=sys.stderr)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
