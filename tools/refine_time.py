"""Cost of the lap-time refinement (raceline_refine.refine_raceline_batch) on the c1 workload of bench.py: 2112 synthetic
closed tracks, N = 1000, started from their minimum-curvature alpha (kappa_bound 0.12, w_veh 2 m), racelines resampled
every STEP m.  CUDA events bracket, per iteration, the line-search trials (create_raceline_batch -> vel_profile_batch),
the forward of the gradient (create_raceline_diff -> vel_profile_diff) and its backward; the rest of the iteration is
the optimizer's own step (elementwise work, row sums, the one host read).  With --metric-length l the refinement runs
in the curvature metric and a fourth part, 'metric', brackets its solve (CurvatureMetric); with --kappa-bound kb as well
the steps stay inside the QP's curvature-limited set and a fifth part, 'projection', brackets the projection QP
(CurvatureProjection, one per iteration).  Prints one JSON line with
the card's name and power limit read in the same run, the per-iteration split, and the mean lap time and running tracks
against iteration.

    python tools/refine_time.py [--batch 2112] [--n 1000] [--max-iters 100] [--metric-length L] [--kappa-bound KB]
                                [--out FILE]
"""
import argparse
import contextlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from sens_time import card  # noqa: E402
from global_racetrajectory_optimization_b200 import batch as B_, raceline_refine as R, synth  # noqa: E402

STEP = 2.0
GGV = np.array([[0.0, 12.0, 12.0], [90.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.3], [40.0, 5.1], [60.0, 2.7], [90.0, 1.5]])
VEH = dict(v_max=70.0, drag_coeff=0.75, m_veh=1200.0)
PARTS = ("trial", "forward", "backward", "metric", "projection")


class Recorder:
    """The objective's timer and spg's callback: CUDA events around every part and at the end of every iteration."""

    def __init__(self):
        self.parts, self.marks = [], []

    def __call__(self, name):
        @contextlib.contextmanager
        def span():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            yield
            e1.record()
            self.parts.append((name, e0, e1))
        return span()

    def callback(self, it, x, f, status):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        running = status == R.ITER_CAP            # (still iterating, or stopped by the cap)
        n_run = running.sum()                     # (no boolean indexing: it would read the device inside the step)
        self.marks.append((it, e, len(self.parts), torch.where(running, f, 0.0).sum() / n_run.clamp(min=1), n_run))

    def iterations(self):
        torch.cuda.synchronize()
        rows = []
        for (_, e_prev, k_prev, _, _), (it, e, k, lap, n_run) in zip(self.marks, self.marks[1:]):
            row = dict(it=it, ms=e_prev.elapsed_time(e), **{p: 0.0 for p in PARTS}, trials=0)
            for name, e0, e1 in self.parts[k_prev:k]:
                row[name] += e0.elapsed_time(e1)
                row["trials"] += name == "trial"
            row["step"] = row["ms"] - sum(row[p] for p in PARTS)
            row.update(mean_laptime=float(lap), running=int(n_run))
            rows.append(row)
        return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=2112)
    ap.add_argument("--n", type=int, default=1000)
    ap.add_argument("--max-iters", type=int, default=R.MAX_ITERS)
    ap.add_argument("--metric-length", type=float, default=None)
    ap.add_argument("--kappa-bound", type=float, default=None)
    ap.add_argument("--relinearise", type=int, default=0, help="outer rounds that re-linearise the curvature rows")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/refine_time.py needs a CUDA device")
    dev = torch.device("cuda")
    rt = torch.tensor(synth.make_batch(10_000, args.batch, args.n), device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    alpha = B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0)["alpha"]
    vp = dict(ggv=GGV, ax_max_machines=MACH, dyn_model_exp=1.0, filt_window=None, **VEH)

    def run(max_iters, rec=None):
        obj = R.LapTime(rt, nv, None, STEP, vp)
        if rec is not None:
            obj.timer = rec
        return R.refine_raceline_batch(rt, nv, alpha, 2.0, GGV, MACH, stepsize_interp=STEP, max_iters=max_iters,
                                       objective=obj, callback=None if rec is None else rec.callback,
                                       metric_length=args.metric_length, kappa_bound=args.kappa_bound,
                                       relinearise=args.relinearise, **VEH)

    run(2)                                                    # warm-up: every launch and allocation size once
    torch.cuda.synchronize()
    rec = Recorder()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    res = run(args.max_iters, rec)
    e1.record()
    rows = rec.iterations()
    total = e0.elapsed_time(e1)
    sums = {p: float(sum(r[p] for r in rows)) for p in PARTS + ("step", "ms")}
    gain = 1.0 - res["laptime"] / res["laptime_start"]
    kept = torch.isfinite(res["laptime"])
    out = dict(card=card(), batch=args.batch, n=args.n, max_iters=args.max_iters, metric_length=args.metric_length,
               kappa_bound=args.kappa_bound,
               total_ms=total,
               iterations=len(rows), per_iteration_ms={k: v / max(len(rows), 1) for k, v in sums.items()},
               step_share=sums["step"] / max(sums["ms"], 1e-30),
               trials_per_iteration=sum(r["trials"] for r in rows) / max(len(rows), 1),
               status={int(k): int(c) for k, c in zip(*torch.unique(res["status"], return_counts=True))},
               iters_median=float(res["iters"].double().median()), evals_median=float(res["evals"].double().median()),
               laptime_start_mean=float(res["laptime_start"][kept].mean()), laptime_mean=float(res["laptime"][kept].mean()),
               metric_fallbacks_median=(float(res["metric_fallbacks"].double().median())
                                        if "metric_fallbacks" in res else None),
               kappa_lin_max=(float(res["kappa_lin_max"][kept].max()) if "kappa_lin_max" in res else None),
               kappa_max=(float(res["kappa_max"][kept].max()) if "kappa_max" in res else None),
               gain_pct=dict(mean=100.0 * float(gain[kept].mean()), min=100.0 * float(gain[kept].min()),
                             max=100.0 * float(gain[kept].max())),
               per_iteration=rows)
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
