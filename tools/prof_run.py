"""Short single-GPU run of the mincurv path for ncu captures: B instances of N points, 1 warm-up + 1 measured call."""
import os, sys, time
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from global_racetrajectory_optimization_b200 import batch as B_, synth
Bn = int(sys.argv[1]) if len(sys.argv) > 1 else 592
N = int(sys.argv[2]) if len(sys.argv) > 2 else 1000
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 2
dev = torch.device("cuda")
base = synth.make_batch(100, 16, N)
rts = np.stack([synth.jitter_widths(base[i % 16], 1000 + i) for i in range(Bn)])
rtd = torch.tensor(rts, device=dev)
cx, cy, nvd, hd = B_.calc_splines_batch(rtd)
for r in range(reps):
    torch.cuda.synchronize(); t0 = time.time()
    res = B_.opt_min_curv_batch(rtd, nvd, hd, 0.12, 2.0)
    torch.cuda.synchronize(); dt = time.time() - t0
st = res["status"].cpu().numpy(); it = res["iters"].cpu().numpy()
print("prof_run", Bn, N, f"{dt*1e3:.2f} ms {Bn/dt:.0f} QP/s status", np.bincount(st[st >= 0], minlength=5).tolist(), "iters", it.min(), float(it.mean()), it.max())

import ctypes
from global_racetrajectory_optimization_b200 import _lib
# the written slots of the cycle counters, in the order of enum ProfSlot in csrc/mincurv_ipm.cu
PROF_TOTAL, PROF_NQP, PROF_ITERS = 9, 11, 12
CYCLE_SLOTS = [(0, "update"), (1, "chain(w0)"), (2, "fwd_sweeps"), (5, "sep_ldlt"), (6, "solve_pred"), (7, "solve_corr"),
               (8, "bwd_sweeps"), (9, "total"), (10, "factor"), (13, "fill(w1)"), (14, "w0_wait_hb"), (15, "steplen"),
               (17, "affine"), (18, "corr_rhs"), (19, "w0_wait_ho_empty"), (20, "w1_wait_ho_full"), (21, "w1_update"),
               (22, "ringwait_w0"), (23, "ringwait_w1")]
buf = (ctypes.c_ulonglong * 24)()
_lib.load().mc_debug_read_profile(ctypes.cast(buf, ctypes.c_void_p), 1)
vals = list(buf)
nq = max(vals[PROF_NQP], 1)
print("profile (cycles per QP of CTA 0, %d QPs, %.1f iters/QP):" % (vals[PROF_NQP], vals[PROF_ITERS] / nq))
for k, nm in CYCLE_SLOTS:
    print("  %-16s %12.0f  %5.1f%%" % (nm, vals[k] / nq, 100.0 * vals[k] / max(vals[PROF_TOTAL], 1)))
