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
buf = (ctypes.c_ulonglong * 24)()
_lib.load().mc_debug_read_profile(ctypes.cast(buf, ctypes.c_void_p), 1)
names = ["v5_update", "chain(w0)", "fwd_sweep", "sep_rhs(w1)", "sep_solve+c(w1)", "sep_ldlt", "solve_pred", "solve_corr", "bwd_sweep", "total", "factor", "nqp", "iters", "fill(w1)", "w0_wait_hb", "v4_steplen", "v1_diag_rhs(in v5_update)", "v2_affine", "v3_corr_rhs", "w0_wait_ltempty", "w1_wait_ltfull", "w1_Supdate", "ringwait_w0", "ringwait_w1"]
vals = list(buf)
nq = max(vals[11], 1)
print("profile (cycles per QP of CTA 0, %d QPs, %.1f iters/QP):" % (vals[11], vals[12] / nq))
for k, nm in enumerate(names):
    if nm != "-" and (k < 11 or k > 12):
        print("  %-9s %12.0f  %5.1f%%" % (nm, vals[k] / nq, 100.0 * vals[k] / max(vals[9], 1)))
