"""Tail of the interior-point launch on the c1 workload of bench.py (2112 instances of N = 1000, 32 shared centre lines):
builds the -DMC_TAIL_TRACE variant of the library into a temporary directory and, for each slice K (MC_DEBUG_PDIP_SLICE;
0 = unsliced), prints the kernel time, the busy-CTA curve, the share of the launch with fewer than 90 % and
50 % of the CTAs busy, the iteration histogram and the ideal time sum(instance time at full load) / CTAs.  From the mu
history of the K = 0 run it also rates the predictor of the remaining iterations for K = 4, 6, 8.

    python tools/ipm_tail.py [--slices 0,4,6,8] [--reps 3] [--json out.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# slots of the V_PARK vector (enum ParkSlot in csrc/mincurv_ipm.cu)
PARK_MU0, PARK_TRACE, PARK_MU_HIST, PARK_LIST = 1, 8, 16, 64
MAX_ITER, MU_REL = 40, 1e-10        # mc_mincurv_pdip_batch's defaults


def build_trace_lib(out_dir: str) -> str:
    from global_racetrajectory_optimization_b200 import build
    out = os.path.join(out_dir, "libmincurv_b200_tail.so")
    subprocess.check_call([build._nvcc(), *build.NVCC_FLAGS, "-DMC_TAIL_TRACE", "-o", out, *build.SOURCES])
    return out


def predicted_remaining(mu_k, mu_k1, target, left):
    """park_bucket of csrc/mincurv_ipm.cu for n == n_max"""
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(mu_k <= target, 1.0,
                     np.where(mu_k < mu_k1, np.ceil(np.log(target / mu_k) / np.log(mu_k / mu_k1)) + 1.0, left))
    return np.clip(np.nan_to_num(r, nan=left), 1.0, left)


def busy_curve(spans, t0, grid, step_ns=20_000):
    """busy CTAs (= instances in flight) sampled every step_ns from t0"""
    ev = np.concatenate([spans[:, 0], spans[:, 1]])
    dv = np.concatenate([np.ones(len(spans)), -np.ones(len(spans))])
    o = np.argsort(ev, kind="stable")
    ev, busy = ev[o], np.cumsum(dv[o])
    t_end = ev[-1]
    ts = np.arange(t0, t_end, step_ns)
    return ts, busy[np.maximum(np.searchsorted(ev, ts, side="right") - 1, 0)], t_end


def analyse(tr, iters, grid, kernel_ms):
    t = tr[:, PARK_TRACE:PARK_TRACE + 4].copy().view(np.int64)
    spans = [t[:, 0:2]]
    parked = t[:, 2] > 0
    if parked.any():
        spans.append(t[parked, 2:4])
    spans = np.concatenate(spans)
    spans = spans[spans[:, 0] > 0]
    t0 = spans[:, 0].min()
    ts, busy, t_end = busy_curve(spans, t0, grid)
    frac = busy / grid
    span_ms = (t_end - t0) * 1e-6
    lo90, lo50 = float(np.mean(frac < 0.9)), float(np.mean(frac < 0.5))
    # per-iteration time at full load: instances that ran whole while >= 90 % of the CTAs were busy
    dur = (t[:, 1] - t[:, 0]).astype(np.float64)
    n1 = np.where(parked, tr[:, PARK_TRACE + 6], iters).astype(np.float64)
    full = np.ones(len(t), bool)
    idx = np.searchsorted(ts, t[:, 1]) - 1
    full &= frac[np.clip(idx, 0, len(frac) - 1)] >= 0.9
    per_it = float(np.median(dur[full & (n1 > 0)] / n1[full & (n1 > 0)]))
    ideal_ms = float(iters.sum()) * per_it / grid * 1e-6
    curve = [(round((ts[i] - t0) * 1e-6, 2), int(busy[i])) for i in range(0, len(ts), max(1, len(ts) // 40))]
    return dict(kernel_ms=kernel_ms, span_ms=span_ms, below90=lo90, below50=lo50, ideal_ms=ideal_ms,
                tail_pct=100.0 * (span_ms - ideal_ms) / span_ms, parked=int(parked.sum()), per_iter_ms=per_it * 1e-6,
                busy_curve=curve)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slices", default="0,4,6,8")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="ipm_tail_")
    os.environ["MC_B200_LIB"] = build_trace_lib(tmp)
    import torch
    import bench
    from global_racetrajectory_optimization_b200 import batch as B_, _lib
    lib = _lib.load()
    dev = torch.device("cuda")
    Bn, n = bench.BATCH_PER_GPU, bench.N_POINTS
    rt = torch.tensor(bench.make_inputs(Bn, n, seed0=10_000), device=dev)       # bench c1, rank 0
    cid = (torch.arange(Bn, device=dev) % bench.N_BASE_LINES).to(torch.int32)
    _, _, nv, h = B_.calc_splines_batch(rt, want_coeffs=False)
    ws = B_._workspace("mincurv", lib.mc_mincurv_workspace_bytes(Bn, n), dev)
    alpha = torch.empty((Bn, n), dtype=torch.float64, device=dev)
    st = torch.empty((Bn,), dtype=torch.int32, device=dev)
    it = torch.empty((Bn,), dtype=torch.int32, device=dev)
    p, s = B_._ptr, B_._stream()
    lay = B_.mincurv_slab_layout(n)
    grid = min(Bn, torch.cuda.get_device_properties(dev).multi_processor_count * 8)      # 8 resident CTAs per SM
    v = B_.SLAB_VECTORS.index("VV") * lay["np"]
    print(f"ipm_tail: {torch.cuda.get_device_name(dev)}, B={Bn} N={n}, {grid} CTAs")
    out = {}
    for k in [int(x) for x in args.slices.split(",")]:
        os.environ["MC_DEBUG_PDIP_SLICE"] = str(k)
        ms = []
        for r in range(args.reps + 1):
            _lib.check(lib.mc_mincurv_setup_batch_shared(Bn, n, None, p(rt), p(nv), p(h), bench.W_VEH, None, B_.F_SCALE,
                                                         p(cid), p(st), p(ws), ws.numel(), s), "setup")
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(lib.mc_mincurv_pdip_batch(Bn, n, None, p(alpha), p(st), p(it), p(ws), ws.numel(), s), "pdip")
            e1.record()
            torch.cuda.synchronize()
            if r > 0:
                ms.append(e0.elapsed_time(e1))
        slabs = ws[:Bn * lay["stride"] * 8].view(torch.float64).view(Bn, lay["stride"])
        tr = slabs[:, v:v + PARK_LIST].cpu().numpy()
        iters = it.cpu().numpy()
        res = analyse(tr, iters, grid, float(np.median(ms)))
        res["kernel_ms_all"] = ms
        res["iters_hist"] = np.bincount(iters, minlength=MAX_ITER + 1).tolist()
        res["iters_mean"] = float(iters.mean())
        res["status"] = np.bincount(st.cpu().numpy().clip(0), minlength=5).tolist()
        print(f"K={k}: kernel {res['kernel_ms']:.3f} ms (runs {', '.join('%.3f' % x for x in ms)}), traced span "
              f"{res['span_ms']:.3f} ms, ideal {res['ideal_ms']:.3f} ms (tail {res['tail_pct']:.1f} %), busy < 90 %: "
              f"{100 * res['below90']:.1f} % of the span, < 50 %: {100 * res['below50']:.1f} %, parked {res['parked']}")
        print("  busy CTAs over time (ms, CTAs):", " ".join(f"{a}:{b}" for a, b in res["busy_curve"]))
        print("  iterations:", {i: c for i, c in enumerate(res["iters_hist"]) if c}, f"mean {res['iters_mean']:.2f}")
        if k == 0:      # the predictor, from the mu history of the unsliced schedule
            from scipy.stats import spearmanr
            mu0 = tr[:, PARK_MU0]
            hist = tr[:, PARK_MU_HIST:PARK_LIST]
            res["predictor"] = {}
            for K in (4, 6, 8):
                m = iters > K
                pred = predicted_remaining(hist[m, K - 1], hist[m, K - 2], MU_REL * mu0[m], MAX_ITER - K)
                act = iters[m] - K
                err = (pred - act).astype(int)
                rho = float(spearmanr(pred, act).correlation)
                eh = {int(e): int(c) for e, c in zip(*np.unique(err, return_counts=True))}
                res["predictor"][K] = dict(spearman=rho, err_hist=eh, mean_abs_err=float(np.abs(err).mean()))
                print(f"  predictor at K={K}: rank correlation {rho:.3f}, mean |error| {np.abs(err).mean():.2f} it, "
                      f"error histogram {eh}")
        out[k] = res
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(device=torch.cuda.get_device_name(dev), grid=grid, runs=out), f, indent=1)


if __name__ == "__main__":
    main()
