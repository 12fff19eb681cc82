"""GPU tests (-m gpu) of the box phase of the minimum-curvature QP (mincurv_pdip_kernel, K2b, csrc/mincurv_ipm.cu)
against the long-double replay of tests/ipm_box_ref.py, on the device's own band, f and box read back from the slab,
so that assembly rounding is not counted twice (test A of test_gpu_edges covers the assembly).  The stages run as
mc_mincurv_solve_batch runs them: mc_mincurv_setup_batch_ex (or _shared), then mc_mincurv_pdip_batch.

Per instance: status and iteration count (equal to the replay's on count-stable cases, one of the three runs' outcomes
otherwise), alpha against the long-double replay at the same iteration, the exact dual residual |H a + f + l_u - l_l|
at the device's final state for status 0 and its gap to the carried V_RD, the carried slacks against UB - AL and
AL - LB, mu recomputed from the slab against the replay's final mu, and the final barrier diagonal V_DD (the width
adjoint's input) against the replay's where the slack is not below 1e-6 of the box."""
import numpy as np
import pytest

import ipm_box_ref as X
import ipm_rows_ref as IR

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402
from test_gpu_ipm_schedule import GOLDEN  # noqa: E402

# bounds, about 10x the largest value measured on an H100 80GB HBM3 (700 W) over all cases of this file (measured)
ALPHA_TOL = 3e-8        # max |alpha_dev - alpha_ld| / max(max |alpha_ld|, 0.01) (2.4e-9, 1:20 spacing)
RD_GAP_TOL = 1e-2       # max |V_RD - (H a + f + l_u - l_l)| / rd_tol (9.2e-4, collapsed boxes)
SLACK_TOL = 1e-14       # max |SU - (UB - AL)|, |SL - (AL - LB)| / (UB - LB) (8.5e-16)
MU_TOL = 1e-6           # |mu_dev - mu_ld| / mu_ld (6.1e-8)
DD_TOL = 5e-5           # |DD_dev - D_ld| / D_ld where min(s_u, s_l) >= 1e-6 (UB - LB) (4.8e-6)
# the exact |H a + f + l_u - l_l| / rd_tol at the device's final state: at most the carried value's test plus the gap
# (converged: 1, mu floor with status 0: 1e3)
RD_EXACT_TOL = dict(converged=1.0 + RD_GAP_TOL, mu_floor=1e3 * (1.0 + RD_GAP_TOL))

DEV = "cuda"
SWEEP_NS = tuple(range(80, 89)) + (96, 97, 103, 104, 127, 128, 129, 255, 256, 257, 1000, 2000, 3203)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _run(tracks, w_veh, monkeypatch, f_scale=B_.F_SCALE, knobs=None, status_in=(), centre_id=None):
    """setup (shared centre lines with centre_id), instances in status_in forced to status 1, then the box phase under
    the MC_DEBUG_PDIP_* knobs; returns status, iters, alpha and per instance the slab's band (the owner's), F, LB, UB
    and final state"""
    for k, v in (knobs or {}).items():
        monkeypatch.setenv(X.KNOB_ENV[k], repr(float(v)))
    n = [t.shape[0] for t in tracks]
    B, n_max = len(tracks), max(n)
    rt = np.zeros((B, n_max, 4))
    for b, t in enumerate(tracks):
        rt[b, :n[b]] = t
    rt = torch.tensor(rt, device=DEV)
    npts = torch.tensor(n, dtype=torch.int32, device=DEV)
    _, _, nv, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    wv = torch.tensor(w_veh, dtype=torch.float64, device=DEV)
    lib = _lib.load()
    p, s = B_._ptr, B_._stream()
    ws = B_._workspace("mincurv", lib.mc_mincurv_workspace_bytes(B, n_max), rt.device)
    st = torch.empty((B,), dtype=torch.int32, device=DEV)
    it = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    alpha = torch.full((B, n_max), np.nan, dtype=torch.float64, device=DEV)
    if centre_id is None:
        _lib.check(lib.mc_mincurv_setup_batch_ex(B, n_max, p(npts), p(rt), p(nv), p(h), 0.0, p(wv), float(f_scale), p(st),
                                                 p(ws), ws.numel(), s), "setup")
    else:
        cid = torch.tensor(centre_id, dtype=torch.int32, device=DEV)
        _lib.check(lib.mc_mincurv_setup_batch_shared(B, n_max, p(npts), p(rt), p(nv), p(h), 0.0, p(wv), float(f_scale),
                                                     p(cid), p(st), p(ws), ws.numel(), s), "setup")
    for b in status_in:
        st[b] = 1
    _lib.check(lib.mc_mincurv_pdip_batch(B, n_max, p(npts), p(alpha), p(st), p(it), p(ws), ws.numel(), s), "pdip")
    torch.cuda.synchronize()
    lay = B_.mincurv_slab_layout(n_max)
    w = ws.view(torch.float64)[:B * lay["stride"]].view(B, lay["stride"]).cpu().numpy()
    V = B_.SLAB_VECTORS

    def vec(b, name):
        o = V.index(name) * lay["np"]
        return w[b, o:o + n[b]]
    inst = []
    for b in range(B):
        owner = int(w[b, V.index("HBSRC") * lay["np"]:].view(np.int32)[0])
        hb = w[owner, lay["o_hb"]:lay["o_hb"] + n[b] * B_.HB_PITCH].reshape(n[b], B_.HB_PITCH)[:, :X.HBW + 1]
        inst.append(dict(n=n[b], owner=owner, q=X.qp(hb, vec(b, "F"), vec(b, "LB"), vec(b, "UB")),
                         **{k.lower(): vec(b, k).copy() for k in ("ALPHA", "LU", "LL", "RD", "SU", "SL", "DD")}))
    return dict(status=st.cpu().numpy(), iters=it.cpu().numpy(), alpha=alpha.cpu().numpy(), inst=inst)


_CACHE = {}


def _stability(q, knobs):
    key = (q["hb"].tobytes(), q["f"].tobytes(), q["lb"].tobytes(), q["ub"].tobytes(), tuple(sorted(knobs.items())))
    if key not in _CACHE:
        _CACHE[key] = X.stability(q, cond=False, **knobs)
    return _CACHE[key]


class _Worst:
    def __init__(self):
        self.v, self.where = {}, {}
        self.tally = {}

    def put(self, k, val, name):
        if not val <= self.v.get(k, -np.inf):
            self.v[k], self.where[k] = float(val), name

    def report(self, tag, bounds):
        for k, val in self.v.items():
            print(f"{tag}: {k} {val:.2e} (bound {bounds[k]:.0e}) at {self.where[k]}")
        print(f"{tag}: count-stable cases per exit {self.tally}")


BOUNDS = dict(alpha=ALPHA_TOL, rd_exact_converged=RD_EXACT_TOL["converged"], rd_exact_mu_floor=RD_EXACT_TOL["mu_floor"],
              rd_gap=RD_GAP_TOL, slack=SLACK_TOL, mu=MU_TOL, dd=DD_TOL)


def _check(out, names, knobs, worst, expect_status1=()):
    """every instance of one launch against its replay; returns {name: (device (status, iters), ld run)}"""
    res = {}
    for b, name in enumerate(names):
        st, it = int(out["status"][b]), int(out["iters"][b])
        d = out["inst"][b]
        if b in expect_status1 or name.startswith("status1"):
            assert (st, it) == (1, 0) and not np.any(out["alpha"][b, :d["n"]]), (name, st, it)
            continue
        q = d["q"]
        r, stable, runs = _stability(q, knobs)
        if stable:
            assert (st, it) == (r["status"], r["iters"]), (name, (st, it), X.outcomes(runs))
            worst.tally[r["exit"]] = worst.tally.get(r["exit"], 0) + 1
        else:
            assert (st, it) in X.outcomes(runs), (name, (st, it), X.outcomes(runs))
        ref = r if it == r["iters"] else X.replay(q, cond=False, **dict(knobs, max_iter=it))
        a = d["alpha"]
        assert np.array_equal(a, out["alpha"][b, :d["n"]]), name
        width = (q["ub"] - q["lb"]).astype(np.float64)
        worst.put("alpha", np.abs(a - ref["alpha"]).max() / max(float(np.abs(ref["alpha"]).max()), 0.01), name)
        rd_tol = ref["rd_tol"]
        exact = X.matvec(q["hb"], a.astype(X.LD)) + q["f"] + d["lu"].astype(X.LD) - d["ll"].astype(X.LD)
        if st == 0:
            worst.put("rd_exact_" + ref["exit"] if ref["exit"] != "cap" else "rd_exact_mu_floor",
                      float(np.abs(exact).max()) / rd_tol, name)
        worst.put("rd_gap", float(np.abs(d["rd"].astype(X.LD) - exact).max()) / rd_tol, name)
        ub, lb = q["ub"].astype(np.float64), q["lb"].astype(np.float64)
        worst.put("slack", max((np.abs(d["su"] - (ub - a)) / width).max(), (np.abs(d["sl"] - (a - lb)) / width).max()), name)
        mu = float((d["su"].astype(X.LD) * d["lu"] + d["sl"].astype(X.LD) * d["ll"]).sum() / (2 * d["n"]))
        mu_ref = float((ref["su"] * ref["lu"] + ref["sl"] * ref["ll"]).sum() / (2 * d["n"]))
        worst.put("mu", abs(mu - mu_ref) / mu_ref, name)
        keep = np.minimum(ref["su"], ref["sl"]).astype(np.float64) >= 1e-6 * width
        if keep.any():
            Dr = ref["D"].astype(np.float64)[keep]
            worst.put("dd", (np.abs(d["dd"][keep] - Dr) / Dr).max(), name)
        res[name] = ((st, it), r, stable)
    return res


def _assert_bounds(worst, tag):
    worst.report(tag, BOUNDS)
    for k, v in worst.v.items():
        assert v <= BOUNDS[k], (tag, k, v, worst.where[k])


def _main_cases(golden):
    """(names, tracks, w_veh): the fixtures, the n sweep, the track variants and the constructed floor case"""
    names, tracks, wv = [], [], []

    def add(name, rt, w):
        names.append(name)
        tracks.append(np.asarray(rt, dtype=np.float64))
        wv.append(float(w))
    for nm in GOLDEN:
        g = golden(nm)
        add(nm, g["reftrack"], g["w_veh"])
    for n in SWEEP_NS:
        add(f"sweep{n}", synth.make_track(n, n), 2.0)
    import mincurv_ref as R
    add("collapsed96", IR.collapsed(96), 2.0)
    add("collapsed200", IR.collapsed(200), 2.0)
    add("uneven96_r5", R.uneven_track(96, 5.0, seed=1), 2.0)
    add("uneven200_r20", R.uneven_track(200, 20.0, seed=1), 2.0)
    add("wveh1.5_n130", synth.make_track(130, 130), 1.5)
    add("wveh2.6_n130", synth.make_track(130, 130), 2.6)
    t, _ = X.exit_cases()["floor_narrow"]
    add("floor_narrow", t["rt"], t["w_veh"])
    rt = synth.make_track(7, 100).copy()
    rt[:, 2:] = 0.5                                      # narrower than the vehicle: status 1 from the setup
    add("status1_narrow", rt, 2.0)
    add("status1_forced", synth.make_track(9, 150), 2.0)
    return names, tracks, wv


def test_fixtures_sweep_and_variants_in_one_ragged_sliced_batch(golden, monkeypatch):
    """every case three times, shuffled, with one resident CTA per SM: more instances than resident CTAs, so that with
    the default slice some are parked after 8 iterations and resumed from their stored state"""
    monkeypatch.setenv("MC_DEBUG_PDIP_CTAS_PER_SM", "1")
    names, tracks, wv = _main_cases(golden)
    order = np.random.default_rng(4).permutation(3 * len(names))
    nm = [names[i % len(names)] for i in order]
    forced = [b for b, x in enumerate(nm) if x == "status1_forced"]
    out = _run([tracks[i % len(names)] for i in order], [wv[i % len(names)] for i in order], monkeypatch,
               status_in=forced)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert len(nm) > sms
    ran = out["iters"][out["status"] != 1]
    assert np.any(ran > 8), "nothing was parked"
    worst = _Worst()
    res = _check(out, nm, {}, worst)
    counts = {x: res[x][0] for x in GOLDEN}
    print("fixtures (status, iters) on the device:", counts)
    assert res["floor_narrow"][1]["exit"] == "converged"
    _assert_bounds(worst, "main batch")


def test_f_scale_1(monkeypatch):
    names = [f"fscale1_n{n}" for n in (96, 130, 333)]
    out = _run([synth.make_track(n, n) for n in (96, 130, 333)], [2.0] * 3, monkeypatch, f_scale=1.0)
    worst = _Worst()
    _check(out, names, {}, worst)
    _assert_bounds(worst, "f_scale 1")


def test_shared_centre_lines_read_the_owners_band(monkeypatch):
    """followers with their own vehicle width on the owner's band"""
    rt0, rt1 = synth.make_track(21, 140), synth.make_track(22, 257)
    tracks = [rt0, rt0, rt1, rt0, rt1]
    cid = [0, 0, 2, 0, 2]
    out = _run(tracks, [2.0, 1.6, 2.0, 2.4, 1.8], monkeypatch, centre_id=cid)
    assert [d["owner"] for d in out["inst"]] == cid
    worst = _Worst()
    _check(out, ["owner140", "follower140_w1.6", "owner257", "follower140_w2.4", "follower257_w1.8"], {}, worst)
    _assert_bounds(worst, "shared centre lines")


@pytest.mark.parametrize("name", ["mu_floor_0", "mu_floor_2"])
def test_mu_floor_exits(name, monkeypatch):
    t, knobs = X.exit_cases()[name]
    out = _run([t["rt"]], [t["w_veh"]], monkeypatch, knobs=knobs)
    worst = _Worst()
    res = _check(out, [name], knobs, worst)
    (st, it), r, stable = res[name]
    assert stable and r["exit"] == "mu_floor" and st == (0 if name == "mu_floor_0" else 2)
    _assert_bounds(worst, name)


def test_iteration_cap(golden, monkeypatch):
    """MC_DEBUG_PDIP_MU_REL=1e-300: status 2 after 40 on the constructed case and two fixtures"""
    t, knobs = X.exit_cases()["cap"]
    tracks = [t["rt"], golden("synth128")["reftrack"], golden("handling")["reftrack"]]
    out = _run(tracks, [t["w_veh"], float(golden("synth128")["w_veh"]), float(golden("handling")["w_veh"])], monkeypatch,
               knobs=knobs)
    assert out["status"].tolist() == [2, 2, 2] and out["iters"].tolist() == [X.MAX_ITER] * 3
    worst = _Worst()
    _check(out, ["cap", "synth128_cap", "handling_cap"], knobs, worst)
    _assert_bounds(worst, "cap")


def test_without_the_step_test_the_fixtures_stop_where_the_replay_says(golden, monkeypatch):
    """MC_DEBUG_PDIP_DX_REL=0: the device stops at the first iteration where the mu and r_d tests pass in the default
    replay, earlier than with the step test exactly where the replay says the step test decided the exit"""
    gs = [golden(nm) for nm in GOLDEN]
    tracks, wv = [g["reftrack"] for g in gs], [float(g["w_veh"]) for g in gs]
    base = _run(tracks, wv, monkeypatch)
    out = _run(tracks, wv, monkeypatch, knobs=dict(dx_rel=0.0))
    worst = _Worst()
    res = _check(out, GOLDEN, dict(dx_rel=0.0), worst)
    step = []
    for b, nm in enumerate(GOLDEN):
        before, after = int(base["iters"][b]), int(out["iters"][b])
        r, stable, _ = _stability(base["inst"][b]["q"], {})
        first = 1 + next(k for k, t in enumerate(r["trace"]) if t["ok"]["mu"] and t["ok"]["rd"])
        print(f"{nm}: {before} iterations, {after} without the step test (the replay: mu and r_d first pass at {first}; "
              f"decided by {r['decided']})")
        assert stable and res[nm][2], nm
        assert after == first, nm
        assert (after < before) == (r["decided"] == ("step",)), nm
        if after < before:
            step.append(nm)
    print(f"the step test decides the exit on {len(step)} of {len(GOLDEN)} fixtures: {step}")
    _assert_bounds(worst, "dx_rel 0")
