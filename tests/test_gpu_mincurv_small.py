"""GPU tests (-m gpu) of the dense small-track solver of the minimum-curvature QP (csrc/mincurv_dense.cu,
opt_min_curv_batch(small_tracks=True), DESIGN.md section 3.14):

A  against the dense oracle (oracle/tph_dense + quadprog_gi) on synthetic tracks of 3 .. 79 points, the handling track
   thinned to every 4th / 6th / 8th point, a collapsed box and curvature limits at which the rows bind: the status
   (oracle RuntimeError <-> 1, ValueError <-> 4, else 0), alpha, kappa_lin_max, curv_error_max and the KKT certificate of
   the full QP (tests/mincurv_ref.py).
B  dense against banded on 80 .. MC_DENSE_N_MAX points (_dense_below), about the centre line and about a given line.
C  a ragged batch from 3 to 1000 points: the long tracks bit for bit as without small_tracks, each short track bit for bit
   as solved alone (also in a batch of 3 x SMs x 8), the refusals, an all-short batch, shared centre lines, and the
   behaviour without small_tracks.
D  iqp_batch and globaltraj_batch with small_tracks against the oracle.
Every measured error is printed next to its tolerance (pytest -s)."""
import numpy as np
import pytest

import mincurv_ref as R
import qp_sens as Q
from conftest import load_golden, rel_max

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import batch as B_, globaltraj, synth  # noqa: E402
from oracle import tph_dense as T  # noqa: E402

# Against the oracle (alpha max|d alpha| / max|alpha|, curvatures relative), measured on an H100 over the cases below:
# alpha 2.8e-7 (handling every 4th point), kappa_lin_max 2.6e-9, curv_error_max 1.1e-6 (synth31, a small value:
# 1.4e-3 1/m).  The project's parity bar (alpha 1e-4, kappa 1e-3) is the ceiling.
ORACLE_TOL = dict(alpha=2e-6, klin=2e-8, cerr=1e-5)
ALPHA_TOL = 1e-4
# KKT certificate of a dense solution with the oracle's H, f, E, k_ref (the stopping rule of the curvature-row phase:
# mu <= 1e-11 mu0, |r_d| <= 1e-8 (|f| + |g0|)); the bars of tests/test_gpu_edges.py.  Measured: stationarity 4.4e-7
# (synth64), 4.9e-11 on the collapsed boxes.
CERT_STAT_TOL = 8e-6
CERT_STAT_TOL_COLLAPSED = 4e-4
CERT_FEAS_TOL = 1e-9
# Dense against banded on 80 .. 108 points (band truncation and the two solvers' stopping rules), measured on an H100:
# alpha 1.0e-7, kappa_lin_max 3.5e-8, curv_error_max 1.4e-7 (n 101 about a given line; about the centre line <= 2e-8).
DVB_TOL = 1e-6
# iqp_batch against tph_dense.iqp_handler (three or more chained QPs and re-sampling), measured on an H100: alpha 3.0e-6,
# reftrack 1.0e-7 m (the handling track re-sampled at 8 m, 208 -> 73 points).
IQP_TOL = dict(alpha=2e-5, reftrack=1e-6)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _closed(rt):
    return np.vstack((rt[:, :2], rt[0, :2]))


def _el(rt):
    return np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1)


def _case(rt, kb, w_veh=2.0):
    """The oracle's normals, h, QP and outcome of a track: status 0 (alpha, curv_error_max, kappa_lin_max), 1 or 4."""
    _, _, A, nv = T.calc_splines(_closed(rt))
    c = dict(rt=rt, nv=nv, h=_el(rt), w_veh=w_veh, kb=kb)
    try:
        alpha, cerr = T.opt_min_curv(rt, nv, A, kb, w_veh)
    except RuntimeError:
        return dict(c, status=1)
    except ValueError:
        return dict(c, status=4)
    qp = T.assemble_min_curv(rt, nv, A, kb, w_veh)
    return dict(c, status=0, qp=qp, alpha=alpha, cerr=cerr, klin=float(np.abs(qp["k_kappa_ref"] + qp["E_kappa"] @ alpha).max()))


def _pack(cases, n_max=None):
    dev = torch.device("cuda")
    n = [c["rt"].shape[0] for c in cases]
    n_max = n_max or max(n)
    rt, nv, h = np.zeros((len(cases), n_max, 4)), np.zeros((len(cases), n_max, 2)), np.ones((len(cases), n_max))
    for b, c in enumerate(cases):
        rt[b, :n[b]], nv[b, :n[b]], h[b, :n[b]] = c["rt"], c["nv"], c["h"]
    f64 = dict(dtype=torch.float64, device=dev)
    return (torch.tensor(rt, **f64), torch.tensor(nv, **f64), torch.tensor(h, **f64),
            torch.tensor(n, dtype=torch.int32, device=dev))


def _np(res):
    return {k: v.cpu().numpy() for k, v in res.items()}


def _collapsed(n):
    rt = synth.make_track(3, n).copy()
    rt[n // 3, 2:] = 1.0                     # w_r + w_l == w_veh: lb == ub == 0 there
    return rt


def _handling(k):
    g = load_golden("handling")
    return g["reftrack"][::k].copy(), float(g["kappa_bound"]), float(g["w_veh"])


ORACLE_CASES = ([(f"synth{n}", lambda n=n: (synth.make_track(1, n), 0.12, 2.0)) for n in (3, 4, 5, 8, 13, 16, 31, 40, 64, 79)]
                + [(f"synth{n}_kb03", lambda n=n: (synth.make_track(1, n), 0.03, 2.0)) for n in (40, 64, 79)]
                + [(f"handling_every{k}", lambda k=k: _handling(k)) for k in (4, 6, 8)]
                + [(f"collapsed{n}", lambda n=n: (_collapsed(n), 0.12, 2.0)) for n in (31, 64)])


def test_against_the_oracle():
    cases = [(name, _case(*make())) for name, make in ORACLE_CASES]
    rt, nv, h, npts = _pack([c for _, c in cases])
    wv = torch.tensor([c["w_veh"] for _, c in cases], dtype=torch.float64, device="cuda")
    kb = torch.tensor([c["kb"] for _, c in cases], dtype=torch.float64, device="cuda")
    res = _np(B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts, small_tracks=True))
    got, want = res["status"].tolist(), [c["status"] for _, c in cases]
    print("statuses:", list(zip([name for name, _ in cases], got, want)))
    assert got == want
    worst = dict(alpha=0.0, klin=0.0, cerr=0.0, stat=0.0)
    for b, (name, c) in enumerate(cases):
        n = c["rt"].shape[0]
        assert not res["alpha"][b, n:].any()
        if c["status"] != 0:
            continue
        a = res["alpha"][b, :n]
        e_a = rel_max(a, c["alpha"])
        e_k = abs(res["kappa_lin_max"][b] - c["klin"]) / c["klin"]
        e_c = abs(res["curv_error_max"][b] - c["cerr"]) / max(c["cerr"], 1e-12)
        lb, ub, _ = Q.bounds(c["rt"], c["w_veh"])
        cert = R.kkt_certificate(c["qp"]["H"], c["qp"]["f"], c["qp"]["E_kappa"], c["qp"]["k_kappa_ref"], lb, ub, c["kb"], a,
                                 act_box=1e-5, act_row=1e-4)
        print(f"{name}: alpha {e_a:.2e}  kappa_lin_max {e_k:.2e}  curv_error_max {e_c:.2e}  stat {cert['stat']:.2e}  "
              f"iters {res['iters'][b]}")
        assert e_a <= ORACLE_TOL["alpha"] and e_k <= ORACLE_TOL["klin"] and e_c <= ORACLE_TOL["cerr"], name
        assert cert["box_viol"] <= CERT_FEAS_TOL and cert["row_viol"] <= CERT_FEAS_TOL, (name, cert)
        assert cert["stat"] <= (CERT_STAT_TOL_COLLAPSED if name.startswith("collapsed") else CERT_STAT_TOL), (name, cert)
        for k, v in (("alpha", e_a), ("klin", e_k), ("cerr", e_c), ("stat", cert["stat"])):
            worst[k] = max(worst[k], v)
    print("worst:", worst)


@pytest.mark.parametrize("lin", [False, True])
def test_dense_against_banded_where_both_apply(lin):
    ns = list(range(B_.N_MIN, B_.N_DENSE_MAX + 1, 7)) + [B_.N_DENSE_MAX]
    cases = [_case(synth.make_track(10 + i, n), 0.12) for i, n in enumerate(ns)]
    rt, nv, h, npts = _pack(cases)
    la = None
    if lin:
        la = 0.3 * torch.sin(torch.arange(h.shape[1], device="cuda", dtype=torch.float64) * 0.37).expand_as(h).contiguous()
    ban = _np(B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, n_pts=npts, lin_alpha=la))
    den = _np(B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, n_pts=npts, lin_alpha=la, _dense_below=B_.N_DENSE_MAX + 1))
    assert den["status"].tolist() == ban["status"].tolist()
    for b, n in enumerate(ns):
        if ban["status"][b] != 0:
            continue
        e_a = rel_max(den["alpha"][b, :n], ban["alpha"][b, :n])
        e_k = abs(den["kappa_lin_max"][b] - ban["kappa_lin_max"][b]) / ban["kappa_lin_max"][b]
        e_c = abs(den["curv_error_max"][b] - ban["curv_error_max"][b]) / ban["curv_error_max"][b]
        print(f"n {n} lin {lin}: alpha {e_a:.2e}  kappa_lin_max {e_k:.2e}  curv_error_max {e_c:.2e}")
        assert e_a <= DVB_TOL and e_k <= DVB_TOL and e_c <= DVB_TOL


def _ragged():
    ns = [3, 1000, 5, 40, 79, 80, 200, 2, 13, 64, 333, 60, 31, 120]
    out = []
    for i, n in enumerate(ns):
        rt = synth.make_track(20 + i, max(n, 3))
        _, _, _, nv = T.calc_splines(_closed(rt))
        out.append(dict(rt=rt, nv=nv, h=_el(rt)) if n >= 3 else None)
    return ns, out


def test_ragged_mixed_batch():
    ns, cs = _ragged()
    base = next(c for c in cs if c is not None)
    cs = [c if c is not None else dict(base, rt=base["rt"][:2], nv=base["nv"][:2], h=base["h"][:2]) for c in cs]
    rt, nv, h, npts = _pack(cs)
    B = len(ns)
    wv = torch.full((B,), 2.0, dtype=torch.float64, device="cuda")
    kb = torch.full((B,), 0.12, dtype=torch.float64, device="cuda")
    small = _np(B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts, small_tracks=True))
    plain = _np(B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts))
    for b, n in enumerate(ns):
        if n >= B_.N_MIN:
            assert all(np.array_equal(small[k][b], plain[k][b]) for k in small), n
        else:
            assert plain["status"][b] == -1
    assert small["status"][ns.index(2)] == -1 and not small["alpha"][ns.index(2)].any()
    # every short track bit for bit as solved alone, and in a batch of 3 x SMs x 8 copies of it
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for b, n in enumerate(ns):
        if not 3 <= n < B_.N_MIN:
            continue
        one = _np(B_.opt_min_curv_batch(rt[b:b + 1, :n], nv[b:b + 1, :n], h[b:b + 1, :n], 0.12, 2.0, small_tracks=True))
        assert all(np.array_equal(one[k][0], small[k][b][:n] if k == "alpha" else small[k][b]) for k in one), n
        if n == 40:
            R_ = 3 * sms * 8
            many = _np(B_.opt_min_curv_batch(rt[b:b + 1, :n].expand(R_, n, 4).contiguous(),
                                             nv[b:b + 1, :n].expand(R_, n, 2).contiguous(),
                                             h[b:b + 1, :n].expand(R_, n).contiguous(), 0.12, 2.0, small_tracks=True))
            assert all((many[k] == one[k][0]).all() for k in many)
    # refusals touch nothing else: a non-finite w_veh, a bad device limit
    wv2, kb2 = wv.clone(), kb.clone()
    i_w, i_k = ns.index(5), ns.index(13)
    wv2[i_w] = float("nan")
    kb2[i_k] = -1.0
    bad = _np(B_.opt_min_curv_batch(rt, nv, h, kb2, wv2, n_pts=npts, small_tracks=True))
    for b in range(B):
        if b in (i_w, i_k):
            assert bad["status"][b] == -1 and not bad["alpha"][b].any()
        else:
            assert all(np.array_equal(bad[k][b], small[k][b]) for k in bad), b


def test_all_short_batch_and_shared_centre_lines():
    cs = [_case(synth.make_track(1, 40), 0.12), _case(synth.make_track(2, 31), 0.12)]
    wide = dict(cs[0], rt=cs[0]["rt"].copy())
    wide["rt"][:, 2:] *= 1.3
    cs = [cs[0], wide, cs[1], cs[0]]
    rt, nv, h, npts = _pack(cs)
    assert rt.shape[1] < B_.N_MIN
    res = _np(B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, n_pts=npts, small_tracks=True))
    cid = torch.tensor([0, 0, 2, 2], dtype=torch.int32, device="cuda")     # the last: another track's n_pts -> -1
    sh = _np(B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, n_pts=npts, small_tracks=True, centre_id=cid))
    assert sh["status"].tolist() == res["status"][:3].tolist() + [-1]
    for b in range(3):
        assert all(np.array_equal(sh[k][b], res[k][b]) for k in sh), b
    with pytest.raises(NotImplementedError):
        B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, n_pts=npts)


def test_iqp_on_short_tracks():
    kb, wv = 0.12, 2.0
    tracks = [(synth.make_track(1, 60), 3.0)]
    rt_h, kb_h, wv_h = _handling(1)
    tracks.append((rt_h, 8.0))                      # re-sampled at 8 m the handling track drops below N_MIN points
    for rt, step in tracks:
        k, w = (kb, wv) if rt is not rt_h else (kb_h, wv_h)
        _, _, A, nv = T.calc_splines(_closed(rt))
        a_o, rt_o, nv_o = T.iqp_handler(rt, nv, A, k, w, False, False, step, 3, 0.01)
        dev = torch.device("cuda")
        res = B_.iqp_batch(torch.tensor(rt[None], device=dev), torch.tensor(nv[None], device=dev),
                           torch.tensor(_el(rt)[None], device=dev), k, w, step, iters_min=3, curv_error_allowed=0.01,
                           small_tracks=True)
        n = int(res["n_pts"][0])
        assert int(res["status"][0]) == 0 and n == rt_o.shape[0], (n, rt_o.shape)
        e_a = rel_max(res["alpha"][0, :n].cpu().numpy(), a_o)
        e_r = np.abs(res["reftrack"][0, :n].cpu().numpy() - rt_o).max()
        print(f"iqp n {rt.shape[0]} -> {n} at {step} m: alpha {e_a:.2e}  reftrack {e_r:.2e} m")
        assert e_a <= IQP_TOL["alpha"] and e_r <= IQP_TOL["reftrack"]


@pytest.mark.parametrize("opt_type", ["mincurv", "mincurv_iqp"])
def test_globaltraj_plans_a_short_track(golden, opt_type):
    v = golden("velprofile")
    pars = globaltraj.default_pars()
    rt = synth.make_track(1, 60)
    dev = torch.device("cuda")
    rt_t = torch.tensor(rt[None], device=dev)
    out = globaltraj.globaltraj_batch(rt_t, opt_type, pars, v["ggv"], v["ax_max_machines"], small_tracks=True, check=False)
    assert int(out["status"][0]) == 0 and np.isfinite(float(out["laptime"][0])) and float(out["laptime"][0]) > 0.0
    if opt_type == "mincurv":
        _, _, A, nv = T.calc_splines(_closed(rt))
        kb, wv = float(pars["veh_params"]["curvlim"]), float(pars["optim_opts"]["width_opt"])
        a_o, _ = T.opt_min_curv(rt, nv, A, kb, wv)
        assert rel_max(out["alpha"][0, :60].cpu().numpy(), a_o) <= ALPHA_TOL
        rl = T.create_raceline(rt[:, :2], nv, a_o, pars["stepsize_opts"]["stepsize_interp_after_opt"])
        m = min(rl[0].shape[0], int(out["n_out"][0]))
        assert abs(rl[0].shape[0] - int(out["n_out"][0])) <= 1
        assert np.abs(out["raceline_interp"][0, :m].cpu().numpy() - rl[0][:m]).max() <= 1e-5
    with pytest.raises(NotImplementedError):        # without the flag a track below N_MIN points is refused
        globaltraj.globaltraj_batch(rt_t, opt_type, pars, v["ggv"], v["ax_max_machines"], check=False)
