"""GPU tests (-m gpu) of the minimum-curvature path where its kernels change code path, against CPU references:

A  the assembled QP (band of H, f, k_ref, x', y', bounds) read back from the workspace after mincurv_setup_kernel alone,
   against the dense oracle, on every golden fixture, every N from 80 to 96 and sizes that are not multiples of 8 or 32,
   strongly non-uniform spacing, and shared centre lines (mincurv_share_kernel);
B  full solves from N_MIN = 80 to 257 (every panel residue), box-only and curvature-row-active, against the oracle and
   the KKT certificate of the full QP (tests/mincurv_ref.py), and the width gradients against tests/qp_sens.py;
C  the curvature-row phase (mincurv_pdip_kappa_kernel) in a mixed batch, unshared and with shared centre lines;
D  the persistent solver kernels with more instances than resident CTAs (a CTA solves many instances of different n);
E  the three algorithms and two scratch placements of closed_spline (splines.cu), against a sparse direct solve.
Measured values are printed next to every tolerance that was set from a measurement (pytest -s)."""
import ctypes

import numpy as np
import pytest

import mincurv_ref as R
import qp_sens as Q
from conftest import rel_max

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402
from oracle import tph_dense as T  # noqa: E402

ALPHA_TOL = 1e-4          # the north-star bar of BASELINE.json
KAPPA_TOL = 1e-3
GRAD_TOL = 1e-5           # tests/test_gpu_sensitivity.py
# The device differentiates the interior-point iterate at which the solver stops (DESIGN.md 3.10): the gradient around a
# bound active with a multiplier of 6e-4 .. 3e-2 |f|_inf is damped by ~H_ii / d there.  Measured (worst component):
# N91 7.5e-5 (weakest active multiplier 6e-4 |f|_inf), N92 1.2e-5 (3e-2), N93 3.6e-5 (2e-3), N95 3.7e-5 (1e-3).
WEAK_TOL = {"N91": 2e-4, "N92": 5e-5, "N93": 1e-4, "N95": 1e-4}
GOLDEN = ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth1000", "synth128",
          "synth160_kappa", "synth200", "synth2000", "synth333", "synth333_kappa", "synth500", "synth500_narrow"]
# Assembly: max|device - oracle| / max|oracle| per quantity.  The band entries are exact sums (no truncation inside the
# band) and the oracle's H beyond half-bandwidth 32 is <= 1.3e-17 max|H|, so what remains is rounding.  Measured on an
# H100: band 9.3e-13, x'/y' 4.6e-13 (both synth2000); f and k_ref below 1e-10 except on the 1:20 track.
ASM_TOL = dict(band=5e-12, f=1e-10, kref=1e-10, xp=4e-12)
# 1:20 spacing: the oracle's dense inverse of the 4N spline system (cond 7e4) is itself off by 5.9e-11 in k_ref there
# (against mincurv_ref.periodic_spline); f = E^T k_ref carries it.  Measured: f 3.6e-10, k_ref 7.1e-11.
ASM_TOL_1_20 = dict(f=2e-9, kref=5e-10)
# KKT certificate of a device solution (mincurv_ref.kkt_certificate with the oracle's H, f, E, k_ref).  The solver stops
# at mu <= 1e-10 mu0 (box phase) / 1e-11 mu0 (curvature-row phase) and |r_d| <= 1e-8 (|f| + |g0|)
# (mincurv_ipm.cu); the multipliers of the constraints the certificate treats as inactive are ~mu / slack.  Measured on an
# H100 over B and C:
# stationarity 8.3e-7 (synth333_kappa), complementarity 4.0e-10 (the collapsed-box instance of C).
CERT_STAT_TOL = 8e-6
CERT_COMP_TOL = 4e-9
# A collapsed box is 2e-8 m wide: the barrier terms l / s there are ~1e8 times those of an ordinary bound and the dual
# residual the solver stops at is that much less balanced.  Measured: 4.3e-5 (alpha within 9.5e-8 of the oracle's).
CERT_STAT_TOL_COLLAPSED = 4e-4
CERT_FEAS_TOL = 1e-9      # box [m] and curvature rows [1/m]: the iterate is interior; what remains is E of device vs oracle


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _closed(rt):
    return np.vstack((rt[:, :2], rt[0, :2]))


def _el(rt):
    return np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1)


def _oracle_case(rt, kb, w_veh=2.0, solve=True):
    """The oracle's normals, h and QP of a track (and its solution with solve=True)."""
    _, _, A, nv = T.calc_splines(_closed(rt))
    qp = T.assemble_min_curv(rt, nv, A, kb, w_veh)
    c = dict(rt=rt, nv=nv, h=_el(rt), qp=qp, w_veh=w_veh, kb=kb)
    if solve:
        alpha, cerr = T.opt_min_curv(rt, nv, A, kb, w_veh)
        c.update(alpha=alpha, cerr=cerr, klin=float(np.abs(qp["k_kappa_ref"] + qp["E_kappa"] @ alpha).max()))
    return c


def _pack(cases, n_max=None):
    """Ragged device batch (reftrack, normvec, h, n_pts, w_veh [B]) from dicts with rt, nv, h, w_veh."""
    dev = torch.device("cuda")
    n = [c["rt"].shape[0] for c in cases]
    n_max = n_max or max(n)
    rt, nv, h = np.zeros((len(cases), n_max, 4)), np.zeros((len(cases), n_max, 2)), np.ones((len(cases), n_max))
    for b, c in enumerate(cases):
        rt[b, :n[b]], nv[b, :n[b]], h[b, :n[b]] = c["rt"], c["nv"], c["h"]
    f64 = dict(dtype=torch.float64, device=dev)
    return (torch.tensor(rt, **f64), torch.tensor(nv, **f64), torch.tensor(h, **f64),
            torch.tensor(n, dtype=torch.int32, device=dev), torch.tensor([c["w_veh"] for c in cases], **f64))


def _certify(c, alpha, rows=True):
    lb, ub, _ = Q.bounds(c["rt"], c["w_veh"])
    qp = c["qp"]
    return R.kkt_certificate(qp["H"], qp["f"], qp["E_kappa"], qp["k_kappa_ref"], lb, ub, c["kb"], alpha, rows=rows,
                             act_box=1e-5, act_row=1e-4)


def _assert_certified(cert, what, collapsed=False):
    assert cert["box_viol"] <= CERT_FEAS_TOL and cert["row_viol"] <= CERT_FEAS_TOL, (what, cert)
    assert cert["stat"] <= (CERT_STAT_TOL_COLLAPSED if collapsed else CERT_STAT_TOL), (what, cert)
    assert cert["comp"] <= CERT_COMP_TOL, (what, cert)


def _res_np(res):
    return {k: v.detach().cpu().numpy() for k, v in res.items()}


# ---------------------------------------------------------------------------------------------------------------------
# A. assembly
# ---------------------------------------------------------------------------------------------------------------------
def _setup_only(cases, n_max, centre_id=None):
    """mc_mincurv_setup_batch_shared alone on a workspace owned here; returns (workspace as float64 numpy, status)."""
    lib = _lib.load()
    rt, nv, h, npts, wv = _pack(cases, n_max)
    B = len(cases)
    nbytes = lib.mc_mincurv_workspace_bytes(B, n_max)
    ws = torch.zeros(nbytes // 8, dtype=torch.float64, device="cuda")
    status = torch.full((B,), -7, dtype=torch.int32, device="cuda")
    cid = None if centre_id is None else torch.tensor(centre_id, dtype=torch.int32, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None      # noqa: E731
    rc = lib.mc_mincurv_setup_batch_shared(B, n_max, p(npts), p(rt), p(nv), p(h), 0.0, p(wv), float(B_.F_SCALE), p(cid),
                                           p(status), p(ws), nbytes, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check(rc, "mc_mincurv_setup_batch_shared")
    torch.cuda.synchronize()
    return ws.cpu().numpy(), status.cpu().numpy()


def _slab(ws, b, lay):
    return ws[b * lay["stride"]:(b + 1) * lay["stride"]]


def _vec(slab, lay, name, n):
    o = B_.SLAB_VECTORS.index(name) * lay["np"]
    return slab[o:o + n]


def _band(slab, lay, n):
    return slab[lay["o_hb"]:lay["o_hb"] + lay["np"] * B_.HB_PITCH].reshape(-1, B_.HB_PITCH)[:n, :33]


def _hbsrc(slab, lay):
    o = B_.SLAB_VECTORS.index("HBSRC") * lay["np"]
    return int(slab[o:o + 1].view(np.int32)[0])


def _band_of(H):
    n = H.shape[0]
    i = np.arange(n)
    return np.stack([H[i, (i + k) % n] for k in range(33)], axis=1)


def _assembly_cases(golden):
    cases = []
    for name in GOLDEN:
        g = golden(name)
        cases.append(dict(name=name, rt=g["reftrack"], nv=g["normvec"], h=g["el_lengths"], w_veh=float(g["w_veh"]),
                          band=g["H_band"], f=g["f"], kref=g["k_kappa_ref"], xp=g["x_prime"], yp=g["y_prime"]))
    live = [(f"synth{n}", synth.make_track(600 + n, n)) for n in list(range(80, 97)) + [103, 111, 119, 127, 129]]
    live += [("spacing1:5", R.uneven_track(260, 5.0, 1)), ("spacing1:20", R.uneven_track(300, 20.0, 2))]
    for name, rt in live:
        c = _oracle_case(rt, 0.12, solve=False)
        qp = c["qp"]
        c.update(name=name, band=_band_of(qp["H"]), f=qp["f"], kref=qp["k_kappa_ref"], xp=qp["x_prime"], yp=qp["y_prime"])
        cases.append(c)
    return cases


def test_assembly_matches_the_dense_oracle(golden):
    cases = _assembly_cases(golden)
    el = _el(cases[-1]["rt"])
    assert el.max() / el.min() > 18.0
    n_max = max(c["rt"].shape[0] for c in cases) + 3
    assert n_max % 8 and n_max % 32
    lay = B_.mincurv_slab_layout(n_max)
    ws, status = _setup_only(cases, n_max)
    assert status.tolist() == [0] * len(cases)
    worst, errs = {}, []
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        s = _slab(ws, b, lay)
        e = dict(band=rel_max(_band(s, lay, n), c["band"]), f=rel_max(_vec(s, lay, "F", n), c["f"]),
                 kref=rel_max(_vec(s, lay, "KREF", n), c["kref"]),
                 xp=float(np.hypot(_vec(s, lay, "XP", n) - c["xp"], _vec(s, lay, "YP", n) - c["yp"]).max()
                          / np.hypot(c["xp"], c["yp"]).max()))
        lb, ub, _ = Q.bounds(c["rt"], c["w_veh"])
        assert np.array_equal(_vec(s, lay, "LB", n), lb) and np.array_equal(_vec(s, lay, "UB", n), ub), c["name"]
        assert _hbsrc(s, lay) == b
        for k, v in e.items():
            if v > worst.get(k, (0.0, ""))[0]:
                worst[k] = (v, c["name"])
        errs.append(e)
    print("assembly, worst max|diff| / max|ref|:", {k: f"{e:.1e} ({name})" for k, (e, name) in worst.items()})
    for c, e in zip(cases, errs):
        tol = dict(ASM_TOL, **ASM_TOL_1_20) if c["name"] == "spacing1:20" else ASM_TOL
        assert all(e[k] <= tol[k] for k in e), (c["name"], e)


def test_assembly_bounds_collapsed_boxes_and_shared_centre_lines(golden):
    """Collapsed boxes get mid -+ FIX_EPS; followers get the owner's vectors bit for bit and point at its band; an owner
    whose own bounds are infeasible still assembles for its followers."""
    g = golden("synth128")
    base = dict(rt=g["reftrack"], nv=g["normvec"], h=g["el_lengths"], w_veh=2.0)
    collapsed = dict(base, rt=g["reftrack"].copy())
    for i in (10, 60, 61):
        collapsed["rt"][i, 3] = 2.0 - collapsed["rt"][i, 2] + 1e-9
    narrow = dict(base, rt=g["reftrack"].copy())
    narrow["rt"][40:44, 2:] = 0.5                                     # 1 m wide for a 2 m vehicle
    wide = dict(base, rt=synth.jitter_widths(g["reftrack"], 3))
    other = _oracle_case(synth.make_track(9, 100), 0.12, solve=False)
    cases = [base, collapsed, narrow, wide, other, dict(base)]
    # groups: {0 (owner), 1, 5}, {2 (owner, infeasible), 3}, {4} alone
    cid = [0, 0, 2, 2, 4, 0]
    n_max, n = 131, 128
    lay = B_.mincurv_slab_layout(n_max)
    ws0, st0 = _setup_only(cases, n_max)
    ws1, st1 = _setup_only(cases, n_max, centre_id=cid)
    assert st0.tolist() == [0, 0, 1, 0, 0, 0] and st1.tolist() == st0.tolist()
    lb, ub, col = Q.bounds(collapsed["rt"], 2.0)
    assert col.sum() == 3 and np.all(ub[col] - lb[col] == pytest.approx(2e-8, rel=1e-6))
    copied = B_.SLAB_VECTORS[:B_.SLAB_VECTORS.index("KREF") + 1] + ["F", "IH"]
    for b, c in enumerate(cases):
        nb = c["rt"].shape[0]
        s0, s1, so = _slab(ws0, b, lay), _slab(ws1, b, lay), _slab(ws1, cid[b], lay)
        lb, ub, _ = Q.bounds(c["rt"], 2.0)
        assert np.array_equal(_vec(s1, lay, "LB", nb), lb) and np.array_equal(_vec(s1, lay, "UB", nb), ub), b
        assert _hbsrc(s1, lay) == cid[b]
        for name in copied:
            assert np.array_equal(_vec(s1, lay, name, nb), _vec(so, lay, name, nb)), (b, name)
            if b != 2:                                                # (unshared, an infeasible instance stops early)
                assert np.array_equal(_vec(s1, lay, name, nb), _vec(s0, lay, name, nb)), (b, name)
        if cid[b] == b:
            assert np.array_equal(_band(s1, lay, nb), _band(_slab(ws0, 0 if b == 2 else b, lay), lay, nb)), b
    # the infeasible owner assembled: its band and f are those of its centre line
    assert np.array_equal(_vec(_slab(ws1, 2, lay), lay, "F", n), _vec(_slab(ws0, 0, lay), lay, "F", n))


# ---------------------------------------------------------------------------------------------------------------------
# B. full solves from N_MIN
# ---------------------------------------------------------------------------------------------------------------------
SMALL_N = list(range(80, 97)) + [97, 103, 111, 119, 127, 129, 255, 257]


def _check_against_oracle(cases, res, tag):
    out = _res_np(res)
    worst = dict(alpha=0.0, stat=0.0, comp=0.0)
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        a = out["alpha"][b, :n]
        what = f"{tag} {c.get('name', b)}"
        assert out["status"][b] == 0, what
        err = rel_max(a, c["alpha"])
        assert err <= ALPHA_TOL, (what, err)
        assert abs(out["curv_error_max"][b] - c["cerr"]) <= 1e-3 * c["cerr"] + 1e-7, what
        assert abs(out["kappa_lin_max"][b] - c["klin"]) <= KAPPA_TOL * c["klin"], what
        cert = _certify(c, a)
        print(f"  {what}: n={n} iters={out['iters'][b]} alpha {err:.1e} stat {cert['stat']:.1e} comp {cert['comp']:.1e} "
              f"n_active {cert['n_active']}")
        _assert_certified(cert, f"{what} iters {out['iters'][b]}", collapsed=bool(Q.bounds(c["rt"], c["w_veh"])[2].any()))
        worst = dict(alpha=max(worst["alpha"], err), stat=max(worst["stat"], cert["stat"]),
                     comp=max(worst["comp"], cert["comp"]))
    print(f"{tag}: worst alpha rel err {worst['alpha']:.1e}, certificate stat {worst['stat']:.1e}, comp {worst['comp']:.1e}")
    return out


def test_full_solves_from_n_min_against_the_oracle_and_the_certificate():
    cases = [dict(_oracle_case(synth.make_track(700 + n, n), 0.12), name=f"N{n}") for n in SMALL_N]
    rt, nv, h, npts, wv = _pack(cases)
    res = B_.opt_min_curv_batch(rt, nv, h, 0.12, wv, n_pts=npts)
    _check_against_oracle(cases, res, "box-only, N 80..257")
    # width gradients of the box-only instances
    widths = rt[:, :, 2:].clone().requires_grad_()
    wvg = wv.clone().requires_grad_()
    d = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, wvg, n_pts=npts)
    assert torch.equal(d["alpha"].detach(), res["alpha"])
    rng = np.random.default_rng(4)
    gbar = np.zeros(rt.shape[:2])
    for b, c in enumerate(cases):
        gbar[b, :c["rt"].shape[0]] = rng.standard_normal(c["rt"].shape[0])
    gw, gv = (t.cpu().numpy() for t in torch.autograd.grad(d["alpha"], (widths, wvg), torch.tensor(gbar, device="cuda")))
    worst, errs = (0.0, ""), []
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        if c["klin"] > 0.12 * (1 + 1e-7):
            continue                                                    # (curvature rows active: no gradient)
        assert int(d["grad_status"][b]) == 0
        ref = Q.width_vjp(c["qp"]["H"], c["qp"]["f"], c["rt"], 2.0, gbar[b, :n], alpha=c["alpha"])
        keep = ~_degenerate(ref, np.abs(c["qp"]["f"]).max())
        e = max(rel_max(gw[b, :n, 0][keep], ref["grad_w_right"][keep]), rel_max(gw[b, :n, 1][keep], ref["grad_w_left"][keep]),
                abs(gv[b] - ref["grad_w_veh"]) / abs(ref["grad_w_veh"]))
        worst = max(worst, (e, c["name"]))
        act = ref["at_ub"] | ref["at_lb"]
        weakest = float(np.where(act, ref["lu"] + ref["ll"], np.inf).min() / np.abs(c["qp"]["f"]).max())
        errs.append((c["name"], e, weakest))
    print(f"width gradients, N 80..257: worst rel err {worst[0]:.1e} ({worst[1]});",
          "above GRAD_TOL (weakest active multiplier / |f|_inf):", [f"{a} {e:.1e} ({w:.0e})" for a, e, w in errs if e > GRAD_TOL])
    for name, e, _ in errs:
        assert e <= WEAK_TOL.get(name, GRAD_TOL), (name, e)


def _degenerate(ref, scale):
    """As in test_gpu_sensitivity.py: bounds active with a multiplier below 1e-6 |f|_inf or inactive within 1e-6 m."""
    weak = (ref["at_ub"] & (ref["lu"] < 1e-6 * scale)) | (ref["at_lb"] & (ref["ll"] < 1e-6 * scale))
    a = ref["alpha"]
    near = ~(ref["at_ub"] | ref["at_lb"]) & (np.minimum(ref["ub"] - a, a - ref["lb"]) < 1e-6)
    return weak | near


@pytest.mark.parametrize("seed,n,kb", [(3, 87, 0.04), (4, 96, 0.03), (5, 100, None)])
def test_curvature_rows_at_small_n(seed, n, kb):
    """kb None: 0.5 % below the largest curvature of the box-only optimum (rows barely active)."""
    rt = synth.make_track(seed, n)
    if kb is None:
        c = _oracle_case(rt, 0.12, solve=False)
        lb, ub, _ = Q.bounds(rt, 2.0)
        box = Q.solve_box_qp(c["qp"]["H"], c["qp"]["f"], lb, ub)
        kb = float(np.abs(c["qp"]["k_kappa_ref"] + c["qp"]["E_kappa"] @ box).max()) / 1.005
    c = dict(_oracle_case(rt, kb), name=f"make_track({seed}, {n})")
    lb, ub, _ = Q.bounds(c["rt"], 2.0)
    box = Q.solve_box_qp(c["qp"]["H"], c["qp"]["f"], lb, ub)
    assert np.abs(c["qp"]["k_kappa_ref"] + c["qp"]["E_kappa"] @ box).max() > kb * 1.004     # the rows cut off the box optimum
    rt, nv, h, npts, wv = _pack([c])
    _check_against_oracle([c], B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts), f"rows active, N={n}")


# ---------------------------------------------------------------------------------------------------------------------
# C. the curvature-row phase in mixed batches
# ---------------------------------------------------------------------------------------------------------------------
KB_MIXED = 0.0185


def _mixed_cases(golden):
    """(cases, centre_id, rows): the mixed batch at KB_MIXED and which instances have active curvature rows."""
    wide = synth.make_track(1, 200, amp=0.15)                          # box-only at KB_MIXED
    narrow = wide.copy()
    narrow[:, 2:] *= 0.45                                              # same centre line, curvature rows active
    flat = synth.make_track(2, 240, amp=0.1)
    infeasible = flat.copy()
    infeasible[100:104, 2:] = 0.5
    collapsed = flat.copy()
    for i in (5, 77, 78):
        collapsed[i, 3] = 2.0 - collapsed[i, 2] + 1e-9
    tracks = [("synth160_kappa", golden("synth160_kappa")["reftrack"]), ("synth333_kappa", golden("synth333_kappa")["reftrack"]),
              ("N1000", synth.make_track(11, 1000)), ("wide owner", wide), ("narrow follower", narrow),
              ("narrow owner", narrow), ("wide follower", wide), ("infeasible", infeasible), ("collapsed", collapsed),
              ("flat", flat)]
    cases = []
    for name, rt in tracks:
        if name == "infeasible":
            c = dict(_oracle_case(flat, KB_MIXED, solve=False), rt=rt)
        else:
            c = _oracle_case(rt, KB_MIXED)
        cases.append(dict(c, name=name))
    centre_id = [0, 1, 2, 3, 3, 5, 5, 7, 8, 9]
    rows = [0, 1, 2, 4, 5]
    return cases, centre_id, rows


def _poison_workspaces():
    """NaN into the cached solver workspaces, so that no call can pass on what an earlier call left in its slabs."""
    torch.cuda.synchronize()
    for k, ws in B_._WS.items():
        if k[0] == "mincurv" and ws is not None:
            ws.fill_(0xFF)


def test_curvature_row_phase_in_a_mixed_batch_unshared_and_shared(golden):
    cases, centre_id, rows = _mixed_cases(golden)
    rt, nv, h, npts, wv = _pack(cases)
    res0 = B_.opt_min_curv_batch(rt, nv, h, KB_MIXED, wv, n_pts=npts)
    _poison_workspaces()
    res1 = B_.opt_min_curv_batch(rt, nv, h, KB_MIXED, wv, n_pts=npts, centre_id=torch.tensor(centre_id, device="cuda"))
    for k in res0:
        assert torch.equal(res0[k], res1[k]), k
    # which instances the curvature-row phase solved: the box phase's status, as the sensitivities report it
    d = B_.opt_min_curv_diff(rt[:, :, :2], rt[:, :, 2:].clone().requires_grad_(), nv, h, KB_MIXED, wv, n_pts=npts,
                             strict=False)
    gs = d["grad_status"].tolist()
    assert [b for b, s in enumerate(gs) if s == 4] == rows, gs
    out = _res_np(res0)
    assert out["status"][7] == 1 and np.all(out["alpha"][7] == 0.0)
    solved = [c for b, c in enumerate(cases) if b != 7]
    _check_against_oracle(solved, {k: v[[b for b in range(len(cases)) if b != 7]] for k, v in res0.items()},
                          "mixed batch at kappa_bound 0.0185")


# ---------------------------------------------------------------------------------------------------------------------
# D. more instances than resident CTAs
# ---------------------------------------------------------------------------------------------------------------------
KB_MANY = 0.04


def _many_cases():
    """~24 distinct instances with N in 80..130 (every residue mod 8): box-only, curvature rows, infeasible, collapsed and
    one group of three width variants of one centre line (group label 100)."""
    spec = [(80, 0.6, 1.0), (81, 0.3, 1.0), (82, 0.15, 1.0), (83, 0.3, 1.0), (84, 0.15, 1.0), (85, 0.3, 1.0),
            (86, 0.15, 1.0), (87, 0.6, 1.0), (94, 0.6, 1.0), (96, 0.3, 1.0), (101, 0.6, 1.0), (103, 0.15, 1.0),
            (108, 0.6, 0.4), (111, 0.3, 1.0), (115, 0.6, 0.4), (119, 0.15, 1.0), (127, 0.3, 1.0), (129, 0.6, 0.4),
            (130, 0.3, 1.0)]
    rts, groups = [], []
    for n, amp, wsc in spec:
        rt = synth.make_track(n, n, amp=amp)
        rt[:, 2:] *= wsc
        rts.append(rt)
    bad = synth.make_track(90, 90, amp=0.3)
    bad[30:33, 2:] = 0.5
    col = synth.make_track(99, 99, amp=0.3)
    for i in (0, 50, 98):
        col[i, 3] = 2.0 - col[i, 2] + 1e-9
    rts += [bad, col]
    groups = list(range(len(rts)))
    base = synth.make_track(122, 122, amp=0.3)
    rts += [base, synth.jitter_widths(base, 1), synth.jitter_widths(base, 2)]
    groups += [100, 100, 100]
    cases = []
    for rt in rts:
        _, _, nv = R.periodic_spline(_closed(rt))
        cases.append(dict(rt=rt, nv=nv, h=_el(rt), w_veh=2.0))
    return cases, groups


def _solve_many(rt, nv, h, npts, wv, cid, gbar):
    B = rt.shape[0]
    res = B_.opt_min_curv_batch(rt, nv, h, KB_MANY, wv, n_pts=npts, centre_id=cid, max_chunk=B)
    widths = rt[:, :, 2:].clone().requires_grad_()
    wvg = wv.clone().requires_grad_()
    d = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, KB_MANY, wvg, n_pts=npts, centre_id=cid, max_chunk=B, strict=False)
    gw, gv = torch.autograd.grad(d["alpha"], (widths, wvg), gbar)
    out = _res_np(res)
    out.update(grad_status=d["grad_status"].cpu().numpy(), gw=gw.cpu().numpy(), gv=gv.cpu().numpy(),
               diff_alpha=d["alpha"].detach().cpu().numpy())
    return out


def test_more_instances_than_resident_ctas_give_bitwise_the_same_results():
    cases, groups = _many_cases()
    ns = sorted({c["rt"].shape[0] for c in cases})
    assert {n % 8 for n in ns} == set(range(8)) and ns[0] == 80 and ns[-1] <= 130
    m = len(cases)
    rt, nv, h, npts, wv = _pack(cases, n_max=130)
    dev = rt.device
    gbar = torch.tensor(np.random.default_rng(8).standard_normal(rt.shape[:2]), device=dev)
    gbar *= (torch.arange(130, device=dev)[None, :] < npts[:, None])
    cid = B_.shared_centre_ids(torch.tensor(groups, device=dev))
    ref = _solve_many(rt, nv, h, npts, wv, cid, gbar)
    assert set(ref["grad_status"].tolist()) == {0, 1, 4}, ref["grad_status"]          # box-only, infeasible, rows
    assert np.all(ref["status"][ref["grad_status"] != 1] == 0)
    # the big batch: every instance repeated, in a seeded shuffled order
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    B = -(-3 * sms * 8 // m) * m
    src = np.random.default_rng(12).permutation(B)
    orig, copy = src % m, src // m
    idx = torch.tensor(orig, device=dev)
    labels = torch.tensor([copy[p] * 1000 + groups[orig[p]] for p in range(B)], device=dev)
    big = [_solve_many(rt[idx], nv[idx], h[idx], npts[idx], wv[idx], B_.shared_centre_ids(labels), gbar[idx]) for _ in range(2)]
    print(f"{B} instances ({sms} SMs) of {m} distinct ones, n_max 130")
    for k in ("alpha", "status", "iters", "curv_error_max", "kappa_lin_max", "grad_status", "gw", "gv", "diff_alpha"):
        assert np.array_equal(big[0][k], big[1][k]), k
        assert np.array_equal(big[0][k], ref[k][orig]), k


# ---------------------------------------------------------------------------------------------------------------------
# E. spline regimes
# ---------------------------------------------------------------------------------------------------------------------
SPLINE_N = [3, 4, 5, 31, 32, 33, 63, 64, 65, 1024, 1025, 2048, 2049, 3000]


def _spline_tracks():
    tr = [R.uneven_track(n, 1.0, n, step=20.0) for n in SPLINE_N if n < 100]
    tr += [synth.make_track(n, n) for n in SPLINE_N if n >= 100]
    tr += [R.uneven_track(400, 20.0, 3), R.uneven_track(2049, 20.0, 4), R.uneven_track(3000, 20.0, 5)]
    return tr


def _spline_run(tracks, n_max):
    dev = torch.device("cuda")
    n = [t.shape[0] for t in tracks]
    xy = np.zeros((len(tracks), n_max, 4))
    for b, t in enumerate(tracks):
        xy[b, :n[b]] = t
    xy = torch.tensor(xy, device=dev)
    npts = torch.tensor(n, dtype=torch.int32, device=dev)
    out = {}
    for ds in (False, True):
        cx, cy, nv, h = B_.calc_splines_batch(xy, n_pts=npts, use_dist_scaling=ds)
        out[ds] = [(cx[b, :n[b]].cpu().numpy(), cy[b, :n[b]].cpu().numpy(), nv[b, :n[b]].cpu().numpy()) for b in range(len(n))]
    alpha = torch.zeros((len(tracks), n_max), dtype=torch.float64, device=dev)
    for b in range(len(n)):
        alpha[b, :n[b]] = 0.3 * torch.sin(torch.arange(n[b], device=dev) * (2.0 * np.pi * 3 / n[b]))
    rl = B_.create_raceline_batch(xy, nv, alpha, 2.0, n_pts=npts)
    m = rl["n_out"].cpu().numpy()
    per_spline = ("coeffs_x", "coeffs_y", "spline_lengths")
    out["rl"] = [{k: v[b, :(n[b] if k in per_spline else m[b])].cpu().numpy() for k, v in rl.items() if k != "n_out"}
                 for b in range(len(n))]
    out["rl_in"] = [(xy[b, :n[b], :2] + alpha[b, :n[b], None] * nv[b, :n[b]]).cpu().numpy() for b in range(len(n))]
    out["n_out"] = m
    return out


def _eval(c, ind, t):
    c = c[ind]
    return c[:, 0] + c[:, 1] * t + c[:, 2] * t ** 2 + c[:, 3] * t ** 3


def test_spline_regimes_shared_and_global_scratch():
    tracks = _spline_tracks()
    runs = [_spline_run(tracks, n_max) for n_max in (3100, 3600)]     # shared-memory scratch / global-memory scratch
    worst = dict(coeffs=0.0, normvec=0.0, raceline=0.0)
    for b, t in enumerate(tracks):
        n = t.shape[0]
        for ds in (True, False):
            for x0, x1 in zip(runs[0][ds][b], runs[1][ds][b]):
                assert np.array_equal(x0, x1), (n, ds)
            cx, cy, nv = runs[0][ds][b]
            rx, ry, rnv = R.periodic_spline(_closed(t), ds)
            e = max(np.abs(cx - rx).max(), np.abs(cy - ry).max())
            worst["coeffs"], worst["normvec"] = max(worst["coeffs"], e), max(worst["normvec"], np.abs(nv - rnv).max())
            assert e < 1e-9 and np.abs(nv - rnv).max() < 1e-11, (n, ds, e)
        r0, r1 = runs[0]["rl"][b], runs[1]["rl"][b]
        for k in r0:
            assert np.array_equal(r0[k], r1[k]), (n, k)
        rx, ry, _ = R.periodic_spline(_closed(runs[0]["rl_in"][b]), False)
        e = max(np.abs(r0["coeffs_x"] - rx).max(), np.abs(r0["coeffs_y"] - ry).max())
        assert e < 1e-9, (n, e)
        ind, tv, xy = r0["spline_inds"], r0["t_values"], r0["raceline_interp"]
        ev = max(np.abs(_eval(r0["coeffs_x"], ind, tv) - xy[:, 0]).max(), np.abs(_eval(r0["coeffs_y"], ind, tv) - xy[:, 1]).max())
        worst["raceline"] = max(worst["raceline"], ev)
        assert ev < 1e-9, (n, ev)
        # the properties of test_gpu_parity.py::test_raceline_batch_properties_at_baseline_size
        m = int(runs[0]["n_out"][b])
        s, el, L = r0["s_interp"], r0["el_lengths_interp"], float(r0["spline_lengths"].sum())
        assert m > 0 and np.all(np.diff(s) > 0) and abs(s[-1] + el[-1] - L) < 1e-8
        assert abs(el[:-1].std()) < 1e-9 and m == int(np.ceil(L / 2.0))
        assert np.all((tv >= 0) & (tv < 1.0 + 1e-12)) and np.all(np.diff(ind) >= 0) and ind[-1] <= n - 1
        # chord ~ arc at 2 m steps where the spline is close to arc-length parametrised: not with three to five splines
        # around a loop (0.23 m at n = 3 in the oracle's create_raceline), nor on the 1:20 tracks (create_raceline uses a
        # uniform parameter, so the steps in t are not equidistant in space, as in tph)
        if 31 <= n and b < len(SPLINE_N):
            assert np.abs(np.linalg.norm(np.diff(xy, axis=0), axis=1) - el[:-1]).max() < 0.15, n
            assert np.abs(r0["kappa"]).max() < 0.5
    print("splines, worst abs err vs the sparse solve:", {k: f"{v:.1e}" for k, v in worst.items()})
