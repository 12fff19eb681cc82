"""GPU tests (-m gpu) of the linear algebra under the interior-point solver and its adjoints, at the matrices they see:
the bordered band LDL^T and its sweeps (csrc/mincurv_ipm.cu factor / solve), the Woodbury correction of the strong
curvature rows (mincurv_adjoint_rows_kernel) and the shortest path's cyclic Thomas + Sherman-Morrison solve
(csrc/shortest_path.cu cyc_solve).  At a final iterate D spans 1e-12 .. 1e12 and cond(M) reaches 1e19, so the measure
is the backward error eta of the diagonally scaled system and the scaled forward error against an extended-precision
solution (tests/linalg_ref.py, which also sets the bounds ETA_MAX and FE_C on CPU).  The solvers' own tests cannot see an
inaccurate factor: the interior-point iteration recomputes its residual every step, and the adjoints are compared with
the exact active-set VJP at bounds that are dominated by the stopping iterate.  Part 5 splits those bounds: the device
gradient against the gradient of the extended solve at the device's own D, and what remains to the active-set VJP."""
import os
import re

import numpy as np
import pytest

import linalg_ref as R
import qp_sens as Q
import qp_sens_rows as QR
import sp_sens as S

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, build as _build, synth  # noqa: E402
from test_gpu_edges import ASM_TOL, KB_MIXED, _mixed_cases, _oracle_case, _pack  # noqa: E402
from test_gpu_factor import _cyclic_band_spd  # noqa: E402
from test_gpu_ipm_schedule import GOLDEN, _ragged  # noqa: E402
from test_gpu_sensitivity import WEAK_TOL as BOX_WEAK_TOL, _cases as _box_cases, _degenerate, _device_batch  # noqa: E402
from test_gpu_sensitivity_rows import WEAK_TOL as ROW_WEAK_TOL  # noqa: E402
from test_gpu_shortest_path_sens import FIXTURES as SP_FIXTURES, _device_batch as _sp_batch  # noqa: E402

DEV = "cuda"
F64 = dict(dtype=torch.float64, device=DEV)
I32 = dict(dtype=torch.int32, device=DEV)
LO, HI = 1e-12, 1e12          # the barrier ratios of an inactive / an active bound at a final iterate
CTAS_PER_SM = 8               # resident CTAs of the interior-point kernels per SM (__launch_bounds__(IP_THREADS, 8))


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _sp_enum():
    """name -> index of enum SpVec (csrc/shortest_path.cu): the interleaved vectors of the shortest-path workspace."""
    body = re.search(r"enum\s+SpVec\b[^{]*\{([^}]*)\}", _lib._c_source(os.path.join(_build.CSRC, "shortest_path.cu"))).group(1)
    out, nxt = {}, 0
    for e in filter(str.strip, body.split(",")):
        name, _, value = e.partition("=")
        nxt = int(value) if value.strip() else nxt
        out[name.strip()] = nxt
        nxt += 1
    return out


def _ws(nbytes):
    return torch.zeros(int(nbytes), dtype=torch.uint8, device=DEV)


def _slabs(ws, lay, B):
    return ws.view(torch.float64)[:B * lay["stride"]].view(B, lay["stride"])


def _vecs(ws, lay, B, n_max, *names):
    w = _slabs(ws, lay, B)
    return [w[:, B_.SLAB_VECTORS.index(nm) * lay["np"]:][:, :n_max].cpu().numpy() for nm in names]


def _bands(ws, lay, B):
    w = _slabs(ws, lay, B)
    return w[:, lay["o_hb"]:lay["o_hb"] + lay["np"] * B_.HB_PITCH].reshape(B, lay["np"], B_.HB_PITCH).cpu().numpy()


def _d_patterns(n, rng):
    """name -> D [n]: the diagonals of a final iterate, placed where the factorisation changes code path (8-column panels,
    the chain / separator boundary at n - 32, the wrap n-1 -> 0)."""
    na = n - 32

    def runs(starts, length):
        D = LO * 10.0 ** rng.uniform(0.0, 1.0, n)
        for s in starts:
            D[(s + np.arange(length)) % n] = HI * 10.0 ** -rng.uniform(0.0, 1.0, length)
        return D
    return {"log-uniform": 10.0 ** rng.uniform(-12.0, 12.0, n),
            "runs on panels": runs(range(0, na, 24), 8),
            "runs off panels": runs(range(3, na, 29), 11),
            "run over the separator": runs([na - 5], 12),
            "run through the wrap": runs([n - 6], 13),
            "all active": HI * 10.0 ** -rng.uniform(0.0, 1.0, n),
            "none active": np.full(n, LO)}


def _debug_factor_solve(bands, D, g1, g2, n, n_max):
    """mc_debug_factor_solve on a workspace of this test's own: bands [B, n_max, 33], D, g1, g2 [B, n_max]; returns
    status [B] and DX, T1, T2 [B, n_max] (M x = g1 through the fused forward half, M x = g2 through the full sweeps, and
    again through a second factorisation)."""
    B = len(n)
    lay = B_.mincurv_slab_layout(n_max)
    ws = _ws(_lib.load().mc_mincurv_workspace_bytes(B, n_max))
    w = _slabs(ws, lay, B)
    hb = torch.zeros((B, lay["np"], B_.HB_PITCH), **F64)
    hb[:, :n_max, :R.HBW + 1] = torch.as_tensor(bands[:, :n_max, :R.HBW + 1], **F64)
    w[:, lay["o_hb"]:lay["o_hb"] + hb[0].numel()] = hb.reshape(B, -1)
    for name, v in (("DD", D), ("RHS", g1), ("T0", g2)):
        o = B_.SLAB_VECTORS.index(name) * lay["np"]
        w[:, o:o + n_max] = torch.as_tensor(v, **F64)
    npts = torch.tensor(n, **I32)
    status = torch.full((B,), -7, **I32)
    B_._call("mc_debug_factor_solve", B, n_max, npts, status, ws=ws)
    torch.cuda.synchronize()
    return (status.cpu().numpy(), *_vecs(ws, lay, B, n_max, "DX", "T1", "T2"))


def _check_factor(tag, names, n, bands, D, g1, g2, out, full=()):
    """eta of DX, T1, T2 for every instance; the scaled forward error too for the instances in full.  An instance whose
    D is 1e-12 everywhere may report status 3 (a pivot rounded to zero or below: H alone is only semidefinite), no other."""
    status, DX, T1, T2 = out
    worst, broke = {}, []
    for b, m in enumerate(n):
        if status[b] == 3 and names[b].endswith("none active"):
            broke.append(names[b])
            continue
        assert status[b] == 0, (tag, names[b], int(status[b]))
        M = R.dense_from_device_band(bands[b], m, D[b])
        eta = max(R.backward_error(M, DX[b, :m], g1[b, :m]), R.backward_error(M, T1[b, :m], g2[b, :m]),
                  R.backward_error(M, T2[b, :m], g2[b, :m]))
        assert eta <= R.ETA_MAX, (tag, names[b], eta)
        kind = names[b].split(": ")[-1]
        worst[kind] = max(worst.get(kind, 0.0), eta)
        if b in full:
            c = R.cond_scaled(M)
            fe = max(R.forward_error(M, DX[b, :m], R.solve_extended(M, g1[b, :m])),
                     R.forward_error(M, T1[b, :m], R.solve_extended(M, g2[b, :m])))
            print(f"{tag} {names[b]}: eta {eta:.1e}, cond(SMS) {c:.1e}, forward {fe:.1e} = {fe / (R.U * c):.2f} u cond")
            assert fe <= R.fe_bound(c), (tag, names[b], fe, c)
    print(f"{tag}: worst eta per D pattern", {k: f"{v:.1e}" for k, v in worst.items()})
    if broke:
        print(f"{tag}: status 3 (non-positive pivot) with D = 1e-12 everywhere: {broke}")


# ---- 1. the factorisation and the sweeps through mc_debug_factor_solve --------------------------------------------------

def test_factor_and_sweeps_on_the_fixtures_h_at_final_iterate_diagonals(golden):
    """H of every golden fixture (n = 128 .. 2000) from mc_mincurv_setup_batch_ex, with the D the real box-phase solve
    exports (sens) and every pattern of _d_patterns."""
    gs = [golden(nm) for nm in GOLDEN]
    rt, nv, h, npts, wv = _ragged([g["reftrack"] for g in gs], [float(g["w_veh"]) for g in gs])
    B, n_max = rt.shape[:2]
    lib = _lib.load()
    lay = B_.mincurv_slab_layout(n_max)
    ws = _ws(lib.mc_mincurv_workspace_bytes(B, n_max))
    res = [torch.zeros((B,), **F64) for _ in range(2)] + [torch.zeros((B,), **I32) for _ in range(3)]
    alpha, sens = torch.zeros((B, n_max), **F64), torch.zeros((B, 2, n_max), **F64)
    B_._call("mc_mincurv_solve_batch_sens", B, n_max, npts, rt, nv, h, 1e3, 0.0, wv, B_.F_SCALE, None, alpha, *res[:2],
             res[2], res[3], sens, res[4], None, None, ws=ws)
    assert res[4].tolist() == [0] * B
    H = _bands(ws, lay, B)
    sens = sens.cpu().numpy()
    rng = np.random.default_rng(1)
    names, n, bands, D = [], [], [], []
    for b, nm in enumerate(GOLDEN):
        m = gs[b]["reftrack"].shape[0]
        pats = dict(sens=sens[b, 0, :m] + sens[b, 1, :m], **_d_patterns(m, rng))
        for p, d in pats.items():
            names.append(f"{nm}: {p}")
            n.append(m)
            bands.append(H[b])
            D.append(np.pad(d, (0, n_max - m)))
    bands, D = np.stack(bands), np.stack(D)
    g1, g2 = rng.standard_normal(D.shape), rng.standard_normal(D.shape)
    for b, m in enumerate(n):
        g1[b, m:] = g2[b, m:] = 0.0
    out = _debug_factor_solve(bands, D, g1, g2, n, n_max)
    _check_factor("fixtures", names, n, bands, D, g1, g2, out, full={b for b, nm in enumerate(names) if nm.endswith("sens")})


def test_factor_and_sweeps_every_size_from_n_min_in_a_batch_of_many_waves():
    """A cyclic band of every n from 80 (N_MIN) to 143 -- every residue of NA = n - 32 modulo the panel of 8, every
    position of the separator in the last panels -- with every D pattern, in one ragged batch of more than three times
    the resident CTAs: each CTA factorises instances of different unit counts in turn (the ring parity across
    instances)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    sizes = list(range(B_.N_MIN, 144))
    rng = np.random.default_rng(2)
    Hs = {m: _cyclic_band_spd(m, rng, 0.0)[0] for m in sizes}
    B = 3 * sms * CTAS_PER_SM + 7 * len(sizes)
    n_max = sizes[-1]
    names, n, bands, D = [], [], [], []
    hb = {m: np.stack([Hs[m][np.arange(m), (np.arange(m) + d) % m] for d in range(R.HBW + 1)], axis=1) for m in sizes}
    while len(n) < B:
        m = int(rng.choice(sizes))
        for p, d in _d_patterns(m, rng).items():
            names.append(f"n={m}: {p}")
            n.append(m)
            bands.append(np.pad(hb[m], ((0, n_max - m), (0, 0))))
            D.append(np.pad(d, (0, n_max - m)))
    names, n, bands, D = names[:B], n[:B], np.stack(bands[:B]), np.stack(D[:B])
    assert set(n) == set(sizes)
    g1, g2 = rng.standard_normal(D.shape), rng.standard_normal(D.shape)
    for b, m in enumerate(n):
        g1[b, m:] = g2[b, m:] = 0.0
    print(f"{len(n)} instances, {sms} SMs x {CTAS_PER_SM} resident CTAs")
    out = _debug_factor_solve(bands, D, g1, g2, n, n_max)
    full = {b for b in range(len(n)) if b < 2 * 7 * 4}
    _check_factor("N_MIN..143", names, n, bands, D, g1, g2, out, full=full)


# ---- 2. and 3. the width adjoints ---------------------------------------------------------------------------------------

def _mincurv_adjoint(rt, nv, h, npts, wv, kb, gbar, centre_id=None, rows=False, given=None):
    """mc_mincurv_solve_batch_sens, then mc_mincurv_adjoint_batch on this test's own workspace; the inputs, outputs and
    the slab contents the adjoint leaves (V_DX = v, V_DD = D, V_ISU = the strong rows, the band) as numpy.  given =
    (sens [B, 2, n_max], sens_rows [B, n_max]): no forward solve, the adjoint runs on these ratios and row weights
    (grad_status 0, n_rows the count of weights > 1)."""
    B, n_max = rt.shape[:2]
    lay = B_.mincurv_slab_layout(n_max)
    ws = _ws(_lib.load().mc_mincurv_workspace_bytes(B, n_max))
    cid = None if centre_id is None else torch.tensor(centre_id, **I32)
    alpha, sens = torch.zeros((B, n_max), **F64), torch.zeros((B, 2, n_max), **F64)
    cerr, kmax = torch.zeros((B,), **F64), torch.zeros((B,), **F64)
    st, it, gs = (torch.zeros((B,), **I32) for _ in range(3))
    sr = torch.zeros((B, n_max), **F64) if rows else None
    nr = torch.zeros((B,), **I32) if rows else None
    if given is None:
        B_._call("mc_mincurv_solve_batch_sens", B, n_max, npts, rt, nv, h, kb, 0.0, wv, B_.F_SCALE, cid, alpha, cerr, kmax,
                 st, it, sens, gs, sr, nr, ws=ws)
    else:
        sens, sr = torch.as_tensor(given[0], **F64), torch.as_tensor(given[1], **F64)
        nr = (sr > 1.0).sum(dim=1).to(torch.int32)
    cap = int(nr.max()) if rows else 0
    schur = torch.zeros((B, max(cap * cap, 1)), **F64) if rows else None
    ga = torch.as_tensor(gbar, **F64)
    gwr, gwl, gwv = torch.zeros((B, n_max), **F64), torch.zeros((B, n_max), **F64), torch.zeros((B,), **F64)
    gs2 = gs.clone()
    B_._call("mc_mincurv_adjoint_batch", B, n_max, npts, rt, nv, h, 0.0, wv, B_.F_SCALE, cid, sens, gs2, ga, gwr, gwl, gwv,
             sr, nr, schur, cap, None, ws=ws)
    torch.cuda.synchronize()
    X, DD = _vecs(ws, lay, B, n_max, "DX", "DD")
    isu = _slabs(ws, lay, B)[:, B_.SLAB_VECTORS.index("ISU") * lay["np"]:][:, :n_max].contiguous().view(torch.int32)
    out = dict(X=X, DD=DD, S=isu.cpu().numpy(), band=_bands(ws, lay, B), sens=sens.cpu().numpy(), gs=gs2.cpu().numpy(),
               status=st.cpu().numpy(), gwr=gwr.cpu().numpy(), gwl=gwl.cpu().numpy(), gwv=gwv.cpu().numpy())
    if rows:
        out.update(sens_rows=sr.cpu().numpy(), n_rows=nr.cpu().numpy())
    return out


def _width_grads(v, du, dl, rt, wv):
    """The width gradients of width_grads (csrc/mincurv_ipm.cu) from v, in the same fp64 operations: (gwr, gwl, the
    w_veh terms)."""
    ub, lb = rt[:, 2] - 0.5 * wv, -(rt[:, 3] - 0.5 * wv)
    coll = ub - lb < 2.0 * Q.FIX_EPS
    gu, gl = du * v, dl * v
    half = 0.5 * (gu + gl)
    return np.where(coll, half, gu), np.where(coll, -half, -gl), np.where(coll, 0.0, 0.5 * (gl - gu))


def _check_adjoint_instance(tag, name, out, b, n, gbar, rt, wv, Kd, rows=None):
    """v of instance b against M = Kd + E_S^T diag(W_S) E_S (rows = (E_S, W_S); Kd alone without rows): eta, the scaled
    forward error against the extended solve (in the scaling of Kd), width_grads from v exactly, and the device gradient
    against the gradient of the extended solve (part 5).  Returns the extended gradients (gwr, gwl, gwv)."""
    v, du, dl = out["X"][b, :n], out["sens"][b, 0, :n], out["sens"][b, 1, :n]
    g = gbar[b, :n]
    assert np.array_equal(out["DD"][b, :n], du + dl), (tag, name)
    eta = R.backward_error(Kd if rows is None else R.with_strong_rows(Kd, *rows), v, g)
    x = R.solve_extended(Kd, g) if rows is None else R.solve_extended_rows(Kd, *rows, g)
    c = R.cond_scaled(Kd)
    fe = R.forward_error(Kd, v, x)
    gwr, gwl, terms = _width_grads(v, du, dl, rt, wv)
    assert np.array_equal(out["gwr"][b, :n].view(np.uint64), gwr.view(np.uint64)), (tag, name)
    assert np.array_equal(out["gwl"][b, :n].view(np.uint64), gwl.view(np.uint64)), (tag, name)
    assert not out["gwr"][b, n:].any() and not out["gwl"][b, n:].any()
    assert abs(out["gwv"][b] - terms.sum()) <= 4.0 * n * R.U * np.abs(terms).sum(), (tag, name)
    xr, xl, xt = _width_grads(x, du.astype(np.longdouble), dl.astype(np.longdouble), rt, wv)
    ge = max(R.rel_err(out["gwr"][b, :n], xr), R.rel_err(out["gwl"][b, :n], xl),
             float(abs(out["gwv"][b] - xt.sum()) / max(abs(xt.sum()), np.abs(xt).max())))
    print(f"{tag} {name}: eta {eta:.1e}, cond(SMS) {c:.1e}, forward {fe:.1e} = {fe / (R.U * c):.2f} u cond, "
          f"gradient vs extended {ge:.1e} = {ge / (R.U * c):.2f} u cond")
    assert eta <= R.ETA_MAX, (tag, name, eta)
    assert fe <= R.fe_bound(c), (tag, name, fe, c)
    assert ge <= R.fe_bound(c), (tag, name, ge, c)
    return np.asarray(xr, dtype=np.float64), np.asarray(xl, dtype=np.float64), float(xt.sum())


def _row_system(tag, name, out, b, n, qp):
    """(K + D, (E_S, W_S)) of a pass-1 instance: K the band the adjoint assembled, checked against the oracle's
    H + E^T W_weak E to the assembly tolerance first; the strong rows S (V_ISU) checked to be those of weight > 1."""
    W = out["sens_rows"][b, :n]
    E = qp["E"]
    K_or = qp["H"] + E.T @ (np.where(W <= 1.0, W, 0.0)[:, None] * E)
    K_dev = R.dense_from_device_band(out["band"][b], n)
    i = np.arange(n)
    asm = max(float(np.abs(K_dev[i, (i + k) % n] - K_or[i, (i + k) % n]).max()) for k in range(R.HBW + 1))
    asm /= np.abs(K_or).max()
    assert asm <= ASM_TOL["band"], (tag, name, asm)
    strong = np.flatnonzero(W > 1.0)
    m = int(out["n_rows"][b])
    assert m == strong.size and np.array_equal(out["S"][b, :m], strong), (tag, name)
    print(f"{tag} {name}: {m} strong rows" + (f" (W {W[strong].min():.1e} .. {W[strong].max():.1e})" if m else "")
          + f", K vs the oracle {asm:.1e}")
    return K_dev + np.diag(out["DD"][b, :n]), (E[strong], W[strong])


def _to_active_set(ref, keep, xr, xl, xv):
    return max(float(np.abs(xr - ref["grad_w_right"])[keep].max() / np.abs(ref["grad_w_right"]).max()),
               float(np.abs(xl - ref["grad_w_left"])[keep].max() / np.abs(ref["grad_w_left"]).max()),
               abs(xv - ref["grad_w_veh"]) / abs(ref["grad_w_veh"]))


def test_box_adjoint_solves_at_the_iterate_and_the_split_of_its_tolerance(golden):
    """mincurv_adjoint_kernel on every box-only fixture and the collapsed-box variant, unshared, and on a batch of shared
    centre lines with jittered widths.  The reference H is the band of the unshared setup of the same batch."""
    cases = _box_cases(golden)
    rts = [c[1] for c in cases]
    names = [c[0] for c in cases]
    share = [0, 3, 5]                                           # owners: berlin, synth128, synth333
    rts += [synth.jitter_widths(rts[k], 40 + k) for k in share]
    names += [f"{names[k]} jittered" for k in share]
    wvs = [c[2] for c in cases] + [cases[k][2] for k in share]
    rt, npts, nv, h = _device_batch(rts, DEV)
    wv = torch.tensor(wvs, **F64)
    B, n_max = rt.shape[:2]
    rng = np.random.default_rng(0)
    gbar = np.zeros((B, n_max))
    for b, r in enumerate(rts):
        gbar[b, :r.shape[0]] = rng.standard_normal(r.shape[0])
    unshared = _mincurv_adjoint(rt, nv, h, npts, wv, 0.12, gbar)
    centre = list(range(len(cases))) + share
    shared = _mincurv_adjoint(rt, nv, h, npts, wv, 0.12, gbar, centre_id=[centre.index(k) for k in centre])
    for tag, out in (("box unshared", unshared), ("box shared", shared)):
        assert out["gs"].tolist() == [0] * B, tag
        for b, r in enumerate(rts):
            n = r.shape[0]
            M = R.dense_from_device_band(unshared["band"][b], n, out["DD"][b])
            xr, xl, xv = _check_adjoint_instance(tag, names[b], out, b, n, gbar, r, wvs[b], M)
            if tag == "box unshared" and b < len(cases):
                name, _, w, H, f, alpha = cases[b]
                ref = Q.width_vjp(H, f, r, w, gbar[b, :n], alpha=alpha)
                keep = ~_degenerate(ref, np.abs(f).max())
                print(f"  {name}: extended solve at the device's D vs the active-set VJP "
                      f"{_to_active_set(ref, keep, xr, xl, xv):.1e} (WEAK_TOL {BOX_WEAK_TOL.get(name, '-')})")


def test_row_adjoint_woodbury_and_pass_order_unshared_and_shared(golden):
    """mincurv_adjoint_rows_kernel on the mixed batch of test_gpu_edges, unshared and shared (followers of a row owner
    read its band in pass 0, before pass 1 overwrites it with K).  Pass-1 instances: K is the band the adjoint assembled,
    checked against the oracle's E^T (I + W_weak) E first; the strong rows S (V_ISU) are those of weight > 1; v solves
    K + D + E_S^T W_S E_S, against the refined Woodbury solve of linalg_ref.solve_extended_rows.  Pass-0 instances: v
    solves H + D with H from the unshared setup."""
    cases, centre_id, rows = _mixed_cases(golden)
    rt, nv, h, npts, wv = _pack(cases)
    B, n_max = rt.shape[:2]
    rng = np.random.default_rng(3)
    gbar = np.zeros((B, n_max))
    for b, c in enumerate(cases):
        gbar[b, :c["rt"].shape[0]] = rng.standard_normal(c["rt"].shape[0])
    qp = [None if c["name"] == "infeasible" else QR.qp_data(c["rt"], c["nv"], KB_MIXED, c["w_veh"]) for c in cases]
    unshared = _mincurv_adjoint(rt, nv, h, npts, wv, KB_MIXED, gbar, rows=True)
    shared = _mincurv_adjoint(rt, nv, h, npts, wv, KB_MIXED, gbar, centre_id=centre_id, rows=True)
    for tag, out in (("rows unshared", unshared), ("rows shared", shared)):
        for b, c in enumerate(cases):
            if c["name"] == "infeasible":
                assert out["gs"][b] == 1
                continue
            assert out["gs"][b] == 0, (tag, c["name"])
            n = c["rt"].shape[0]
            if out["sens_rows"][b, :n].max() > 0.0:
                assert b in rows, (tag, c["name"])
                Kd, strong = _row_system(tag, c["name"], out, b, n, qp[b])
            else:
                assert b not in rows, (tag, c["name"])
                Kd, strong = R.dense_from_device_band(unshared["band"][b], n, out["DD"][b]), None
            xr, xl, xv = _check_adjoint_instance(tag, c["name"], out, b, n, gbar, c["rt"], c["w_veh"], Kd, strong)
            if tag == "rows unshared":
                ref = QR.width_vjp_rows(qp[b], c["rt"], c["w_veh"], KB_MIXED, gbar[b, :n])
                keep = ~QR.degenerate(ref, np.abs(qp[b]["f"]).max())
                top = max(np.abs(ref["grad_w_right"]).max(), np.abs(ref["grad_w_left"]).max())
                dist = max(float(np.abs(xr - ref["grad_w_right"])[keep].max() / top),
                           float(np.abs(xl - ref["grad_w_left"])[keep].max() / top),
                           abs(xv - ref["grad_w_veh"]) / max(abs(ref["grad_w_veh"]), 1e-300))
                print(f"  {c['name']}: extended solve at the device's D vs the active-set VJP {dist:.1e} "
                      f"(WEAK_TOL {ROW_WEAK_TOL.get(c['name'], '-')})")


def test_row_adjoint_on_given_weights_around_the_split():
    """mincurv_adjoint_rows_kernel on given ratios and row weights: weights just below, at and just above the split at 1
    and through 1 .. 1e3 (the weights a final iterate of the mixed batch does not have: its strong rows weigh 6e7 and
    more), strong rows only of moderate weight, no strong row (m = 0), and no row weight at all (pass 0)."""
    wide, flat = synth.make_track(1, 200, amp=0.15), synth.make_track(2, 240, amp=0.1)
    cases = [_oracle_case(rt, KB_MIXED, solve=False) for rt in (wide, flat, wide, flat)]
    rng = np.random.default_rng(6)
    B, n_max = len(cases), 240
    sens, sr, gbar = np.zeros((B, 2, n_max)), np.zeros((B, n_max)), np.zeros((B, n_max))
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        d = 10.0 ** rng.uniform(-12.0, 12.0, n)
        up = rng.random(n) < 0.5
        sens[b, 0, :n], sens[b, 1, :n] = np.where(up, d, 0.5 * LO), np.where(up, 0.5 * LO, d)
        gbar[b, :n] = rng.standard_normal(n)
        w = 10.0 ** rng.uniform(-6.0, -0.5, n)
        if b == 0:          # every regime around the split, and a few strong rows of a final iterate
            pts = rng.choice(n, 16, replace=False)
            w[pts] = (1.0 - 1e-12, 1.0, 1.0, 1.0 + 1e-12, 1.0 + 1e-9, 1.5, 3.0, 20.0, 150.0, 700.0, 999.0, 1e3, 1e6,
                      1e9, 1e12, 1e15)
        elif b == 1:        # strong rows of moderate weight only
            w[::5] = 10.0 ** rng.uniform(0.0, 3.0, w[::5].size)
        elif b == 2:        # weak rows only, up to exactly 1 (m = 0)
            w[::7] = 1.0
        else:               # no row weight: pass 0
            w[:] = 0.0
        sr[b, :n] = w
    rt, nv, h, npts, wv = _pack(cases)
    out = _mincurv_adjoint(rt, nv, h, npts, wv, KB_MIXED, gbar, rows=True, given=(sens, sr))
    assert out["gs"].tolist() == [0] * B
    assert out["n_rows"].tolist()[2:] == [0, 0] and min(out["n_rows"][:2]) > 10
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        if b < 3:
            Kd, strong = _row_system("given weights", f"instance {b}", out, b, n,
                                     QR.qp_data(c["rt"], c["nv"], KB_MIXED, c["w_veh"]))
        else:
            Kd, strong = R.dense_from_device_band(out["band"][b], n, out["DD"][b]), None
        _check_adjoint_instance("given weights", f"instance {b}", out, b, n, gbar, c["rt"], c["w_veh"], Kd, strong)


# ---- 4. the shortest path's cyclic solve ----------------------------------------------------------------------------

def _sp_grads(v, rt, nv, a, du, dl, wv):
    """grad_reftrack [n, 4] and grad_normvec [n, 2] of shortest_path_adjoint_kernel from v (any float type)."""
    vm, vp = np.roll(v, 1), np.roll(v, -1)
    nm, npl = np.roll(nv, 1, axis=0), np.roll(nv, -1, axis=0)
    am, ap = np.roll(a, 1), np.roll(a, -1)
    gxy = [-(4.0 * nv[:, k] * v - 2.0 * nm[:, k] * vm - 2.0 * npl[:, k] * vp) for k in (0, 1)]
    gub = np.where(rt[:, 2] - 0.5 * wv < 0.001, 0.0, du * v)
    glb = np.where(rt[:, 3] - 0.5 * wv < 0.001, 0.0, dl * v)
    gd, go, gom = -v * a, -(v * ap + vp * a), -(vm * a + v * am)
    c = [2.0 * rt[:, k] - np.roll(rt[:, k], -1) - np.roll(rt[:, k], 1) for k in (0, 1)]
    gnv = [8.0 * nv[:, k] * gd - 2.0 * npl[:, k] * go - 2.0 * nm[:, k] * gom - 2.0 * c[k] * v for k in (0, 1)]
    return np.column_stack(gxy + [gub, -glb]), np.column_stack(gnv), (0.5 * (glb - gub)).sum()


def _sp_adjoint(rt, nv, npts, wv, gbar, alpha=None, sens=None):
    """mc_shortest_path_adjoint_batch (after mc_shortest_path_solve_batch_sens unless alpha and sens are given) on this
    test's own workspace; returns its outputs and M's diagonal, off-diagonal, D and x from the workspace."""
    B, n_max = rt.shape[:2]
    lib = _lib.load()
    ws = _ws(lib.mc_shortest_path_workspace_bytes(B, n_max))
    gs = torch.zeros((B,), **I32)
    if sens is None:
        alpha, sens = torch.zeros((B, n_max), **F64), torch.zeros((B, 2, n_max), **F64)
        st, it = torch.zeros((B,), **I32), torch.zeros((B,), **I32)
        B_._call("mc_shortest_path_solve_batch_sens", B, n_max, npts, rt, nv, 0.0, wv, alpha, st, it, sens, gs, ws=ws)
    grt, gnv, gwv = torch.zeros((B, n_max, 4), **F64), torch.zeros((B, n_max, 2), **F64), torch.zeros((B,), **F64)
    B_._call("mc_shortest_path_adjoint_batch", B, n_max, npts, rt, nv, 0.0, wv, alpha, sens, gs, torch.as_tensor(gbar, **F64),
             grt, gnv, gwv, ws=ws)
    torch.cuda.synchronize()
    sp = _sp_enum()
    w = ws.view(torch.float64)[:sp["SP_NUM"] * n_max * B].view(sp["SP_NUM"], n_max, B)
    vec = {k: w[sp[f"SP_{k}"]].T.cpu().numpy() for k in ("DG", "OFF", "DD", "X")}
    return dict(vec, gs=gs.cpu().numpy(), grt=grt.cpu().numpy(), gnv=gnv.cpu().numpy(), gwv=gwv.cpu().numpy(),
                alpha=alpha.cpu().numpy(), sens=sens.cpu().numpy())


def _check_sp(tag, out, b, n, gbar, rt, nv, wv):
    M = R.cyclic_tridiag(out["DG"][b, :n], out["OFF"][b, :n], out["DD"][b, :n])
    v, g = out["X"][b, :n], gbar[b, :n]
    du, dl = out["sens"][b, 0, :n], out["sens"][b, 1, :n]
    assert np.array_equal(out["DD"][b, :n], du + dl), tag
    eta = R.backward_error(M, v, g)
    x = R.solve_extended(M, g)
    c = R.cond_scaled(M)
    fe = R.forward_error(M, v, x)
    a = out["alpha"][b, :n]
    grt, gnv, gwv = _sp_grads(x, rt, nv, a.astype(np.longdouble), du.astype(np.longdouble), dl.astype(np.longdouble), wv)
    sx = 8.0 * float(np.abs(x).max())                     # (x, y and the normals: second differences of v)
    ge = max(float(np.abs(out["grt"][b, :n, :2] - grt[:, :2]).max()) / sx,
             R.rel_err(out["grt"][b, :n, 2:], grt[:, 2:]) if np.abs(grt[:, 2:]).max() > 0 else 0.0)
    print(f"{tag}: eta {eta:.1e}, cond(SMS) {c:.1e}, forward {fe:.1e} = {fe / (R.U * c):.2f} u cond, "
          f"gradient vs extended {ge:.1e}")
    assert eta <= R.ETA_MAX, (tag, eta)
    assert fe <= R.fe_bound(c), (tag, fe, c)
    assert ge <= R.fe_bound(c), (tag, ge, c)
    return np.asarray(grt, dtype=np.float64), np.asarray(gnv, dtype=np.float64)


def test_shortest_path_adjoint_on_every_fixture(golden):
    rt, nv, npts, wv = _sp_batch(golden, SP_FIXTURES, DEV)
    B, n_max = rt.shape[:2]
    rng = np.random.default_rng(4)
    gbar = np.zeros((B, n_max))
    for b, m in enumerate(npts.tolist()):
        gbar[b, :m] = rng.standard_normal(m)
    out = _sp_adjoint(rt, nv, npts, wv, gbar)
    assert out["gs"].tolist() == [0] * B
    for b, name in enumerate(SP_FIXTURES):
        g = golden(name)
        n = g["reftrack"].shape[0]
        grt, _ = _check_sp(name, out, b, n, gbar, g["reftrack"], g["normvec"], float(g["w_veh"]))
        ref = S.vjp(g["reftrack"], g["normvec"], float(g["w_veh"]), gbar[b, :n], alpha=g["alpha_shpath"])
        bad = S.degenerate(ref, np.abs(ref["f"]).max())
        keep = ~(bad | np.roll(bad, 1) | np.roll(bad, -1))
        r = ref["grad_reftrack"]
        scale = [np.abs(r[:, 0]).max(), np.abs(r[:, 1]).max()] + [np.abs(r[:, 2:]).max()] * 2     # (as device_vs_oracle)
        dist = max(float(np.abs(grt[:, k] - r[:, k])[keep].max() / scale[k]) for k in range(4))
        print(f"  {name}: extended solve at the device's D vs the active-set VJP {dist:.1e}")


@pytest.mark.parametrize("n", [3, 4, 5, 7])
def test_shortest_path_adjoint_small_tracks_with_either_end_active(n):
    """Constructed tracks of n points with point 0 and point n-1 each active (D = 1e12: gamma = -d_0 of the
    Sherman-Morrison split becomes -1e12) or inactive (1e-12), the corner M[n-1][0] = cN included; the adjoint runs on
    given ratios, the interior points' log-uniform."""
    rng = np.random.default_rng(50 + n)
    combos = [(a0, an) for a0 in (HI, LO) for an in (HI, LO)] * 3
    B = len(combos)
    rt, nv, du, dl = np.zeros((B, n, 4)), np.zeros((B, n, 2)), np.zeros((B, n)), np.zeros((B, n))
    for b, (a0, an) in enumerate(combos):
        th = np.sort(rng.uniform(0.0, 2.0 * np.pi, n))
        rt[b, :, 0], rt[b, :, 1] = 30.0 * np.cos(th), 30.0 * np.sin(th)
        rt[b, :, 2:] = rng.uniform(2.0, 5.0, (n, 2))
        phi = th + rng.uniform(-0.5, 0.5, n)
        nv[b] = np.column_stack((np.cos(phi), np.sin(phi)))
        d = 10.0 ** rng.uniform(-12.0, 12.0, n)
        d[0], d[n - 1] = a0, an
        up = rng.random(n) < 0.5
        du[b], dl[b] = np.where(up, d, 0.5 * LO), np.where(up, 0.5 * LO, d)
    gbar = rng.standard_normal((B, n))
    sens = torch.tensor(np.stack((du, dl), axis=1), **F64)
    out = _sp_adjoint(torch.tensor(rt, **F64), torch.tensor(nv, **F64), None, torch.full((B,), 2.0, **F64), gbar,
                      alpha=torch.tensor(rng.uniform(-1.0, 1.0, (B, n)), **F64), sens=sens)
    assert out["gs"].tolist() == [0] * B
    for b, (a0, an) in enumerate(combos):
        _check_sp(f"n={n} d_0 {a0:.0e} d_n-1 {an:.0e}", out, b, n, gbar, rt[b], nv[b], 2.0)
