"""GPU tests (-m gpu) of the width sensitivities of small closed tracks (opt_min_curv_diff(small_tracks=True,
curvature_rows=True): the row export of the dense small-track kernel and the dense adjoint K2e-d, DESIGN.md section 3.14):

A  against the exact active-set VJP with rows (tests/qp_sens_rows.py) on 3 .. 79 points: synthetic tracks, the handling
   track thinned to every 4th / 6th / 8th point, a collapsed box, limits at which the rows bind, a [B] kappa_bound and a
   tensor w_veh; points where the derivative is ill-conditioned are excluded by qp_sens_rows.degenerate and counted.
B  the linear algebra alone: the device's gradients against an extended-precision solve (linalg_ref.solve_extended_rows)
   at the device's own exported D and W.
C  dense against banded gradients on 80 .. 108 points (_dense_below).
D  a ragged batch from 3 to 1000 points with shared centre ids and max_chunk: the long tracks, the forward, each short
   track alone, an all-short batch and a batch of 3 x SMs x 8, bit for bit.
E  the unsupported instances, and central differences through the device solver.
Every measured error is printed next to its tolerance (pytest -s)."""
import numpy as np
import pytest

import ipm_rows_ref as IR
import linalg_ref as LR
import qp_sens as Q
import qp_sens_rows as QR
from conftest import load_golden

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import batch as B_, synth  # noqa: E402
from oracle import tph_dense as T  # noqa: E402

DEV = "cuda"
# Against the exact VJP (max error over the non-degenerate points / the largest width gradient), measured on an H100
# 80GB HBM3: 1.1e-5 (synth64, box only).  The device differentiates the final interior-point iterate, not the
# exact active set: a weakly active bound keeps a finite weight there and damps the gradient around it.  synth31 has a
# bound active with a multiplier of 1.2e-4 |f|: 1.0e-3 measured.
GRAD_TOL = 5e-5
WEAK_TOL = {"synth31": 5e-3}
# Against the extended-precision solve at the device's own D and W (the linear algebra alone), measured on an H100:
# 2.5e-10 (uneven64_r50, rows binding) at weights up to 5e15.  The regime at kb_min (1 + 1e-3) of ipm_rows_ref is left
# out: the feasible set is nearly a point, up to 72 of 79 rows are strongly active together with bounds, and the
# weights reach 1e19, so the system's condition is beyond what either solve resolves (measured errors 1e-11 to 1).
LINALG_TOL = 2e-9
# Dense against banded on 80 .. 108 points (band truncation, two stopping rules), measured on an H100: 7.0e-7.
DVB_TOL = 1e-5
# Central differences through the device solver (delta 1 cm), measured on an H100: 1.2e-7.
FD_TOL = 1e-4


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _closed(rt):
    return np.vstack((rt[:, :2], rt[0, :2]))


def _case(name, rt, kb, w_veh=2.0):
    _, _, _, nv = T.calc_splines(_closed(rt))
    return dict(name=name, rt=np.asarray(rt, dtype=np.float64), nv=nv,
                h=np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1), kb=kb, w_veh=w_veh)


def _pack(cases, n_max=None):
    n = [c["rt"].shape[0] for c in cases]
    n_max = n_max or max(n)
    rt, nv, h = np.zeros((len(cases), n_max, 4)), np.zeros((len(cases), n_max, 2)), np.ones((len(cases), n_max))
    for b, c in enumerate(cases):
        rt[b, :n[b]], nv[b, :n[b]], h[b, :n[b]] = c["rt"], c["nv"], c["h"]
    f64 = dict(dtype=torch.float64, device=DEV)
    return (torch.tensor(rt, **f64), torch.tensor(nv, **f64), torch.tensor(h, **f64),
            torch.tensor(n, dtype=torch.int32, device=DEV), torch.tensor([c["w_veh"] for c in cases], **f64),
            torch.tensor([c["kb"] for c in cases], **f64))


def _gbar(cases, seed, n_max=None):
    n_max = n_max or max(c["rt"].shape[0] for c in cases)
    rng = np.random.default_rng(seed)
    g = np.zeros((len(cases), n_max))
    for b, c in enumerate(cases):
        g[b, :c["rt"].shape[0]] = rng.standard_normal(c["rt"].shape[0])
    return g


def _grads(cases, gbar, n_max=None, **kw):
    """(result dict as numpy, dL/dwidths [B, n_max, 2], dL/dw_veh [B]) of L = sum gbar * alpha."""
    rt, nv, h, npts, wv, kb = _pack(cases, n_max)
    widths = rt[:, :, 2:].clone().requires_grad_()
    wvg = wv.clone().requires_grad_()
    kw = dict(dict(small_tracks=True, curvature_rows=True, strict=False), **kw)
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, wvg, n_pts=npts, **kw)
    gw, gv = torch.autograd.grad(res["alpha"], (widths, wvg), torch.as_tensor(gbar, device=DEV))
    return {k: v.detach().cpu().numpy() for k, v in res.items()}, gw.cpu().numpy(), gv.cpu().numpy()


def _wide(rt):
    rt = np.asarray(rt, dtype=np.float64).copy()
    rt[:, 2:] = np.maximum(rt[:, 2:], 1.6)             # (the widths of tiny synthetic tracks fit a 2 m car)
    return rt


def _collapsed(n):
    rt = _wide(synth.make_track(3, n))
    rt[n // 3, 2:] = 1.0                               # w_r + w_l == w_veh: lb == ub there
    return rt


def _kb_binding(c):
    """A limit at which the rows bind but can be met: 0.9 of the box-only optimum's largest |kappa|, or just above the
    smallest limit the box allows (bisection on the oracle) if that is higher."""
    d = QR.qp_data(c["rt"], c["nv"], 1.0, c["w_veh"])
    lb, ub, _ = Q.bounds(c["rt"], c["w_veh"])
    kmax = float(np.abs(d["k_ref"] + d["E"] @ QR.solve(d, lb, ub, 1e6)[0]).max())
    lo, hi = 0.0, kmax
    for _ in range(40):
        mid = 0.5 * (lo + hi)
        try:
            QR.solve(d, lb, ub, mid)
            hi = mid
        except ValueError:
            lo = mid
    return max(0.9 * kmax, 1.05 * hi)


def _oracle_cases():
    g = load_golden("handling")
    out = [_case(f"synth{n}", _wide(synth.make_track(1, n)), 0.12) for n in (3, 4, 5, 8, 16, 31, 40, 64, 79)]
    out += [_case(f"handling_every{k}", g["reftrack"][::k].copy(), float(g["kappa_bound"]), float(g["w_veh"]))
            for k in (4, 6, 8)]
    out += [_case("collapsed31", _collapsed(31), 0.12)]
    for n in (16, 40, 79):
        c = _case(f"synth{n}_rows", _wide(synth.make_track(5, n)), 1.0)
        c["kb"] = _kb_binding(c)
        out.append(c)
    out[-1]["w_veh"] = 1.8                             # (a different vehicle width per track: w_veh is a tensor)
    return out


def _reference(c, gbar):
    """The exact VJP with rows, or None where the oracle refuses the QP (with the status it stands for)."""
    d = QR.qp_data(c["rt"], c["nv"], c["kb"], c["w_veh"])
    try:
        return d, QR.width_vjp_rows(d, c["rt"], c["w_veh"], c["kb"], gbar), 0
    except RuntimeError:
        return d, None, 1
    except ValueError:
        return d, None, 4


def test_against_the_exact_vjp_on_short_tracks():
    cases = _oracle_cases()
    gbar = _gbar(cases, 0)
    res, gw, gv = _grads(cases, gbar)
    worst, failed = 0.0, []
    for b, c in enumerate(cases):
        n = c["rt"].shape[0]
        assert not gw[b, n:].any()
        d, ref, st = _reference(c, gbar[b, :n])
        if ref is None:
            print(f"{c['name']}: oracle status {st}, device status {res['status'][b]} grad_status {res['grad_status'][b]}")
            assert res["status"][b] == st and res["grad_status"][b] == st
            assert not gw[b].any() and gv[b] == 0.0
            continue
        if not (res["status"][b] == 0 and res["grad_status"][b] == 0):
            print(f"{c['name']}: device status {res['status'][b]} grad_status {res['grad_status'][b]}, oracle 0")
            failed.append(c["name"])
            continue
        keep = ~QR.degenerate(ref, np.abs(d["f"]).max())
        top = max(np.abs(ref["grad_w_right"]).max(), np.abs(ref["grad_w_left"]).max(), 1e-300)
        e = max(float(np.abs(gw[b, :n, 0] - ref["grad_w_right"])[keep].max(initial=0.0) / top),
                float(np.abs(gw[b, :n, 1] - ref["grad_w_left"])[keep].max(initial=0.0) / top),
                abs(float(gv[b]) - ref["grad_w_veh"]) / max(abs(ref["grad_w_veh"]), top))
        rows = int((ref["row_hi"] | ref["row_lo"]).sum())
        tol = WEAK_TOL.get(c["name"], GRAD_TOL)
        print(f"{c['name']}: grad {e:.2e} (tol {tol:.0e})  rows {rows}  excluded {int((~keep).sum())}  "
              f"iters {int(res['iters'][b])}")
        worst = max(worst, e)
        failed += [c["name"]] if not e <= tol else []
    print("worst:", worst)
    assert not failed, failed
    assert any("rows" in c["name"] for c in cases)


def _export(cases, f_scale):
    """The forward's row export (sens, grad_status, sens_rows, n_rows) through mc_mincurv_solve_batch_ex, as numpy."""
    rt, nv, h, npts, wv, kb = _pack(cases)
    B, n = h.shape
    out = B_._mincurv_results(B, n, h.device)
    f64 = dict(dtype=torch.float64, device=DEV)
    exp = (torch.empty((B, 2, n), **f64), torch.empty((B,), dtype=torch.int32, device=DEV), torch.empty((B, n), **f64),
           torch.empty((B,), dtype=torch.int32, device=DEV))
    B_._mincurv_per_instance(B, npts, rt, nv, h, kb, 0.0, wv, f_scale, None, out.values(), exp, dense_below=B_.N_MIN)
    return [t.cpu().numpy() for t in exp]


def test_the_linear_algebra_at_the_exported_iterate():
    """v = (E^T E + D + E^T W E)^-1 g in extended precision at the device's exported D and W, against the device's
    gradients (d_u v, -d_l v), over the dense kernel's box and rows regimes.  exit_pivot_late0, where the long-double
    replay takes the late-accept exit (status 0 at a failed pivot), ends with status 3 in float64 on the device, so it
    checks only that such an instance gets its status and zero gradients."""
    picked = [(name, t, kb) for name, t, kb in IR.dense_cases()
              if t["lin_alpha"] is None and t["f_scale"] == 2.0 and not name.endswith("feasible")
              and t["rt"].shape[0] < B_.N_MIN] + \
             [(name, t, kb) for name, t, kb in IR.dense_cases() if name.startswith("exit_pivot_late0")]
    cases = [dict(name=name, rt=t["rt"], nv=t["nv"], h=t["h"], kb=kb, w_veh=t["w_veh"], f_scale=t["f_scale"])
             for name, t, kb in picked]
    worst, failed = 0.0, []
    for fs in sorted({c["f_scale"] for c in cases}):
        group = [c for c in cases if c["f_scale"] == fs]
        gbar = _gbar(group, 1)
        res, gw, _ = _grads(group, gbar, f_scale=fs)
        sens, gs, srows, nrows = _export(group, fs)
        for b, c in enumerate(group):
            n = c["rt"].shape[0]
            if gs[b] != 0:
                print(f"{c['name']}: status {res['status'][b]} grad_status {gs[b]}")
                assert res["grad_status"][b] == gs[b] and not gw[b].any(), c["name"]
                continue
            d = QR.qp_data(c["rt"], c["nv"], c["kb"], c["w_veh"])
            du, dl, w = sens[b, 0, :n], sens[b, 1, :n], srows[b, :n]
            strong = w > 1.0
            assert int(strong.sum()) == nrows[b]
            E = d["E"]
            K = E.T @ ((1.0 + np.where(strong, 0.0, w))[:, None] * E) + np.diag(du + dl)
            v = np.asarray(LR.solve_extended_rows(K, E[strong], w[strong], gbar[b, :n]), dtype=np.float64)
            lb, ub, coll = Q.bounds(c["rt"], c["w_veh"])
            gr = np.where(coll, 0.5 * (du + dl) * v, du * v)
            gl = np.where(coll, -0.5 * (du + dl) * v, -dl * v)
            top = max(np.abs(gr).max(), np.abs(gl).max(), 1e-300)
            e = max(np.abs(gw[b, :n, 0] - gr).max(), np.abs(gw[b, :n, 1] - gl).max()) / top
            print(f"{c['name']}: linalg {e:.2e} (tol {LINALG_TOL:.0e})  n_rows {nrows[b]}  max W {w.max():.1e}")
            worst = max(worst, e)
            failed += [c["name"]] if not e <= LINALG_TOL else []
    print("worst:", worst)
    assert not failed, failed


@pytest.mark.parametrize("kind", ["box", "rows"])
def test_dense_against_banded_where_both_apply(kind):
    cases = [_case(f"synth{n}", synth.make_track(20 + n, n), 0.12) for n in (80, 90, 101, 108)]
    if kind == "rows":
        for c in cases:
            c["kb"] = _kb_binding(c)
    gbar = _gbar(cases, 2)
    ref, gw_b, gv_b = _grads(cases, gbar, small_tracks=False)
    res, gw_d, gv_d = _grads(cases, gbar, _dense_below=B_.N_DENSE_MAX + 1, small_tracks=False)
    for b, c in enumerate(cases):
        assert ref["grad_status"][b] == 0 and res["grad_status"][b] == 0, c["name"]
        top = np.abs(gw_b[b]).max()
        e = max(np.abs(gw_d[b] - gw_b[b]).max() / top, abs(gv_d[b] - gv_b[b]) / max(abs(gv_b[b]), top))
        print(f"{c['name']} {kind}: dense vs banded {e:.2e} (tol {DVB_TOL:.0e})")
        assert e <= DVB_TOL, c["name"]


def _ragged(n_list, seed=0):
    return [_case(f"n{n}", _wide(synth.make_track(seed + i, n)) if n < B_.N_MIN else synth.make_track(seed + i, n), 0.12)
            for i, n in enumerate(n_list)]


def test_a_ragged_batch_bit_for_bit():
    ns = [3, 1000, 40, 79, 120, 5, 80, 16, 250, 64]
    cases = _ragged(ns)
    n_max = max(ns)
    gbar = _gbar(cases, 3, n_max)
    cid = torch.arange(len(ns), dtype=torch.int32, device=DEV)
    res, gw, gv = _grads(cases, gbar, centre_id=cid, max_chunk=4)
    base, gw0, gv0 = _grads(cases, gbar, small_tracks=False, centre_id=cid, max_chunk=4)
    rt, nv, h, npts, wv, kb = _pack(cases)
    fwd = {k: v.cpu().numpy() for k, v in B_.opt_min_curv_batch(rt, nv, h, kb, wv, n_pts=npts, small_tracks=True,
                                                                 centre_id=cid, max_chunk=4).items()}
    for k in fwd:
        assert np.array_equal(res[k], fwd[k], equal_nan=True), k
    for b, n in enumerate(ns):
        if n >= B_.N_MIN:
            for k in fwd:
                assert np.array_equal(res[k][b], base[k][b], equal_nan=True), (k, n)
            assert np.array_equal(gw[b], gw0[b]) and gv[b] == gv0[b], n
        elif n >= 3:
            one, gw1, gv1 = _grads([cases[b]], gbar[b:b + 1, :n])
            assert np.array_equal(gw[b, :n], gw1[0]) and gv[b] == gv1[0], n
            assert not gw[b, n:].any()
    print("grad_status:", res["grad_status"].tolist())
    assert res["grad_status"][ns.index(40)] == 0
    assert (res["grad_status"] == res["status"]).all() and res["status"][ns.index(3)] != 0
    # an all-short batch (n_max < N_MIN) and a batch larger than the resident CTAs: each track as alone
    short = [c for c in cases if c["rt"].shape[0] < B_.N_MIN]
    s_res, s_gw, s_gv = _grads(short, _gbar(short, 4))
    assert s_gw.shape[1] < B_.N_MIN
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    many = [short[i % len(short)] for i in range(3 * sms * 8)]
    m_res, m_gw, m_gv = _grads(many, np.tile(_gbar(short, 4), (3 * sms * 8 // len(short) + 1, 1))[:len(many)])
    for b in range(len(many)):
        k = b % len(short)
        assert np.array_equal(m_gw[b], s_gw[k]) and m_gv[b] == s_gv[k] and m_res["grad_status"][b] == s_res["grad_status"][k]


def test_unsupported_instances():
    ok = _case("ok", _wide(synth.make_track(7, 40)), 0.12)
    two = _case("n2", _wide(synth.make_track(8, 40)), 0.12)
    narrow = _case("narrow", _wide(synth.make_track(9, 40)), 0.12)
    narrow["rt"][5, 2:] = 0.2                                 # w_r + w_l < w_veh: status 1
    unmet = _case("unmet", _wide(synth.make_track(10, 40)), 1e-4)    # rows that cannot be met: status 4
    nan_veh = _case("nan_wveh", _wide(synth.make_track(11, 40)), 0.12)
    cases = [ok, two, narrow, unmet, nan_veh]
    rt, nv, h, npts, wv, kb = _pack(cases)
    npts[1] = 2
    wv[4] = float("nan")
    widths = rt[:, :, 2:].clone().requires_grad_()
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, wv, n_pts=npts, small_tracks=True, curvature_rows=True,
                               strict=False)
    (gw,) = torch.autograd.grad(res["alpha"], (widths,), torch.ones_like(res["alpha"]))
    st, gs = res["status"].tolist(), res["grad_status"].tolist()
    print("status", st, "grad_status", gs)
    assert st == gs and st[0] == 0 and st[1] == -1 and st[2] == 1 and st[3] == 4 and st[4] == -1
    assert gw[0].abs().max() > 0 and not gw[1:].any()
    res = B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, wv, n_pts=npts, small_tracks=True, curvature_rows=True)
    with pytest.raises(B_._lib.MinCurvLibError):
        torch.autograd.grad(res["alpha"], (widths,), torch.ones_like(res["alpha"]))


def test_directional_difference_through_the_device_solver():
    cases = [_case("synth40_rows", _wide(synth.make_track(5, 40)), 1.0), _case("synth16", _wide(synth.make_track(1, 16)), 0.12)]
    cases[0]["kb"] = _kb_binding(cases[0])
    gbar = _gbar(cases, 5)
    res, gw, gv = _grads(cases, gbar)
    rt, nv, h, npts, wv, kb = _pack(cases)
    rng = np.random.default_rng(6)
    dw = torch.tensor(rng.uniform(-1.0, 1.0, tuple(rt[:, :, 2:].shape)), dtype=torch.float64, device=DEV)
    dv = torch.tensor(rng.uniform(-1.0, 1.0, len(cases)), dtype=torch.float64, device=DEV)
    for b in range(len(cases)):
        n = cases[b]["rt"].shape[0]
        dw[b, n:] = 0.0
    delta = 0.01

    def loss(sign):
        w = rt[:, :, 2:] + sign * delta * dw
        out = B_.opt_min_curv_diff(rt[:, :, :2], w, nv, h, kb, wv + sign * delta * dv, n_pts=npts, small_tracks=True,
                                   curvature_rows=True)
        return (torch.as_tensor(gbar, device=DEV) * out["alpha"]).sum(dim=1).cpu().numpy()
    fd = (loss(1.0) - loss(-1.0)) / (2 * delta)
    ad = (gw * dw.cpu().numpy()).sum(axis=(1, 2)) + gv * dv.cpu().numpy()
    for b, c in enumerate(cases):
        e = abs(fd[b] - ad[b]) / max(abs(ad[b]), 1e-12)
        print(f"{c['name']}: fd {fd[b]:.6e} ad {ad[b]:.6e} rel {e:.2e} (tol {FD_TOL:.0e})")
        assert e <= FD_TOL, c["name"]
