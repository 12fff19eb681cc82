"""GPU tests of the minimum-curvature QP linearised about a given line (lin_alpha of opt_min_curv_batch and of the C-ABI
entries; DESIGN.md sections 3.2 and 3.13): lin_alpha = 0 is the centre-line QP bit for bit; about the line P + a n the
finalize stage at alpha = a has no linearisation error, H's band and f match the dense QP about the line
(lin_ref.dense_qp_about), the solution matches its Goldfarb-Idnani solve, a follower of a shared centre line is solved
about its owner's row, the curvature metric about the line matches dense numpy; and the refinement with re-linearised
rows returns lines whose knot curvature honours the limit up to curv_error_max."""
import numpy as np
import pytest
import torch

import lin_ref
from conftest import rel_max
from global_racetrajectory_optimization_b200 import _lib, batch as B_, raceline_refine as R
from test_gpu_raceline_refine_metric import _fresh, _veh

pytestmark = pytest.mark.gpu
DEV = "cuda"
CURVLIM = 0.12              # tests/golden/racecar_ini.json veh_params.curvlim
ASM_TOL = dict(band=5e-12, f=1e-10, kref=1e-10)      # test_gpu_edges.py's assembly tolerances (max |diff| / max |ref|)
ALPHA_TOL = 1e-4            # test_gpu_parity.py's
SOLVE_TOL = 1e-10           # test_gpu_raceline_refine_metric.py's metric solve


def _track(g):
    rt = torch.tensor(g["reftrack"], dtype=torch.float64, device=DEV)[None].contiguous()
    nv = torch.tensor(g["normvec"], dtype=torch.float64, device=DEV)[None].contiguous()
    _, _, _, h = B_.calc_splines_batch(rt, want_coeffs=False)
    return rt, nv, h


@pytest.mark.parametrize("name", ["handling", "synth160_kappa", "synth333_kappa"])
def test_zero_linearisation_point_is_the_centre_line_qp(golden, name):
    g = golden(name)
    rt, nv, h = _track(g)
    kb, wv = float(g["kappa_bound"]), float(g["w_veh"])
    for k in (kb, CURVLIM):
        ref = B_.opt_min_curv_batch(rt, nv, h, k, wv)
        out = B_.opt_min_curv_batch(rt, nv, h, k, wv, lin_alpha=torch.zeros_like(h))
        print(f"LIN zero {name} kb {k}: status {out['status'].tolist()}, iters {out['iters'].tolist()}")
        for key in ("alpha", "curv_error_max", "kappa_lin_max", "status", "iters"):
            assert torch.equal(out[key], ref[key]), (k, key)


@pytest.mark.parametrize("name", ["handling", "berlin", "synth1000", "synth333_kappa"])
def test_assembly_about_a_line(golden, name):
    """Linearised about a = the minimum-curvature alpha: finalize at alpha = a gives curv_error_max <= 1e-9 and
    kappa_lin_max = the knot curvature of the spline through P + a n; finalize at alpha = 0 measures the curvature of
    the centre line against the same linearisation."""
    g = golden(name)
    rt, nv, h = _track(g)
    wv = float(g["w_veh"])
    a = B_.opt_min_curv_batch(rt, nv, h, 10.0, wv)["alpha"]
    n_max = h.shape[1]
    lib = _lib.load()
    ws = B_._workspace("mincurv", lib.mc_mincurv_workspace_bytes(1, n_max), rt.device)
    out = B_._mincurv_results(1, n_max, rt.device)
    for x in (a, torch.zeros_like(a)):
        B_._call("mc_mincurv_setup_batch_ex", 1, n_max, None, rt, nv, h, wv, None, B_.F_SCALE, out["status"], a, ws=ws)
        B_._call("mc_mincurv_finalize_batch", 1, n_max, None, x, 10.0, out["curv_error_max"], out["kappa_lin_max"],
                 out["status"], 1, ws=ws)
        assert int(out["status"]) == 0
        p, nvec, hh, av = (t.cpu().numpy()[0] for t in (rt, nv, h, a))
        xv = x.cpu().numpy()[0]
        k_lin = lin_ref.linearised_curvature(p[:, :2], nvec, hh, av, xv)
        k_true = lin_ref.knot_curvature(p[:, :2] + xv[:, None] * nvec, hh)
        kl, ce = float(out["kappa_lin_max"]), float(out["curv_error_max"])
        print(f"LIN about a {name}: |x| {np.abs(xv).max():.3f} kappa_lin_max {kl:.6g} (ref {np.abs(k_lin).max():.6g}), "
              f"curv_error_max {ce:.3g} (ref {np.abs(k_true - k_lin).max():.3g})")
        assert abs(kl - np.abs(k_lin).max()) <= 1e-9 * np.abs(k_lin).max()
        assert abs(ce - np.abs(k_true - k_lin).max()) <= 1e-9 * max(np.abs(k_true).max(), 1.0)
        if x is a:
            assert ce <= 1e-9
            assert np.allclose(k_lin, k_true, rtol=0, atol=1e-10)


@pytest.mark.parametrize("name", ["handling", "synth160_kappa"])
def test_solution_about_a_line_keeps_its_rows(golden, name):
    """opt_min_curv_batch(lin_alpha = a) with active rows: the linearised rows hold at the solution (status 0), and the
    returned curv_error_max and kappa_lin_max are those of its linearisation (lin_ref.py)."""
    g = golden(name)
    rt, nv, h = _track(g)
    wv = float(g["w_veh"])
    kb = CURVLIM if name == "handling" else float(g["kappa_bound"])
    a = B_.opt_min_curv_batch(rt, nv, h, kb, wv)["alpha"]
    out = B_.opt_min_curv_batch(rt, nv, h, kb, wv, lin_alpha=a)
    print(f"LIN solve {name} kb {kb}: status {out['status'].tolist()}, iters {out['iters'].tolist()}, "
          f"kappa_lin_max {out['kappa_lin_max'].tolist()}, curv_error_max {out['curv_error_max'].tolist()}")
    assert int(out["status"]) == 0
    p, nvec, hh, av, x = (t.cpu().numpy()[0] for t in (rt, nv, h, a, out["alpha"]))
    k_lin = lin_ref.linearised_curvature(p[:, :2], nvec, hh, av, x)
    k_true = lin_ref.knot_curvature(p[:, :2] + x[:, None] * nvec, hh)
    assert np.abs(k_lin).max() <= kb * (1 + 1e-7)
    assert abs(float(out["kappa_lin_max"]) - np.abs(k_lin).max()) <= 1e-9
    assert abs(float(out["curv_error_max"]) - np.abs(k_true - k_lin).max()) <= 1e-9


def _dense_case(g, rt, nv, h, a, kb):
    wv = float(g["w_veh"])
    d = lin_ref.dense_qp_about(g["reftrack"], nv[0].cpu().numpy(), a, kb, wv)
    lb, ub, _ = R.box(rt.cpu(), wv)
    return d, lb[0].numpy(), ub[0].numpy(), wv


@pytest.mark.parametrize("name", ["handling", "berlin", "synth1000", "synth333_kappa"])
def test_assembled_band_and_f_match_the_dense_qp_about_the_line(golden, name):
    g = golden(name)
    rt, nv, h = _track(g)
    n = h.shape[1]
    a = B_.opt_min_curv_batch(rt, nv, h, 10.0, float(g["w_veh"]))["alpha"]
    d, _, _, wv = _dense_case(g, rt, nv, h, a[0].cpu().numpy(), CURVLIM)
    lay = B_.mincurv_slab_layout(n)
    ws = B_._workspace("mincurv", _lib.load().mc_mincurv_workspace_bytes(1, n), rt.device)
    st = torch.empty(1, dtype=torch.int32, device=DEV)
    B_._call("mc_mincurv_setup_batch_ex", 1, n, None, rt, nv, h, wv, None, B_.F_SCALE, st, a, ws=ws)
    torch.cuda.synchronize()
    slab = ws.view(torch.float64)[:lay["stride"]].cpu().numpy()
    vec = lambda nm: slab[B_.SLAB_VECTORS.index(nm) * lay["np"]:][:n]          # noqa: E731
    band = slab[lay["o_hb"]:lay["o_hb"] + lay["np"] * B_.HB_PITCH].reshape(-1, B_.HB_PITCH)[:n, :33]
    i = np.arange(n)
    band_ref = np.stack([d["H"][i, (i + k) % n] for k in range(33)], axis=1)
    e = dict(band=rel_max(band, band_ref), f=rel_max(vec("F"), d["f"]), kref=rel_max(vec("KREF"), d["k_ref"]))
    print(f"LIN assembly {name}: " + ", ".join(f"{k} {v:.1e}" for k, v in e.items()))
    assert int(st) == 0 and all(e[k] <= ASM_TOL[k] for k in e), e


@pytest.mark.parametrize("name,kb", [("handling", None), ("handling", CURVLIM), ("synth160_kappa", None),
                                     ("synth160_kappa", "golden")])
def test_solution_about_a_line_matches_the_dense_qp(golden, name, kb):
    """Box only (kb None: a limit no row reaches) and with active rows, linearised about the minimum-curvature alpha at
    the same limit (about which the rows bind)."""
    g = golden(name)
    rt, nv, h = _track(g)
    wv = float(g["w_veh"])
    k = 10.0 if kb is None else (float(g["kappa_bound"]) if kb == "golden" else kb)
    a = B_.opt_min_curv_batch(rt, nv, h, k, wv)["alpha"]
    out = B_.opt_min_curv_batch(rt, nv, h, k, wv, lin_alpha=a)
    d, lb, ub, _ = _dense_case(g, rt, nv, h, a[0].cpu().numpy(), k)
    ref = lin_ref.solve_dense(d, lb, ub, k, rows=kb is not None)
    x = out["alpha"][0].cpu().numpy()
    act = int((np.abs(d["k_ref"] + d["E"] @ ref) >= k * (1 - 1e-6)).sum())
    err = rel_max(x, ref)
    print(f"LIN dense {name} kb {k}: status {out['status'].tolist()}, active rows {act}, alpha rel err {err:.1e}")
    assert int(out["status"]) == 0 and err <= ALPHA_TOL
    if kb is not None:
        assert act > 0


def test_a_follower_is_solved_about_its_owners_row(golden):
    g = golden("synth160_kappa")
    rt, nv, h = _track(g)
    wv, kb = float(g["w_veh"]), float(g["kappa_bound"])
    a = B_.opt_min_curv_batch(rt, nv, h, kb, wv)["alpha"]
    rt3, nv3, h3 = (t.repeat(3, *([1] * (t.dim() - 1))).contiguous() for t in (rt, nv, h))
    rt3[1, :, 2:] *= 0.9                                                     # a width variant
    lin = torch.stack((a[0], torch.zeros_like(a[0]), 0.5 * a[0]))            # the follower's own row is not used
    out = B_.opt_min_curv_batch(rt3, nv3, h3, kb, wv, lin_alpha=lin, centre_id=torch.tensor([0, 0, 2], device=DEV))
    ref = B_.opt_min_curv_batch(rt3[1:2].contiguous(), nv, h, kb, wv, lin_alpha=a)
    for key in ("alpha", "curv_error_max", "kappa_lin_max", "status", "iters"):
        assert torch.equal(out[key][1:2], ref[key]), key


@pytest.mark.parametrize("name", ["handling", "synth1000"])
def test_the_metric_about_a_line_matches_dense_numpy(golden, name):
    g = golden(name)
    rt, nv, h = _track(g)
    n = h.shape[1]
    a = B_.opt_min_curv_batch(rt, nv, h, 10.0, float(g["w_veh"]))["alpha"]
    H = lin_ref.dense_qp_about(g["reftrack"], nv[0].cpu().numpy(), a[0].cpu().numpy(), CURVLIM, 0.0)["H"]
    i = np.arange(n)
    dist = np.abs(i[:, None] - i[None, :])
    M = np.eye(n) + 10.0 ** 4 * np.where(np.minimum(dist, n - dist) <= 32, H, 0.0)
    met = R.CurvatureMetric(rt, nv, None, 10.0, lin_alpha=a)
    rng = np.random.default_rng(5)
    gv, yv = rng.standard_normal(n) * 0.01, rng.standard_normal(n) * 0.01
    u, w, ok = met(torch.tensor(gv, device=DEV)[None], torch.zeros((1, n), dtype=torch.bool, device=DEV),
                   torch.tensor(yv, device=DEV)[None], torch.ones(1, dtype=torch.bool, device=DEV))
    eu = rel_max(u[0].cpu().numpy(), np.linalg.solve(M, gv))
    ew = rel_max(w[0].cpu().numpy(), np.linalg.solve(M, yv))
    print(f"LIN metric {name}: rel err u {eu:.1e}, w {ew:.1e}")
    assert ok.tolist() == [True] and max(eu, ew) <= SOLVE_TOL


def test_refinement_with_relinearised_rows(golden):
    """handling at kb 0.12, l = 10 m, relinearise = 3: the knot curvature of the returned line (the h-spline through
    P + alpha n) stays within kb (1 + 1e-6) + curv_error_max, and the lap time is a fresh evaluation bit for bit."""
    g = golden("handling")
    rt, nv, h = _track(g)
    wv = float(g["w_veh"])
    al = B_.opt_min_curv_batch(rt, nv, h, CURVLIM, wv)["alpha"]
    veh = _veh(golden)
    res = R.refine_raceline_batch(rt, nv, al, wv, stepsize_interp=2.0, metric_length=10.0, kappa_bound=CURVLIM,
                                  relinearise=3, **veh)
    print(f"LIN refine handling: rounds {res['rounds'].tolist()}, status {res['status'].tolist()}, iters "
          f"{res['iters'].tolist()}, laptime {res['laptime'].tolist()}, kappa_max {res['kappa_max'].tolist()}, "
          f"kappa_lin_max {res['kappa_lin_max'].tolist()}, curv_error_max {res['curv_error_max'].tolist()}")
    assert not (res["status"] == R.NO_PROJECTION).logical_and(res["evals"] == 0).any()
    x = res["alpha"][0].cpu().numpy()
    k = lin_ref.knot_curvature(g["reftrack"][:, :2] + x[:, None] * nv[0].cpu().numpy(), h[0].cpu().numpy())
    assert np.abs(k).max() <= CURVLIM * (1 + 1e-6) + float(res["curv_error_max"][0])
    lt, _ = _fresh(rt, nv, res["alpha"], None, veh)
    assert torch.equal(lt, res["laptime"])
