"""CPU tests (-m "not gpu") of a vehicle per track through the flow: the MC_OPTIONAL3 parameters of the C-ABI as the
binding reads them and their short forms without a GPU, and against the recording stand-in of the library: the float
path's launches unchanged, the stage sequence, chunking and centre-id re-indexing of a [B] curvature limit, the
Vehicles fields, check_traj_flags(vehicles=) and the wiring of globaltraj_batch(vehicles=)."""
import ctypes

import numpy as np
import pytest
import torch

from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_, globaltraj

TABLES = dict(ggv=[np.array([[0.0, 5.0, 6.0], [80.0, 4.0, 7.0]])] * 2, ax_max_machines=[np.array([[0.0, 8.0], [80.0, 3.0]])] * 2)


def test_the_vehicle_parameters_are_parsed_from_the_header():
    assert _lib._OPTIONAL3 == {"mc_mincurv_solve_batch_ex": (19, 6), "mc_mincurv_finalize_batch": (9, 1),
                               "mc_mincurv_kappa_batch": (7, 1), "mc_min_bound_dists_batch": (15, 2),
                               "mc_traj_extrema_batch": (10, 2)}
    assert len(_lib.EXPORTED_SYMBOLS) == 47
    assert _lib._SIGS["mc_mincurv_solve_batch_ex"][1][19:25] == [ctypes.c_void_p] * 6


def test_short_forms_without_gpu():
    """Each changed entry without its MC_OPTIONAL3 parameters and with them NULL passes the same checks in the same
    order: an undersized workspace gives -3, a NULL input -1."""
    lib = _lib.load()
    d = ctypes.c_void_p(4096)
    head = [1, 100, None, d, d, d]
    for tail in ([], [None] * 6):
        ex = head + [0.12, 2.0, None, 2.0, d, d, None, d, None, 0.0, None, None, None] + tail
        assert lib.mc_mincurv_solve_batch_ex(*ex, None, 0, None) == -3
        assert lib.mc_mincurv_solve_batch_ex(*ex[:3], None, *ex[4:], None, 0, None) == -1
    for tail in ([], [None]):
        assert lib.mc_mincurv_finalize_batch(1, 100, None, d, 0.12, d, None, d, 0, *tail, None, 0, None) == -3
        assert lib.mc_mincurv_finalize_batch(1, 100, None, None, 0.12, d, None, d, 0, *tail, None, 0, None) == -1
        assert lib.mc_mincurv_kappa_batch(1, 100, None, 0.12, d, d, None, *tail, None, 0, None) == -3
        assert lib.mc_mincurv_kappa_batch(1, 100, None, 0.12, None, d, None, *tail, None, 0, None) == -1
    for tail in ([], [None, None]):
        assert lib.mc_min_bound_dists_batch(1, 10, None, None, d, 4, None, d, 4, None, d, 2, 4.7, 2.0, d, *tail, None) == -1
        assert lib.mc_traj_extrema_batch(1, 10, None, None, d, d, None, 0.75, 1200.0, d, *tail, None) == -1
        assert lib.mc_traj_extrema_batch(1, 10, None, d, d, d, None, 0.75, 0.0, None, *tail, None) == -1
    # the sensitivity export of the extended entry: sens and grad_status together, the rows only with them
    ex = head + [0.12, 2.0, None, 2.0, d, d, None, d, None, 0.0, None, None, None, None, None]
    assert lib.mc_mincurv_solve_batch_ex(*ex, d, None, None, None, None, 0, None) == -1
    assert lib.mc_mincurv_solve_batch_ex(*ex, d, d, None, None, None, 0, None) == -3
    assert lib.mc_mincurv_solve_batch_ex(*ex, None, None, d, d, None, 0, None) == -1
    assert lib.mc_mincurv_solve_batch_ex(*ex, d, d, d, d, None, 0, None) == -3


def _qp(B=4, n=100):
    g = torch.Generator().manual_seed(1)
    return (torch.rand((B, n, 4), dtype=torch.float64, generator=g), torch.rand((B, n, 2), dtype=torch.float64, generator=g),
            torch.ones((B, n), dtype=torch.float64))


def test_the_float_path_launches_as_before(fake):
    rt, nv, h = _qp()
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0)
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, lin_alpha=torch.zeros((4, 100), dtype=torch.float64))
    widths = rt[:, :, 2:].clone().requires_grad_()
    B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, 2.0, strict=False)["alpha"].sum().backward()
    names = [c[0] for c in fake.calls if c[0].startswith("mc_mincurv") and not c[0].endswith("_bytes")]
    assert names == (["mc_mincurv_solve_batch_shared"] * 2 + ["mc_mincurv_solve_batch_ex"] * 2
                     + ["mc_mincurv_solve_batch_sens"] * 2 + ["mc_mincurv_adjoint_batch"] * 2)
    for name, a in fake.calls:
        if name in ("mc_mincurv_solve_batch_shared", "mc_mincurv_solve_batch_sens", "mc_mincurv_solve_batch_ex"):
            assert a[6] == 0.12
        if name == "mc_mincurv_solve_batch_ex":
            assert a[19:25] == (None,) * 6


def test_a_limit_per_instance_goes_through_the_extended_entry_per_chunk(fake, monkeypatch):
    """A [B] limit: mc_mincurv_solve_batch_ex on each chunk (the solve of mc_mincurv_solve_batch_shared) with the chunk's
    rows of the limits, the centre ids re-indexed inside the chunk and no export; the scalar kappa_bound is 0."""
    rt, nv, h = _qp()
    chunk_ids = []
    real = B_.shared_centre_ids
    monkeypatch.setattr(B_, "shared_centre_ids", lambda g: chunk_ids.append(real(g)) or chunk_ids[-1])
    kb = torch.tensor([0.12, 0.05, 0.12, 0.03], dtype=torch.float64)
    B_.opt_min_curv_batch(rt, nv, h, kb, 2.0, centre_id=torch.tensor([0, 0, 0, 2]))
    calls = [(n, a) for n, a in fake.calls if n.startswith("mc_mincurv") and not n.endswith("_bytes")]
    assert [n for n, _ in calls] == ["mc_mincurv_solve_batch_ex"] * 2                 # chunks of two, one workspace
    assert len({a[-3].value for _, a in calls}) == 1
    for k, (_, a) in enumerate(calls):
        assert a[0] == 2 and a[6] == 0.0 and a[15] == 0.0 and a[16:19] == (None,) * 3
        assert a[19].value == kb[2 * k:2 * k + 2].data_ptr() and a[21:25] == (None,) * 4
    # centre ids re-indexed inside each chunk: [0, 0] and, for owners 0 and 2 of the chunk 2:4, [0, 1]
    assert [c.tolist() for c in chunk_ids] == [[0, 0], [0, 1]]
    assert [a[20].value for _, a in calls] == [c.data_ptr() for c in chunk_ids]
    with pytest.raises(ValueError, match="finite curvature"):
        B_.opt_min_curv_batch(rt, nv, h, torch.tensor([0.12, 0.0, 0.1, 0.1], dtype=torch.float64), 2.0)
    with pytest.raises(ValueError, match="one entry per track"):
        B_.opt_min_curv_batch(rt, nv, h, torch.tensor([0.12, 0.1], dtype=torch.float64), 2.0)


def test_the_sensitivities_and_the_projection_take_the_limits(fake):
    rt, nv, h = _qp()
    kb = torch.tensor([0.12, 0.05, 0.12, 0.03], dtype=torch.float64)
    widths = rt[:, :, 2:].clone().requires_grad_()
    B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, kb, 2.0, strict=False, curvature_rows=True)["alpha"].sum().backward()
    ex = [a for n, a in fake.calls if n == "mc_mincurv_solve_batch_ex"]
    assert len(ex) == 2 and not any(n == "mc_mincurv_solve_batch_sens" for n, _ in fake.calls)
    for k, a in enumerate(ex):
        assert a[19].value == kb[2 * k:2 * k + 2].data_ptr() and all(x is not None for x in a[21:25])
    fake.calls.clear()
    from global_racetrajectory_optimization_b200 import raceline_refine as R
    p = R.CurvatureProjection(rt, nv, None, 2.0, kb, 10.0)
    p(torch.zeros((4, 100), dtype=torch.float64), torch.zeros((4, 100), dtype=torch.float64), torch.ones(4, dtype=torch.bool))
    p.evaluate(torch.zeros((4, 100), dtype=torch.float64), torch.ones(4, dtype=torch.bool))
    assert [a[19].value for n, a in fake.calls if n == "mc_mincurv_solve_batch_ex"] == [kb[:2].data_ptr(), kb[2:].data_ptr()]
    assert [a[9].value for n, a in fake.calls if n == "mc_mincurv_finalize_batch"] == [kb[:2].data_ptr(), kb[2:].data_ptr()]


def test_check_traj_wrappers_pass_the_arrays(fake):
    B, n = 4, 50
    z = torch.zeros((B, n), dtype=torch.float64)
    length = torch.tensor([4.7, 4.2, 5.0, 4.7], dtype=torch.float64)
    B_.min_bound_dists_batch(torch.zeros((B, n, 2), dtype=torch.float64), z, torch.zeros((B, 8, 4), dtype=torch.float64),
                             torch.zeros((B, 8, 4), dtype=torch.float64), length, 2.0)
    B_.traj_extrema_batch(z, z, z, 0.75, torch.full((B,), 1200.0, dtype=torch.float64))
    B_.traj_extrema_batch(z, z, z, 0.75, 1200.0)
    (_, mb), (_, e1), (_, e2) = [c for c in fake.calls if c[0] in ("mc_min_bound_dists_batch", "mc_traj_extrema_batch")]
    assert mb[12] == 0.0 and mb[13] == 2.0 and mb[15].value == length.data_ptr() and mb[16] is None
    assert e1[8] == 0.0 and e1[10] is None and e1[11] is not None
    assert e2[8] == 1200.0 and e2[10] is None and e2[11] is None
    with pytest.raises(ValueError, match="mass_veh"):
        B_.traj_extrema_batch(z, z, z, 0.75, torch.tensor([1200.0, 0.0, 1.0, 1.0], dtype=torch.float64))


def test_vehicles_fields_and_flags():
    v = B_.Vehicles(**TABLES, v_max=[70.0, 60.0], drag_coeff=0.75, m_veh=[1200.0, 1300.0], device="cpu", curvlim=[0.12, 0.05],
                    length=4.7)
    assert v.curvlim == [0.12, 0.05] and v.length == [4.7, 4.7] and v.width_opt is None and v.width is None
    ids = torch.tensor([1, 0, 1, 7], dtype=torch.int32)              # (a device veh_id is not range-checked)
    kb = v.per_track("curvlim", ids)
    assert kb[:3].tolist() == [0.05, 0.12, 0.05] and bool(torch.isnan(kb[3]))
    assert v.per_track("m_veh", ids)[:3].tolist() == [1300.0, 1200.0, 1300.0]
    with pytest.raises(ValueError, match="not set"):
        v.per_track("width", ids)
    for bad in (dict(curvlim=[0.1, 0.0]), dict(width=[2.0, float("nan")]), dict(length=[1.0])):
        with pytest.raises(ValueError):
            B_.Vehicles(**TABLES, v_max=70.0, drag_coeff=0.75, m_veh=1200.0, device="cpu", **bad)
    chk = {k: torch.tensor(x, dtype=torch.float64) for k, x in dict(
        min_dist=[2.0, 0.5, 2.0], kappa_abs_max=[0.1, 0.1, 0.01], vx_max=[65.0, 65.0, 50.0], ay_max=[6.95, 7.2, 1.0],
        ax_wo_drag_max=[5.05, 5.2, 1.0], ax_wo_drag_min=[-5.05, -5.2, -1.0], a_tot_max=[1.0, 7.2, 1.0]).items()}
    f = B_.check_traj_flags(chk, vehicles=v, veh_id=[0, 1, 1])
    assert f["curvature"].tolist() == [False, True, False] and f["v_max"].tolist() == [False, True, False]
    assert f["min_dist"].tolist() == [False, True, False] and f["ay"].tolist() == [False, True, False]
    assert f["ax_pos"].tolist() == [False, True, False] and f["ax_neg"].tolist() == [False, True, False]
    ref = B_.check_traj_flags(chk, TABLES["ggv"][0], TABLES["ax_max_machines"][0], 70.0, 0.12)
    assert all(f[k][0] == ref[k][0] for k in ref)
    with pytest.raises(ValueError, match="must be None"):
        B_.check_traj_flags(chk, TABLES["ggv"][0], vehicles=v, veh_id=[0, 1, 1])


@pytest.mark.parametrize("opt_type,refine", [("mincurv", None), ("mincurv_iqp", None), ("shortest_path", None),
                                             ("mincurv", {"metric_length": 10.0})])
def test_globaltraj_wiring(fake, monkeypatch, opt_type, refine):
    """Each stage gets the per-track tensors (curvlim and width_opt from the Vehicles, length and width from pars where
    unset) and the velocity profile and the refinement get vehicles= and the device veh_id."""
    seen = {}
    rec = lambda name, out: (lambda *a, **k: seen.setdefault(name, (a, k)) and out(*a, **k))   # noqa: E731
    B, n = 4, 100
    f64 = dict(dtype=torch.float64)
    qp = lambda *a, **k: dict(alpha=torch.zeros((B, n), **f64), status=torch.zeros(B, dtype=torch.int32),    # noqa: E731
                              reftrack=a[0], normvec=a[1], n_pts=torch.full((B,), n, dtype=torch.int32))
    monkeypatch.setattr(B_, "opt_min_curv_batch", rec("qp", qp))
    monkeypatch.setattr(B_, "iqp_batch", rec("qp", qp))
    monkeypatch.setattr(B_, "opt_shortest_path_batch", rec("sp", qp))
    from global_racetrajectory_optimization_b200 import raceline_refine as R
    monkeypatch.setattr(R, "refine_raceline_batch", rec("refine", lambda *a, **k: dict(
        alpha=a[2], laptime_start=torch.zeros(B, **f64), status=torch.zeros(B, dtype=torch.int32),
        iters=torch.zeros(B, dtype=torch.int32), evals=torch.zeros(B, dtype=torch.int32))))
    monkeypatch.setattr(B_, "vel_profile_batch", rec("vp", lambda *a, **k: dict(
        vx=torch.zeros((B, 1, n), **f64), ax=torch.zeros((B, 1, n), **f64), t=torch.zeros((B, 1, n + 1), **f64),
        laptime=torch.zeros((B, 1), **f64), status=torch.zeros((B, 1), dtype=torch.int32))))
    monkeypatch.setattr(B_, "check_traj_batch", rec("check", lambda *a, **k: {}))
    v = B_.Vehicles(**TABLES, v_max=[70.0, 60.0], drag_coeff=[0.75, 0.9], m_veh=[1200.0, 1300.0], device="cpu",
                    curvlim=[0.12, 0.05], width_opt=[3.4, 2.6])
    rt = torch.rand((B, n, 4), **f64) + torch.tensor([0.0, 0.0, 5.0, 5.0], **f64)
    globaltraj.globaltraj_batch(rt, opt_type, globaltraj.default_pars(), vehicles=v, veh_id=[1, 0, 0, 1], refine=refine)
    ids = [1, 0, 0, 1]
    if opt_type == "shortest_path":
        assert seen["sp"][0][2].tolist() == [[3.4, 2.6][i] for i in ids]
    else:
        assert seen["qp"][0][3].tolist() == [[0.12, 0.05][i] for i in ids]
        assert seen["qp"][0][4].tolist() == [[3.4, 2.6][i] for i in ids]
    vp = seen["vp"][1]
    assert vp["vehicles"] is v and vp["veh_id"].tolist() == ids and "ggv" not in vp
    chk = seen["check"][0]
    assert chk[7:9] == (4.7, 2.0) and chk[9].tolist() == [[0.75, 0.9][i] for i in ids]
    assert chk[10].tolist() == [[1200.0, 1300.0][i] for i in ids]
    if refine is not None:
        a, k = seen["refine"]
        assert a[3].tolist() == [[3.4, 2.6][i] for i in ids] and k["vehicles"] is v and k["metric_length"] == 10.0
    with pytest.raises(ValueError, match="must be None"):
        globaltraj.globaltraj_batch(rt, opt_type, globaltraj.default_pars(), TABLES["ggv"][0], vehicles=v, veh_id=ids)
    with pytest.raises(ValueError, match="needs vehicles"):
        globaltraj.globaltraj_batch(rt, opt_type, globaltraj.default_pars(), TABLES["ggv"][0], TABLES["ax_max_machines"][0],
                                    veh_id=ids)
