"""CPU tests (-m "not gpu") of the host logic above the C-ABI: every batched wrapper is run against the recording stand-in
of libmincurv_b200.so in fake_lib.py, with CPU tensors in place of device buffers.  Catches arity / ordering / chunking
mistakes in batch.py and globaltraj.py without a GPU; the numerical behaviour is covered by the -m gpu tests."""
import numpy as np
import pytest
import torch

from fake_lib import FakeLib, fake  # noqa: F401  (fake: the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_, globaltraj


def _names(lib):
    return [c[0] for c in lib.calls]


def test_every_wrapper_matches_the_signature_table(fake):
    B, n = 5, 120
    rt = torch.rand((B, n, 4), dtype=torch.float64) + 3.0
    npts = torch.full((B,), n, dtype=torch.int32)
    cx, cy, nv, h = B_.calc_splines_batch(rt, n_pts=npts)
    res = B_.opt_min_curv_batch(rt, nv, h, 0.12, torch.full((B,), 2.0, dtype=torch.float64), n_pts=npts)
    assert _names(fake).count("mc_mincurv_solve_batch_shared") == 3                     # 5 tracks in chunks of 2
    assert res["alpha"].shape == (B, n)
    widths = rt[:, :, 2:].clone().requires_grad_()
    B_.opt_min_curv_diff(rt[:, :, :2], widths, nv, h, 0.12, 2.0, n_pts=npts)["alpha"].sum().backward()
    assert widths.grad.shape == (B, n, 2)
    alpha = torch.zeros((B, n), dtype=torch.float64)      # (the stand-in library writes nothing: outputs are uninitialised)
    B_.opt_shortest_path_batch(rt, nv, 2.0, n_pts=npts)
    rl = B_.create_raceline_batch(rt, nv, alpha, 2.0, n_pts=npts)
    B_.calc_head_curv_batch(rl["coeffs_x"], rl["coeffs_y"], rl["spline_inds"], rl["t_values"], n_eval=rl["n_out"])
    B_.iqp_relinearise_batch(rt, nv, alpha, 3.0, n_pts=npts)
    B_.scale_alpha_batch(alpha, 0.5)
    ggv = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
    mach = np.array([[0.0, 5.0], [80.0, 5.0]])
    kap, el = torch.rand((B, 200), dtype=torch.float64), torch.ones((B, 200), dtype=torch.float64)
    vp = B_.vel_profile_batch(kap, el, ggv, mach, 70.0, 0.75, 1200.0, n_pts=torch.full((B,), 200, dtype=torch.int32))
    assert vp["vx"].shape == (B, 1, 200) and vp["t"].shape == (B, 1, 201) and _names(fake).count("mc_vel_profile_batch_ex") == 3
    ltm = B_.lap_time_matrix_batch(kap, el, ggv, mach, [0.5, 1.0], [30.0, 40.0, 50.0], 0.75, 1200.0)
    assert ltm.shape == (B, 3, 2)
    last = [c for c in fake.calls if c[0] == "mc_vel_profile_batch_ex"][-1][1]
    assert last[6] == 6                                                              # V = 3 top speeds x 2 ggv scales
    B_.calc_ax_t_profile_batch(torch.rand((B, 201), dtype=torch.float64), el)
    out, n_out = B_.interp_track_batch(rt, 1.0, n_pts=npts)
    assert out.shape[0] == B and out.shape[2] == 4
    chk = B_.check_traj_batch(rt, nv, torch.rand((B, 200, 2), dtype=torch.float64), kap, kap, kap, kap, 4.7, 2.0, 0.75, 1200.0,
                              n_pts=npts)
    assert set(B_.EXTREMA) <= set(chk) and chk["min_dists"].shape == (B, 200)
    flags = B_.check_traj_flags(chk, ggv, mach, 70.0, 0.12)
    assert set(flags) == {"min_dist", "curvature", "v_max", "ay", "ax_pos", "ax_neg", "a_tot", "ax_machines"}
    B_.assemble_trajectory_batch(kap, torch.rand((B, 200, 2), dtype=torch.float64), kap, kap, kap, kap,
                                 torch.rand((B, n), dtype=torch.float64))
    assert B_.check_normals_crossing_batch(rt, nv, 10, n_pts=npts).shape == (B,)
    with pytest.raises(RuntimeError, match="too large"):
        B_.check_normals_crossing_batch(rt, nv, n, n_pts=npts)
    raw = torch.rand((B, 300, 4), dtype=torch.float64) + 3.0
    smoothed, n_smoothed, lam = B_.spline_approximation_batch(raw, k_reg=3, s_reg=10.0, stepsize_prep=1.0, stepsize_reg=3.0)
    assert smoothed.shape[0] == B and smoothed.shape[2] == 4 and n_smoothed.shape == (B,) and lam.shape == (B,)
    used = set(_names(fake))
    assert used >= set(_lib.EXPORTED_SYMBOLS) - {"mc_version", "mc_last_error", "mc_debug_read_profile", "mc_debug_factor_solve",
                                                 "mc_mincurv_setup_batch", "mc_mincurv_setup_batch_ex", "mc_mincurv_setup_batch_shared",
                                                 "mc_mincurv_solve_batch", "mc_mincurv_solve_batch_ex",
                                                 "mc_vel_profile_batch", "mc_mincurv_pdip_batch", "mc_mincurv_finalize_batch",
                                                 "mc_mincurv_kappa_batch", "mc_iqp_finish_batch", "mc_jitter_widths_batch"}


def test_shared_centre_ids_and_their_chunking(fake, monkeypatch):
    """centre_id: owners are the first instance of every group; inside a chunk the first instance of the chunk with the
    same owner takes the role (the owner itself may live in another chunk)."""
    group = torch.tensor([7, 3, 7, 3, 3, 9], dtype=torch.int64)
    cid = B_.shared_centre_ids(group)
    assert cid.dtype == torch.int32 and cid.tolist() == [0, 1, 0, 1, 1, 5]
    B, n = 6, 120
    rt = torch.rand((B, n, 4), dtype=torch.float64) + 3.0
    cx, cy, nv, h = B_.calc_splines_batch(rt)
    fake.calls.clear()
    local, real = [], B_.shared_centre_ids
    monkeypatch.setattr(B_, "shared_centre_ids", lambda g: local.append(real(g)) or local[-1])
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, centre_id=cid)           # the fixture forces chunks of 3
    calls = [c[1] for c in fake.calls if c[0] == "mc_mincurv_solve_batch_shared"]
    assert [c[0] for c in calls] == [3, 3]
    assert [t.tolist() for t in local] == [[0, 1, 0], [0, 0, 2]]           # local owners of [0, 1, 0] and [1, 1, 5]
    assert [c[10].value for c in calls] == [t.data_ptr() for t in local]
    with pytest.raises(ValueError, match="centre_id"):
        B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, centre_id=cid[:4])


def test_launches_with_the_track_index_on_grid_y_are_chunked(fake, monkeypatch):
    monkeypatch.setattr(B_, "_GRID_Y_MAX", 2)
    B, n = 5, 100
    rt = torch.rand((B, n, 4), dtype=torch.float64)
    nv = torch.rand((B, n, 2), dtype=torch.float64)
    B_.check_normals_crossing_batch(rt, nv, 10)
    B_.min_bound_dists_batch(torch.rand((B, 50, 2), dtype=torch.float64), torch.rand((B, 50), dtype=torch.float64), rt, rt,
                             4.7, 2.0)
    sizes = [c[1][0] for c in fake.calls if c[0] == "mc_check_normals_crossing_batch"]
    assert sizes == [2, 2, 1]
    assert [c[1][0] for c in fake.calls if c[0] == "mc_min_bound_dists_batch"] == [2, 2, 1]


@pytest.mark.parametrize("opt_type", ["mincurv", "shortest_path"])
def test_globaltraj_batch_wires_the_stages_in_the_reference_order(fake, opt_type):
    B, n = 3, 150
    rt = torch.rand((B, n, 4), dtype=torch.float64) + 3.0
    ggv = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
    mach = np.array([[0.0, 5.0], [80.0, 5.0]])
    out = globaltraj.globaltraj_batch(rt, opt_type, globaltraj.default_pars(), ggv, mach)
    order = [nm for nm in _names(fake) if not nm.endswith("_workspace_bytes")]
    qp = "mc_mincurv_solve_batch_shared" if opt_type == "mincurv" else "mc_shortest_path_solve_batch"
    want = ["mc_calc_splines_batch", qp, "mc_create_raceline_batch", "mc_vel_profile_batch_ex", "mc_assemble_trajectory_batch",
            "mc_interp_track_batch", "mc_min_bound_dists_batch", "mc_traj_extrema_batch"]
    staged = [nm for nm in order if nm in want]                   # (helper launches such as mc_polygon_length_batch aside)
    stages = [nm for k, nm in enumerate(staged) if k == 0 or staged[k - 1] != nm]                  # chunked launches collapse
    assert stages == want
    assert out["trajectory"].shape[2] == 7 and out["laptime"].shape == (B,) and "min_dist" in out
    with pytest.raises(IOError):
        globaltraj.globaltraj_batch(rt, "mintime", globaltraj.default_pars(), ggv, mach)


def test_iqp_batch_grows_its_buffers_when_a_resampled_track_does_not_fit(fake, monkeypatch):
    """mc_iqp_relinearise_batch reports -(required points) for a track that exceeds the capacity; iqp_batch must enlarge
    every per-track buffer and repeat the step.  The stand-in writes those counts into the (CPU) n_pts_new tensor."""
    import ctypes
    B, n = 2, 100
    state = {"calls": 0, "caps": []}
    real_getattr = FakeLib.__getattr__

    def patched(self, name):
        fn = real_getattr(self, name)
        if name == "mc_mincurv_solve_batch_shared":
            def solve(*a):
                fn(*a)
                bq, nmax = a[0], a[1]
                ctypes.memset(a[11].value, 0, bq * nmax * 8)                     # alpha = 0
                ctypes.memset(a[12].value, 0, bq * 8)                            # curv_error_max = 0 (converged once iter >= iters_min)
                ctypes.memset(a[14].value, 0, bq * 4)                            # status = 0
                return 0
            return solve
        if name == "mc_iqp_finish_batch":
            def finish(*a):        # stand-in of the device-side termination test: curv_error_max = 0, so done once iter >= iters_min
                fn(*a)
                bq, it, iters_min = a[0], a[3], a[4]
                done = it >= iters_min
                i32 = lambda ptr, k: (ctypes.c_int32 * k).from_address(ptr.value)
                counters, active = i32(a[22], 2), i32(a[8], bq)
                counters[0], counters[1] = (0, bq) if done else (bq, 0)
                if done:
                    npts = i32(a[11], bq)
                    for b in range(bq):
                        active[b] = 0
                        i32(a[18], bq)[b] = npts[b]          # fin_n_pts
                        i32(a[19], bq)[b] = it               # fin_outer_iters
                return 0
            return finish
        if name != "mc_iqp_relinearise_batch":
            return fn

        def relin(*a):
            fn(*a)
            state["calls"] += 1
            cap = a[8]
            state["caps"].append(cap)
            need = -(cap + 40) if state["calls"] == 1 else cap - 5              # first answer: does not fit
            arr = (ctypes.c_int32 * B)(*([need] * B))
            ctypes.memmove(a[11].value, arr, 4 * B)
            return 0
        return relin
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    rt = torch.rand((B, n, 4), dtype=torch.float64) + 3.0
    nv = torch.rand((B, n, 2), dtype=torch.float64)
    h = torch.ones((B, n), dtype=torch.float64)
    res = B_.iqp_batch(rt, nv, h, 0.12, 2.0, 3.0, iters_min=2, curv_error_allowed=0.01)
    # grown, then accepted; the third launch follows the iteration in which every track finished (the host learns that from
    # the same single read as the point counts, so the launch is already queued: its kernels skip inactive tracks)
    assert state["calls"] == 3 and state["caps"][1] == state["caps"][0] + 40 + 64 and state["caps"][2] == state["caps"][1]
    cap = state["caps"][1]
    assert res["alpha"].shape == (B, cap) and res["reftrack"].shape == (B, cap, 4) and res["normvec"].shape == (B, cap, 2)
    assert res["outer_iters"].tolist() == [2, 2] and res["n_pts"].tolist() == [cap - 5, cap - 5] and res["qp_solves"] == 4


def test_iqp_batch_with_a_fixed_iteration_count_checks_the_capacity_once_at_the_end(fake, monkeypatch):
    """fixed_iters: the iterations are queued without host reads; an overflow reported by mc_iqp_relinearise_batch in any of
    them makes the call repeat once with room for the largest track."""
    import ctypes
    B, n = 2, 100
    state = {"caps": []}
    real_getattr = FakeLib.__getattr__

    def patched(self, name):
        fn = real_getattr(self, name)
        if name != "mc_iqp_relinearise_batch":
            return fn

        def relin(*a):
            fn(*a)
            cap = a[8]
            state["caps"].append(cap)
            need = -(cap + 30) if len(state["caps"]) == 2 else cap - 5          # the second re-sampling of the first pass overflows
            ctypes.memmove(a[11].value, (ctypes.c_int32 * B)(*([need] * B)), 4 * B)
            return 0
        return relin
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    rt = torch.rand((B, n, 4), dtype=torch.float64) + 3.0
    nv = torch.rand((B, n, 2), dtype=torch.float64)
    h = torch.ones((B, n), dtype=torch.float64)
    res = B_.iqp_batch(rt, nv, h, 0.12, 2.0, 3.0, fixed_iters=4)
    first = state["caps"][0]
    # 3 re-samplings per pass (4 iterations), two passes; the second pass runs with the capacity the overflow asked for
    assert len(state["caps"]) == 6 and state["caps"][:3] == [first] * 3 and state["caps"][3:] == [first + 30 + 64] * 3
    assert res["alpha"].shape == (B, first + 30 + 64) and res["qp_solves"] == 4 * B
    assert _names(fake).count("mc_mincurv_solve_batch_shared") == 2 * 4 * 2        # (the fixture forces chunks of one track)
