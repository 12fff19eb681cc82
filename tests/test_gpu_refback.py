"""GPU parity tests (-m gpu) of the trajectory back end (SURVEY.md 8f-3/8f-4) through the C-ABI against fixtures made by
the reference's own in-tree helpers (tests/golden/refback_*.npz; parity PINNED, see tools/make_golden_ref.py).
Tolerances: interp_track and the boundaries repeat numpy's statements (1e-12 absolute on coordinates of O(1e2..1e3) m);
calc_min_bound_dists differs only by device sin/cos and numpy's matmul rounding (1e-11 m)."""
import contextlib
import io

import numpy as np
import pytest
import torch

from global_racetrajectory_optimization_b200 import batch as B_
from global_racetrajectory_optimization_b200 import helper_funcs_glob as hf

pytestmark = pytest.mark.gpu
NAMES = ["berlin", "handling", "synth333"]


def _pad(rows, width=None, fill=0.0):
    n_max = max(r.shape[0] for r in rows) + 3
    shape = (len(rows), n_max) + rows[0].shape[1:]
    out = np.full(shape, fill)
    for i, r in enumerate(rows):
        out[i, :r.shape[0]] = r
    return out


def test_interp_track_and_boundaries_on_a_ragged_batch(golden):
    dev = torch.device("cuda")
    gs, rs = [golden(n) for n in NAMES], [golden("refback_" + n) for n in NAMES]
    rt = torch.tensor(_pad([g["reftrack"] for g in gs]), device=dev)
    nv = torch.tensor(_pad([g["normvec"] for g in gs]), device=dev)
    npts = torch.tensor([g["reftrack"].shape[0] for g in gs], dtype=torch.int32, device=dev)
    for step in (1.0, 2.5):
        out, n_out = B_.interp_track_batch(rt, step, n_pts=npts)
        for i, r in enumerate(rs):
            want = r[f"interp_track_{step}"]
            assert int(n_out[i]) == want.shape[0]
            assert np.abs(out[i, :want.shape[0]].cpu().numpy() - want).max() <= 1e-12
    out, n_out = B_.interp_track_batch(rt, 1.0, n_pts=npts, n_out_max=100)          # too small: grows to the required size
    assert int(n_out[0]) == rs[0]["interp_track_1.0"].shape[0]
    for sign, col, key in ((1.0, 2, "bound_r_interp"), (-1.0, 3, "bound_l_interp")):
        out, n_out = B_.interp_track_batch(rt, 1.0, n_pts=npts, normvec=nv, normal_sign=sign, width_col=col)
        for i, r in enumerate(rs):
            want = r[key]
            assert int(n_out[i]) == want.shape[0]
            assert np.abs(out[i, :want.shape[0]].cpu().numpy() - want).max() <= 1e-12


def test_check_traj_batch_matches_the_reference_helpers(golden):
    dev = torch.device("cuda")
    gs, rs = [golden(n) for n in NAMES], [golden("refback_" + n) for n in NAMES]
    r0 = rs[0]
    rt = torch.tensor(_pad([g["reftrack"] for g in gs]), device=dev)
    nv = torch.tensor(_pad([g["normvec"] for g in gs]), device=dev)
    npts = torch.tensor([g["reftrack"].shape[0] for g in gs], dtype=torch.int32, device=dev)
    trs = [r["trajectory_opt"] for r in rs]
    ntr = torch.tensor([t.shape[0] for t in trs], dtype=torch.int32, device=dev)
    tr = torch.tensor(_pad(trs), device=dev)
    chk = B_.check_traj_batch(rt, nv, tr[:, :, 1:3].contiguous(), tr[:, :, 3].contiguous(), tr[:, :, 4].contiguous(),
                              tr[:, :, 5].contiguous(), tr[:, :, 6].contiguous(), float(r0["length_veh"]),
                              float(r0["width_veh"]), float(r0["dragcoeff"]), float(r0["mass"]), n_pts=npts, n_traj=ntr)
    for i, r in enumerate(rs):
        n = trs[i].shape[0]
        md = chk["min_dists"][i, :n].cpu().numpy()
        assert np.abs(md - r["min_dists_full"]).max() <= 1e-11                  # calc_min_bound_dists, all boundary points
        assert abs(float(chk["min_dist"][i]) - r["min_dists_full"].min()) <= 1e-11
        k, v, a = trs[i][:, 4], trs[i][:, 5], trs[i][:, 6]
        radii = np.abs(np.divide(1.0, k, out=np.full(k.size, np.inf), where=k != 0))
        ay = np.divide(np.power(v, 2), radii)
        ax_wo = a - (-np.power(v, 2) * float(r0["dragcoeff"]) / float(r0["mass"]))
        want = dict(kappa_abs_max=np.abs(k).max(), ay_max=ay.max(), ax_wo_drag_max=ax_wo.max(), ax_wo_drag_min=ax_wo.min(),
                    a_tot_max=np.sqrt(np.power(ax_wo, 2) + np.power(ay, 2)).max(), vx_max=v.max(), n_points=float(n))
        for key, val in want.items():
            assert abs(float(chk[key][i]) - val) <= 1e-12 * max(1.0, abs(val)), key
    flags = B_.check_traj_flags(chk, r0["ggv"], r0["ax_max_machines"], float(r0["v_max"]), float(r0["curvlim"]))
    assert flags["min_dist"].cpu().tolist() == [True, True, True]              # corners within 1 m of the boundary
    assert flags["curvature"].cpu().tolist() == [False, True, False]           # handling track: 0.167 rad/m > 0.12
    assert not any(flags[k].any().item() for k in ("ay", "ax_pos", "ax_neg", "a_tot", "ax_machines", "v_max"))
    tight = B_.check_traj_flags(chk, r0["tight_ggv"], r0["tight_ax_max_machines"], float(r0["tight_v_max"]),
                                float(r0["tight_curvlim"]))
    assert all(tight[k].all().item() for k in ("ay", "ax_neg", "a_tot", "ax_machines"))


@pytest.mark.parametrize("name", NAMES)
def test_single_track_mirrors_print_and_return_what_the_reference_does(golden, name):
    g, r = golden(name), golden("refback_" + name)
    tr = r["trajectory_opt"]
    args = dict(reftrack=g["reftrack"], reftrack_normvec_normalized=g["normvec"], length_veh=float(r["length_veh"]),
                width_veh=float(r["width_veh"]), debug=True, trajectory=tr, ggv=r["ggv"],
                ax_max_machines=r["ax_max_machines"], v_max=float(r["v_max"]), curvlim=float(r["curvlim"]),
                mass_veh=float(r["mass"]), dragcoeff=float(r["dragcoeff"]))
    for tag, kw in (("stock", {}), ("tight", dict(v_max=float(r["tight_v_max"]), curvlim=float(r["tight_curvlim"]),
                                                  ggv=r["tight_ggv"], ax_max_machines=r["tight_ax_max_machines"]))):
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            b1, b2 = hf.src.check_traj.check_traj(**{**args, **kw})
        assert buf.getvalue() == str(r[f"check_traj_{tag}_stdout"])
        assert np.array_equal(b1, r[f"check_traj_{tag}_bound_r"]) and np.array_equal(b2, r[f"check_traj_{tag}_bound_l"])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        hf.src.check_traj.check_traj(**{**args, "ggv": None, "ax_max_machines": None, "debug": False})
    assert "Since ggv-diagram was not given" in buf.getvalue()
    it = hf.src.interp_track.interp_track(reftrack=g["reftrack"], stepsize_approx=2.5)
    assert it.shape == r["interp_track_2.5"].shape and np.abs(it - r["interp_track_2.5"]).max() <= 1e-12
    md = hf.src.calc_min_bound_dists.calc_min_bound_dists(trajectory=tr, bound1=r["bound_r_interp"], bound2=r["bound_l_interp"],
                                                          length_veh=float(r["length_veh"]), width_veh=float(r["width_veh"]))
    assert np.abs(md - r["min_dists_full"]).max() <= 1e-11


def test_assemble_trajectory_matches_main_globaltraj(golden):
    dev = torch.device("cuda")
    gs, rs = [golden(n) for n in NAMES], [golden("refback_" + n) for n in NAMES]
    trs = [r["trajectory_opt"] for r in rs]
    ntr = torch.tensor([t.shape[0] for t in trs], dtype=torch.int32, device=dev)
    tr = torch.tensor(_pad(trs), device=dev)
    spl = torch.tensor(_pad([g["rl_spline_lengths"] for g in gs]), device=dev)
    nsp = torch.tensor([g["rl_spline_lengths"].shape[0] for g in gs], dtype=torch.int32, device=dev)
    out = B_.assemble_trajectory_batch(tr[:, :, 0].contiguous(), tr[:, :, 1:3].contiguous(), tr[:, :, 3].contiguous(),
                                       tr[:, :, 4].contiguous(), tr[:, :, 5].contiguous(), tr[:, :, 6].contiguous(), spl,
                                       n_traj=ntr, n_spl=nsp)
    for i, r in enumerate(rs):
        want = r["traj_race_cl"]
        got = out[i, :want.shape[0]].cpu().numpy()
        assert np.array_equal(got[:-1], want[:-1]) and np.array_equal(got[-1, 1:], want[-1, 1:])
        assert abs(got[-1, 0] - want[-1, 0]) <= 1e-12 * want[-1, 0]              # sum(spline_lengths): summation order
        assert np.all(out[i, want.shape[0]:].cpu().numpy() == 0.0)


def _ring_tracks(B, K=7):
    """B small closed tracks cycling through K ring shapes of 16 points (radius 10-11 m, outward normals): even shapes are
    narrow, odd ones reach past the centre on the left, where the normals cross.  7 does not divide 65535, so the rows
    after a 65535-track chunk boundary differ from the first rows of the batch, and so do the per-track counts."""
    g = torch.Generator().manual_seed(5)
    ang = torch.arange(16, dtype=torch.float64) * (2 * np.pi / 16)
    normal = torch.stack((ang.cos(), ang.sin()), dim=1).expand(K, 16, 2)
    centre = normal * (10.0 + torch.rand((K, 16, 1), generator=g, dtype=torch.float64))
    w_left = torch.where(torch.arange(K) % 2 == 1, 12.0, 2.0).to(torch.float64)[:, None].expand(K, 16)
    widths = torch.stack((torch.full((K, 16), 2.0, dtype=torch.float64), w_left), dim=2)
    psi = torch.rand((K, 8), generator=g, dtype=torch.float64) * 6.0 - 3.0
    k = torch.arange(B) % K
    b = torch.arange(B, dtype=torch.int32)
    dev = torch.device("cuda")
    return dict(track=torch.cat((centre, widths), dim=2)[k].to(dev), normvec=normal[k].contiguous().to(dev),
                xy=centre[:, ::2][k].contiguous().to(dev), psi=psi[k].to(dev),
                bound_r=(centre + normal * widths[:, :, :1])[k].to(dev), bound_l=(centre - normal * widths[:, :, 1:])[k].to(dev),
                n_pts=(12 + b % 4).to(dev), n_traj=(5 + b % 4).to(dev), nb1=(16 - b % 11).to(dev), nb2=(16 - b % 9).to(dev))


def _ring_checks(t, rows=slice(None)):
    r = {k: v[rows].contiguous() for k, v in t.items()}
    md = B_.min_bound_dists_batch(r["xy"], r["psi"], r["bound_r"], r["bound_l"], 4.7, 2.0, n_traj=r["n_traj"], nb1=r["nb1"],
                                  nb2=r["nb2"])
    return md, B_.check_normals_crossing_batch(r["track"], r["normvec"], 3, n_pts=r["n_pts"])


def test_batches_beyond_the_grid_y_limit_match_a_small_batch():
    """min_bound_dists and check_normals_crossing put the track index on gridDim.y, at most 65535 per launch; the library
    runs larger batches in chunks.  The rows on both sides of the chunk boundary equal a run of the same rows alone."""
    B = 65535 + 7
    t = _ring_tracks(B)
    md, crossing = _ring_checks(t)
    rows = slice(65535 - 3, B)
    md_small, crossing_small = _ring_checks(t, rows)
    assert torch.equal(md[rows], md_small) and torch.equal(crossing[rows], crossing_small)
    assert bool((md_small[:, :5] > 0).all()) and bool(crossing_small.any()) and not bool(crossing_small.all())


def test_check_normals_crossing_batch_vs_oracle(golden):
    """tph.check_normals_crossing (prep_track.py:57-59; tph restatement, parity unpinned) on widened fixtures."""
    import global_racetrajectory_optimization_b200 as tph
    from oracle import tph_prep
    dev = torch.device("cuda")
    gs = [golden(n) for n in NAMES]
    scales = (1.0, 2.0, 3.0, 4.0)
    rows, nvs, want = [], [], []
    for g in gs:
        for sc in scales:
            rt = g["reftrack"].copy()
            rt[:, 2:] *= sc
            rows.append(rt)
            nvs.append(g["normvec"])
            want.append(tph_prep.check_normals_crossing(rt, g["normvec"], 10))
    rt = torch.tensor(_pad(rows), device=dev)
    nv = torch.tensor(_pad(nvs), device=dev)
    npts = torch.tensor([r.shape[0] for r in rows], dtype=torch.int32, device=dev)
    got = B_.check_normals_crossing_batch(rt, nv, 10, n_pts=npts).cpu().tolist()
    assert got == want and any(want) and not all(want)
    assert tph.check_normals_crossing.check_normals_crossing(track=rows[0], normvec_normalized=nvs[0], horizon=10) is False
    assert tph.check_normals_crossing.check_normals_crossing(track=rows[3], normvec_normalized=nvs[3], horizon=10) is True
    with pytest.raises(RuntimeError, match="too large"):
        tph.check_normals_crossing.check_normals_crossing(track=rows[0][:8], normvec_normalized=nvs[0][:8], horizon=10)
