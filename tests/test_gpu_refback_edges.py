"""GPU tests (-m gpu) of the trajectory back end (K6, csrc/traj_check.cu) where its kernels change code path, against the
reference's own helpers on constructed cases (tests/golden/refback_edges.npz; tests/test_refback_edges_host.py shows the
same statements on the host reproduce every case bit for bit and that each case reaches its path).

interp_track, the extrema and the assembly run the same correctly rounded statements as the host, and min_bound_dists at
psi = 0 has exact corners (cos 0 = 1, sin 0 = 0), so all of these are compared bit for bit.  Only rotated corners carry a
tolerance (test_min_bound_dists_rotated_within_the_sin_cos_bound)."""
import contextlib
import io

import numpy as np
import pytest
import torch

import refback_edge_cases as E
from refback_edge_cases import same
from global_racetrajectory_optimization_b200 import batch as B_
from global_racetrajectory_optimization_b200 import helper_funcs_glob as hf

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
SENTINEL = 7.0e7          # padding that would show in any distance, sum or extremum it leaked into


@pytest.fixture(scope="module")
def edges(golden):
    return golden("refback_edges")


def _pad(rows, n_max=None, fill=np.nan):
    n_max = n_max or max(r.shape[0] for r in rows)
    out = np.full((len(rows), n_max) + rows[0].shape[1:], fill)
    for i, r in enumerate(rows):
        out[i, :r.shape[0]] = r
    return torch.tensor(out, device=DEV)


def _counts(rows):
    return torch.tensor([r.shape[0] for r in rows], dtype=torch.int32, device=DEV)


def _it_cases(edges):
    """(name, track, normvec, step, want) for every fixture interp_track run"""
    out = []
    for name in edges["it_names"]:
        for i, step in enumerate(edges[f"it_{name}_steps"]):
            out.append((str(name), edges[f"it_{name}_track"], edges[f"it_{name}_normvec"], float(step), edges[f"it_{name}_{i}"]))
    return out


def _raw_interp(pts, n_pts, step, n_out_max, normvec=None, sign=0.0, col=2):
    """mc_interp_track_batch with a fixed n_out_max (the wrapper regrows it): out and the raw n_out (-m: too small)"""
    B, n_max, stride = pts.shape
    out = torch.full((B, n_out_max, 4), SENTINEL, dtype=torch.float64, device=DEV)
    n_out = torch.full((B,), 12345, dtype=torch.int32, device=DEV)
    ws = B_._workspace("interp_track", B_._lib.load().mc_interp_track_workspace_bytes(B, n_max), DEV)
    B_._call("mc_interp_track_batch", B, n_max, n_pts, pts.contiguous(), stride, normvec, float(sign), int(col), float(step),
             int(n_out_max), out, n_out, ws=ws)
    return out, n_out


def test_interp_track_alone_and_in_a_ragged_batch_bit_for_bit(edges):
    cases = _it_cases(edges)
    for step in sorted({c[3] for c in cases}):
        group = [c for c in cases if c[3] == step]
        rows = [c[1] for c in group]
        pts, npts = _pad(rows, max(r.shape[0] for r in rows) + 3), _counts(rows)            # NaN in every padding row
        for stride in (4, 2):
            out, n_out = B_.interp_track_batch(pts[:, :, :stride].contiguous(), step, n_pts=npts)
            for i, (name, rt, _, _, want) in enumerate(group):
                m = want.shape[0]
                assert int(n_out[i]) == m, (name, step)
                got = out[i, :m].cpu().numpy()
                assert same(got[:, :stride], want[:, :stride]), (name, step, stride)
                assert stride == 4 or not got[:, 2:].any()
        for name, rt, _, _, want in group:                                                       # alone
            out, n_out = B_.interp_track_batch(torch.tensor(rt, device=DEV)[None], step)
            assert int(n_out[0]) == want.shape[0] and same(out[0, :want.shape[0]].cpu().numpy(), want), (name, step)


def test_interp_track_boundary_form_bit_for_bit(edges):
    names = [str(n) for n in edges["it_names"]]
    rows = [edges[f"it_{n}_track"] for n in names]
    pts, npts = _pad(rows, max(r.shape[0] for r in rows) + 2), _counts(rows)
    nv = _pad([edges[f"it_{n}_normvec"] for n in names], pts.shape[1])
    for sign, col, side in ((1.0, 2, "r"), (-1.0, 3, "l")):                                      # check_traj.py:50-61
        out, n_out = B_.interp_track_batch(pts, 1.0, n_pts=npts, normvec=nv, normal_sign=sign, width_col=col)
        for i, n in enumerate(names):
            want = edges[f"it_{n}_bound_{side}"]
            assert int(n_out[i]) == want.shape[0] and same(out[i, :want.shape[0]].cpu().numpy(), want), (n, side)


def test_interp_track_capacity_and_refused_tracks(edges):
    names = ["ring127", "n2", "square10", "repeat"]
    rows = [edges[f"it_{n}_track"] for n in names]
    want = [edges[f"it_{n}_0"] for n in names]                                                   # step 1.0
    m = [w.shape[0] for w in want]
    big = int(np.argmax(m))
    pts, npts = _pad(rows, 140), _counts(rows)
    for cap, expect_big in ((m[big] - 1, -m[big]), (m[big], m[big])):
        out, n_out = _raw_interp(pts, npts, 1.0, cap)
        assert int(n_out[big]) == expect_big
        for i in range(len(names)):
            if i != big:
                assert int(n_out[i]) == m[i] and same(out[i, :m[i]].cpu().numpy(), want[i])
    out, n_out = B_.interp_track_batch(pts, 1.0, n_pts=npts, n_out_max=3)                      # the wrapper regrows
    assert [int(x) for x in n_out] == m and all(same(out[i, :m[i]].cpu().numpy(), want[i]) for i in range(len(names)))
    # refused: n = 1, n > n_max, a lap of zero length, a NaN point; their neighbours are their lone runs
    zero = np.tile(np.array([[3.0, 4.0, 1.0, 1.0]]), (5, 1))
    nan = rows[2].copy()
    nan[1, 0] = np.nan
    mixed = [rows[0], rows[2], zero, rows[3], nan, rows[1], rows[2]]
    pts = _pad(mixed, 140, SENTINEL)
    npts = _counts(mixed)
    npts[1], npts[6] = 1, 141
    out, n_out = B_.interp_track_batch(pts, 1.0, n_pts=npts)
    assert [int(x) for x in n_out] == [m[0], 0, 0, m[3], 0, m[1], 0]
    for i, k in ((0, 0), (3, 3), (5, 1)):
        assert same(out[i, :m[k]].cpu().numpy(), want[k])


def _mb_cases(edges):
    return [dict(tag=str(edges[f"mb_{i}_tag"]), xy=edges[f"mb_{i}_xy"], psi=edges[f"mb_{i}_psi"], bounds=edges[f"mb_{i}_bounds"],
                 splits=edges[f"mb_{i}_splits"], out=edges[f"mb_{i}_out"], veh=edges[f"mb_{i}_veh"])
            for i in range(int(edges["mb_count"]))]


def _mb_batch(cases, split_of, pad=0, fill=SENTINEL, veh=None):
    """min_bound_dists_batch of the cases in one ragged batch, case c split at split_of(c); padding filled with fill"""
    b1 = [c["bounds"][:split_of(c)] for c in cases]
    b2 = [c["bounds"][split_of(c):] for c in cases]
    nb1_max, nb2_max = max(1, max(len(b) for b in b1)) + pad, max(1, max(len(b) for b in b2)) + pad
    b1t = _pad([b if len(b) else np.zeros((0, 2)) for b in b1], nb1_max, fill) if any(len(b) for b in b1) else \
        torch.full((len(cases), nb1_max, 2), fill, dtype=torch.float64, device=DEV)
    b2t = _pad([b if len(b) else np.zeros((0, 2)) for b in b2], nb2_max, fill) if any(len(b) for b in b2) else \
        torch.full((len(cases), nb2_max, 2), fill, dtype=torch.float64, device=DEV)
    xy, psi = _pad([c["xy"] for c in cases], None, fill), _pad([c["psi"] for c in cases], None, fill)
    length, width = veh if veh is not None else (float(cases[0]["veh"][0]), float(cases[0]["veh"][1]))
    return B_.min_bound_dists_batch(xy, psi, b1t, b2t, length, width, n_traj=_counts([c["xy"] for c in cases]),
                                    nb1=_counts(b1), nb2=_counts(b2)).cpu().numpy()


def test_min_bound_dists_psi0_bit_for_bit_under_any_split_and_padding(edges):
    """Every psi = 0 case (tile edges at 511 / 512 / 513 / 1024 / 1025 / 1537 boundary points, the nearest point at each
    tile slot, 1 to 257 trajectory points so that whole CTAs lie beyond short tracks, NaN points) in one ragged batch, for
    every split of the boundary points between the sides and with extra padding: bit for bit the reference."""
    cases = [c for c in _mb_cases(edges) if not c["psi"].any() and c["veh"][0] == 4.7]
    for j in range(max(len(c["splits"]) for c in cases)):
        split_of = lambda c: int(c["splits"][min(j, len(c["splits"]) - 1)])        # noqa: E731
        for pad in (0, 37):
            got = _mb_batch(cases, split_of, pad)
            for i, c in enumerate(cases):
                n = c["xy"].shape[0]
                assert same(got[i, :n], c["out"][min(j, len(c["splits"]) - 1)]), (c["tag"], j, pad)
    z = [c for c in _mb_cases(edges) if c["tag"] == "zero_vehicle"]
    for s in z[0]["splits"]:
        got = _mb_batch(z, lambda c: int(s), veh=(0.0, 0.0))
        assert same(got[0], z[0]["out"][list(z[0]["splits"]).index(s)])


def test_min_bound_dists_rotated_within_the_sin_cos_bound(edges):
    """psi = +-pi/2, +-pi, 3 and mixed headings.  The device's cos/sin are within 2 ulp (CUDA C Programming Guide,
    double-precision functions), the reference's libm within 1, so each of c, s differs by at most 3 * 2^-53.  A corner
    x + (c ox - s oy) then moves by at most (|ox| + |oy|) 3 * 2^-53 before the add, plus one ulp of the coordinate after
    it (the rounded sum can land on the neighbouring double); both coordinates of a corner move, so its distance to any
    boundary point moves by at most sqrt(2) times that, and so does the minimum (1-Lipschitz).  The differences, squares,
    sum and sqrt round differently on the two sides: at most 4 ulp of the distance.  Measured on an H100: printed below, a small fraction of the bound."""
    worst = 0.0
    for c in (c for c in _mb_cases(edges) if c["psi"].any()):
        got = _mb_batch([c], lambda c: int(c["splits"][0]))[0]
        want = c["out"][0]
        x = float(np.abs(c["xy"]).max()) + float(c["veh"].sum())
        bound = np.sqrt(2.0) * (float(c["veh"].sum()) / 2 * 3 * 2.0 ** -53 + np.spacing(x)) + 4 * np.spacing(want)
        err = np.abs(got - want)
        assert np.all(err <= bound), (c["tag"], float(err.max()))
        worst = max(worst, float(err.max()))
    print(f"min_bound_dists, rotated corners: max |device - reference| = {worst:.3e} m")


def test_min_bound_dists_per_track_vehicle_is_the_scalar_call(edges):
    cases = [c for c in _mb_cases(edges) if c["tag"] in ("spread", "psi_mixed", "nb1537_k513", "nb513_k512")]
    sizes = [(4.7, 2.0), (0.0, 0.0), (5.5, 1.2), (3.0, 3.0)]
    split_of = lambda c: int(c["splits"][len(c["splits"]) // 2])                  # noqa: E731  (both sides non-empty)
    got = _mb_batch(cases, split_of, veh=(torch.tensor([s[0] for s in sizes], dtype=torch.float64),
                                                  torch.tensor([s[1] for s in sizes], dtype=torch.float64)))
    for i, c in enumerate(cases):
        n = c["xy"].shape[0]
        assert same(got[i, :n], _mb_batch([c], split_of, veh=sizes[i])[0]), c["tag"]


def test_traj_extrema_every_size_bit_for_bit(edges):
    v_max, length, width, mass, drag, curvlim = (float(x) for x in edges["ct_veh"])
    names = [str(n) for n in edges["ct_names"]]
    trs = [edges[f"ct_{n}"] for n in names]
    mds = []
    for t in trs:
        md = np.abs(t[:, 1]).copy()
        mds.append(md)
    mds[names.index("nan_vx")][3] = np.nan                                           # a NaN distance too
    n_max = max(t.shape[0] for t in trs) + 5
    col = lambda c: _pad([t[:, c] for t in trs], n_max, SENTINEL)                    # noqa: E731
    ntr = _counts(trs)
    ext = B_.traj_extrema_batch(col(4), col(5), col(6), drag, mass, min_dists=_pad(mds, n_max, SENTINEL), n_traj=ntr).cpu().numpy()
    for i, t in enumerate(trs):
        assert same(ext[i], E.reference_extrema(t[:, 4], t[:, 5], t[:, 6], mds[i], drag, mass)), names[i]
    # per-track drag and mass are the scalar calls; a device mass <= 0 refuses its track alone, a host one raises
    drags = torch.tensor([0.75, 0.0, 1.3, 0.75, 2.0, 0.5, 0.75, 0.9, 0.1][:len(trs)], dtype=torch.float64)
    masses = torch.tensor([1200.0, 800.0, 1500.0, 1e4, 950.0, 1200.0, 700.0, 1100.0, 2000.0][:len(trs)], dtype=torch.float64)
    per = B_.traj_extrema_batch(col(4), col(5), col(6), drags, masses, n_traj=ntr).cpu().numpy()
    for i, t in enumerate(trs):
        assert same(per[i], E.reference_extrema(t[:, 4], t[:, 5], t[:, 6], None, float(drags[i]), float(masses[i])))
    bad = masses.clone()
    bad[2] = 0.0
    ref = B_.traj_extrema_batch(col(4), col(5), col(6), drags.to(DEV), bad.to(DEV), n_traj=ntr).cpu().numpy()
    assert np.isnan(ref[2, :7]).all() and ref[2, 7] == trs[2].shape[0]
    assert same(np.delete(ref, 2, axis=0), np.delete(per, 2, axis=0))
    with pytest.raises(ValueError, match="mass_veh"):
        B_.traj_extrema_batch(col(4), col(5), col(6), drags, bad, n_traj=ntr)


def test_assemble_trajectory_thousands_of_splines():
    rng = np.random.default_rng(7)
    n_spl = [3000, 1, 2048, 4097]
    n_tr = [50, 1, 17, 300]
    spl = [rng.uniform(0.1, 3.0, k) for k in n_spl]
    spl[2][::5] *= 1e6                                                # magnitudes that make the order show
    trs = [rng.uniform(-100.0, 100.0, (k, 7)) for k in n_tr]
    n_max = max(n_tr) + 4
    col = lambda c: _pad([t[:, c] for t in trs], n_max, SENTINEL)                   # noqa: E731
    xy = _pad([t[:, 1:3] for t in trs], n_max, SENTINEL)
    out = B_.assemble_trajectory_batch(col(0), xy, col(3), col(4), col(5), col(6), _pad(spl, max(n_spl) + 9, SENTINEL),
                                       n_traj=_counts(trs), n_spl=_counts(spl)).cpu().numpy()
    for i, t in enumerate(trs):
        acc = 0.0
        for v in spl[i]:
            acc += float(v)                                                       # left to right
        n = n_tr[i]
        assert same(out[i, :n], t) and same(out[i, n, 1:], t[0, 1:]) and same(out[i, n, 0], acc)
        assert abs(acc - np.sum(spl[i])) <= n_spl[i] * np.spacing(acc)
        assert not out[i, n + 1:].any()                                           # rows beyond stay untouched


def test_normals_crossing_constructed_cases():
    from oracle import tph_prep
    pairs = E.normals_pairs()
    tracks = [E.pair_track(c) for c in pairs]
    rings = [(12, (11, 0), 1), (12, (5, 6), 1), (12, None, 1), (12, (11, 1), 1), (12, (11, 1), 2), (9, (0, 4), 8),
             (9, (0, 4), 3)]
    for h in (1, 2, 8):
        rows = [t for t in tracks] + [E.ring_track(n, p) for n, p, hz in rings if hz == h]
        rows = [r for r in rows if r[0].shape[0] > h]
        track, nv = _pad([r[0] for r in rows], 13, SENTINEL), _pad([r[1] for r in rows], 13, SENTINEL)
        with contextlib.redirect_stdout(io.StringIO()):
            want = [tph_prep.check_normals_crossing(r[0], r[1], h) for r in rows]
        got = B_.check_normals_crossing_batch(track, nv, h, n_pts=_counts([r[0] for r in rows])).cpu().tolist()
        assert got == want, h
    for c, (t, _) in zip(pairs, tracks):
        assert bool(c["expect"] & (1 << 6)) == tph_prep.check_normals_crossing(t, E.pair_track(c)[1], 1)
    # n_pts == horizon + 1 in a ragged batch: the crossing pair of the 9-point ring is only reached with horizon 8
    rows = [E.ring_track(9, (0, 4)), E.ring_track(12, (11, 0)), E.ring_track(12, None)]
    track, nv = _pad([r[0] for r in rows], 12, SENTINEL), _pad([r[1] for r in rows], 12, SENTINEL)
    assert B_.check_normals_crossing_batch(track, nv, 8, n_pts=_counts([r[0] for r in rows])).cpu().tolist() == \
        [True, True, False]


@pytest.mark.parametrize("tag", ["stock", "tight"])
def test_single_track_check_traj_prints_what_the_reference_prints(edges, tag):
    v_max, length, width, mass, drag, curvlim = (float(x) for x in edges["ct_veh"])
    kw = dict(v_max=v_max, curvlim=curvlim, ggv=edges["ct_ggv"], ax_max_machines=edges["ct_ax_max_machines"])
    if tag == "tight":
        kw = dict(v_max=float(edges["ct_tight_v_max"]), curvlim=float(edges["ct_tight_curvlim"]), ggv=edges["ct_tight_ggv"],
                  ax_max_machines=edges["ct_tight_ax_max_machines"])
    for name in edges["ct_names"]:
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            hf.src.check_traj.check_traj(reftrack=edges["ct_reftrack"], reftrack_normvec_normalized=edges["ct_normvec"],
                                         trajectory=edges[f"ct_{name}"], length_veh=length, width_veh=width, debug=True,
                                         mass_veh=mass, dragcoeff=drag, **kw)
        assert buf.getvalue() == str(edges[f"ct_{name}_{tag}_stdout"]), name
    assert "nan" in str(edges[f"ct_nan_vx_{tag}_stdout"]) or tag == "stock"


def test_counts_beyond_the_row_refuse_their_track_alone(edges):
    cases = [c for c in _mb_cases(edges) if c["tag"] in ("spread", "nb513_k512", "nb1025_k0", "nb1537_k513")]
    split_of = lambda c: int(c["splits"][len(c["splits"]) // 2])                  # noqa: E731  (both sides non-empty)
    lone = [_mb_batch([c], split_of) for c in cases]
    b1 = [c["bounds"][:split_of(c)] for c in cases]
    b2 = [c["bounds"][split_of(c):] for c in cases]
    xy, psi = _pad([c["xy"] for c in cases], None, SENTINEL), _pad([c["psi"] for c in cases], None, SENTINEL)
    b1t, b2t = _pad(b1, None, SENTINEL), _pad(b2, None, SENTINEL)
    for which in ("n_traj", "nb1", "nb2"):
        cnt = dict(n_traj=_counts([c["xy"] for c in cases]), nb1=_counts(b1), nb2=_counts(b2))
        cap = dict(n_traj=xy.shape[1], nb1=b1t.shape[1], nb2=b2t.shape[1])[which]
        cnt[which][1] = cap + 1
        got = B_.min_bound_dists_batch(xy, psi, b1t, b2t, 4.7, 2.0, **cnt).cpu().numpy()
        assert np.isnan(got[1]).all(), which
        for i in (0, 2, 3):
            n = cases[i]["xy"].shape[0]
            assert same(got[i, :n], lone[i][0]), which
        with pytest.raises(ValueError, match=which):
            B_.min_bound_dists_batch(xy, psi, b1t, b2t, 4.7, 2.0, **{k: (v.cpu() if k == which else v) for k, v in cnt.items()})
    # the extrema: a row of NaN but for n_points
    trs = [edges[f"ct_{n}"] for n in ("n255", "n1", "kappa_zero")]
    col = lambda c: _pad([t[:, c] for t in trs], 256, SENTINEL)                      # noqa: E731
    ntr = _counts(trs)
    ntr[1] = 257
    ext = B_.traj_extrema_batch(col(4), col(5), col(6), 0.75, 1200.0, n_traj=ntr).cpu().numpy()
    assert np.isnan(ext[1, :7]).all() and ext[1, 7] == 257
    for i in (0, 2):
        t = trs[i]
        assert same(ext[i], E.reference_extrema(t[:, 4], t[:, 5], t[:, 6], None, 0.75, 1200.0))
    with pytest.raises(ValueError, match="n_traj"):
        B_.traj_extrema_batch(col(4), col(5), col(6), 0.75, 1200.0, n_traj=ntr.cpu())
    # the assembly: the track's rows stay untouched
    rng = np.random.default_rng(3)
    trs = [rng.uniform(-10.0, 10.0, (k, 7)) for k in (20, 30, 25)]
    spl = [rng.uniform(0.5, 1.5, k) for k in (20, 30, 25)]
    col = lambda c: _pad([t[:, c] for t in trs], 32, SENTINEL)                       # noqa: E731
    xy = _pad([t[:, 1:3] for t in trs], 32, SENTINEL)
    spt = _pad(spl, 31, SENTINEL)
    for which in ("n_traj", "n_spl"):
        cnt = dict(n_traj=_counts(trs), n_spl=_counts(spl))
        cnt[which][1] = 33 if which == "n_traj" else 32
        out = B_.assemble_trajectory_batch(col(0), xy, col(3), col(4), col(5), col(6), spt, **cnt).cpu().numpy()
        assert not out[1].any(), which
        for i in (0, 2):
            n = trs[i].shape[0]
            assert same(out[i, :n], trs[i]) and same(out[i, n, 0], float(np.cumsum(spl[i])[-1]))
        with pytest.raises(ValueError, match=which):
            B_.assemble_trajectory_batch(col(0), xy, col(3), col(4), col(5), col(6), spt,
                                         **{k: (v.cpu() if k == which else v) for k, v in cnt.items()})
