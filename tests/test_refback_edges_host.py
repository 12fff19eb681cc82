"""CPU tests (-m "not gpu") of the trajectory back end where its kernels change code path, against the reference's own
helpers run on constructed cases (tests/golden/refback_edges.npz, tools/make_golden_ref.py edges): the statements of
csrc/traj_check_core.cuh, compiled for the host by tests/host_harness/tc_host.cpp, reproduce every case bit for bit.

Each case also shows that it reaches its path: stations landing exactly on a cumulative distance (interp_closed's
dc[j] == d), the nearest boundary point at each position of min_bound_dists_kernel's 512-point tiles, and which pivot
branch and which inclusive width comparison decided a normals-crossing pair."""
import numpy as np
import pytest

import refback_edge_cases as E
from refback_edge_cases import ptr, same

MB_TILE = 512


@pytest.fixture(scope="module")
def tc(tmp_path_factory):
    lib = E.load_tc_host(tmp_path_factory.mktemp("tc_edges"))
    if lib is None:
        pytest.skip("g++ not available")
    return lib


@pytest.fixture(scope="module")
def edges(golden):
    return golden("refback_edges")


def _interp(tc, rt, step, n_out_max, nv=None, sign=0.0, col=2):
    out = np.zeros((max(n_out_max, 1), 4))
    m = tc.tc_host_interp_track(rt.shape[0], ptr(rt), 4, ptr(nv), sign, col, step, n_out_max, ptr(out))
    return m, out


def test_interp_track_cases_bit_for_bit(tc, edges):
    hits = {}
    for name in edges["it_names"]:
        rt, nv = np.ascontiguousarray(edges[f"it_{name}_track"]), np.ascontiguousarray(edges[f"it_{name}_normvec"])
        for i, step in enumerate(edges[f"it_{name}_steps"]):
            want = edges[f"it_{name}_{i}"]
            m, out = _interp(tc, rt, float(step), want.shape[0])
            assert m == want.shape[0] and same(out[:m], want), (name, step)
            assert _interp(tc, rt, float(step), m - 1)[0] == (-m if m > 1 else 0) or m == 1, (name, step)
            hits[(str(name), float(step))] = tc.tc_host_interp_exact_hits(rt.shape[0], ptr(rt), 4, float(step))
        for sign, col, side in ((1.0, 2, "r"), (-1.0, 3, "l")):                          # check_traj.py:50-61
            want = edges[f"it_{name}_bound_{side}"]
            m, out = _interp(tc, rt, 1.0, want.shape[0] + 2, nv, sign, col)
            assert m == want.shape[0] and same(out[:m], want), (name, side)
    # the paths: stations on the cumulative distances of exact-multiple laps (station 0 always is one), the zero-length
    # element, a step longer than the lap (one station), n = 2
    assert hits[("square10", 2.5)] == 4 and hits[("square10", 1.0)] == 4 and hits[("offset", 2.5)] == 4
    assert hits[("n2", 1.0)] == 2 and hits[("n2", 2.5)] == 2 and hits[("n3", 1.0)] == 3
    assert hits[("repeat", 1.0)] == 4                # 0, 4 (on the repeated point: the later of two equal distances), 7, 11
    assert edges["it_n2_3"].shape[0] == 1 and edges["it_ring127_3"].shape[0] == 1
    assert edges["it_ring3000_track"].shape[0] == 3000 and edges["it_ring_offset_track"][0, 0] > 9e4


def _mb_case(edges, i):
    g = lambda k: np.ascontiguousarray(edges[f"mb_{i}_{k}"])          # noqa: E731
    return dict(xy=g("xy"), psi=g("psi"), bounds=g("bounds"), splits=g("splits"), out=g("out"), veh=g("veh"),
                near=int(edges[f"mb_{i}_near"]), tag=str(edges[f"mb_{i}_tag"]))


def _host_mb(tc, c, s):
    n = c["xy"].shape[0]
    b1, b2 = np.ascontiguousarray(c["bounds"][:s]), np.ascontiguousarray(c["bounds"][s:])
    md, nearest = np.zeros(n), np.zeros(n, dtype=np.int32)
    tc.tc_host_min_bound_dists(n, ptr(c["xy"]), ptr(c["psi"]), b1.shape[0], ptr(b1) if b1.size else ptr(np.zeros(2)),
                               b2.shape[0], ptr(b2) if b2.size else ptr(np.zeros(2)), 2, float(c["veh"][0]),
                               float(c["veh"][1]), ptr(md), ptr(nearest))
    return md, nearest


def test_min_bound_dists_cases_bit_for_bit(tc, edges):
    """Every case at psi = 0, psi = +-pi/2, +-pi, 3 and mixed headings, with every split of its boundary points between
    bound1 and bound2.  The host sin/cos are the reference's (libm through math.sin/cos), so even the rotated cases
    match bit for bit; the device's are not (tests/test_gpu_refback_edges.py)."""
    tile_pos, ntraj, nbs = set(), set(), set()
    for i in range(int(edges["mb_count"])):
        c = _mb_case(edges, i)
        ntraj.add(c["xy"].shape[0])
        nbs.add(c["bounds"].shape[0])
        for j, s in enumerate(c["splits"]):
            md, nearest = _host_mb(tc, c, int(s))
            assert same(md, c["out"][j]), (c["tag"], s)
            if c["near"] >= 0:                     # the planted point decides every trajectory point: side and tile slot
                side, k = (0, c["near"]) if c["near"] < s else (1, c["near"] - s)
                assert np.all(nearest == (side << 20) + k), (c["tag"], s)
                tile_pos.add((k // MB_TILE, k % MB_TILE))
    assert {(0, 0), (0, 511), (1, 0), (1, 1), (2, 0), (2, 511)} <= tile_pos
    assert {1, 127, 128, 129, 257} <= ntraj and {1, 511, 512, 513, 1024, 1025, 1537} <= nbs
    by_tag = {str(edges[f"mb_{i}_tag"]): _mb_case(edges, i) for i in range(int(edges["mb_count"]))}
    assert np.isnan(by_tag["nan_bound"]["out"]).all()                                  # np.amin propagates NaN
    nt = by_tag["nan_traj"]["out"]
    assert np.isnan(nt[:, 5]).all() and not np.isnan(np.delete(nt, 5, axis=1)).any()
    z = by_tag["zero_vehicle"]                                       # a point car: the distance of the point itself
    d = np.sqrt(((z["xy"] - z["bounds"][z["near"]]) ** 2).sum(axis=1))
    assert same(z["out"][0], d)


def test_extrema_match_the_quantities_check_traj_forms(tc, edges):
    """traj_extrema_kernel's statements on every check_traj fixture trajectory (kappa exactly 0, all-negative ax_wo_drag,
    v = 0, 1 / 255 / 256 / 257 points, a NaN kappa, a NaN vx), with a NaN minimum distance too."""
    v_max, length, width, mass, drag, curvlim = edges["ct_veh"]
    for name in edges["ct_names"]:
        tr = edges[f"ct_{name}"]
        k, v, a = (np.ascontiguousarray(tr[:, c]) for c in (4, 5, 6))
        for md in (np.ascontiguousarray(np.abs(tr[:, 1])), None):
            e = np.zeros(8)
            tc.tc_host_extrema(k.size, ptr(k), ptr(v), ptr(a), ptr(md), drag, mass, ptr(e))
            assert same(e, E.reference_extrema(k, v, a, md, drag, mass)), name
        md = np.ascontiguousarray(np.abs(tr[:, 1]))
        md[-1] = np.nan
        tc.tc_host_extrema(k.size, ptr(k), ptr(v), ptr(a), ptr(md), drag, mass, ptr(e))
        assert np.isnan(e[0]) and same(e[1:], E.reference_extrema(k, v, a, md, drag, mass)[1:])
    e = np.zeros(8)
    tr = edges["ct_nan_kappa"]
    k, v, a = (np.ascontiguousarray(tr[:, c]) for c in (4, 5, 6))
    tc.tc_host_extrema(k.size, ptr(k), ptr(v), ptr(a), None, drag, mass, ptr(e))
    assert np.isnan(e[1]) and np.isfinite(e[2:7]).all()             # |kappa| max is NaN, ay max skips the NaN point


@pytest.mark.parametrize("c", E.normals_pairs(), ids=lambda c: c["tag"])
def test_normals_cross_pairs_take_their_branch_and_match_the_oracle(tc, c):
    from oracle import tph_prep
    info = tc.tc_host_normals_cross_info(ptr(c["p"]), ptr(c["n1"]), ptr(c["q"]), ptr(c["n2"]))
    assert info == c["expect"]
    track, nv = E.pair_track(c)
    want = tph_prep.check_normals_crossing(track, nv, 1)
    assert bool(tc.tc_host_normals_crossing(3, ptr(track), ptr(nv), 1)) == want
    assert want == bool(info & (1 << 6))


def test_normals_crossing_across_index_0_and_at_horizon_n_minus_1(tc, capsys):
    from oracle import tph_prep
    cases = [(12, (11, 0), 1, True), (12, (5, 6), 1, True), (12, None, 1, False), (12, (11, 1), 1, False),
             (12, (11, 1), 2, True), (9, (0, 4), 8, True), (9, (0, 4), 3, False)]
    for n, pair, horizon, want in cases:
        track, nv = E.ring_track(n, pair)
        assert tph_prep.check_normals_crossing(track, nv, horizon) == want
        assert bool(tc.tc_host_normals_crossing(n, ptr(track), ptr(nv), horizon)) == want, (n, pair, horizon)
    capsys.readouterr()
