"""CPU tests (-m "not gpu") of the trajectory back end (SURVEY.md 8f-3/8f-4) against fixtures produced by the reference's
OWN in-tree helpers (tests/golden/refback_*.npz, tools/make_golden_ref.py runs helper_funcs_glob/src/*.py
unmodified): this row is parity-PINNED.

* the arithmetic of the K6 kernels (csrc/traj_check_core.cuh) compiled for the host by tests/host_harness/tc_host.cpp;
* the host-side mirrors that do no device work: import_track and the two CSV exports (byte-for-byte, the random UUID
  line aside)."""
import contextlib
import ctypes
import io

import numpy as np
import pytest

from global_racetrajectory_optimization_b200 import helper_funcs_glob as hf
from refback_edge_cases import load_tc_host

DP = ctypes.POINTER(ctypes.c_double)
NAMES = ["berlin", "handling", "synth333"]


def _p(a):
    return a.ctypes.data_as(DP) if a is not None else None


@pytest.fixture(scope="module")
def tc(tmp_path_factory):
    lib = load_tc_host(tmp_path_factory.mktemp("tc_host"))
    if lib is None:
        pytest.skip("g++ not available")
    return lib


@pytest.mark.parametrize("name", NAMES)
def test_interp_track_statements_reproduce_the_reference_bit_for_bit(golden, tc, name):
    g, r = golden(name), golden("refback_" + name)
    rt, nv = np.ascontiguousarray(g["reftrack"]), np.ascontiguousarray(g["normvec"])
    for step in (1.0, 2.5):
        want = r[f"interp_track_{step}"]
        out = np.zeros((want.shape[0] + 5, 4))
        m = tc.tc_host_interp_track(rt.shape[0], _p(rt), 4, None, 0.0, 2, step, out.shape[0], _p(out))
        assert m == want.shape[0] and np.array_equal(out[:m], want)
        assert tc.tc_host_interp_track(rt.shape[0], _p(rt), 4, None, 0.0, 2, step, m - 1, _p(out)) == -m   # too small
    for sign, col, key in ((1.0, 2, "bound_r_interp"), (-1.0, 3, "bound_l_interp")):      # check_traj.py:50-61
        want = r[key]
        out = np.zeros((want.shape[0] + 5, 4))
        m = tc.tc_host_interp_track(rt.shape[0], _p(rt), 4, _p(nv), sign, col, 1.0, out.shape[0], _p(out))
        assert m == want.shape[0] and np.array_equal(out[:m], want)


@pytest.mark.parametrize("name", NAMES)
def test_min_bound_dists_and_extrema_statements_reproduce_the_reference(golden, tc, name):
    r = golden("refback_" + name)
    tr = r["trajectory_opt"]
    xy, psi = np.ascontiguousarray(tr[:, 1:3]), np.ascontiguousarray(tr[:, 3])
    br, bl = np.ascontiguousarray(r["bound_r_interp"]), np.ascontiguousarray(r["bound_l_interp"])
    md = np.zeros(tr.shape[0])
    tc.tc_host_min_bound_dists(tr.shape[0], _p(xy), _p(psi), br.shape[0], _p(br), bl.shape[0], _p(bl), 4,
                               float(r["length_veh"]), float(r["width_veh"]), _p(md), None)
    assert np.abs(md - r["min_dists_full"]).max() <= 1e-12
    b1, b2 = np.ascontiguousarray(br[:1]), np.ascontiguousarray(bl[:1])                     # what check_traj.py:58-68 passes
    tc.tc_host_min_bound_dists(tr.shape[0], _p(xy), _p(psi), 1, _p(b1), 1, _p(b2), 4, float(r["length_veh"]),
                               float(r["width_veh"]), _p(md), None)
    assert np.abs(md - r["min_dists_as_called"]).max() <= 1e-12
    # the quantities of check_traj.py:93-131, formed exactly like the reference forms them
    k, v, a = (np.ascontiguousarray(tr[:, c]) for c in (4, 5, 6))
    e = np.zeros(8)
    tc.tc_host_extrema(tr.shape[0], _p(k), _p(v), _p(a), _p(md), float(r["dragcoeff"]), float(r["mass"]), _p(e))
    radii = np.abs(np.divide(1.0, k, out=np.full(k.size, np.inf), where=k != 0))
    ay = np.divide(np.power(v, 2), radii)
    ax_wo = a - (-np.power(v, 2) * float(r["dragcoeff"]) / float(r["mass"]))
    want = [md.min(), np.abs(k).max(), ay.max(), ax_wo.max(), ax_wo.min(), np.sqrt(np.power(ax_wo, 2) + np.power(ay, 2)).max(),
            v.max(), k.size]
    assert np.array_equal(e, np.array(want))


def test_import_track_matches_the_reference(golden, tmp_path):
    g = golden("refback_import_track")
    for csv in ("berlin_2018", "handling_track", "rounded_rectangle"):
        o = g[csv + "_opts"]
        opts = dict(flip_imp_track=bool(o[0]), set_new_start=bool(o[1]), new_start=np.array([o[2], o[3]]), num_laps=int(o[4]))
        path = tmp_path / (csv + ".csv")
        path.write_bytes(g[csv + "_csv"].tobytes())
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            track = hf.src.import_track.import_track(file_path=str(path), imp_opts=opts, width_veh=2.0)
        assert np.array_equal(track, g[csv]) and buf.getvalue() == str(g[csv + "_stdout"])
    bad = tmp_path / "bad.csv"
    bad.write_text("1.0,2.0\n3.0,4.0\n")
    with pytest.raises(IOError, match="cannot be read"):
        hf.src.import_track.import_track(str(bad), dict(flip_imp_track=False, set_new_start=False, new_start=None, num_laps=1), 2.0)
    narrow = tmp_path / "narrow.csv"
    narrow.write_text("0.0,0.0,2.2\n1.0,0.0,2.2\n1.0,1.0,2.2\n")
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        hf.src.import_track.import_track(str(narrow), dict(flip_imp_track=False, set_new_start=False, new_start=None, num_laps=1), 2.0)
    assert buf.getvalue() == "WARNING: Minimum track width 2.20m is close to or smaller than vehicle width!\n"


@pytest.mark.parametrize("name", NAMES)
def test_exports_are_byte_identical_to_the_reference(golden, tmp_path, name):
    g, r = golden(name), golden("refback_" + name)
    ggv_path = tmp_path / "ggv.csv"
    ggv_path.write_bytes(r["ggv_file_bytes"].tobytes())
    fp = dict(ggv_file=str(ggv_path), traj_race_export=str(tmp_path / "race.csv"), traj_ltpl_export=str(tmp_path / "ltpl.csv"))
    hf.src.export_traj_race.export_traj_race(file_paths=fp, traj_race=r["traj_race_cl"])
    hf.src.export_traj_ltpl.export_traj_ltpl(file_paths=fp, spline_lengths_opt=g["rl_spline_lengths"],
                                             trajectory_opt=r["trajectory_opt"], reftrack=g["reftrack"],
                                             normvec_normalized=g["normvec"], alpha_opt=g["alpha_mincurv"])
    for key in ("traj_race_export", "traj_ltpl_export"):
        first, rest = open(fp[key]).read().split("\n", 1)
        want = str(r[key])
        assert len(first) == 2 + 36 and first.startswith("# ")                       # "# " + uuid4
        assert rest[:len(want)] == want and (name == "berlin" or len(rest) == len(want))
    fp2 = dict(traj_race_export=str(tmp_path / "race2.csv"))                       # no ggv file: SHA1 of an empty buffer
    hf.src.export_traj_race.export_traj_race(file_paths=fp2, traj_race=r["traj_race_cl"][:3])
    assert open(fp2["traj_race_export"]).read().split("\n", 1)[1] == str(r["traj_race_export_noggv"])


def test_normals_crossing_statements_match_the_oracle(golden, tc):
    """tph.check_normals_crossing is NOT in the reference tree (parity unpinned, oracle/tph_prep.py); the kernel's
    statements are compared with that restatement on the fixtures with widened tracks (crossings appear from ~2x)."""
    from oracle import tph_prep
    positives = 0
    for name in ("berlin", "handling", "synth333", "synth200"):
        g = golden(name)
        nv = np.ascontiguousarray(g["normvec"])
        for scale in (1.0, 1.5, 2.0, 3.0, 4.0):
            for horizon in (3, 10, 25):
                rt = np.ascontiguousarray(g["reftrack"].copy())
                rt[:, 2:] *= scale
                want = tph_prep.check_normals_crossing(rt, nv, horizon)
                assert bool(tc.tc_host_normals_crossing(rt.shape[0], _p(rt), _p(nv), horizon)) == want
                positives += want
    assert 10 < positives < 60                                   # both outcomes are exercised
    with pytest.raises(RuntimeError, match="too large"):
        tph_prep.check_normals_crossing(np.zeros((8, 4)), np.zeros((8, 2)), 10)
