"""Generates tests/golden/refback_*.npz by executing the UNMODIFIED in-tree reference helpers

    helper_funcs_glob/src/interp_track.py          interp_track
    helper_funcs_glob/src/calc_min_bound_dists.py  calc_min_bound_dists
    helper_funcs_glob/src/check_traj.py            check_traj   (stdout captured)
    helper_funcs_glob/src/export_traj_race.py      export_traj_race
    helper_funcs_glob/src/export_traj_ltpl.py      export_traj_ltpl
    helper_funcs_glob/src/import_track.py          import_track

imported from a checkout of the reference (MC_REFERENCE_DIR) -- so, unlike the tph-based rows, the fixtures of this row are
PINNED to the reference's own code.  The package's __init__ also imports prep_track / result_plots, which need
trajectory_planning_helpers and matplotlib (absent offline); both are stubbed with empty modules -- none of the functions
executed here touches them.

Inputs: the raceline of the committed fixtures (tests/golden/<name>.npz, made by tools/make_golden.py) with the velocity
profile of oracle/tph_velprofile.py, assembled into the trajectory array exactly like
the reference's main_globaltraj.py:501-512.

    MC_REFERENCE_DIR=<reference checkout> python tools/make_golden_ref.py [edges]

With ``edges`` only tests/golden/refback_edges.npz is written: constructed cases where the K6 kernels change code path
(see edges() below), each run through the same unmodified helpers.
"""
from __future__ import annotations

import contextlib
import io
import os
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("MC_REFERENCE_DIR", "")
GOLD = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)


def load_reference_helpers():
    for name in ("trajectory_planning_helpers", "matplotlib", "matplotlib.pyplot", "mpl_toolkits", "mpl_toolkits.mplot3d"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
    sys.modules["mpl_toolkits.mplot3d"].Axes3D = object
    if not os.path.isdir(os.path.join(REF, "helper_funcs_glob")):
        raise SystemExit("set MC_REFERENCE_DIR to a checkout of the reference")
    sys.path.insert(0, REF)
    import helper_funcs_glob  # noqa: E402  (the reference's own package)
    return helper_funcs_glob


def main():
    hf = load_reference_helpers()
    from oracle import tph_velprofile as VP
    ggv_file = os.path.join(REF, "inputs", "veh_dyn_info", "ggv.csv")
    ggv, axm = VP.import_veh_dyn_info(ggv_file, os.path.join(REF, "inputs", "veh_dyn_info", "ax_max_machines.csv"))
    veh = dict(v_max=70.0, length=4.7, width=2.0, mass=1200.0, dragcoeff=0.75, curvlim=0.12)   # params/racecar.ini:44-50
    for name in ("berlin", "handling", "synth333"):
        g = np.load(os.path.join(GOLD, name + ".npz"))
        rt, nv, alpha = g["reftrack"], g["normvec"], g["alpha_mincurv"]
        kappa, el = g["rl_kappa"], g["rl_el_lengths"]
        vx = VP.calc_vel_profile(ggv=ggv, ax_max_machines=axm, v_max=veh["v_max"], kappa=kappa, el_lengths=el, closed=True,
                                 drag_coeff=veh["dragcoeff"], m_veh=veh["mass"])
        ax = VP.calc_ax_profile(np.append(vx, vx[0]), el)
        # main_globaltraj.py:501-512
        trajectory_opt = np.column_stack((g["rl_s"], g["rl_raceline_interp"], g["rl_psi"], kappa, vx, ax))
        spline_data_opt = np.column_stack((g["rl_spline_lengths"], g["rl_coeffs_x"], g["rl_coeffs_y"]))
        traj_race_cl = np.vstack((trajectory_opt, trajectory_opt[0, :]))
        traj_race_cl[-1, 0] = np.sum(spline_data_opt[:, 0])
        out = dict(trajectory_opt=trajectory_opt, traj_race_cl=traj_race_cl, length_veh=veh["length"], width_veh=veh["width"],
                   v_max=veh["v_max"], dragcoeff=veh["dragcoeff"], mass=veh["mass"], curvlim=veh["curvlim"],
                   ggv=ggv, ax_max_machines=axm)
        # interp_track on the reftrack itself (prep_track.py:32-34 uses it on the imported track) and on the bounds
        for step in (1.0, 2.5):
            out[f"interp_track_{step}"] = hf.src.interp_track.interp_track(reftrack=rt, stepsize_approx=step)
        bound_r = rt[:, :2] + nv * np.expand_dims(rt[:, 2], 1)
        bound_l = rt[:, :2] - nv * np.expand_dims(rt[:, 3], 1)
        br = hf.src.interp_track.interp_track(np.column_stack((bound_r, np.zeros((rt.shape[0], 2)))), 1.0)
        bl = hf.src.interp_track.interp_track(np.column_stack((bound_l, np.zeros((rt.shape[0], 2)))), 1.0)
        out.update(bound_r_interp=br, bound_l_interp=bl)
        # calc_min_bound_dists against the full interpolated boundaries (what check_traj intends) ...
        out["min_dists_full"] = hf.src.calc_min_bound_dists.calc_min_bound_dists(
            trajectory=trajectory_opt, bound1=br, bound2=bl, length_veh=veh["length"], width_veh=veh["width"])
        # ... and what check_traj.py:58-69 actually passes: interp_track(...)[0], i.e. the FIRST point of each boundary
        out["min_dists_as_called"] = hf.src.calc_min_bound_dists.calc_min_bound_dists(
            trajectory=trajectory_opt, bound1=br[0], bound2=bl[0], length_veh=veh["length"], width_veh=veh["width"])
        # check_traj: messages + returned boundaries, for the stock car and for limits that trigger every warning
        for tag, kw in (("stock", {}), ("tight", dict(v_max=30.0, curvlim=0.05, ggv=ggv * np.array([1.0, 0.5, 0.5]),
                                                      ax_max_machines=axm * np.array([1.0, 0.5])))):
            args = dict(reftrack=rt, reftrack_normvec_normalized=nv, length_veh=veh["length"], width_veh=veh["width"],
                        debug=True, trajectory=trajectory_opt, ggv=ggv, ax_max_machines=axm, v_max=veh["v_max"],
                        curvlim=veh["curvlim"], mass_veh=veh["mass"], dragcoeff=veh["dragcoeff"])
            args.update(kw)
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf):
                b1, b2 = hf.src.check_traj.check_traj(**args)
            out[f"check_traj_{tag}_stdout"] = np.array(buf.getvalue())
            out[f"check_traj_{tag}_bound_r"], out[f"check_traj_{tag}_bound_l"] = b1, b2
            if kw:
                out["tight_ggv"], out["tight_ax_max_machines"], out["tight_v_max"], out["tight_curvlim"] = \
                    kw["ggv"], kw["ax_max_machines"], kw["v_max"], kw["curvlim"]
        # exports (first line = random UUID, dropped; second line = SHA1 of the ggv file)
        with tempfile.TemporaryDirectory() as d:
            fp = dict(ggv_file=ggv_file, traj_race_export=os.path.join(d, "race.csv"), traj_ltpl_export=os.path.join(d, "ltpl.csv"))
            hf.src.export_traj_race.export_traj_race(file_paths=fp, traj_race=traj_race_cl)
            hf.src.export_traj_ltpl.export_traj_ltpl(file_paths=fp, spline_lengths_opt=g["rl_spline_lengths"],
                                                     trajectory_opt=trajectory_opt, reftrack=rt, normvec_normalized=nv,
                                                     alpha_opt=alpha)
            for key in ("traj_race_export", "traj_ltpl_export"):
                txt = open(fp[key]).read().split("\n", 1)[1]
                out[key] = np.array(txt if name != "berlin" else txt[:20000])       # keep the fixture small
            fp2 = dict(traj_race_export=os.path.join(d, "race2.csv"))                # no ggv file: hash of an empty array
            hf.src.export_traj_race.export_traj_race(file_paths=fp2, traj_race=traj_race_cl[:3])
            out["traj_race_export_noggv"] = np.array(open(fp2["traj_race_export"]).read().split("\n", 1)[1])
        out["ggv_file_bytes"] = np.frombuffer(open(ggv_file, "rb").read(), dtype=np.uint8)
        np.savez_compressed(os.path.join(GOLD, f"refback_{name}.npz"), **out)
        print(f"  refback_{name}: traj {trajectory_opt.shape}, bounds {br.shape[0]}+{bl.shape[0]} points, "
              f"min dist full {out['min_dists_full'].min():.3f} m / as called {out['min_dists_as_called'].min():.3f} m")
        print("   ", str(out["check_traj_stock_stdout"]).strip().replace("\n", "\n    "))
        print("   ", str(out["check_traj_tight_stdout"]).strip().replace("\n", "\n    "))
    # import_track on the reference's own CSVs (3-, 4-column forms; flip / new start / laps options)
    imp = {}
    for csv, opts in (("berlin_2018", dict(flip_imp_track=False, set_new_start=False, new_start=np.array([0.0, -47.0]), num_laps=1)),
                      ("handling_track", dict(flip_imp_track=True, set_new_start=True, new_start=np.array([0.0, -47.0]), num_laps=2)),
                      ("rounded_rectangle", dict(flip_imp_track=False, set_new_start=True, new_start=np.array([10.0, 5.0]), num_laps=1)),
                      ("modena_2019", dict(flip_imp_track=False, set_new_start=False, new_start=np.array([0.0, 0.0]), num_laps=1))):
        path = os.path.join(REF, "inputs", "tracks", csv + ".csv")
        buf = io.StringIO()
        with contextlib.redirect_stdout(buf):
            imp[csv] = hf.src.import_track.import_track(file_path=path, imp_opts=opts, width_veh=2.0)
        imp[csv + "_csv"] = np.frombuffer(open(path, "rb").read(), dtype=np.uint8)
        imp[csv + "_stdout"] = np.array(buf.getvalue())
        imp[csv + "_opts"] = np.array([float(opts["flip_imp_track"]), float(opts["set_new_start"]), opts["new_start"][0],
                                       opts["new_start"][1], float(opts["num_laps"])])
        print(f"  import_track {csv}: {imp[csv].shape}")
    np.savez_compressed(os.path.join(GOLD, "refback_import_track.npz"), **imp)


def _normals(xy):
    """Unit normals (tangent of the neighbours turned right) of a closed polyline; any unit vectors would do."""
    t = np.roll(xy, -1, axis=0) - np.roll(xy, 1, axis=0)
    for alt in (np.roll(xy, -1, axis=0) - xy, xy - np.roll(xy, 1, axis=0)):     # 2 points, repeated points
        t = np.where(np.all(t == 0.0, axis=1)[:, None], alt, t)
    n = np.column_stack((t[:, 1], -t[:, 0]))
    return n / np.sqrt(np.sum(n * n, axis=1))[:, None]


def _ring(rng, n, r, jitter, smooth=False):
    """n points around a circle of radius r (radius jittered by a factor up to 1 +- jitter), random widths 1 .. 3 m (with
    smooth, the same at every point, so that the boundaries stay as short as the ring)"""
    ang = 2.0 * np.pi * np.arange(n) / n
    rad = r * (1.0 + jitter * rng.uniform(-1.0, 1.0, n))
    xy = np.round(np.column_stack((rad * np.cos(ang), rad * np.sin(ang))) * 4096.0) / 4096.0    # (a smaller fixture)
    w = np.round(rng.uniform(1.0, 3.0, (1 if smooth else n, 2)) * 64.0) / 64.0
    return np.column_stack((xy, np.broadcast_to(w, (n, 2))))


IT_STEPS = (1.0, 2.5, 0.1 / 3)


def edge_interp_tracks(rng):
    """name -> (track [n, 4], its steps: IT_STEPS, and a step longer than the lap for some)"""
    sq = np.array([[0.0, 0.0, 1.0, 2.0], [10.0, 0.0, 1.5, 1.0], [10.0, 10.0, 2.0, 1.5], [0.0, 10.0, 1.0, 1.0]])
    return {
        "n2": (np.array([[0.0, 0.0, 1.0, 2.0], [3.0, 4.0, 1.5, 2.5]]), IT_STEPS + (1000.0,)),          # lap 10 m: multiples of 1, 2.5
        "n3": (np.array([[0.0, 0.0, 1.0, 1.0], [4.0, 0.0, 1.2, 0.8], [0.0, 3.0, 0.9, 1.1]]), IT_STEPS),  # lap 12 m
        "ring127": (_ring(rng, 127, 3.0, 0.1), IT_STEPS + (1000.0,)),
        "ring128": (_ring(rng, 128, 3.0, 0.1), IT_STEPS),
        "ring129": (_ring(rng, 129, 3.0, 0.1), IT_STEPS),
        "ring3000": (_ring(rng, 3000, 20.0, 0.0, smooth=True) , (1.0, 2.5, 0.7)),        # lap ~126 m
        "square10": (sq, IT_STEPS),                                                               # lap 40 m
        "repeat": (np.array([[0.0, 0.0, 1.0, 1.0], [4.0, 0.0, 1.0, 1.0], [4.0, 0.0, 2.0, 3.0], [4.0, 3.0, 1.5, 1.0],
                             [0.0, 3.0, 1.0, 2.0]]), IT_STEPS),                             # zero-length element
        "offset": (sq + np.array([1e5, 1e5, 0.0, 0.0]), IT_STEPS),
        "ring_offset": (_ring(rng, 16, 3.0, 0.1) + np.array([1e5, -1e5, 0.0, 0.0]), IT_STEPS),
    }


MB_SIZES = (1, 511, 512, 513, 1024, 1025, 1537)
MB_NTRAJ = (1, 127, 128, 129, 257)
MB_PSI = {"p_half_pi": np.pi / 2, "m_half_pi": -np.pi / 2, "p_pi": np.pi, "m_pi": -np.pi, "three": 3.0}


def edge_min_bound_dists_cases(rng):
    """list of dicts: xy [n, 2], psi [n], bounds [nb, 2] (split into bound1 = bounds[:s], bound2 = bounds[s:] for every s
    in splits), length, width, near (index of the planted nearest boundary point, -1 for none)."""
    ang = 2.0 * np.pi * np.arange(1537) / 1537
    base = np.round(np.column_stack((60.0 * np.cos(ang), 60.0 * np.sin(ang))) * 64.0) / 64.0     # far from the car
    near = np.array([0.15625, 0.3125])                                  # closer to every corner than any base point
    cases, c = [], 0
    for nb in MB_SIZES:
        for k in sorted({0, 511, 512, 513, nb - 1} & set(range(nb))):
            n = MB_NTRAJ[c % len(MB_NTRAJ)]
            c += 1
            b = base[:nb].copy()
            b[k] = near
            cases.append(dict(tag=f"nb{nb}_k{k}", xy=np.round(rng.uniform(-0.5, 0.5, (n, 2)) * 256.0) / 256.0,
                              psi=np.zeros(n), bounds=b, length=4.7, width=2.0, near=k,
                              splits=sorted({nb, nb // 2, 1, min(512, nb), 0} & set(range(nb + 1)))))
    b = base[:1025].copy()
    b[700] = near
    for tag, psi in MB_PSI.items():
        cases.append(dict(tag="psi_" + tag, xy=rng.uniform(-0.5, 0.5, (257, 2)), psi=np.full(257, psi), bounds=b,
                          length=4.7, width=2.0, near=700, splits=[600]))
    cases.append(dict(tag="psi_mixed", xy=rng.uniform(-40.0, 40.0, (257, 2)), psi=rng.uniform(-np.pi, np.pi, 257),
                      bounds=base, length=4.7, width=2.0, near=-1, splits=[768]))
    cases.append(dict(tag="spread", xy=np.round(rng.uniform(-50.0, 50.0, (257, 2)) * 256.0) / 256.0, psi=np.zeros(257),
                      bounds=base, length=4.7, width=2.0, near=-1, splits=[0, 511, 1025, 1537]))
    b = base[:513].copy()
    b[512] = near
    cases.append(dict(tag="zero_vehicle", xy=np.round(rng.uniform(-0.5, 0.5, (129, 2)) * 256.0) / 256.0, psi=np.zeros(129),
                      bounds=b, length=0.0, width=0.0, near=512, splits=[513, 200]))
    b = base[:513].copy()
    b[300, 0] = np.nan
    cases.append(dict(tag="nan_bound", xy=rng.uniform(-0.5, 0.5, (129, 2)), psi=np.zeros(129), bounds=b, length=4.7,
                      width=2.0, near=-1, splits=[513, 300, 301]))
    xy = rng.uniform(-0.5, 0.5, (128, 2))
    xy[5, 1] = np.nan
    cases.append(dict(tag="nan_traj", xy=xy, psi=np.zeros(128), bounds=base[:1024], length=4.7, width=2.0, near=-1,
                      splits=[1024, 512]))
    return cases


def edge_check_traj_cases(rng):
    """(reftrack, normvec, name -> trajectory [n, 7]): trajectories along a 30 m circle inside the reftrack's corridor."""
    rt = _ring(rng, 40, 30.0, 0.0)
    rt[:, 2:] = rng.uniform(3.0, 4.0, (40, 2))
    nv = _normals(rt[:, :2])

    def lap(n, v_lo=20.0, v_hi=40.0):
        a = 2.0 * np.pi * np.arange(n) / max(n, 1)
        s = 30.0 * a
        return np.column_stack((s, 30.0 * np.cos(a), 30.0 * np.sin(a), a + np.pi / 2, np.full(n, 1.0 / 30.0),
                                rng.uniform(v_lo, v_hi, n), rng.uniform(-8.0, 6.0, n)))

    tr = {}
    t = lap(100)
    t[::7, 4] = 0.0                                                     # kappa exactly 0: radius inf, ay 0
    tr["kappa_zero"] = t
    t = lap(100)
    t[:, 6] = rng.uniform(-12.0, -2.0, 100)                             # ax_wo_drag < 0 everywhere
    tr["ax_negative"] = t
    t = lap(100)
    t[:, 5] = 0.0
    t[::3, 4] = 0.0                                                     # v = 0 (and 0 / inf)
    tr["v_zero"] = t
    for n in (1, 255, 256, 257):
        tr[f"n{n}"] = lap(n)
    t = lap(100)
    t[10, 4] = np.nan
    tr["nan_kappa"] = t
    t = lap(100, 20.0, 80.0)
    t[20, 5] = np.nan
    tr["nan_vx"] = t
    return rt, nv, tr


def edges():
    """tests/golden/refback_edges.npz: the reference's interp_track, calc_min_bound_dists and check_traj on constructed
    cases (tile edges, block-reduction sizes, exact-multiple laps, zero-length elements, NaN)."""
    hf = load_reference_helpers()
    from oracle import tph_velprofile as VP
    rng = np.random.default_rng(20261018)
    out = dict(numpy_version=np.array(np.__version__))
    names = []
    for name, (rt, steps) in edge_interp_tracks(rng).items():
        names.append(name)
        nv = _normals(rt[:, :2])
        out[f"it_{name}_track"], out[f"it_{name}_normvec"] = rt, nv
        out[f"it_{name}_steps"] = np.array(steps)
        for i, step in enumerate(steps):
            out[f"it_{name}_{i}"] = hf.src.interp_track.interp_track(reftrack=rt, stepsize_approx=step)
        for side, bound in (("r", rt[:, :2] + nv * np.expand_dims(rt[:, 2], 1)),          # check_traj.py:50-55
                            ("l", rt[:, :2] - nv * np.expand_dims(rt[:, 3], 1))):
            out[f"it_{name}_bound_{side}"] = hf.src.interp_track.interp_track(
                reftrack=np.column_stack((bound, np.zeros((bound.shape[0], 2)))), stepsize_approx=1.0)
    out["it_names"] = np.array(names)
    cases = edge_min_bound_dists_cases(rng)
    for i, c in enumerate(cases):
        traj = np.column_stack((np.zeros(c["xy"].shape[0]), c["xy"], c["psi"]))
        res = [hf.src.calc_min_bound_dists.calc_min_bound_dists(trajectory=traj, bound1=c["bounds"][:s],
                                                                bound2=c["bounds"][s:], length_veh=c["length"],
                                                                width_veh=c["width"]) for s in c["splits"]]
        out.update({f"mb_{i}_xy": c["xy"], f"mb_{i}_psi": c["psi"], f"mb_{i}_bounds": c["bounds"],
                    f"mb_{i}_splits": np.array(c["splits"], dtype=np.int64), f"mb_{i}_out": np.array(res),
                    f"mb_{i}_veh": np.array([c["length"], c["width"]]), f"mb_{i}_near": np.array(c["near"]),
                    f"mb_{i}_tag": np.array(c["tag"])})
    out["mb_count"] = np.array(len(cases))
    ggv_file = os.path.join(REF, "inputs", "veh_dyn_info", "ggv.csv")
    ggv, axm = VP.import_veh_dyn_info(ggv_file, os.path.join(REF, "inputs", "veh_dyn_info", "ax_max_machines.csv"))
    veh = dict(v_max=70.0, length=4.7, width=2.0, mass=1200.0, dragcoeff=0.75, curvlim=0.12)   # params/racecar.ini:44-50
    tight = dict(v_max=30.0, curvlim=0.02, ggv=ggv * np.array([1.0, 0.5, 0.5]), ax_max_machines=axm * np.array([1.0, 0.5]))
    rt, nv, trs = edge_check_traj_cases(rng)
    out.update(ct_reftrack=rt, ct_normvec=nv, ct_names=np.array(list(trs)), ct_ggv=ggv, ct_ax_max_machines=axm,
               ct_veh=np.array([veh[k] for k in ("v_max", "length", "width", "mass", "dragcoeff", "curvlim")]),
               ct_tight_ggv=tight["ggv"], ct_tight_ax_max_machines=tight["ax_max_machines"],
               ct_tight_v_max=np.array(tight["v_max"]), ct_tight_curvlim=np.array(tight["curvlim"]))
    for name, tr in trs.items():
        out[f"ct_{name}"] = tr
        for tag, kw in (("stock", {}), ("tight", tight)):
            args = dict(reftrack=rt, reftrack_normvec_normalized=nv, length_veh=veh["length"], width_veh=veh["width"],
                        debug=True, trajectory=tr, ggv=ggv, ax_max_machines=axm, v_max=veh["v_max"],
                        curvlim=veh["curvlim"], mass_veh=veh["mass"], dragcoeff=veh["dragcoeff"])
            args.update(kw)
            buf = io.StringIO()
            with contextlib.redirect_stdout(buf), np.errstate(all="ignore"):
                hf.src.check_traj.check_traj(**args)
            out[f"ct_{name}_{tag}_stdout"] = np.array(buf.getvalue())
    path = os.path.join(GOLD, "refback_edges.npz")
    np.savez_compressed(path, **out)
    print(f"  refback_edges: {len(names)} interp_track tracks, {len(cases)} calc_min_bound_dists cases, {len(trs)} "
          f"check_traj trajectories, {os.path.getsize(path)} bytes (numpy {np.__version__})")


if __name__ == "__main__":
    if sys.argv[1:] == ["edges"]:
        edges()
    else:
        main()
        edges()
