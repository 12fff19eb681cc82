"""Batched driver of the reference's main flow between prep_track and the exports
(main_globaltraj.py:252-532 for opt_type 'mincurv', 'mincurv_iqp' and 'shortest_path'): every stage runs
on the device for a whole batch of prepared reference tracks; nothing here computes on the host.

    reftrack -> calc_splines -> QP (min. curvature / iterative / shortest path) -> create_raceline + heading/curvature
             -> velocity / acceleration / time profile -> trajectory_opt / traj_race_cl -> check_traj quantities

The parameter names are those of params/racecar.ini (``pars["veh_params"]``, ``pars["optim_opts"]``,
``pars["stepsize_opts"]``, ``pars["vel_calc_opts"]``); ``default_pars()`` returns the stock values."""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional

import torch

from . import batch as _b, raceline_refine as _refine


def default_pars() -> dict:
    """Stock values of params/racecar.ini (:13-15 step sizes, :44-50 vehicle, :56-57 velocity profile,
    :65-74 optimisation)."""
    return {"veh_params": {"v_max": 70.0, "length": 4.7, "width": 2.0, "mass": 1200.0, "dragcoeff": 0.75, "curvlim": 0.12},
            "stepsize_opts": {"stepsize_prep": 1.0, "stepsize_reg": 3.0, "stepsize_interp_after_opt": 2.0},
            "vel_calc_opts": {"dyn_model_exp": 1.0, "vel_profile_conv_filt_window": None},
            "optim_opts": {"width_opt": 3.4, "iqp_iters_min": 3, "iqp_curverror_allowed": 0.01}}


def globaltraj_batch(reftrack: torch.Tensor, opt_type: str, pars: dict, ggv=None, ax_max_machines=None,
                     n_pts: Optional[torch.Tensor] = None, check: bool = True, refine: Optional[dict] = None,
                     vehicles: Optional[_b.Vehicles] = None, veh_id=None, small_tracks: bool = False) -> dict:
    """Runs the flow for every track of ``reftrack`` [B, n_max, 4] (prepared tracks: what prep_track returns).

    Returns a dict of device tensors: alpha, reftrack / normvec / n_pts (of the last QP: they change for 'mincurv_iqp'),
    status, the create_raceline outputs (raceline_interp, psi, kappa, s_interp, el_lengths_interp, spline_lengths, n_out,
    ...), vx / ax / t profiles [B, n_out_max(+1)], laptime [B], trajectory [B, n_out_max + 1, 7] (traj_race_cl rows) and,
    with ``check``, the check_traj quantities (min_dists, the EXTREMA, bound_r / bound_l).

    ``refine``: None, or a dict of options of raceline_refine.refine_raceline_batch (e.g. ``{"max_iters": 50}``, ``{}``
    for its defaults).  The QP's alpha is then refined for the lap time inside the QP's box before the raceline is built,
    and every later stage uses the refined alpha; ``qp_alpha``, ``laptime_start`` (the lap time at the QP's alpha),
    ``refine_status``, ``refine_iters`` and ``refine_evals`` are added.  A track whose QP failed (status != 0) is not
    refined: it keeps the QP's alpha and gets refine_status -1.  Not for 'mincurv_iqp', whose reftrack changes per
    iteration.

    ``vehicles``, ``veh_id``: a car per track (batch.Vehicles; veh_id [B] host or device integers, None for one vehicle
    per track), so that one call sweeps cars.  Every stage runs with each track's car: the QPs with its curvlim and
    width_opt, the velocity profile (and the refinement's lap time) with its tables, v_max, dragcoeff and mass, and the
    check_traj quantities with its length, width, dragcoeff and mass.  A field the Vehicles object leaves unset
    (curvlim, width_opt, length, width) is taken from ``pars`` for every track.  ggv and ax_max_machines are then None.
    The refinement plans with each track's width_opt and drives each track's car.  Its curvature limit is, as with
    ``pars``, refine's own ``kappa_bound`` and not curvlim: with ``pars`` the refinement enforces no limit unless refine
    asks for one, and the vehicles path keeps that meaning, so that a track's outputs stay those of the call with its
    car's scalar ``pars`` and tables alone.  For each car's limit pass it per track, e.g.
    ``refine={"metric_length": 10.0, "kappa_bound": vehicles.per_track("curvlim", vehicles.veh_id(veh_id, B, dev))}``.
    Still one per call: dyn_model_exp, the filter window, the step sizes and the iterative
    QP's options.

    ``small_tracks``: the 'mincurv' and 'mincurv_iqp' QPs also solve the tracks below batch.N_MIN points (the dense
    small-track solver, batch.opt_min_curv_batch); without it those get status -1.  'shortest_path' takes every size
    anyway.  With ``refine`` a solved short track is refined as the refinement documents for tracks below N_MIN: in the
    curvature metric and under a curvature limit only with the refinement's own flag as well,
    ``refine={"small_tracks": True, "metric_length": 10.0, "kappa_bound": 0.12}`` (the dense kernels then give such a
    track its metric and projection; without it the metric falls back to the identity step and the projection fails)."""
    if opt_type not in ("mincurv", "mincurv_iqp", "shortest_path"):
        raise IOError("Unknown optimization type!" if opt_type != "mintime" else
                      "opt_type 'mintime' (CasADi/IPOPT NLP) is outside the CUDA path")
    if refine is not None and not isinstance(refine, dict):
        raise TypeError("refine must be None or a dict of refine_raceline_batch options")
    if refine is not None and opt_type == "mincurv_iqp":
        raise NotImplementedError("refine: not for 'mincurv_iqp' (its reftrack changes per iteration)")
    veh, opt, steps, vel = pars["veh_params"], pars["optim_opts"], pars["stepsize_opts"], pars["vel_calc_opts"]
    car = _car(reftrack, veh, opt, ggv, ax_max_machines, vehicles, veh_id)
    cx, cy, nv, h = _b.calc_splines_batch(reftrack, n_pts=n_pts, want_coeffs=False)
    rt_used, nv_used, n_used = reftrack, nv, n_pts
    if opt_type == "mincurv":
        qp = _b.opt_min_curv_batch(reftrack, nv, h, car.curvlim, car.width_opt, n_pts=n_pts, small_tracks=small_tracks)
        alpha, status = qp["alpha"], qp["status"]
    elif opt_type == "mincurv_iqp":
        qp = _b.iqp_batch(reftrack, nv, h, car.curvlim, car.width_opt, steps["stepsize_reg"],
                          iters_min=opt["iqp_iters_min"], curv_error_allowed=opt["iqp_curverror_allowed"], n_pts=n_pts,
                          small_tracks=small_tracks)
        alpha, status = qp["alpha"], qp["status"]
        rt_used, nv_used, n_used = qp["reftrack"], qp["normvec"], qp["n_pts"]
    else:
        qp = _b.opt_shortest_path_batch(reftrack, nv, car.width_opt, n_pts=n_pts)
        alpha, status = qp["alpha"], qp["status"]
    refined = {}
    if refine is not None:
        n_all = n_pts if n_pts is not None else torch.full_like(status, reftrack.shape[1])
        ref = _refine.refine_raceline_batch(reftrack, nv, alpha, car.width_opt, stepsize_interp=steps["stepsize_interp_after_opt"],
                                            n_pts=torch.where(status == 0, n_all.to(status), torch.zeros_like(status)),
                                            dyn_model_exp=vel["dyn_model_exp"],
                                            filt_window=vel["vel_profile_conv_filt_window"], **car.vp, **refine)
        refined = dict(qp_alpha=alpha, laptime_start=ref["laptime_start"], refine_status=ref["status"],
                       refine_iters=ref["iters"], refine_evals=ref["evals"])
        alpha = ref["alpha"]
    rl = _b.create_raceline_batch(rt_used, nv_used, alpha, steps["stepsize_interp_after_opt"], n_pts=n_used)
    n_out = rl["n_out"]
    vp = _b.vel_profile_batch(rl["kappa"], rl["el_lengths_interp"], dyn_model_exp=vel["dyn_model_exp"],
                              filt_window=vel["vel_profile_conv_filt_window"], n_pts=n_out, **car.vp)
    vx, ax, t = vp["vx"][:, 0].contiguous(), vp["ax"][:, 0].contiguous(), vp["t"][:, 0].contiguous()
    traj = _b.assemble_trajectory_batch(rl["s_interp"], rl["raceline_interp"], rl["psi"], rl["kappa"], vx, ax,
                                        rl["spline_lengths"], n_traj=n_out, n_spl=n_used)
    out = dict(alpha=alpha, status=status, reftrack=rt_used, normvec=nv_used, n_pts=n_used, vx=vx, ax=ax, t=t,
               laptime=vp["laptime"][:, 0], vel_status=vp["status"][:, 0], trajectory=traj)
    out.update(rl)
    out.update(refined)
    if check:
        out.update(_b.check_traj_batch(rt_used, nv_used, rl["raceline_interp"], rl["psi"], rl["kappa"], vx, ax,
                                       car.length, car.width, car.dragcoeff, car.mass, n_pts=n_used, n_traj=n_out))
    return out


def _car(reftrack, veh: dict, opt: dict, ggv, ax_max_machines, vehicles, veh_id) -> SimpleNamespace:
    """The vehicle parameters of globaltraj_batch's stages: curvlim, width_opt, length, width, dragcoeff, mass (a number
    from pars, or with vehicles a [B] device tensor gathered by veh_id, pars where the Vehicles leave a field unset) and
    vp, the vehicle arguments of the velocity profile and the refinement."""
    if vehicles is None:
        if veh_id is not None:
            raise ValueError("veh_id needs vehicles=")
        if ggv is None or ax_max_machines is None:
            raise TypeError("globaltraj_batch needs ggv and ax_max_machines (or vehicles=)")
        return SimpleNamespace(curvlim=veh["curvlim"], width_opt=opt["width_opt"], length=veh["length"], width=veh["width"],
                               dragcoeff=veh["dragcoeff"], mass=veh["mass"],
                               vp=dict(ggv=ggv, ax_max_machines=ax_max_machines, v_max=float(veh["v_max"]),
                                       drag_coeff=veh["dragcoeff"], m_veh=veh["mass"]))
    if ggv is not None or ax_max_machines is not None:
        raise ValueError("globaltraj_batch: with vehicles= ggv and ax_max_machines must be None (each vehicle has its own)")
    if not isinstance(vehicles, _b.Vehicles):
        raise TypeError("vehicles must be a batch.Vehicles")
    ids = vehicles.veh_id(veh_id, reftrack.shape[0], reftrack.device)
    field = lambda name, default: default if getattr(vehicles, name) is None else vehicles.per_track(name, ids)  # noqa: E731
    return SimpleNamespace(curvlim=field("curvlim", veh["curvlim"]), width_opt=field("width_opt", opt["width_opt"]),
                           length=field("length", veh["length"]), width=field("width", veh["width"]),
                           dragcoeff=vehicles.per_track("drag_coeff", ids), mass=vehicles.per_track("m_veh", ids),
                           vp=dict(vehicles=vehicles, veh_id=ids))
