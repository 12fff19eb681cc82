"""Batched driver of the reference's main flow between prep_track and the exports
(main_globaltraj.py:252-532 for opt_type 'mincurv', 'mincurv_iqp' and 'shortest_path'): every stage runs
on the device for a whole batch of prepared reference tracks; nothing here computes on the host.

    reftrack -> calc_splines -> QP (min. curvature / iterative / shortest path) -> create_raceline + heading/curvature
             -> velocity / acceleration / time profile -> trajectory_opt / traj_race_cl -> check_traj quantities

The parameter names are those of params/racecar.ini (``pars["veh_params"]``, ``pars["optim_opts"]``,
``pars["stepsize_opts"]``, ``pars["vel_calc_opts"]``); ``default_pars()`` returns the stock values."""
from __future__ import annotations

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


def globaltraj_batch(reftrack: torch.Tensor, opt_type: str, pars: dict, ggv, ax_max_machines,
                     n_pts: Optional[torch.Tensor] = None, check: bool = True, refine: Optional[dict] = None) -> dict:
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
    iteration."""
    if opt_type not in ("mincurv", "mincurv_iqp", "shortest_path"):
        raise IOError("Unknown optimization type!" if opt_type != "mintime" else
                      "opt_type 'mintime' (CasADi/IPOPT NLP) is outside the CUDA path")
    if refine is not None and not isinstance(refine, dict):
        raise TypeError("refine must be None or a dict of refine_raceline_batch options")
    if refine is not None and opt_type == "mincurv_iqp":
        raise NotImplementedError("refine: not for 'mincurv_iqp' (its reftrack changes per iteration)")
    veh, opt, steps, vel = pars["veh_params"], pars["optim_opts"], pars["stepsize_opts"], pars["vel_calc_opts"]
    cx, cy, nv, h = _b.calc_splines_batch(reftrack, n_pts=n_pts, want_coeffs=False)
    rt_used, nv_used, n_used = reftrack, nv, n_pts
    if opt_type == "mincurv":
        qp = _b.opt_min_curv_batch(reftrack, nv, h, veh["curvlim"], opt["width_opt"], n_pts=n_pts)
        alpha, status = qp["alpha"], qp["status"]
    elif opt_type == "mincurv_iqp":
        qp = _b.iqp_batch(reftrack, nv, h, veh["curvlim"], opt["width_opt"], steps["stepsize_reg"],
                          iters_min=opt["iqp_iters_min"], curv_error_allowed=opt["iqp_curverror_allowed"], n_pts=n_pts)
        alpha, status = qp["alpha"], qp["status"]
        rt_used, nv_used, n_used = qp["reftrack"], qp["normvec"], qp["n_pts"]
    else:
        qp = _b.opt_shortest_path_batch(reftrack, nv, opt["width_opt"], n_pts=n_pts)
        alpha, status = qp["alpha"], qp["status"]
    refined = {}
    if refine is not None:
        n_all = n_pts if n_pts is not None else torch.full_like(status, reftrack.shape[1])
        ref = _refine.refine_raceline_batch(reftrack, nv, alpha, opt["width_opt"], ggv, ax_max_machines, float(veh["v_max"]),
                                            veh["dragcoeff"], veh["mass"], stepsize_interp=steps["stepsize_interp_after_opt"],
                                            n_pts=torch.where(status == 0, n_all.to(status), torch.zeros_like(status)),
                                            dyn_model_exp=vel["dyn_model_exp"],
                                            filt_window=vel["vel_profile_conv_filt_window"], **refine)
        refined = dict(qp_alpha=alpha, laptime_start=ref["laptime_start"], refine_status=ref["status"],
                       refine_iters=ref["iters"], refine_evals=ref["evals"])
        alpha = ref["alpha"]
    rl = _b.create_raceline_batch(rt_used, nv_used, alpha, steps["stepsize_interp_after_opt"], n_pts=n_used)
    n_out = rl["n_out"]
    vp = _b.vel_profile_batch(rl["kappa"], rl["el_lengths_interp"], ggv, ax_max_machines, float(veh["v_max"]),
                              veh["dragcoeff"], veh["mass"], dyn_model_exp=vel["dyn_model_exp"],
                              filt_window=vel["vel_profile_conv_filt_window"], n_pts=n_out)
    vx, ax, t = vp["vx"][:, 0].contiguous(), vp["ax"][:, 0].contiguous(), vp["t"][:, 0].contiguous()
    traj = _b.assemble_trajectory_batch(rl["s_interp"], rl["raceline_interp"], rl["psi"], rl["kappa"], vx, ax,
                                        rl["spline_lengths"], n_traj=n_out, n_spl=n_used)
    out = dict(alpha=alpha, status=status, reftrack=rt_used, normvec=nv_used, n_pts=n_used, vx=vx, ax=ax, t=t,
               laptime=vp["laptime"][:, 0], vel_status=vp["status"][:, 0], trajectory=traj)
    out.update(rl)
    out.update(refined)
    if check:
        out.update(_b.check_traj_batch(rt_used, nv_used, rl["raceline_interp"], rl["psi"], rl["kappa"], vx, ax,
                                       veh["length"], veh["width"], veh["dragcoeff"], veh["mass"], n_pts=n_used,
                                       n_traj=n_out))
    return out
