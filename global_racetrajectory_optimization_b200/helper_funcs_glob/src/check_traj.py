"""check_traj -- call site main_globaltraj.py:520-532.  Prints what the reference prints."""
import numpy as np

from ... import batch as _b
from ._dev import up
from . import calc_min_bound_dists as _cmbd
from . import interp_track as _it

_DIST = "Minimum distance to boundaries is estimated to %.2fm. Keep in mind that the distance can also lie on the " \
        "outside of the track!"


def check_traj(reftrack: np.ndarray, reftrack_normvec_normalized: np.ndarray, trajectory: np.ndarray, ggv: np.ndarray,
               ax_max_machines: np.ndarray, v_max: float, length_veh: float, width_veh: float, debug: bool,
               dragcoeff: float, mass_veh: float, curvlim: float) -> tuple:
    """Distance / curvature / acceleration / speed checks of the final trajectory
    [s, x, y, psi, kappa, vx, ax]; returns (bound_r, bound_l) like the reference."""
    reftrack = np.asarray(reftrack, dtype=np.float64)
    nvec = np.asarray(reftrack_normvec_normalized, dtype=np.float64)
    traj = np.asarray(trajectory, dtype=np.float64)
    bound_r = reftrack[:, :2] + nvec * reftrack[:, 2:3]
    bound_l = reftrack[:, :2] - nvec * reftrack[:, 3:4]
    # The reference re-samples both boundaries at 1 m and then hands only element [0] of each result -- the first
    # boundary point -- to calc_min_bound_dists (check_traj.py:58-68); reproduced so that the printed distance is the
    # reference's.  batch.check_traj_batch measures against every boundary point instead.
    zeros = np.zeros((reftrack.shape[0], 2))
    first_r = _it.interp_track(np.column_stack((bound_r, zeros)), 1.0)[0]
    first_l = _it.interp_track(np.column_stack((bound_l, zeros)), 1.0)[0]
    min_dist = float(np.amin(_cmbd.calc_min_bound_dists(traj, first_r, first_l, length_veh, width_veh)))
    if min_dist < 1.0:
        print("WARNING: " + _DIST % min_dist)
    elif debug:
        print("INFO: " + _DIST % min_dist)

    ext = _b.traj_extrema_batch(up(traj[:, 4]), up(traj[:, 5]), up(traj[:, 6]), dragcoeff, mass_veh)[0].cpu().numpy()
    kappa_max, ay_max, ax_max, ax_min, a_tot_max, vx_max = ext[1:7]

    # The device maxima of ay, ax, a_tot and vx skip NaN points, as the reference's np.any(x > limit) tests do.  Its
    # messages print np.amax / np.amin, which is nan if a point is, so a printed value is NaN where the trajectory's
    # quantity has a NaN point.
    def shown(x, q):
        return np.nan if np.isnan(q).any() else x

    k, v, a = traj[:, 4], traj[:, 5], traj[:, 6]
    with np.errstate(divide="ignore", invalid="ignore"):
        ay = np.power(v, 2) / np.abs(np.divide(1.0, k, out=np.full(k.shape[0], np.inf), where=k != 0))
        ax_wo = a - (-np.power(v, 2) * dragcoeff / mass_veh)
        a_tot = np.sqrt(np.power(ax_wo, 2) + np.power(ay, 2))

    if kappa_max > curvlim:
        print("WARNING: Curvature limit is exceeded: %.3frad/m" % kappa_max)
    if ggv is not None:
        ggv = np.asarray(ggv, dtype=np.float64)
        if ay_max > np.amax(ggv[:, 2]) + 0.1:
            print("WARNING: Lateral ggv acceleration limit is exceeded: %.2fm/s2" % shown(ay_max, ay))
        if ax_max > np.amax(ggv[:, 1]) + 0.1:
            print("WARNING: Longitudinal ggv acceleration limit (positive) is exceeded: %.2fm/s2" % shown(ax_max, ax_wo))
        if ax_min < np.amin(-ggv[:, 1]) - 0.1:
            print("WARNING: Longitudinal ggv acceleration limit (negative) is exceeded: %.2fm/s2" % shown(ax_min, ax_wo))
        if a_tot_max > np.amax(ggv[:, 1:]) + 0.1:
            print("WARNING: Total ggv acceleration limit is exceeded: %.2fm/s2" % shown(a_tot_max, a_tot))
    else:
        print("WARNING: Since ggv-diagram was not given the according checks cannot be performed!")
    if ax_max_machines is not None:
        if ax_max > np.amax(np.asarray(ax_max_machines, dtype=np.float64)[:, 1]) + 0.1:
            print("WARNING: Longitudinal acceleration machine limits are exceeded: %.2fm/s2" % shown(ax_max, ax_wo))
    if vx_max > v_max + 0.1:
        print("WARNING: Maximum velocity of final trajectory exceeds the maximal velocity of the vehicle: %.2fm/s!"
              % shown(vx_max, v))
    return bound_r, bound_l
