/*
 * mincurv_sens.h -- width sensitivities of the minimum-curvature QP: the two entry points of libmincurv_b200.so
 * behind batch.opt_min_curv_diff.  Conventions as in include/mincurv_b200.h (device pointers, float64, batch-major,
 * n_pts may be NULL, stream-ordered, 0 / -1 / -2 / -3 return codes).  DESIGN.md section 3.10 has the derivation.
 *
 * Only instances solved by the box-only phase have a gradient here.  grad_status[b] (int32):
 *   0  solved by the box-only phase (status 0): gradients are computed
 *   4  the box-only optimum violated the curvature rows and the curvature-row phase re-solved it: not supported
 *   1, 2, 3, -1  the forward solve's status (infeasible, iteration cap, breakdown, unsupported size)
 *   3  also: a non-positive pivot in the adjoint factorisation
 * Every unsupported instance gets zero gradients.  The widths are differentiated, the centre line, h, f_scale and
 * kappa_bound are constants.
 */
#ifndef MINCURV_SENS_H
#define MINCURV_SENS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* mc_mincurv_solve_batch_shared (same arguments, bit-identical alpha, curv_error_max, kappa_lin_max, status, iters) that
 * also exports what the backward pass needs, 16 bytes per point:
 *   sens        [B][2][n_max] : lu / su and ll / sl, the box phase's final multiplier-to-slack ratios of the upper and
 *                               lower bounds (zero beyond n_pts[b] and for grad_status != 0)
 *   grad_status [B]           : see above; recorded after the box phase, before the curvature-row phase */
int mc_mincurv_solve_batch_sens(int B, int n_max, const int32_t *n_pts,
                                const double *reftrack, const double *normvec, const double *h,
                                double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                const int32_t *centre_id,
                                double *alpha, double *curv_error_max, double *kappa_lin_max,
                                int32_t *status, int32_t *iters, double *sens, int32_t *grad_status,
                                void *workspace, size_t workspace_bytes, void *stream);

/* Vector-Jacobian product of alpha with respect to the widths: for an upstream gradient grad_alpha [B][n_max] of a
 * loss L,
 *   grad_w_right [B][n_max] = dL / dw_tr_right,  grad_w_left [B][n_max] = dL / dw_tr_left,  grad_w_veh [B] = dL / dw_veh
 * (per instance; the scalar w_veh's gradient is their sum).  Geometry, widths, w_veh / w_veh_batch, f_scale and centre_id
 * must be those of the mc_mincurv_solve_batch_sens call that produced sens and grad_status.  The assembly is re-run in
 * the workspace, then one factorisation of H + diag(sens[0] + sens[1]) and one solve per instance; nothing has to
 * survive in the workspace between the two calls.  grad_status is read, and set to 3 where the factorisation breaks
 * down.  grad_w_right also serves as scratch of the assembly's status words before it is written. */
int mc_mincurv_adjoint_batch(int B, int n_max, const int32_t *n_pts,
                             const double *reftrack, const double *normvec, const double *h,
                             double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                             const double *sens, int32_t *grad_status, const double *grad_alpha,
                             double *grad_w_right, double *grad_w_left, double *grad_w_veh,
                             void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MINCURV_SENS_H */
