/*
 * lap_time_sens.h -- sensitivities of the lap time: the entry points of libmincurv_b200.so behind batch.create_raceline_diff
 * and batch.vel_profile_diff.
 * Conventions as in include/mincurv_b200.h (device pointers, float64, batch-major, n_pts may be NULL, stream-ordered,
 * 0 / -1 / -2 / -3 return codes).  DESIGN.md section 3.12 has the derivation.
 *
 * The velocity profile (closed track, ggv branch, one profile per track, no mu) is differentiated with respect to kappa
 * and el_lengths as the forward evaluates it, with every discrete decision frozen as the forward took it.  grad_status[b]
 * (int32):
 *   0  the gradient is computed
 *   3  non-finite lap time (the forward's status) or a non-finite gradient
 *   for n_pts[b] < 2 (an inactive slot) the forward's status (0 for n_pts 0, 3 otherwise)
 * Every such instance gets zero gradients.
 */
#ifndef LAP_TIME_SENS_H
#define LAP_TIME_SENS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Workspace of mc_create_raceline_adjoint_batch: 25 (n_max rounded up to 32, + 32) doubles per track. */
size_t mc_create_raceline_adjoint_workspace_bytes(int B, int n_max);

/* Vector-Jacobian product of mc_create_raceline_batch (unit parameter scales, the raceline refline + alpha normvec): for
 * upstream gradients grad_raceline [B][n_out_max][2], grad_kappa [B][n_out_max] and grad_el_lengths [B][n_out_max]
 * (each may be NULL: zero) of a loss L,
 *   grad_alpha   [B][n_max]          = dL / dalpha
 *   grad_refline [B][n_max][2] or NULL = dL / d(x, y) of the reference line
 *   grad_normvec [B][n_max][2] or NULL = dL / dnormvec
 * all zero beyond n_pts[b], and zero for a track with n_out[b] <= 0 (overflow or inactive) or n_pts[b] < 3.  n_out and the
 * segment of every station are held: coeffs_x / coeffs_y, spline_lengths, n_out, spline_inds and t_values are the
 * forward call's outputs (n_out_max its capacity); normvec and alpha its inputs. */
int mc_create_raceline_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *normvec, const double *alpha,
                                     int n_out_max, const double *coeffs_x, const double *coeffs_y,
                                     const double *spline_lengths, const int32_t *n_out, const int32_t *spline_inds,
                                     const double *t_values, const double *grad_raceline, const double *grad_kappa,
                                     const double *grad_el_lengths, double *grad_alpha, double *grad_refline,
                                     double *grad_normvec, void *workspace, size_t workspace_bytes, void *stream);

/* Workspace of mc_vel_profile_adjoint_batch: 17 n_max + 1 doubles per track (the forward's scratch vectors, its tape and
 * the adjoint vectors). */
size_t mc_vel_profile_adjoint_workspace_bytes(int B, int n_max);

/* Vector-Jacobian product of mc_vel_profile_batch_ex with V = 1 (no ggv scales, no per-variant top speed, no mu): for
 * upstream gradients grad_laptime [B] and grad_vx [B][n_max] (either may be NULL: zero) of a loss L,
 *   grad_kappa      [B][n_max] or NULL = dL / dkappa
 *   grad_el_lengths [B][n_max] or NULL = dL / del_lengths
 * both zero beyond n_pts[b].  The other arguments are those of the forward call; the forward is run again inside (its
 * outputs are not inputs here). */
int mc_vel_profile_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                                 double v_max, int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines,
                                 double dyn_model_exp, double drag_coeff, double m_veh, int filt_window,
                                 int decel_slice_upper, const double *grad_laptime, const double *grad_vx,
                                 double *grad_kappa, double *grad_el_lengths, int32_t *grad_status,
                                 void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* LAP_TIME_SENS_H */
