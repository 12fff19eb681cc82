/*
 * shortest_path_sens.h -- sensitivities of the shortest-path QP: the two entry points of libmincurv_b200.so behind
 * batch.opt_shortest_path_diff.  Conventions as in include/mincurv_b200.h (device pointers, float64, batch-major, n_pts may
 * be NULL, stream-ordered, 0 / -1 / -2 / -3 return codes).  DESIGN.md section 3.11 has the derivation.
 *
 * H and f of this QP are explicit in the centre line and the normals, so alpha is differentiated with respect to all of
 * them: x, y, w_tr_right, w_tr_left, the normal vectors and w_veh.  grad_status[b] (int32):
 *   0  the solve converged (status 0): gradients are computed
 *   2, 3, -1  the solve's status (iteration cap, breakdown, unsupported size)
 *   3  also: a non-finite adjoint solution
 * Every unsupported instance gets zero gradients.  A bound clamped to 0.001 m (tph's clamp of w - w_veh / 2) does not
 * move with the widths: its width gradients are zero.
 */
#ifndef SHORTEST_PATH_SENS_H
#define SHORTEST_PATH_SENS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* mc_shortest_path_solve_batch (same arguments, bit-identical alpha, status, iters) that also exports what the backward
 * pass needs, 16 bytes per point:
 *   sens        [B][2][n_max] : lu / su and ll / sl, the final multiplier-to-slack ratios of the upper and lower bounds
 *                               (zero beyond n_pts[b] and for grad_status != 0)
 *   grad_status [B]           : see above */
int mc_shortest_path_solve_batch_sens(int B, int n_max, const int32_t *n_pts,
                                      const double *reftrack, const double *normvec,
                                      double w_veh, const double *w_veh_batch,
                                      double *alpha, int32_t *status, int32_t *iters, double *sens, int32_t *grad_status,
                                      void *workspace, size_t workspace_bytes, void *stream);

/* Vector-Jacobian product of alpha: for an upstream gradient grad_alpha [B][n_max] of a loss L,
 *   grad_reftrack [B][n_max][4]        = dL / d(x, y, w_tr_right, w_tr_left)   (x, y at fixed normals)
 *   grad_normvec  [B][n_max][2] or NULL = dL / dnormvec
 *   grad_w_veh    [B] or NULL           = dL / dw_veh per instance (the scalar w_veh's gradient is their sum)
 * reftrack, normvec, w_veh / w_veh_batch, alpha, sens and grad_status are those of the mc_shortest_path_solve_batch_sens
 * call.  One cyclic tridiagonal factorisation of H + diag(sens[0] + sens[1]) and one solve per instance in a workspace of
 * mc_shortest_path_workspace_bytes(B, n_max); nothing has to survive in it between the two calls.  grad_status is read,
 * and set to 3 where the adjoint solution is not finite. */
int mc_shortest_path_adjoint_batch(int B, int n_max, const int32_t *n_pts,
                                   const double *reftrack, const double *normvec,
                                   double w_veh, const double *w_veh_batch,
                                   const double *alpha, const double *sens, int32_t *grad_status, const double *grad_alpha,
                                   double *grad_reftrack, double *grad_normvec, double *grad_w_veh,
                                   void *workspace, size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SHORTEST_PATH_SENS_H */
