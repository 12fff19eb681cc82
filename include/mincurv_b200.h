/*
 * mincurv_b200.h -- C-ABI of the H100-native (sm_90a) batched minimum-curvature / shortest-path raceline QP path.
 *
 * Every entry point replaces one function of the third-party package the reference calls
 * (trajectory_planning_helpers==0.76, requirements.txt:3); the reference-side
 * call site that fixes its meaning is cited on each declaration.  The reference has no native
 * boundary of its own on this path (it is pure Python above quadprog's Cython shim), so this header
 * is what a ctypes binding inside tph would bind -- see INTEGRATION.md.
 *
 * Conventions
 *   - all pointers are DEVICE pointers (e.g. torch.Tensor.data_ptr()); nothing is allocated or freed
 *     by the library: the caller passes a workspace of mc_*_workspace_bytes() bytes;
 *   - all arrays are float64 unless stated, batch-major, row-major, padded to n_max points per track;
 *     n_pts[b] (int32, may be NULL => every track has n_max points) is the true size of track b;
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous and stream-ordered;
 *   - arguments are int, double, size_t or pointers: the package's ctypes binding is parsed from these declarations;
 *   - return value: 0 = ok, <0 = bad argument (-1), CUDA error (-2), workspace too small (-3);
 *   - per-instance results are reported in status[b] (int32):
 *       0 ok | 1 track too narrow ("Problem not solvable, track might be too small ...", tph RuntimeError)
 *       2 iteration cap reached | 3 numerical breakdown (non-positive pivot)
 *       4 (transient) curvature rows |k_ref + E alpha| <= kappa_bound violated by the box-only optimum: set by the
 *         finalize stage, consumed by mc_mincurv_kappa_batch, which re-solves the instance with the rows.
 */
#ifndef MINCURV_B200_H
#define MINCURV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MC_OK 0
#define MC_EINVAL (-1)
#define MC_ECUDA (-2)
#define MC_EWORKSPACE (-3)

/* MC_OPTIONAL marks parameters added to an entry point after its first release.  They are NULL-able (an int among them
 * may be 0), and NULL gives the entry's earlier behaviour exactly.  The package's ctypes binding lets a call leave them
 * out altogether, so code written for the earlier signature keeps working; C callers pass NULL / 0. */
#define MC_OPTIONAL
/* MC_OPTIONAL2 marks parameters added after the MC_OPTIONAL ones, alike NULL-able.  The binding lets a call leave out
 * the MC_OPTIONAL2 parameters alone (the signature before they were added), or them and the MC_OPTIONAL ones. */
#define MC_OPTIONAL2

#define MC_STATUS_OK 0
#define MC_STATUS_TOO_NARROW 1
#define MC_STATUS_MAXITER 2
#define MC_STATUS_BREAKDOWN 3
#define MC_STATUS_KAPPA_ACTIVE 4

/* The two constants of the third-party package that cannot be confirmed offline (parity unpinned, DESIGN.md section 2).
 * They are RUN-TIME parameters of the *_ex entry points; the plain entry points use these defaults.
 * tools/pin_against_tph.py determines both from the real trajectory_planning_helpers when it is importable.
 *   f_scale            tph.opt_min_curv: f = f_scale * E^T k_ref (tph as recalled: the linear term carries a factor 2 the
 *                      quadratic term does not; 1.0 would be the consistent Gauss-Newton scaling)
 *   decel_slice_upper  tph.calc_vel_profile (closed): which half of the doubled lap is kept after the backward pass */
#define MC_F_SCALE_DEFAULT 2.0
#define MC_VP_DECEL_SLICE_UPPER_DEFAULT 1

/* library version (major*10000 + minor*100 + patch) and last CUDA error text of this thread */
int mc_version(void);
const char *mc_last_error(void);

/* -------------------------------------------------------------------------------------------------
 * tph.calc_splines.calc_splines(path, el_lengths=None, psi_s=None, psi_e=None, use_dist_scaling=True)
 * closed-path branch -- call sites helper_funcs_glob/src/prep_track.py:48-51,
 * main_globaltraj.py:568.
 *   xy        [B][n_max][xy_stride] : points (x at +0, y at +1); xy_stride = 2 (a path) or 4 (a reftrack)
 *   el_lengths[B][n_max] or NULL    : segment lengths |p_{i+1}-p_i| override (tph's el_lengths argument)
 *   use_dist_scaling                : 1 => chord-length scaling between neighbouring segments, 0 => none
 *   coeffs_x/y[B][n_max][4]         : a0..a3 of every segment, local parameter t in [0,1]
 *   normvec   [B][n_max][2]         : right-pointing unit normals (t = 0 derivative rotated by -90 deg)
 *   h_out     [B][n_max]            : the per-segment parameter scale the system matrix M encodes
 *                                     (scaling_i = h_i / h_{i+1}; all ones without dist scaling) --
 *                                     replaces the dense 4N x 4N matrix tph returns as `M`
 * workspace: mc_calc_splines_workspace_bytes(B, n_max)
 */
size_t mc_calc_splines_workspace_bytes(int B, int n_max);
int mc_calc_splines_batch(int B, int n_max, const int32_t *n_pts,
                          const double *xy, int xy_stride, const double *el_lengths, int use_dist_scaling,
                          double *coeffs_x, double *coeffs_y, double *normvec, double *h_out,
                          void *workspace, size_t workspace_bytes, void *stream);

/* -------------------------------------------------------------------------------------------------
 * tph.opt_min_curv.opt_min_curv(reftrack, normvectors, A, kappa_bound, w_veh, ...)  (closed=True)
 * -- call sites main_globaltraj.py:264-271 and :344-350; the QP it hands to
 * quadprog.solve_qp (SURVEY.md A.3) is solved here by a primal-dual interior-point method.
 *   reftrack  [B][n_max][4]  : x, y, w_tr_right, w_tr_left
 *   normvec   [B][n_max][2]
 *   h         [B][n_max]     : parameter scales of the spline system (h_out of mc_calc_splines_batch;
 *                              what the reference passes as the dense matrix `A`)
 *   w_veh_batch [B] or NULL  : per-instance vehicle width; NULL => the scalar w_veh for all
 *   alpha     [B][n_max]     : lateral shift of every point along its normal [m]
 *   curv_error_max [B]       : tph's linearisation error (second tuple element of opt_min_curv)
 *   kappa_lin_max  [B] or NULL : max |k_ref + E alpha| of the linearised curvature at the solution
 *   iters     [B] or NULL    : interior-point iterations used (int32)
 */
size_t mc_mincurv_workspace_bytes(int B, int n_max);
int mc_mincurv_solve_batch(int B, int n_max, const int32_t *n_pts,
                           const double *reftrack, const double *normvec, const double *h,
                           double kappa_bound, double w_veh, const double *w_veh_batch,
                           double *alpha, double *curv_error_max, double *kappa_lin_max,
                           int32_t *status, int32_t *iters,
                           void *workspace, size_t workspace_bytes, void *stream);

/* the same with an explicit f_scale (see MC_F_SCALE_DEFAULT) and, with prox_x, the projection onto the QP's feasible set
 * P = {lb <= alpha <= ub, |k_ref + E alpha| <= kappa_bound} in the metric H + prox_mu I (raceline_refine.CurvatureProjection,
 * DESIGN.md section 3.13):
 *   prox_x == NULL : the call above, bit for bit (prox_mu and prox_q are not read)
 *   prox_x, prox_q [B][n_max] : solves  min 1/2 alpha^T (H + prox_mu I) alpha + c^T alpha  over P,
 *                    c = prox_mu prox_q - (H + prox_mu I) prox_x,  i.e.  argmin_{alpha in P} 1/2 |alpha - x|^2_{I + H / prox_mu}
 *                    + q^T (alpha - x);  prox_mu > 0 and finite, prox_q required.  f_scale is checked but does not enter
 *                    the objective; the stages are those of mc_mincurv_solve_batch (assembly, box phase, finalize,
 *                    curvature-row phase, finalize) on H + prox_mu I, without shared centre lines.  kappa_lin_max and
 *                    curv_error_max are those of the result; status as above (4: the rows are still violated).
 *   lin_alpha [B][n_max] or NULL : the linearisation point a (DESIGN.md section 3.2), with or without prox_x.  NULL: the
 *                    QP as tph builds it, its curvature rows linearised about the centre line P.  Otherwise about the line
 *                    P + a n on the same grid (the step of tph's iterative QP, without re-sampling): the first
 *                    derivatives x', y' in S_x, S_y are those of the spline through P + a n, k_ref = S_y m_y - S_x m_x
 *                    keeps the centre line's moments, so that k_ref + E a is the knot curvature of the spline through
 *                    P + a n.  H, f and the rows follow from these; the variable is still alpha about P.  curv_error_max
 *                    and kappa_lin_max refer to this linearisation. */
int mc_mincurv_solve_batch_ex(int B, int n_max, const int32_t *n_pts,
                              const double *reftrack, const double *normvec, const double *h,
                              double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                              double *alpha, double *curv_error_max, double *kappa_lin_max,
                              int32_t *status, int32_t *iters,
                              double prox_mu, const double *prox_x, const double *prox_q,
                              MC_OPTIONAL2 const double *lin_alpha,
                              void *workspace, size_t workspace_bytes, void *stream);

/* the same for batches in which several instances share a centreline (x, y, normal vectors, h and n_pts identical, only
 * the track widths / vehicle width differ -- e.g. the width variants of one track, main_globaltraj.py:264-271
 * called in a sweep): H, f and k_ref depend on the centreline only, so they are assembled once per centreline; f and
 * k_ref are copied to the followers, and the solver reads the owner's band of H (it stays in the owner's workspace slab).
 *   centre_id [B] or NULL : centre_id[b] = index (in this batch) of the instance that owns b's centreline; owners have
 *                           centre_id[b] == b.  NULL: every instance is assembled on its own.  A follower whose owner is
 *                           not an owner itself, is out of range or has another n_pts gets status -1.
 * The results are identical to the unshared call (the shared quantities are bitwise the same). */
int mc_mincurv_solve_batch_shared(int B, int n_max, const int32_t *n_pts,
                                  const double *reftrack, const double *normvec, const double *h,
                                  double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                  const int32_t *centre_id,
                                  double *alpha, double *curv_error_max, double *kappa_lin_max,
                                  int32_t *status, int32_t *iters,
                                  void *workspace, size_t workspace_bytes, void *stream);
int mc_mincurv_setup_batch_shared(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                  const double *h, double w_veh, const double *w_veh_batch, double f_scale,
                                  const int32_t *centre_id, int32_t *status,
                                  void *workspace, size_t workspace_bytes, void *stream);

/* The three stages of mc_mincurv_solve_batch as separate stream-ordered calls on the same workspace
 * (assembly of the banded QP, interior-point solve, post-solve curvature check / linearisation error);
 * mc_mincurv_solve_batch is exactly setup -> pdip -> finalize.  Exposed so that a caller can time or
 * overlap the stages; arguments as above.  The finalize stage of a workspace assembled about a linearisation point
 * (lin_alpha of mc_mincurv_setup_batch_ex) needs linearised = 1: the line P + alpha n takes the centre line's first
 * derivatives, the linearised curvature those of the linearisation point. */
int mc_mincurv_setup_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                           const double *h, double w_veh, const double *w_veh_batch, int32_t *status,
                           void *workspace, size_t workspace_bytes, void *stream);
int mc_mincurv_setup_batch_ex(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double w_veh, const double *w_veh_batch, double f_scale, int32_t *status,
                              MC_OPTIONAL2 const double *lin_alpha,
                              void *workspace, size_t workspace_bytes, void *stream);
int mc_mincurv_pdip_batch(int B, int n_max, const int32_t *n_pts, double *alpha, int32_t *status, int32_t *iters,
                          void *workspace, size_t workspace_bytes, void *stream);
int mc_mincurv_finalize_batch(int B, int n_max, const int32_t *n_pts, const double *alpha, double kappa_bound,
                              double *curv_error_max, double *kappa_lin_max, int32_t *status,
                              MC_OPTIONAL2 int linearised,
                              void *workspace, size_t workspace_bytes, void *stream);

/* Width sensitivities of this QP: alpha differentiated with respect to w_tr_right, w_tr_left and w_veh by one more
 * factorisation per instance (batch.opt_min_curv_diff; DESIGN.md section 3.10 has the derivation).
 * Without the curvature-row export (sens_rows NULL) only instances solved by the box-only phase have a gradient.
 * grad_status[b] (int32):
 *   0  solved by the box-only phase (status 0), or with sens_rows by the curvature-row phase: gradients are computed
 *   4  without sens_rows: the box-only optimum violated the curvature rows and the curvature-row phase re-solved it:
 *      not supported
 *   1, 2, 3, -1  the forward solve's status (infeasible, iteration cap, breakdown, unsupported size; with sens_rows
 *      also 4: rows still violated after the curvature-row phase)
 *   3  also: a non-positive pivot in the adjoint factorisation (or in its Schur complement of the strong rows), or more
 *      strong rows than n_rows_cap
 * Every unsupported instance gets zero gradients.  The widths are differentiated, the centre line, h, f_scale and
 * kappa_bound are constants.
 *
 * mc_mincurv_solve_batch_sens: mc_mincurv_solve_batch_shared (same arguments, bit-identical alpha, curv_error_max,
 * kappa_lin_max, status, iters) that also exports what the backward pass needs, 16 bytes per point:
 *   sens        [B][2][n_max] : lu / su and ll / sl, the box phase's final multiplier-to-slack ratios of the upper and
 *                               lower bounds (zero beyond n_pts[b] and for grad_status != 0)
 *   grad_status [B]           : see above; recorded after the box phase, before the curvature-row phase
 * and with sens_rows and n_rows (both or neither; NULL: the call above), 8 more bytes per point, from the final
 * iterate of the curvature-row phase for the instances it solved:
 *   sens        [B][2][n_max] : that phase's final lu / su and ll / sl
 *   sens_rows   [B][n_max]    : the row weights l3 / s3 + l4 / s4 (zero for the other instances and beyond n_pts[b])
 *   n_rows      [B] (int32)   : the strong rows (weight > 1), the Schur complement size of the adjoint (0 elsewhere)
 *   grad_status [B]           : the final solve status
 *
 * mc_mincurv_adjoint_batch: vector-Jacobian product of alpha with respect to the widths: for an upstream gradient
 * grad_alpha [B][n_max] of a loss L,
 *   grad_w_right [B][n_max] = dL / dw_tr_right,  grad_w_left [B][n_max] = dL / dw_tr_left,  grad_w_veh [B] = dL / dw_veh
 * (per instance; the scalar w_veh's gradient is their sum).  Geometry, widths, w_veh / w_veh_batch, f_scale and centre_id
 * must be those of the mc_mincurv_solve_batch_sens call that produced sens and grad_status.  The assembly is re-run in
 * the workspace, then one factorisation of H + diag(sens[0] + sens[1]) and one solve per instance; nothing has to
 * survive in the workspace between the two calls.  grad_status is read, and set to 3 where the factorisation breaks
 * down.  grad_w_right also serves as scratch of the assembly's status words before it is written.
 * sens_rows, n_rows (NULL: the call above): those of the mc_mincurv_solve_batch_sens call.  An instance with row weights
 * is differentiated at the curvature-row phase's iterate: one factorisation of H + diag(sens[0] + sens[1]) + E^T W E
 * with the weak rows (W <= 1) in the band, and the n_rows[b] strong rows through their Schur complement, a dense
 * n_rows[b]^2 matrix kept in schur [B][n_rows_cap][n_rows_cap] (required with sens_rows); an instance with
 * n_rows[b] > n_rows_cap gets grad_status 3.
 * lin_alpha (NULL: the centre line): the linearisation point of H, as for mc_mincurv_solve_batch_ex; with centre_id a
 * follower is linearised about its owner's row (the assembly is shared); alpha is not
 * differentiated with respect to it. */
int mc_mincurv_solve_batch_sens(int B, int n_max, const int32_t *n_pts,
                                const double *reftrack, const double *normvec, const double *h,
                                double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                const int32_t *centre_id,
                                double *alpha, double *curv_error_max, double *kappa_lin_max,
                                int32_t *status, int32_t *iters, double *sens, int32_t *grad_status,
                                MC_OPTIONAL double *sens_rows, MC_OPTIONAL int32_t *n_rows,
                                void *workspace, size_t workspace_bytes, void *stream);
int mc_mincurv_adjoint_batch(int B, int n_max, const int32_t *n_pts,
                             const double *reftrack, const double *normvec, const double *h,
                             double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                             const double *sens, int32_t *grad_status, const double *grad_alpha,
                             double *grad_w_right, double *grad_w_left, double *grad_w_veh,
                             MC_OPTIONAL const double *sens_rows, MC_OPTIONAL const int32_t *n_rows,
                             MC_OPTIONAL double *schur, MC_OPTIONAL int n_rows_cap,
                             MC_OPTIONAL2 const double *lin_alpha,
                             void *workspace, size_t workspace_bytes, void *stream);

/* Fourth stage, run by mc_mincurv_solve_batch between two finalize passes: re-solves every instance flagged
 * status 4 (curvature rows violated by the box-only optimum) as the full QP tph hands to quadprog, rows
 * |k_ref + E alpha| <= kappa_bound included; leaves all other instances untouched. */
int mc_mincurv_kappa_batch(int B, int n_max, const int32_t *n_pts, double kappa_bound, double *alpha, int32_t *status,
                           int32_t *iters, void *workspace, size_t workspace_bytes, void *stream);

/* -------------------------------------------------------------------------------------------------
 * tph.opt_shortest_path.opt_shortest_path(reftrack, normvectors, w_veh, print_debug)
 * -- call site main_globaltraj.py:286-290 (SURVEY.md A.4).
 */
size_t mc_shortest_path_workspace_bytes(int B, int n_max);
int mc_shortest_path_solve_batch(int B, int n_max, const int32_t *n_pts,
                                 const double *reftrack, const double *normvec,
                                 double w_veh, const double *w_veh_batch,
                                 double *alpha, int32_t *status, int32_t *iters,
                                 void *workspace, size_t workspace_bytes, void *stream);

/* Sensitivities of this QP (batch.opt_shortest_path_diff; DESIGN.md section 3.11 has the derivation).  H and f are
 * explicit in the centre line and the normals, so alpha is differentiated with respect to all of them: x, y, w_tr_right,
 * w_tr_left, the normal vectors and w_veh.  grad_status[b] (int32):
 *   0  the solve converged (status 0): gradients are computed
 *   2, 3, -1  the solve's status (iteration cap, breakdown, unsupported size)
 *   3  also: a non-finite adjoint solution
 * Every unsupported instance gets zero gradients.  A bound clamped to 0.001 m (tph's clamp of w - w_veh / 2) does not
 * move with the widths: its width gradients are zero.
 *
 * mc_shortest_path_solve_batch_sens: mc_shortest_path_solve_batch (same arguments, bit-identical alpha, status, iters)
 * that also exports what the backward pass needs, 16 bytes per point:
 *   sens        [B][2][n_max] : lu / su and ll / sl, the final multiplier-to-slack ratios of the upper and lower bounds
 *                               (zero beyond n_pts[b] and for grad_status != 0)
 *   grad_status [B]           : see above
 *
 * mc_shortest_path_adjoint_batch: vector-Jacobian product of alpha: for an upstream gradient grad_alpha [B][n_max] of a
 * loss L,
 *   grad_reftrack [B][n_max][4]        = dL / d(x, y, w_tr_right, w_tr_left)   (x, y at fixed normals)
 *   grad_normvec  [B][n_max][2] or NULL = dL / dnormvec
 *   grad_w_veh    [B] or NULL           = dL / dw_veh per instance (the scalar w_veh's gradient is their sum)
 * reftrack, normvec, w_veh / w_veh_batch, alpha, sens and grad_status are those of the mc_shortest_path_solve_batch_sens
 * call.  One cyclic tridiagonal factorisation of H + diag(sens[0] + sens[1]) and one solve per instance in a workspace of
 * mc_shortest_path_workspace_bytes(B, n_max); nothing has to survive in it between the two calls.  grad_status is read,
 * and set to 3 where the adjoint solution is not finite. */
int mc_shortest_path_solve_batch_sens(int B, int n_max, const int32_t *n_pts,
                                      const double *reftrack, const double *normvec,
                                      double w_veh, const double *w_veh_batch,
                                      double *alpha, int32_t *status, int32_t *iters, double *sens, int32_t *grad_status,
                                      void *workspace, size_t workspace_bytes, void *stream);
int mc_shortest_path_adjoint_batch(int B, int n_max, const int32_t *n_pts,
                                   const double *reftrack, const double *normvec,
                                   double w_veh, const double *w_veh_batch,
                                   const double *alpha, const double *sens, int32_t *grad_status, const double *grad_alpha,
                                   double *grad_reftrack, double *grad_normvec, double *grad_w_veh,
                                   void *workspace, size_t workspace_bytes, void *stream);

/* -------------------------------------------------------------------------------------------------
 * tph.create_raceline.create_raceline(refline, normvectors, alpha, stepsize_interp)
 * -- call site main_globaltraj.py:371-376 (9-tuple; the dense A_raceline is replaced
 * by nothing: without distance scaling every parameter scale is 1) fused with
 * tph.calc_head_curv_an.calc_head_curv_an(coeffs_x, coeffs_y, ind_spls, t_spls)
 * -- call site main_globaltraj.py:383-387 (SURVEY.md A.6/A.7).
 *   refline [B][n_max][ref_stride] (x at +0, y at +1), normvec [B][n_max][2], alpha [B][n_max]
 *   outputs per track: coeffs_x/y [B][n_max][4], spline_lengths [B][n_max],
 *   n_out [B] (int32) and, padded to n_out_max: raceline_interp [.][2], spline_inds (int32), t_values,
 *   s_interp, el_lengths_interp, psi, kappa (psi/kappa may be NULL).
 *   A track whose n_out would exceed n_out_max gets n_out = -(required size) and no resampled output.
 */
size_t mc_create_raceline_workspace_bytes(int B, int n_max);
int mc_create_raceline_batch(int B, int n_max, const int32_t *n_pts,
                             const double *refline, int ref_stride, const double *normvec, const double *alpha,
                             double stepsize_interp, int n_out_max,
                             double *coeffs_x, double *coeffs_y, double *spline_lengths,
                             int32_t *n_out, double *raceline_interp, int32_t *spline_inds, double *t_values,
                             double *s_interp, double *el_lengths_interp, double *psi, double *kappa,
                             void *workspace, size_t workspace_bytes, void *stream);

/* Sensitivities of create_raceline (batch.create_raceline_diff; DESIGN.md section 3.12 has the derivation).
 *
 * mc_create_raceline_adjoint_workspace_bytes: 25 (n_max rounded up to 32, + 32) doubles per track.
 *
 * mc_create_raceline_adjoint_batch: vector-Jacobian product of mc_create_raceline_batch (unit parameter scales, the
 * raceline refline + alpha normvec): for upstream gradients grad_raceline [B][n_out_max][2], grad_kappa [B][n_out_max]
 * and grad_el_lengths [B][n_out_max] (each may be NULL: zero) of a loss L,
 *   grad_alpha   [B][n_max]          = dL / dalpha
 *   grad_refline [B][n_max][2] or NULL = dL / d(x, y) of the reference line
 *   grad_normvec [B][n_max][2] or NULL = dL / dnormvec
 * all zero beyond n_pts[b], and zero for a track with n_out[b] <= 0 (overflow or inactive) or n_pts[b] < 3.  n_out and the
 * segment of every station are held: coeffs_x / coeffs_y, spline_lengths, n_out, spline_inds and t_values are the
 * forward call's outputs (n_out_max its capacity); normvec and alpha its inputs. */
size_t mc_create_raceline_adjoint_workspace_bytes(int B, int n_max);
int mc_create_raceline_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *normvec, const double *alpha,
                                     int n_out_max, const double *coeffs_x, const double *coeffs_y,
                                     const double *spline_lengths, const int32_t *n_out, const int32_t *spline_inds,
                                     const double *t_values, const double *grad_raceline, const double *grad_kappa,
                                     const double *grad_el_lengths, double *grad_alpha, double *grad_refline,
                                     double *grad_normvec, void *workspace, size_t workspace_bytes, void *stream);

/* tph.calc_head_curv_an.calc_head_curv_an stand-alone (any (spline index, t) pairs), call site
 * main_globaltraj.py:383-387.  dkappa may be NULL (calc_dcurv=False). */
int mc_calc_head_curv_batch(int B, int n_max, const double *coeffs_x, const double *coeffs_y,
                            int n_eval_max, const int32_t *n_eval, const int32_t *ind_spls, const double *t_spls,
                            double *psi, double *kappa, double *dkappa, void *stream);

/* -------------------------------------------------------------------------------------------------
 * One re-linearisation step of tph.iqp_handler.iqp_handler (call site
 * main_globaltraj.py:273-284, SURVEY.md A.5): given alpha on the current reftrack,
 * build the next reftrack on the re-sampled raceline (create_raceline with stepsize_interp, widths
 * shifted by alpha and interpolated linearly in t) and its splines without distance scaling.
 *   in : reftrack [B][n_max][4], normvec [B][n_max][2], alpha [B][n_max], n_pts [B]
 *   out: reftrack_new [B][n_max_new][4], normvec_new [B][n_max_new][2], n_pts_new [B]
 *        (n_pts_new[b] = -(required) if it would exceed n_max_new)
 *   active [B] (int32) or NULL: tracks with active[b] == 0 are copied through unchanged.
 */
size_t mc_iqp_relinearise_workspace_bytes(int B, int n_max, int n_max_new);
int mc_iqp_relinearise_batch(int B, int n_max, const int32_t *n_pts, const int32_t *active,
                             const double *reftrack, const double *normvec, const double *alpha,
                             double stepsize_interp, int n_max_new,
                             double *reftrack_new, double *normvec_new, int32_t *n_pts_new,
                             void *workspace, size_t workspace_bytes, void *stream);

/* alpha[b][:] *= scale_batch[b] (or the scalar `scale` when scale_batch is NULL): the damping
 * `alpha *= iter / iters_min` of tph.iqp_handler (SURVEY.md A.5). */
int mc_scale_alpha_batch(int B, int n_max, double *alpha, const double *scale_batch, double scale, void *stream);

/* -------------------------------------------------------------------------------------------------
 * tph.calc_vel_profile.calc_vel_profile(ggv, ax_max_machines, v_max, kappa, el_lengths, closed=True, filt_window,
 * dyn_model_exp, drag_coeff, m_veh[, mu]) followed by tph.calc_ax_profile.calc_ax_profile(vx_cl, el_lengths) and
 * tph.calc_t_profile.calc_t_profile(vx, ax, el_lengths) -- call sites main_globaltraj.py:400-421
 * -- for B closed racelines x V variants per raceline.  A variant is one cell of the reference's lap-time
 * matrix (main_globaltraj.py:442-496): ggv_mod[:, 1:] = ggv[:, 1:] * ggv_scale[v], v_max = v_max_batch[v].
 *   kappa, el_lengths [B][n_max] : curvature and element lengths of the (re-sampled) raceline, n_pts[b] valid entries
 *                                  (the kappa / el_lengths_interp outputs of mc_create_raceline_batch, n_pts = n_out)
 *   mu [B][n_max] or NULL        : friction scaling per point (NULL => ones)
 *   ggv_scale [V] or NULL (=> 1), v_max_batch [V] or NULL (=> the scalar v_max)
 *   ggv [n_ggv][3] (v, ax_max, ay_max), ax_max_machines [n_mach][2] (v, ax): device arrays, <= 256 rows each
 *   filt_window                  : odd width of tph's moving-average filter, <= 1 => none (filt_window=None)
 *   outputs (profile p = b * V + v): vx [B*V][n_max], ax [B*V][n_max], t [B*V][n_max + 1] (each may be NULL),
 *   laptime [B*V] (= t[n_pts]), status [B*V] (0 ok, 3 non-finite result) or NULL
 * workspace: mc_vel_profile_workspace_bytes(B, V, n_max)
 */
#define MC_VP_VEHICLES (-1)
/* The vehicles of a call with n_ggv = MC_VP_VEHICLES (in host memory; every pointer in it is a device array):
 * K = n_veh >= 1 vehicles, their tables back to back in ggv [n_ggv][3] (v, ax_max, ay_max) and ax_max_machines
 * [n_mach][2] (v, ax); veh_rows [K + 1][2] the prefix row offsets (vehicle k has ggv rows veh_rows[k][0] ..
 * veh_rows[k + 1][0] - 1 and machine rows veh_rows[k][1] .. veh_rows[k + 1][1] - 1, 1 to 256 of each); veh_par [K][3]
 * its v_max, drag_coeff, m_veh; veh_id [B] the vehicle of each track of the call. */
typedef struct {
    int n_veh, n_ggv, n_mach;
    const double *ggv, *ax_max_machines;
    const int32_t *veh_rows;
    const double *veh_par;
    const int32_t *veh_id;
} mc_vp_vehicles;
size_t mc_vel_profile_workspace_bytes(int B, int V, int n_max);
int mc_vel_profile_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                         const double *mu, int V, const double *ggv_scale, const double *v_max_batch, double v_max,
                         int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines,
                         double dyn_model_exp, double drag_coeff, double m_veh, int filt_window,
                         double *vx, double *ax, double *t, double *laptime, int32_t *status,
                         void *workspace, size_t workspace_bytes, void *stream);
/* The same with an explicit decel_slice_upper (see MC_VP_DECEL_SLICE_UPPER_DEFAULT) and, optionally, the
 * vector-Jacobian product of the lap times (the lap-time matrix for V > 1; batch.lap_time_matrix_diff, DESIGN.md
 * section 3.12):
 *   grad_laptime [B][V] or NULL : NULL => the forward above, nothing else is read or written.  Otherwise the upstream
 *                                 gradient dL/dlaptime of a loss L, and the call writes only
 *   grad_kappa [B][n_max] or NULL, grad_el_lengths [B][n_max] or NULL : dL/dkappa, dL/del_lengths, the sum of the V
 *                                 profiles' gradients of a track in variant order (zero beyond n_pts[b]);
 *   grad_status [B][V] (required) : per profile, the codes of mc_vel_profile_adjoint_batch below (a profile whose code
 *                                 is not 0 adds nothing to its track's sum).
 *   In this mode vx, ax, t, laptime and status are not written (they may be NULL), mu must be NULL (the adjoint has no
 *   mu), and the forward is run again inside: the other arguments are those of the forward call.
 * workspace: mc_vel_profile_workspace_bytes(B, V, n_max) for the forward,
 *            mc_vel_profile_adjoint_workspace_bytes(B * V, n_max) with grad_laptime (the tape of every profile; the
 *            sum over the variants reads it and needs nothing more)
 *
 * A vehicle per track (here, in mc_vel_profile_batch, which forwards to this entry, and in
 * mc_vel_profile_adjoint_batch): n_ggv = MC_VP_VEHICLES and ggv = (const double *) a HOST pointer to an mc_vp_vehicles
 * below, which the entry reads before it returns; n_mach and ax_max_machines are then not read, nor are the scalar
 * v_max, drag_coeff and m_veh.  A variant's top speed is v_max_batch[v] if given, else its vehicle's v_max;
 * ggv_scale[v] scales its vehicle's ggv.  A track's results are bit for bit those of a call with its vehicle's tables
 * and scalars alone.  A track whose veh_id is outside 0 .. n_veh - 1, or whose vehicle has rows outside the tables or
 * outside 1 .. 256, m_veh <= 0 or (without v_max_batch) v_max <= 0, is refused alone: lap time 0, zero gradients and
 * status / grad_status 5 (an inactive slot, n_pts 0, stays status 0).  The workspace sizes are those above (the
 * kernels read the tables in place). */
int mc_vel_profile_batch_ex(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                            const double *mu, int V, const double *ggv_scale, const double *v_max_batch, double v_max,
                            int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines,
                            double dyn_model_exp, double drag_coeff, double m_veh, int filt_window, int decel_slice_upper,
                            double *vx, double *ax, double *t, double *laptime, int32_t *status,
                            const double *grad_laptime, double *grad_kappa, double *grad_el_lengths,
                            int32_t *grad_status, void *workspace, size_t workspace_bytes, void *stream);

/* Sensitivities of the lap time (batch.vel_profile_diff; DESIGN.md section 3.12 has the derivation).  The velocity
 * profile (closed track, ggv branch, one profile per track, no mu) is differentiated with respect to kappa and el_lengths
 * as the forward evaluates it, with every discrete decision frozen as the forward took it.  grad_status[b] (int32):
 *   0  the gradient is computed
 *   3  non-finite lap time (the forward's status) or a non-finite gradient
 *   for n_pts[b] < 2 (an inactive slot) the forward's status (0 for n_pts 0, 3 otherwise)
 * Every such instance gets zero gradients.
 *
 * mc_vel_profile_adjoint_workspace_bytes: 17 n_max + 1 doubles per profile (the forward's scratch vectors, its tape and
 * the adjoint vectors); B here counts profiles (B * V for mc_vel_profile_batch_ex).
 *
 * mc_vel_profile_adjoint_batch: vector-Jacobian product of mc_vel_profile_batch_ex with V = 1 (no ggv scales, no
 * per-variant top speed, no mu): for upstream gradients grad_laptime [B] and grad_vx [B][n_max] (either may be NULL:
 * zero) of a loss L,
 *   grad_kappa      [B][n_max] or NULL = dL / dkappa
 *   grad_el_lengths [B][n_max] or NULL = dL / del_lengths
 * both zero beyond n_pts[b].  The other arguments are those of the forward call; the forward is run again inside (its
 * outputs are not inputs here).  n_ggv = MC_VP_VEHICLES: a vehicle per track, as for mc_vel_profile_batch_ex. */
size_t mc_vel_profile_adjoint_workspace_bytes(int B, int n_max);
int mc_vel_profile_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                                 double v_max, int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines,
                                 double dyn_model_exp, double drag_coeff, double m_veh, int filt_window,
                                 int decel_slice_upper, const double *grad_laptime, const double *grad_vx,
                                 double *grad_kappa, double *grad_el_lengths, int32_t *grad_status,
                                 void *workspace, size_t workspace_bytes, void *stream);

/* tph.calc_ax_profile.calc_ax_profile(vx_profile, el_lengths, eq_length_output=False) and
 * tph.calc_t_profile.calc_t_profile(vx_profile, el_lengths, t_start, ax_profile) stand-alone
 * (call sites main_globaltraj.py:413-421) for P profiles.
 *   vx [P][vx_pitch] (vx_pitch >= n_max + 1 when ax_in is NULL: ax is derived from vx[0..n]), el_lengths [P][n_max],
 *   ax_in [P][n_max] or NULL, ax_out [P][n_max] or NULL, t_out [P][n_max + 1] or NULL (t_out[0] = t_start).
 */
int mc_calc_ax_t_profile_batch(int P, int n_max, const int32_t *n_pts, const double *vx, int vx_pitch,
                               const double *el_lengths, const double *ax_in, double t_start,
                               double *ax_out, double *t_out, void *stream);

/* -------------------------------------------------------------------------------------------------
 * The reference's in-tree trajectory back end (these helpers live in the reference tree itself, so their fixtures are
 * produced by the reference's own code -- tools/make_golden_ref.py).
 *
 * helper_funcs_glob.src.interp_track.interp_track(reftrack, stepsize_approx)
 * -- helper_funcs_glob/src/interp_track.py:5-49; call sites prep_track.py:32-34 (the imported track) and
 * check_traj.py:58-61 (the boundary polylines).  Linear re-sampling of a closed polyline at equal arc length.
 *   pts [B][n_max][stride] (stride 2: x, y; stride 4: x, y, w_tr_right, w_tr_left), n_pts [B] or NULL
 *   normvec [B][n_max][2] or NULL: if given, the polyline is pts.xy + normal_sign * normvec * pts[width_col]
 *     (check_traj.py:50-51: bound_r = +normvec * w_tr_right (width_col 2), bound_l = -normvec * w_tr_left (width_col 3))
 *     and the two width columns of the output are zero, as in check_traj.py:54-55
 *   out [B][n_out_max][4], n_out [B]: points written (the closing point is dropped); -(required) if > n_out_max
 * workspace: mc_interp_track_workspace_bytes(B, n_max)
 */
size_t mc_interp_track_workspace_bytes(int B, int n_max);
int mc_interp_track_batch(int B, int n_max, const int32_t *n_pts, const double *pts, int stride, const double *normvec,
                          double normal_sign, int width_col, double stepsize_approx, int n_out_max, double *out,
                          int32_t *n_out, void *workspace, size_t workspace_bytes, void *stream);

/* helper_funcs_glob.src.calc_min_bound_dists.calc_min_bound_dists(trajectory, bound1, bound2, length_veh, width_veh)
 * -- helper_funcs_glob/src/calc_min_bound_dists.py:5-66, call site check_traj.py:64-68: for every
 * trajectory point the smallest distance of the four vehicle corners (vehicle heading = psi) to any boundary point.
 *   xy [B][n_traj_max][2], psi [B][n_traj_max], n_traj [B] or NULL
 *   bound1/bound2 [B][nb*_max][bound_stride] (x at +0, y at +1), nb1/nb2 [B] or NULL
 *   min_dists [B][n_traj_max]
 */
int mc_min_bound_dists_batch(int B, int n_traj_max, const int32_t *n_traj, const double *xy, const double *psi,
                             int nb1_max, const int32_t *nb1, const double *bound1, int nb2_max, const int32_t *nb2,
                             const double *bound2, int bound_stride, double length_veh, double width_veh,
                             double *min_dists, void *stream);

/* The quantities helper_funcs_glob.src.check_traj.check_traj compares with its limits
 * (helper_funcs_glob/src/check_traj.py:74-139; call site main_globaltraj.py:520-532), per trajectory:
 *   extrema [B][8] = min(min_dists) (inf if min_dists is NULL), max |kappa|, max ay = vx^2 / radius,
 *                    max and min of ax_wo_drag = ax + vx^2 dragcoeff / mass_veh, max sqrt(ax_wo_drag^2 + ay^2), max vx,
 *                    number of points
 */
int mc_traj_extrema_batch(int B, int n_max, const int32_t *n_traj, const double *kappa, const double *vx, const double *ax,
                          const double *min_dists, double dragcoeff, double mass_veh, double *extrema, void *stream);

/* trajectory_opt / traj_race_cl of main_globaltraj.py:501-512: rows [s, x, y, psi, kappa, vx, ax];
 * row n_traj[b] closes the lap (copy of row 0 with s = sum(spline_lengths)).  traj [B][n_max + 1][7].
 */
int mc_assemble_trajectory_batch(int B, int n_max, const int32_t *n_traj, const double *s, const double *xy,
                                 const double *psi, const double *kappa, const double *vx, const double *ax,
                                 int n_spl_max, const int32_t *n_spl, const double *spline_lengths, double *traj,
                                 void *stream);

/* tph.check_normals_crossing.check_normals_crossing(track, normvec_normalized, horizon)
 * -- call site helper_funcs_glob/src/prep_track.py:57-59: do normals of points at most `horizon` apart
 * cross inside the track (which would make the QP's parametrisation ambiguous)?
 *   track [B][n_max][4] (x, y, w_tr_right, w_tr_left), normvec [B][n_max][2], crossing [B] (int32): 1 = crossing found
 *   tracks with n_pts[b] <= horizon are left at 0 (tph raises for them; the Python surface does too)
 */
int mc_check_normals_crossing_batch(int B, int n_max, const int32_t *n_pts, const double *track, const double *normvec,
                                    int horizon, int32_t *crossing, void *stream);

/* -------------------------------------------------------------------------------------------------
 * Sweep inputs generated on the device (no counterpart in tph: the reference builds its parameter sweeps in Python
 * loops around one prepared track, main_globaltraj.py:442-496): V width-jitter variants of n_base
 * prepared tracks, w <- w (1 + rel g(s)) with a smooth g, |g| <= 1, drawn from the 64-bit seed of the variant by a
 * stateless hash (splitmix64) that global_racetrajectory_optimization_b200/synth.py mirrors in numpy.
 *   base [n_base][n_max][4], n_pts_base [n_base] or NULL, centre_id [V] (int32) or NULL => variant v uses track v % n_base,
 *   seed [V] (int64), out [V][n_max][4], n_pts_out [V] or NULL
 */
int mc_jitter_widths_batch(int V, int n_max, const int32_t *n_pts_base, int n_base, const double *base,
                           const int32_t *centre_id, const int64_t *seed, double rel, double *out, int32_t *n_pts_out,
                           void *stream);

/* -------------------------------------------------------------------------------------------------
 * tph.spline_approximation.spline_approximation(track, k_reg, s_reg, stepsize_prep, stepsize_reg) followed by prep_track's
 * min-width inflation -- call sites helper_funcs_glob/src/prep_track.py:39-45 and :89-98 (SURVEY.md 8f-2).
 * Every statement of tph.spline_approximation is kept except scipy's splprep (FITPACK), which is replaced by the periodic
 * cubic smoothing spline of Reinsch with the same residual budget s_reg (see csrc/prep_track.cu; the distance to the
 * FITPACK route is reported by tests/test_gpu_prep.py).
 *   track [B][n_raw_max][4]       : imported tracks x, y, w_tr_right, w_tr_left (unclosed), n_raw[b] points each
 *   n_int_max                     : capacity for the pre-interpolated closed track (>= ceil(length / stepsize_prep) + 1)
 *   min_width                     : <= 0 => no inflation (prep_track's min_width=None)
 *   reftrack_interp [B][n_out_max][4], n_out [B]: the prepared tracks, with n_out[b] telling three outcomes apart:
 *     n_out[b] >= 0                          points written (0: an inactive slot, n_raw[b] == 0)
 *     -MC_PREP_REFUSED < n_out[b] < 0        a capacity is too small: -(points needed) for n_int_max or n_out_max
 *     n_out[b] == -MC_PREP_REFUSED - reason  the track is refused (nothing is written to its row), reason one of
 *                                            MC_PREP_R_*; every count the kernel needs is below MC_PREP_REFUSED
 *   smoothing_lambda [B] or NULL  : the smoothing parameter found for every track (0 if refused before the fit)
 */
#define MC_PREP_REFUSED (1 << 30)
#define MC_PREP_R_N_RAW 1         /* n_raw[b] < 0 or n_raw[b] > n_raw_max */
#define MC_PREP_R_TOO_FEW 2       /* 1 <= n_raw[b] < 5, or fewer than 5 points after the pre-interpolation */
#define MC_PREP_R_NONFINITE 3     /* a coordinate or width is inf or NaN, or a length overflows */
#define MC_PREP_R_COUNT 4         /* a point count (length / step) does not fit below MC_PREP_REFUSED */
#define MC_PREP_R_BUDGET 5        /* the residual budget s_reg is not reached: s_reg >= F(inf), or the bracket or the
                                     iteration cap of the root search runs out */
#define MC_PREP_R_FEW_OUT 6       /* fewer than 3 re-sampled points */
size_t mc_prep_track_workspace_bytes(int B, int n_raw_max, int n_int_max);
int mc_prep_track_batch(int B, int n_raw_max, const int32_t *n_raw, const double *track, int k_reg, double s_reg,
                        double stepsize_prep, double stepsize_reg, double min_width, int n_int_max, int n_out_max,
                        double *reftrack_interp, int32_t *n_out, double *smoothing_lambda, void *workspace,
                        size_t workspace_bytes, void *stream);

/* Length [B] of the closed polygon through the first n_pts[b] points of every track; with normvec and shift the points are
 * p_i + sign * shift_i * n_i (shift: alpha [B][n_max] with shift_stride 1, or a width column &track[0][0][2] with
 * shift_stride 4).  Used by the host to size the re-sampling buffers of create_raceline / interp_track / iqp_handler. */
int mc_polygon_length_batch(int B, int n_max, const int32_t *n_pts, const double *pts, int stride, const double *normvec,
                            const double *shift, int shift_stride, double sign, double *length, void *stream);

/* tph.iqp_handler's per-track termination test (SURVEY.md A.5; call site main_globaltraj.py:273-284) for
 * outer iteration `iter` (1-based): an active track is finished when iter >= iters_min and curv_error_max <=
 * curv_error_allowed, when its QP failed (status != 0), or when iter >= iter_limit (then fin_status = 2: cap reached before
 * the tolerance).  fixed_iters > 0 replaces the test by iter >= fixed_iters.  Finished tracks get their alpha / reftrack /
 * normvec rows of this iteration copied into the fin_* buffers (row pitch n_cap >= n_max) and active[b] = 0.
 * counters [2] (int32, device): [0] tracks still active afterwards, [1] tracks finished by this call. */
int mc_iqp_finish_batch(int B, int n_max, int n_cap, int iter, int iters_min, double curv_error_allowed, int fixed_iters,
                        int iter_limit, int32_t *active, const int32_t *status, const double *curv_error_max,
                        const int32_t *n_pts, const double *alpha, const double *reftrack, const double *normvec,
                        double *fin_alpha, double *fin_reftrack, double *fin_normvec, int32_t *fin_n_pts,
                        int32_t *fin_outer_iters, int32_t *fin_status, double *fin_curv_error_max, int32_t *counters,
                        void *stream);

/* Debug aid (synchronous): reads (and optionally clears) 24 cycle counters that CTA 0 of mincurv_pdip_kernel
 * accumulates per phase -- used by tools/prof_run.py to attribute time inside the kernel. Host pointer. */
int mc_debug_read_profile(unsigned long long *host_out24, int reset);

/* Debug aid (tests/test_gpu_factor.py): runs the linear algebra of one interior-point iteration of
 * mincurv_pdip_kernel -- the bordered LDL^T factorisation of M = H + D and both kinds of solve -- on slabs whose
 * H band, D (slab vector DD), and right-hand sides (slab vectors RHS, T0) the caller has filled in; the solutions
 * M^-1 RHS, M^-1 T0 (full sweeps), M^-1 T0 (forward sweep fused into a second factorisation) are left in the slab
 * vectors DX, T1, T2.  status[b] = 3 on a non-positive pivot.  Workspace as for mc_mincurv_solve_batch. */
int mc_debug_factor_solve(int B, int n_max, const int32_t *n_pts, int32_t *status, void *workspace, size_t workspace_bytes,
                          void *stream);

#ifdef __cplusplus
}
#endif
#endif /* MINCURV_B200_H */
