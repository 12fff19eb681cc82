// extern "C" boundary of libmincurv_b200.so -- see include/mincurv_b200.h for the contract and the
// reference call sites each entry point replaces.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../include/mincurv_b200.h"
#include "mincurv_ws.cuh"

namespace mc {
size_t spline_ws_doubles(int n_max);
int pdip_ctas_per_sm();
int pdip_kappa_ctas_per_sm();
int debug_factor_solve_ctas_per_sm();
int adjoint_ctas_per_sm();
int launch_mincurv_adjoint(int, int, const int32_t *, const double *, double, const double *, double *, const Layout &,
                           const double *, const double *, int32_t *, double *, double *, double *, int, int *, cudaStream_t);
void launch_mincurv_sens_export(int, int, const int32_t *, double *, const Layout &, const int32_t *, double *, int32_t *,
                                cudaStream_t);
int launch_debug_factor_solve(int, int, const int32_t *, double *, const Layout &, int32_t *, int, cudaStream_t);
int debug_read_profile(unsigned long long *, int);
void launch_mincurv_setup(int, int, const int32_t *, const double *, const double *, const double *, double,
                          const double *, double, const int32_t *, double *, const Layout &, int32_t *, cudaStream_t);
int launch_mincurv_pdip(int, int, const int32_t *, double *, const Layout &, const PdipParams &, int, double *, int32_t *,
                        int32_t *, int, int *, cudaStream_t);
int launch_mincurv_pdip_kappa(int, int, const int32_t *, double *, const Layout &, const PdipParams &, double, double *,
                              int32_t *, int32_t *, int, int *, cudaStream_t);
void launch_mincurv_finalize(int, int, const int32_t *, double *, const Layout &, const double *, double, double *,
                             double *, int32_t *, cudaStream_t);
void launch_calc_splines(int, int, const int32_t *, const double *, int, const double *, int, double *, double *,
                         double *, double *, double *, cudaStream_t);
void launch_create_raceline(int, int, const int32_t *, const double *, int, const double *, const double *, double, int,
                            double *, double *, double *, int32_t *, double *, int32_t *, double *, double *, double *,
                            double *, double *, double *, cudaStream_t);
void launch_head_curv(int, int, const double *, const double *, int, const int32_t *, const int32_t *, const double *,
                      double *, double *, double *, cudaStream_t);
void launch_iqp_new_reftrack(int, int, const int32_t *, const int32_t *, const double *, const double *, const double *,
                             int, const int32_t *, const double *, const int32_t *, const double *, double *, double *,
                             int32_t *, cudaStream_t);
void launch_scale_alpha(int, int, double *, const double *, double, cudaStream_t);
void launch_iqp_finish(int, int, int, int, int, double, int, int, int32_t *, const int32_t *, const double *, const int32_t *,
                       const double *, const double *, const double *, double *, double *, double *, int32_t *, int32_t *,
                       int32_t *, double *, int32_t *, cudaStream_t);
size_t shortest_path_ws_doubles(int n_max);
int launch_shortest_path(int, int, const int32_t *, const double *, const double *, double, const double *, double *,
                         int32_t *, int32_t *, double *, cudaStream_t);
void launch_shortest_path_sens_export(int, int, const int32_t *, const int32_t *, const double *, double *, int32_t *,
                                      cudaStream_t);
void launch_shortest_path_adjoint(int, int, const int32_t *, const double *, const double *, double, const double *,
                                  const double *, const double *, int32_t *, const double *, double *, double *, double *,
                                  double *, cudaStream_t);
size_t vel_profile_ws_doubles(int n_max);
int launch_vel_profile(int, int, int, const int32_t *, const double *, const double *, const double *, const double *,
                       const double *, double, int, const double *, int, const double *, double, double, double, int, int,
                       double *, double *, double *, double *, int32_t *, double *, cudaStream_t);
void launch_ax_t_profile(int, int, const int32_t *, const double *, int, const double *, const double *, double, double *,
                         double *, cudaStream_t);
size_t vel_profile_adjoint_ws_doubles(int n_max);
size_t create_raceline_adjoint_ws_doubles(int n_max);
void launch_create_raceline_adjoint(int, int, const int32_t *, const double *, const double *, int, const double *,
                                    const double *, const double *, const int32_t *, const int32_t *, const double *,
                                    const double *, const double *, const double *, double *, double *, double *, double *,
                                    cudaStream_t);
int launch_vel_profile_adjoint(int, int, const int32_t *, const double *, const double *, double, int, const double *, int,
                               const double *, double, double, double, int, int, const double *, const double *, double *,
                               double *, int32_t *, double *, cudaStream_t);
size_t interp_track_ws_doubles(int n_max);
void launch_interp_track(int, int, const int32_t *, const double *, int, const double *, double, int, double, int, double *,
                         int32_t *, double *, cudaStream_t);
void launch_min_bound_dists(int, int, const int32_t *, const double *, const double *, int, const int32_t *, const double *,
                            int, const int32_t *, const double *, int, double, double, double *, cudaStream_t);
void launch_traj_extrema(int, int, const int32_t *, const double *, const double *, const double *, const double *, double,
                         double, double *, cudaStream_t);
void launch_assemble_trajectory(int, int, const int32_t *, const double *, const double *, const double *, const double *,
                                const double *, const double *, int, const int32_t *, const double *, double *, cudaStream_t);
void launch_normals_crossing(int, int, const int32_t *, const double *, const double *, int, int32_t *, cudaStream_t);
size_t prep_track_ws_doubles(int, int);
void launch_prep_track(int, int, const int32_t *, const double *, double, double, double, double, int, int, double *, int32_t *,
                       double *, double *, cudaStream_t);
void launch_polygon_length(int, int, const int32_t *, const double *, int, const double *, const double *, int, double, double *,
                           cudaStream_t);
void launch_jitter_widths(int, int, const int32_t *, int, const double *, const int32_t *, const int64_t *, double, double *,
                          int32_t *, cudaStream_t);
}  // namespace mc

static thread_local char g_err[256] = "";

static int check_cuda(const char *what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        snprintf(g_err, sizeof(g_err), "%s: %s", what, cudaGetErrorString(e));
        return MC_ECUDA;
    }
    return MC_OK;
}
__attribute__((format(printf, 1, 2))) static int bad(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return MC_EINVAL;
}
static int small_workspace(const char *who) {
    snprintf(g_err, sizeof(g_err), "%s: workspace too small", who);
    return MC_EWORKSPACE;
}
static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
static constexpr int PDIP_SLICE_DEFAULT = 8;      // DESIGN.md section 3.3: the predictor of the remaining iterations is
                                                  // no better than chance after 4 iterations, within one iteration after 8

extern "C" {

int mc_version(void) { return 100; }
const char *mc_last_error(void) { return g_err; }

// ------------------------------------------------------------------------------------------------
size_t mc_calc_splines_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max <= 0) return 0;
    return align256((size_t)B * mc::spline_ws_doubles(n_max) * sizeof(double));
}

int mc_calc_splines_batch(int B, int n_max, const int32_t *n_pts, const double *xy, int xy_stride,
                          const double *el_lengths, int use_dist_scaling, double *coeffs_x, double *coeffs_y,
                          double *normvec, double *h_out, void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 3 || !xy || (xy_stride != 2 && xy_stride != 4)) return bad("mc_calc_splines_batch: bad argument");
    if ((coeffs_x == nullptr) != (coeffs_y == nullptr)) return bad("mc_calc_splines_batch: coeffs_x/coeffs_y must both be given or both NULL");
    if (!workspace || workspace_bytes < mc_calc_splines_workspace_bytes(B, n_max))
        return small_workspace("mc_calc_splines_batch");
    mc::launch_calc_splines(B, n_max, n_pts, xy, xy_stride, el_lengths, use_dist_scaling, coeffs_x, coeffs_y, normvec,
                            h_out, (double *)workspace, (cudaStream_t)stream);
    return check_cuda("mc_calc_splines_batch");
}

// ------------------------------------------------------------------------------------------------
static size_t mincurv_slabs_bytes(int B, int n_max) { return align256((size_t)B * mc::make_layout(n_max).stride * sizeof(double)); }

static_assert(mc::SCHED_INTS * sizeof(int) <= 256, "the counters behind the slabs");
size_t mc_mincurv_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < mc::N_MIN) return 0;
    return mincurv_slabs_bytes(B, n_max) + 256;      // + the work counters of the persistent solver kernels (SCHED_INTS)
}

static int mincurv_args(const char *who, int B, int n_max, void *workspace, size_t workspace_bytes) {
    if (B <= 0) return bad("mincurv: B <= 0");
    if (n_max < mc::N_MIN) return bad("mincurv: n_max below the supported minimum (%d points)", mc::N_MIN);
    if (!workspace || workspace_bytes < mc_mincurv_workspace_bytes(B, n_max)) return small_workspace(who);
    return MC_OK;
}

// launch shape of a persistent solver kernel: per_sm resident CTAs on every SM, but no more CTAs than instances; the counter
// that hands out the instances sits behind the slabs
struct SolverGrid {
    int grid;
    int *counter;
};
static SolverGrid solver_grid(int B, int n_max, void *workspace, int per_sm) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int grid = sms * (per_sm > 0 ? per_sm : 1);
    if (grid > B) grid = B;
    return {grid, (int *)((char *)workspace + mincurv_slabs_bytes(B, n_max))};
}

int mc_mincurv_setup_batch_shared(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                  const double *h, double w_veh, const double *w_veh_batch, double f_scale,
                                  const int32_t *centre_id, int32_t *status, void *workspace, size_t workspace_bytes,
                                  void *stream) {
    if (!reftrack || !normvec || !h || !status) return bad("mc_mincurv_setup_batch: NULL argument");
    if (!(f_scale > 0.0)) return bad("mc_mincurv_setup_batch: f_scale must be positive");
    int rc = mincurv_args("mc_mincurv_setup_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    mc::launch_mincurv_setup(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, (double *)workspace,
                             mc::make_layout(n_max), status, (cudaStream_t)stream);
    return check_cuda("mincurv_setup_kernel");
}

int mc_mincurv_setup_batch_ex(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double w_veh, const double *w_veh_batch, double f_scale, int32_t *status,
                              void *workspace, size_t workspace_bytes, void *stream) {
    return mc_mincurv_setup_batch_shared(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, nullptr, status,
                                         workspace, workspace_bytes, stream);
}

int mc_mincurv_setup_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                           const double *h, double w_veh, const double *w_veh_batch, int32_t *status, void *workspace,
                           size_t workspace_bytes, void *stream) {
    return mc_mincurv_setup_batch_ex(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, MC_F_SCALE_DEFAULT, status,
                                     workspace, workspace_bytes, stream);
}

int mc_mincurv_pdip_batch(int B, int n_max, const int32_t *n_pts, double *alpha, int32_t *status, int32_t *iters,
                          void *workspace, size_t workspace_bytes, void *stream) {
    if (!alpha || !status) return bad("mc_mincurv_pdip_batch: NULL argument");
    int rc = mincurv_args("mc_mincurv_pdip_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    mc::PdipParams prm;
    prm.max_iter = 40;
    prm.mu_rel = 1e-10;
    prm.rd_rel = 1e-8;
    prm.eta = 0.995;
    prm.dx_rel = 1e-5;
    prm.lam0_rel = 1e-2;
    if (const char *e = getenv("MC_DEBUG_PDIP_LAM0")) { const double v = atof(e); if (v > 0.0) prm.lam0_rel = v; }   // start-point experiments only
    if (const char *e = getenv("MC_DEBUG_PDIP_ETA")) { const double v = atof(e); if (v > 0.5 && v < 1.0) prm.eta = v; }
    if (const char *e = getenv("MC_DEBUG_PDIP_DX_REL")) { const double v = atof(e); if (v >= 0.0) prm.dx_rel = v; }
    if (const char *e = getenv("MC_DEBUG_PDIP_MU_REL")) { const double v = atof(e); if (v > 0.0) prm.mu_rel = v; }   // tolerance experiments only
    int per_sm = mc::pdip_ctas_per_sm();
    if (const char *e = getenv("MC_DEBUG_PDIP_CTAS_PER_SM")) {      // occupancy experiments only (tools/prof_run.py)
        const int v = atoi(e);
        if (v > 0 && v < per_sm) per_sm = v;
    }
    // iterations before an instance is parked in the sliced schedule (DESIGN.md section 3.3); 0: every instance to the end
    int slice = PDIP_SLICE_DEFAULT;
    if (const char *e = getenv("MC_DEBUG_PDIP_SLICE")) { const int v = atoi(e); if (v >= 0) slice = v; }   // A/B runs and tests
    const SolverGrid g = solver_grid(B, n_max, workspace, per_sm);
    if (mc::launch_mincurv_pdip(B, n_max, n_pts, (double *)workspace, mc::make_layout(n_max), prm, slice, alpha, status, iters,
                                g.grid, g.counter, (cudaStream_t)stream) != 0) {
        snprintf(g_err, sizeof(g_err), "mincurv_pdip_kernel: cudaFuncSetAttribute failed");
        return MC_ECUDA;
    }
    return check_cuda("mincurv_pdip_kernel");
}

int mc_mincurv_finalize_batch(int B, int n_max, const int32_t *n_pts, const double *alpha, double kappa_bound,
                              double *curv_error_max, double *kappa_lin_max, int32_t *status, void *workspace,
                              size_t workspace_bytes, void *stream) {
    if (!alpha || !curv_error_max || !status) return bad("mc_mincurv_finalize_batch: NULL argument");
    int rc = mincurv_args("mc_mincurv_finalize_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    mc::launch_mincurv_finalize(B, n_max, n_pts, (double *)workspace, mc::make_layout(n_max), alpha, kappa_bound,
                                curv_error_max, kappa_lin_max, status, (cudaStream_t)stream);
    return check_cuda("mincurv_finalize_kernel");
}

int mc_mincurv_solve_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                           const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double *alpha,
                           double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                           void *workspace, size_t workspace_bytes, void *stream) {
    return mc_mincurv_solve_batch_ex(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, MC_F_SCALE_DEFAULT,
                                     alpha, curv_error_max, kappa_lin_max, status, iters, workspace, workspace_bytes, stream);
}

int mc_mincurv_solve_batch_ex(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                              double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                              void *workspace, size_t workspace_bytes, void *stream) {
    return mc_mincurv_solve_batch_shared(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, nullptr,
                                         alpha, curv_error_max, kappa_lin_max, status, iters, workspace, workspace_bytes, stream);
}

// setup -> pdip -> finalize -> (export of the sensitivity data) -> kappa -> finalize; sens == NULL: no export.  Every
// argument is checked before the first launch: the pointers here, f_scale and the sizes by the setup stage.
static int mincurv_solve(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec, const double *h,
                         double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                         double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                         double *sens, int32_t *grad_status, void *workspace, size_t workspace_bytes, void *stream) {
    if (!reftrack || !normvec || !h || !alpha || !curv_error_max || !status)
        return bad("mc_mincurv_solve_batch: NULL argument");
    int rc = mc_mincurv_setup_batch_shared(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, status,
                                           workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc_mincurv_pdip_batch(B, n_max, n_pts, alpha, status, iters, workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc_mincurv_finalize_batch(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, workspace,
                                   workspace_bytes, stream);
    if (rc) return rc;
    if (sens) {
        // the box phase's final iterate, before the curvature-row phase takes over the status-4 slabs
        mc::launch_mincurv_sens_export(B, n_max, n_pts, (double *)workspace, mc::make_layout(n_max), status, sens, grad_status,
                                       (cudaStream_t)stream);
        rc = check_cuda("mincurv_sens_export_kernel");
        if (rc) return rc;
    }
    // instances whose box-only optimum violates the curvature rows (status 4) are re-solved with the rows
    rc = mc_mincurv_kappa_batch(B, n_max, n_pts, kappa_bound, alpha, status, iters, workspace, workspace_bytes, stream);
    if (rc) return rc;
    return mc_mincurv_finalize_batch(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, workspace,
                                     workspace_bytes, stream);
}

int mc_mincurv_solve_batch_shared(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                  const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                  const int32_t *centre_id, double *alpha, double *curv_error_max, double *kappa_lin_max,
                                  int32_t *status, int32_t *iters, void *workspace, size_t workspace_bytes, void *stream) {
    return mincurv_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, centre_id, alpha,
                         curv_error_max, kappa_lin_max, status, iters, nullptr, nullptr, workspace, workspace_bytes, stream);
}

int mc_mincurv_solve_batch_sens(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                const int32_t *centre_id, double *alpha, double *curv_error_max, double *kappa_lin_max,
                                int32_t *status, int32_t *iters, double *sens, int32_t *grad_status, void *workspace,
                                size_t workspace_bytes, void *stream) {
    if (!sens || !grad_status) return bad("mc_mincurv_solve_batch_sens: NULL argument");
    return mincurv_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, centre_id, alpha,
                         curv_error_max, kappa_lin_max, status, iters, sens, grad_status, workspace, workspace_bytes, stream);
}

int mc_mincurv_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                             const double *h, double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                             const double *sens, int32_t *grad_status, const double *grad_alpha, double *grad_w_right,
                             double *grad_w_left, double *grad_w_veh, void *workspace, size_t workspace_bytes, void *stream) {
    if (!sens || !grad_status || !grad_alpha || !grad_w_right || !grad_w_left || !grad_w_veh)
        return bad("mc_mincurv_adjoint_batch: NULL argument");
    // the band of H and the bounds are rebuilt in the slabs; the assembly's status words (the forward pass's, recorded in
    // grad_status) go to grad_w_right, which the adjoint kernel overwrites
    int rc = mc_mincurv_setup_batch_shared(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id,
                                           reinterpret_cast<int32_t *>(grad_w_right), workspace, workspace_bytes, stream);
    if (rc) return rc;
    const SolverGrid g = solver_grid(B, n_max, workspace, mc::adjoint_ctas_per_sm());
    if (mc::launch_mincurv_adjoint(B, n_max, n_pts, reftrack, w_veh, w_veh_batch, (double *)workspace, mc::make_layout(n_max),
                                   sens, grad_alpha, grad_status, grad_w_right, grad_w_left, grad_w_veh, g.grid, g.counter,
                                   (cudaStream_t)stream) != 0) {
        snprintf(g_err, sizeof(g_err), "mincurv_adjoint_kernel: cudaFuncSetAttribute failed");
        return MC_ECUDA;
    }
    return check_cuda("mincurv_adjoint_kernel");
}

int mc_mincurv_kappa_batch(int B, int n_max, const int32_t *n_pts, double kappa_bound, double *alpha, int32_t *status,
                           int32_t *iters, void *workspace, size_t workspace_bytes, void *stream) {
    if (!alpha || !status) return bad("mc_mincurv_kappa_batch: NULL argument");
    int rc = mincurv_args("mc_mincurv_kappa_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    mc::PdipParams prm;
    prm.max_iter = 40;
    prm.mu_rel = 1e-11;
    prm.rd_rel = 1e-8;
    prm.eta = 0.995;
    prm.dx_rel = 0.0;
    prm.lam0_rel = 1e-2;
    const SolverGrid g = solver_grid(B, n_max, workspace, mc::pdip_kappa_ctas_per_sm());
    if (mc::launch_mincurv_pdip_kappa(B, n_max, n_pts, (double *)workspace, mc::make_layout(n_max), prm, kappa_bound, alpha,
                                      status, iters, g.grid, g.counter, (cudaStream_t)stream) != 0) {
        snprintf(g_err, sizeof(g_err), "mincurv_pdip_kappa_kernel: cudaFuncSetAttribute failed");
        return MC_ECUDA;
    }
    return check_cuda("mincurv_pdip_kappa_kernel");
}

// ------------------------------------------------------------------------------------------------
size_t mc_shortest_path_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < 3) return 0;
    return align256((size_t)B * mc::shortest_path_ws_doubles(n_max) * sizeof(double));
}

int mc_shortest_path_solve_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                 double w_veh, const double *w_veh_batch, double *alpha, int32_t *status, int32_t *iters,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 3 || !reftrack || !normvec || !alpha || !status)
        return bad("mc_shortest_path_solve_batch: bad argument");
    if (!workspace || workspace_bytes < mc_shortest_path_workspace_bytes(B, n_max))
        return small_workspace("mc_shortest_path_solve_batch");
    if (mc::launch_shortest_path(B, n_max, n_pts, reftrack, normvec, w_veh, w_veh_batch, alpha, status, iters,
                                 (double *)workspace, (cudaStream_t)stream) != 0) {
        snprintf(g_err, sizeof(g_err), "shortest_path_kernel: launch configuration failed");
        return MC_ECUDA;
    }
    return check_cuda("shortest_path_kernel");
}

int mc_shortest_path_solve_batch_sens(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                      double w_veh, const double *w_veh_batch, double *alpha, int32_t *status, int32_t *iters,
                                      double *sens, int32_t *grad_status, void *workspace, size_t workspace_bytes,
                                      void *stream) {
    if (!sens || !grad_status) return bad("mc_shortest_path_solve_batch_sens: NULL argument");
    int rc = mc_shortest_path_solve_batch(B, n_max, n_pts, reftrack, normvec, w_veh, w_veh_batch, alpha, status, iters,
                                          workspace, workspace_bytes, stream);
    if (rc) return rc;
    // the workspace still holds the final iterate
    mc::launch_shortest_path_sens_export(B, n_max, n_pts, status, (const double *)workspace, sens, grad_status,
                                         (cudaStream_t)stream);
    return check_cuda("shortest_path_sens_export_kernel");
}

int mc_shortest_path_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                   double w_veh, const double *w_veh_batch, const double *alpha, const double *sens,
                                   int32_t *grad_status, const double *grad_alpha, double *grad_reftrack, double *grad_normvec,
                                   double *grad_w_veh, void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 3 || !reftrack || !normvec || !alpha || !sens || !grad_status || !grad_alpha || !grad_reftrack)
        return bad("mc_shortest_path_adjoint_batch: bad argument");
    if (!workspace || workspace_bytes < mc_shortest_path_workspace_bytes(B, n_max))
        return small_workspace("mc_shortest_path_adjoint_batch");
    mc::launch_shortest_path_adjoint(B, n_max, n_pts, reftrack, normvec, w_veh, w_veh_batch, alpha, sens, grad_status,
                                     grad_alpha, grad_reftrack, grad_normvec, grad_w_veh, (double *)workspace,
                                     (cudaStream_t)stream);
    return check_cuda("shortest_path_adjoint_kernel");
}

// ------------------------------------------------------------------------------------------------
size_t mc_create_raceline_workspace_bytes(int B, int n_max) { return mc_calc_splines_workspace_bytes(B, n_max); }

int mc_create_raceline_batch(int B, int n_max, const int32_t *n_pts, const double *refline, int ref_stride,
                             const double *normvec, const double *alpha, double stepsize_interp, int n_out_max,
                             double *coeffs_x, double *coeffs_y, double *spline_lengths, int32_t *n_out,
                             double *raceline_interp, int32_t *spline_inds, double *t_values, double *s_interp,
                             double *el_lengths_interp, double *psi, double *kappa, void *workspace,
                             size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 3 || n_out_max <= 0 || !refline || (ref_stride != 2 && ref_stride != 4) || !normvec || !alpha ||
        !(stepsize_interp > 0.0) || !coeffs_x || !coeffs_y || !spline_lengths || !n_out || !raceline_interp ||
        !spline_inds || !t_values || !s_interp || !el_lengths_interp)
        return bad("mc_create_raceline_batch: bad argument");
    if (!workspace || workspace_bytes < mc_create_raceline_workspace_bytes(B, n_max))
        return small_workspace("mc_create_raceline_batch");
    mc::launch_create_raceline(B, n_max, n_pts, refline, ref_stride, normvec, alpha, stepsize_interp, n_out_max,
                               coeffs_x, coeffs_y, spline_lengths, n_out, raceline_interp, spline_inds, t_values,
                               s_interp, el_lengths_interp, psi, kappa, (double *)workspace, (cudaStream_t)stream);
    return check_cuda("create_raceline_kernel");
}

int mc_calc_head_curv_batch(int B, int n_max, const double *coeffs_x, const double *coeffs_y, int n_eval_max,
                            const int32_t *n_eval, const int32_t *ind_spls, const double *t_spls, double *psi,
                            double *kappa, double *dkappa, void *stream) {
    if (B <= 0 || n_max <= 0 || n_eval_max <= 0 || !coeffs_x || !coeffs_y || !ind_spls || !t_spls || !psi)
        return bad("mc_calc_head_curv_batch: bad argument");
    if (dkappa && !kappa) return bad("dkappa cannot be calculated without kappa!");
    mc::launch_head_curv(B, n_max, coeffs_x, coeffs_y, n_eval_max, n_eval, ind_spls, t_spls, psi, kappa, dkappa,
                         (cudaStream_t)stream);
    return check_cuda("head_curv_kernel");
}

// ------------------------------------------------------------------------------------------------
// workspace of the IQP re-linearisation: spline scratch + the create_raceline outputs it discards
static size_t iqp_ws_parts(int B, int n_max, int n_max_new, size_t off[10]) {
    size_t o = 0;
    const size_t spl = align256((size_t)B * mc::spline_ws_doubles(n_max > n_max_new ? n_max : n_max_new) * sizeof(double));
    off[0] = o; o += spl;                                                    // spline scratch
    off[1] = o; o += align256((size_t)B * n_max * 4 * sizeof(double));       // coeffs_x
    off[2] = o; o += align256((size_t)B * n_max * 4 * sizeof(double));       // coeffs_y
    off[3] = o; o += align256((size_t)B * n_max * sizeof(double));           // spline_lengths
    off[4] = o; o += align256((size_t)B * sizeof(int32_t));                  // n_out
    off[5] = o; o += align256((size_t)B * n_max_new * 2 * sizeof(double));   // raceline_interp
    off[6] = o; o += align256((size_t)B * n_max_new * sizeof(int32_t));      // spline_inds
    off[7] = o; o += align256((size_t)B * n_max_new * sizeof(double));       // t_values
    off[8] = o; o += align256((size_t)B * n_max_new * sizeof(double));       // s_interp
    off[9] = o; o += align256((size_t)B * n_max_new * sizeof(double));       // el_lengths
    return o;
}

size_t mc_iqp_relinearise_workspace_bytes(int B, int n_max, int n_max_new) {
    if (B <= 0 || n_max < 3 || n_max_new < 3) return 0;
    size_t off[10];
    return iqp_ws_parts(B, n_max, n_max_new, off);
}

int mc_iqp_relinearise_batch(int B, int n_max, const int32_t *n_pts, const int32_t *active, const double *reftrack,
                             const double *normvec, const double *alpha, double stepsize_interp, int n_max_new,
                             double *reftrack_new, double *normvec_new, int32_t *n_pts_new, void *workspace,
                             size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 3 || n_max_new < 3 || !reftrack || !normvec || !alpha || !(stepsize_interp > 0.0) ||
        !reftrack_new || !normvec_new || !n_pts_new)
        return bad("mc_iqp_relinearise_batch: bad argument");
    size_t off[10];
    const size_t need = iqp_ws_parts(B, n_max, n_max_new, off);
    if (!workspace || workspace_bytes < need) return small_workspace("mc_iqp_relinearise_batch");
    char *w = (char *)workspace;
    cudaStream_t s = (cudaStream_t)stream;
    double *spl = (double *)(w + off[0]);
    int32_t *n_out = (int32_t *)(w + off[4]);
    mc::launch_create_raceline(B, n_max, n_pts, reftrack, 4, normvec, alpha, stepsize_interp, n_max_new,
                               (double *)(w + off[1]), (double *)(w + off[2]), (double *)(w + off[3]), n_out,
                               (double *)(w + off[5]), (int32_t *)(w + off[6]), (double *)(w + off[7]),
                               (double *)(w + off[8]), (double *)(w + off[9]), nullptr, nullptr, spl, s);
    int rc = check_cuda("create_raceline_kernel");
    if (rc) return rc;
    mc::launch_iqp_new_reftrack(B, n_max, n_pts, active, reftrack, normvec, alpha, n_max_new, n_out,
                                (double *)(w + off[5]), (int32_t *)(w + off[6]), (double *)(w + off[7]), reftrack_new,
                                normvec_new, n_pts_new, s);
    rc = check_cuda("iqp_new_reftrack_kernel");
    if (rc) return rc;
    // splines of the new reference line without distance scaling -> new normal vectors
    mc::launch_calc_splines(B, n_max_new, n_pts_new, reftrack_new, 4, nullptr, 0, nullptr, nullptr, normvec_new, nullptr,
                            spl, s);
    return check_cuda("calc_splines_kernel");
}

// ------------------------------------------------------------------------------------------------
size_t mc_vel_profile_workspace_bytes(int B, int V, int n_max) {
    if (B <= 0 || V <= 0 || n_max < 2) return 0;
    return align256((size_t)B * V * mc::vel_profile_ws_doubles(n_max) * sizeof(double));
}

int mc_vel_profile_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                         const double *mu, int V, const double *ggv_scale, const double *v_max_batch, double v_max,
                         int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines, double dyn_model_exp,
                         double drag_coeff, double m_veh, int filt_window, double *vx, double *ax, double *t,
                         double *laptime, int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    return mc_vel_profile_batch_ex(B, n_max, n_pts, kappa, el_lengths, mu, V, ggv_scale, v_max_batch, v_max, n_ggv, ggv, n_mach,
                                   ax_max_machines, dyn_model_exp, drag_coeff, m_veh, filt_window, MC_VP_DECEL_SLICE_UPPER_DEFAULT,
                                   vx, ax, t, laptime, status, workspace, workspace_bytes, stream);
}

int mc_vel_profile_batch_ex(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                            const double *mu, int V, const double *ggv_scale, const double *v_max_batch, double v_max,
                            int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines, double dyn_model_exp,
                            double drag_coeff, double m_veh, int filt_window, int decel_slice_upper, double *vx, double *ax,
                            double *t, double *laptime, int32_t *status, void *workspace, size_t workspace_bytes,
                            void *stream) {
    if (B <= 0 || V <= 0 || n_max < 2 || !kappa || !el_lengths || !ggv || !ax_max_machines || !laptime || n_ggv < 1 ||
        n_mach < 1 || !(m_veh > 0.0) || !(dyn_model_exp > 0.0) || (!v_max_batch && !(v_max > 0.0)))
        return bad("mc_vel_profile_batch: bad argument");
    if (filt_window > 1 && (filt_window % 2 == 0 || filt_window >= n_max))
        return bad("mc_vel_profile_batch: filt_window must be odd (tph: 'Window width of moving average filter must be odd!')");
    if ((size_t)B * V > (size_t)0x7fffffff - 256) return bad("mc_vel_profile_batch: too many profiles in one call");
    if (!workspace || workspace_bytes < mc_vel_profile_workspace_bytes(B, V, n_max))
        return small_workspace("mc_vel_profile_batch");
    if (mc::launch_vel_profile(B, V, n_max, n_pts, kappa, el_lengths, mu, ggv_scale, v_max_batch, v_max, n_ggv, ggv, n_mach,
                               ax_max_machines, dyn_model_exp, drag_coeff, m_veh, filt_window, decel_slice_upper != 0, vx, ax, t,
                               laptime, status, (double *)workspace, (cudaStream_t)stream) != 0)
        return bad("mc_vel_profile_batch: ggv / ax_max_machines tables are limited to 256 rows");
    return check_cuda("vel_profile_kernel");
}

size_t mc_create_raceline_adjoint_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < 3) return 0;
    return align256((size_t)B * mc::create_raceline_adjoint_ws_doubles(n_max) * sizeof(double));
}

int mc_create_raceline_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *normvec, const double *alpha,
                                     int n_out_max, const double *coeffs_x, const double *coeffs_y,
                                     const double *spline_lengths, const int32_t *n_out, const int32_t *spline_inds,
                                     const double *t_values, const double *grad_raceline, const double *grad_kappa,
                                     const double *grad_el_lengths, double *grad_alpha, double *grad_refline,
                                     double *grad_normvec, void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 3 || n_out_max < 1 || !normvec || !alpha || !coeffs_x || !coeffs_y || !spline_lengths ||
        !n_out || !spline_inds || !t_values || !grad_alpha)
        return bad("mc_create_raceline_adjoint_batch: bad argument");
    if (B > 65535 * 1024) return bad("mc_create_raceline_adjoint_batch: too many tracks in one call");
    if (!workspace || workspace_bytes < mc_create_raceline_adjoint_workspace_bytes(B, n_max))
        return small_workspace("mc_create_raceline_adjoint_batch");
    mc::launch_create_raceline_adjoint(B, n_max, n_pts, normvec, alpha, n_out_max, coeffs_x, coeffs_y, spline_lengths, n_out,
                                       spline_inds, t_values, grad_raceline, grad_kappa, grad_el_lengths, grad_alpha,
                                       grad_refline, grad_normvec, (double *)workspace, (cudaStream_t)stream);
    return check_cuda("create_raceline_adjoint_kernel");
}

size_t mc_vel_profile_adjoint_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < 2) return 0;
    return align256((size_t)B * mc::vel_profile_adjoint_ws_doubles(n_max) * sizeof(double));
}

int mc_vel_profile_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                                 double v_max, int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines,
                                 double dyn_model_exp, double drag_coeff, double m_veh, int filt_window,
                                 int decel_slice_upper, const double *grad_laptime, const double *grad_vx,
                                 double *grad_kappa, double *grad_el_lengths, int32_t *grad_status,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 2 || !kappa || !el_lengths || !ggv || !ax_max_machines || !grad_status || n_ggv < 1 ||
        n_mach < 1 || !(m_veh > 0.0) || !(dyn_model_exp > 0.0) || !(v_max > 0.0))
        return bad("mc_vel_profile_adjoint_batch: bad argument");
    if (filt_window > 1 && (filt_window % 2 == 0 || filt_window >= n_max))
        return bad("mc_vel_profile_adjoint_batch: filt_window must be odd and smaller than n_max");
    if ((size_t)B > (size_t)0x7fffffff - 256) return bad("mc_vel_profile_adjoint_batch: too many profiles in one call");
    if (!workspace || workspace_bytes < mc_vel_profile_adjoint_workspace_bytes(B, n_max))
        return small_workspace("mc_vel_profile_adjoint_batch");
    if (mc::launch_vel_profile_adjoint(B, n_max, n_pts, kappa, el_lengths, v_max, n_ggv, ggv, n_mach, ax_max_machines,
                                       dyn_model_exp, drag_coeff, m_veh, filt_window, decel_slice_upper != 0, grad_laptime,
                                       grad_vx, grad_kappa, grad_el_lengths, grad_status, (double *)workspace,
                                       (cudaStream_t)stream) != 0)
        return bad("mc_vel_profile_adjoint_batch: ggv / ax_max_machines tables are limited to 256 rows");
    return check_cuda("vel_profile_adjoint_kernel");
}

int mc_calc_ax_t_profile_batch(int P, int n_max, const int32_t *n_pts, const double *vx, int vx_pitch,
                               const double *el_lengths, const double *ax_in, double t_start, double *ax_out,
                               double *t_out, void *stream) {
    if (P <= 0 || n_max < 1 || !vx || !el_lengths || (!ax_out && !t_out) || vx_pitch < n_max + (ax_in ? 0 : 1))
        return bad("mc_calc_ax_t_profile_batch: bad argument");
    mc::launch_ax_t_profile(P, n_max, n_pts, vx, vx_pitch, el_lengths, ax_in, t_start, ax_out, t_out, (cudaStream_t)stream);
    return check_cuda("ax_t_profile_kernel");
}

// ------------------------------------------------------------------------------------------------
size_t mc_interp_track_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < 2) return 0;
    return align256((size_t)B * mc::interp_track_ws_doubles(n_max) * sizeof(double));
}

int mc_interp_track_batch(int B, int n_max, const int32_t *n_pts, const double *pts, int stride, const double *normvec,
                          double normal_sign, int width_col, double stepsize_approx, int n_out_max, double *out,
                          int32_t *n_out, void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 2 || !pts || (stride != 2 && stride != 4) || !(stepsize_approx > 0.0) || n_out_max <= 0 || !out ||
        !n_out || (normvec && (stride != 4 || (width_col != 2 && width_col != 3))))
        return bad("mc_interp_track_batch: bad argument");
    if (!workspace || workspace_bytes < mc_interp_track_workspace_bytes(B, n_max))
        return small_workspace("mc_interp_track_batch");
    mc::launch_interp_track(B, n_max, n_pts, pts, stride, normvec, normal_sign, normvec ? width_col : 2, stepsize_approx,
                            n_out_max, out, n_out, (double *)workspace, (cudaStream_t)stream);
    return check_cuda("interp_track_kernel");
}

int mc_min_bound_dists_batch(int B, int n_traj_max, const int32_t *n_traj, const double *xy, const double *psi, int nb1_max,
                             const int32_t *nb1, const double *bound1, int nb2_max, const int32_t *nb2, const double *bound2,
                             int bound_stride, double length_veh, double width_veh, double *min_dists, void *stream) {
    if (B <= 0 || n_traj_max <= 0 || !xy || !psi || !bound1 || !bound2 || nb1_max <= 0 || nb2_max <= 0 ||
        bound_stride < 2 || !min_dists)
        return bad("mc_min_bound_dists_batch: bad argument");
    mc::launch_min_bound_dists(B, n_traj_max, n_traj, xy, psi, nb1_max, nb1, bound1, nb2_max, nb2, bound2, bound_stride,
                               length_veh, width_veh, min_dists, (cudaStream_t)stream);
    return check_cuda("min_bound_dists_kernel");
}

int mc_traj_extrema_batch(int B, int n_max, const int32_t *n_traj, const double *kappa, const double *vx, const double *ax,
                          const double *min_dists, double dragcoeff, double mass_veh, double *extrema, void *stream) {
    if (B <= 0 || n_max <= 0 || !kappa || !vx || !ax || !extrema || !(mass_veh > 0.0))
        return bad("mc_traj_extrema_batch: bad argument");
    mc::launch_traj_extrema(B, n_max, n_traj, kappa, vx, ax, min_dists, dragcoeff, mass_veh, extrema, (cudaStream_t)stream);
    return check_cuda("traj_extrema_kernel");
}

int mc_assemble_trajectory_batch(int B, int n_max, const int32_t *n_traj, const double *s, const double *xy,
                                 const double *psi, const double *kappa, const double *vx, const double *ax, int n_spl_max,
                                 const int32_t *n_spl, const double *spline_lengths, double *traj, void *stream) {
    if (B <= 0 || n_max <= 0 || !s || !xy || !psi || !kappa || !vx || !ax || n_spl_max <= 0 || !spline_lengths || !traj)
        return bad("mc_assemble_trajectory_batch: bad argument");
    mc::launch_assemble_trajectory(B, n_max, n_traj, s, xy, psi, kappa, vx, ax, n_spl_max, n_spl, spline_lengths, traj,
                                   (cudaStream_t)stream);
    return check_cuda("assemble_trajectory_kernel");
}

int mc_check_normals_crossing_batch(int B, int n_max, const int32_t *n_pts, const double *track, const double *normvec,
                                    int horizon, int32_t *crossing, void *stream) {
    if (B <= 0 || n_max < 3 || !track || !normvec || horizon < 1 || !crossing)
        return bad("mc_check_normals_crossing_batch: bad argument");
    mc::launch_normals_crossing(B, n_max, n_pts, track, normvec, horizon, crossing, (cudaStream_t)stream);
    return check_cuda("normals_crossing_kernel");
}

size_t mc_prep_track_workspace_bytes(int B, int n_raw_max, int n_int_max) {
    if (B <= 0 || n_raw_max < 5 || n_int_max < 6) return 0;
    return align256((size_t)B * mc::prep_track_ws_doubles(n_raw_max, n_int_max) * sizeof(double));
}

int mc_prep_track_batch(int B, int n_raw_max, const int32_t *n_raw, const double *track, int k_reg, double s_reg,
                        double stepsize_prep, double stepsize_reg, double min_width, int n_int_max, int n_out_max,
                        double *reftrack_interp, int32_t *n_out, double *smoothing_lambda, void *workspace,
                        size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_raw_max < 5 || !track || !(s_reg > 0.0) || !(stepsize_prep > 0.0) || !(stepsize_reg > 0.0) || n_int_max < 6 ||
        n_out_max < 4 || !reftrack_interp || !n_out)
        return bad("mc_prep_track_batch: bad argument");
    if (k_reg != 3) return bad("mc_prep_track_batch: only cubic splines (k_reg = 3, the reference's setting) are implemented");
    if (!workspace || workspace_bytes < mc_prep_track_workspace_bytes(B, n_raw_max, n_int_max))
        return small_workspace("mc_prep_track_batch");
    mc::launch_prep_track(B, n_raw_max, n_raw, track, s_reg, stepsize_prep, stepsize_reg, min_width, n_int_max, n_out_max,
                          reftrack_interp, n_out, smoothing_lambda, (double *)workspace, (cudaStream_t)stream);
    return check_cuda("prep_track_kernel");
}

int mc_polygon_length_batch(int B, int n_max, const int32_t *n_pts, const double *pts, int stride, const double *normvec,
                            const double *shift, int shift_stride, double sign, double *length, void *stream) {
    if (B <= 0 || n_max <= 0 || !pts || stride < 2 || !length || ((normvec == nullptr) != (shift == nullptr)) ||
        (shift && shift_stride < 1))
        return bad("mc_polygon_length_batch: bad argument");
    mc::launch_polygon_length(B, n_max, n_pts, pts, stride, normvec, shift, shift_stride, sign, length, (cudaStream_t)stream);
    return check_cuda("polygon_length_kernel");
}

int mc_jitter_widths_batch(int V, int n_max, const int32_t *n_pts_base, int n_base, const double *base,
                           const int32_t *centre_id, const int64_t *seed, double rel, double *out, int32_t *n_pts_out,
                           void *stream) {
    if (V <= 0 || n_max <= 0 || n_base <= 0 || !base || !seed || !out || !(rel >= 0.0) || rel >= 1.0)
        return bad("mc_jitter_widths_batch: bad argument");
    mc::launch_jitter_widths(V, n_max, n_pts_base, n_base, base, centre_id, seed, rel, out, n_pts_out, (cudaStream_t)stream);
    return check_cuda("jitter_widths_kernel");
}

/* debug aid (tests/test_gpu_factor.py): one factorisation + the two kinds of solve of the interior-point kernel on slabs
 * whose H band, V_DD, V_RHS and V_T0 the caller has filled in; results in V_DX, V_T1, V_T2 */
int mc_debug_factor_solve(int B, int n_max, const int32_t *n_pts, int32_t *status, void *workspace, size_t workspace_bytes,
                          void *stream) {
    if (!status) return bad("mc_debug_factor_solve: NULL argument");
    int rc = mincurv_args("mc_debug_factor_solve", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    const SolverGrid g = solver_grid(B, n_max, workspace, mc::debug_factor_solve_ctas_per_sm());
    if (mc::launch_debug_factor_solve(B, n_max, n_pts, (double *)workspace, mc::make_layout(n_max), status, g.grid,
                                      (cudaStream_t)stream) != 0)
        return bad("mc_debug_factor_solve: cudaFuncSetAttribute failed");
    return check_cuda("debug_factor_solve_kernel");
}

// debug aid: the cycle counters of CTA 0 of mincurv_pdip_kernel, slots as in enum ProfSlot of mincurv_ipm.cu
int mc_debug_read_profile(unsigned long long *host_out24, int reset) {
    return mc::debug_read_profile(host_out24, reset) == 0 ? MC_OK : MC_ECUDA;
}

int mc_iqp_finish_batch(int B, int n_max, int n_cap, int iter, int iters_min, double curv_error_allowed, int fixed_iters,
                        int iter_limit, int32_t *active, const int32_t *status, const double *curv_error_max,
                        const int32_t *n_pts, const double *alpha, const double *reftrack, const double *normvec,
                        double *fin_alpha, double *fin_reftrack, double *fin_normvec, int32_t *fin_n_pts,
                        int32_t *fin_outer_iters, int32_t *fin_status, double *fin_curv_error_max, int32_t *counters,
                        void *stream) {
    if (B <= 0 || n_max <= 0 || n_cap < n_max || iter < 1 || !active || !status || !curv_error_max || !alpha || !reftrack ||
        !normvec || !fin_alpha || !fin_reftrack || !fin_normvec || !fin_n_pts || !fin_outer_iters || !fin_status ||
        !fin_curv_error_max || !counters)
        return bad("mc_iqp_finish_batch: bad argument");
    mc::launch_iqp_finish(B, n_max, n_cap, iter, iters_min, curv_error_allowed, fixed_iters, iter_limit, active, status,
                          curv_error_max, n_pts, alpha, reftrack, normvec, fin_alpha, fin_reftrack, fin_normvec, fin_n_pts,
                          fin_outer_iters, fin_status, fin_curv_error_max, counters, (cudaStream_t)stream);
    return check_cuda("iqp_finish_kernel");
}

int mc_scale_alpha_batch(int B, int n_max, double *alpha, const double *scale_batch, double scale, void *stream) {
    if (B <= 0 || n_max <= 0 || !alpha) return bad("mc_scale_alpha_batch: bad argument");
    mc::launch_scale_alpha(B, n_max, alpha, scale_batch, scale, (cudaStream_t)stream);
    return check_cuda("scale_alpha_kernel");
}

}  // extern "C"
