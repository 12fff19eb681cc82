// K2c -- post-solve quantities of tph.opt_min_curv (SURVEY.md A.3, call site
// main_globaltraj.py:264-271): the linearised curvature k_ref + E alpha (checked
// against kappa_bound) and the linearisation error curv_error_max, both through the O(N) operator
// form E a = S_y Z (n_y a) - S_x Z (n_x a) (one periodic tridiagonal solve with two right-hand sides).
#include "capi.cuh"
#include "mincurv_ops.cuh"

namespace mc {

__global__ void __launch_bounds__(256)
mincurv_finalize_kernel(int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                        const double *__restrict__ alpha, double kappa_bound,
                        double *__restrict__ curv_error_max, double *__restrict__ kappa_lin_max,
                        int32_t *__restrict__ status) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    __shared__ double red[32];
    const int st = status[b];
    if (st == 1 || st < 0) {
        if (threadIdx.x == 0) {
            curv_error_max[b] = 0.0;
            if (kappa_lin_max) kappa_lin_max[b] = 0.0;
        }
        return;
    }
    double *slab = ws + (size_t)b * L.stride;
    const double *al = alpha + (size_t)b * n_max;
    const double *H = vec(slab, L, V_H), *LFW = vec(slab, L, V_LFW), *INVD = vec(slab, L, V_INVD);
    const double *NX = vec(slab, L, V_NX), *NY = vec(slab, L, V_NY), *MX = vec(slab, L, V_MX), *MY = vec(slab, L, V_MY);
    const double *XP = vec(slab, L, V_XP), *YP = vec(slab, L, V_YP), *SX = vec(slab, L, V_SX), *SY = vec(slab, L, V_SY);
    const double *KREF = vec(slab, L, V_KREF);
    double *T0 = vec(slab, L, V_T0), *T1 = vec(slab, L, V_T1), *T2 = vec(slab, L, V_T2), *T3 = vec(slab, L, V_T3);
    double *ZX = vec(slab, L, V_T4), *ZY = vec(slab, L, V_T5);

    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], him = H[im1];
        const double vx = NX[i] * al[i], vxm = NX[im1] * al[im1], vxp = NX[ip1] * al[ip1];
        const double vy = NY[i] * al[i], vym = NY[im1] * al[im1], vyp = NY[ip1] * al[ip1];
        T0[i] = 6.0 * ((vxp - vx) / hi - (vx - vxm) / him);
        T1[i] = 6.0 * ((vyp - vy) / hi - (vy - vym) / him);
    }
    __syncthreads();
    tri_solve2(LFW, INVD, H, T0, T1, T2, T3, ZX, ZY, n);
    double kmax = 0.0, emax = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], h2 = hi * hi;
        const double zx = ZX[i], zy = ZY[i];
        const double klin = KREF[i] + SY[i] * zy - SX[i] * zx;
        kmax = fmax(kmax, fabs(klin));
        const double ddx = h2 * (MX[i] + zx), ddy = h2 * (MY[i] + zy);
        const double xp = XP[i], yp = YP[i];
        const double xpt = xp + (NX[ip1] * al[ip1] - NX[i] * al[i]) - h2 * (2.0 * zx + ZX[ip1]) * (1.0 / 6.0);
        const double ypt = yp + (NY[ip1] * al[ip1] - NY[i] * al[i]) - h2 * (2.0 * zy + ZY[ip1]) * (1.0 / 6.0);
        const double q0 = xp * xp + yp * yp, q1 = xpt * xpt + ypt * ypt;
        const double c0 = (xp * ddy - yp * ddx) / (q0 * sqrt(q0));
        const double c1 = (xpt * ddy - ypt * ddx) / (q1 * sqrt(q1));
        emax = fmax(emax, fabs(c1 - c0));
    }
    kmax = block_reduce<1>(kmax, red);
    emax = block_reduce<1>(emax, red);
    if (threadIdx.x == 0) {
        curv_error_max[b] = emax;
        if (kappa_lin_max) kappa_lin_max[b] = kmax;
        if (st == 0 && kmax > kappa_bound * (1.0 + 1e-7)) status[b] = 4;
    }
}

// Export for the width sensitivities (K2d, mincurv_ipm.cu), run between the first finalize pass and the curvature-row
// phase: the box phase's final ratios sens[b][0][i] = lu / su, sens[b][1][i] = ll / sl, and grad_status[b] = the status
// at that point (0: solved by the box phase; 4: goes to the curvature-row phase; otherwise the solve's failure status).
// Zeros for every instance with grad_status != 0 and beyond n.
__global__ void __launch_bounds__(256)
mincurv_sens_export_kernel(int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                           const int32_t *__restrict__ status, double *__restrict__ sens, int32_t *__restrict__ grad_status) {
    const int b = blockIdx.x;
    const int st = status[b];
    const int n = (st == 0) ? (n_pts ? n_pts[b] : n_max) : 0;
    double *slab = ws + (size_t)b * L.stride;
    const double *LU = vec(slab, L, V_LU), *LL = vec(slab, L, V_LL), *SU = vec(slab, L, V_SU), *SL = vec(slab, L, V_SL);
    double *du = sens + (size_t)b * 2 * n_max, *dl = du + n_max;
    for (int i = threadIdx.x; i < n_max; i += blockDim.x) {
        du[i] = (i < n) ? LU[i] / SU[i] : 0.0;
        dl[i] = (i < n) ? LL[i] / SL[i] : 0.0;
    }
    if (threadIdx.x == 0) grad_status[b] = st;
}

// The projection QP of mc_mincurv_solve_batch_ex, run after the assembly: Hessian H + mu I and linear term
// c = mu q - (H + mu I) x.  mu goes onto the diagonal of the instance's band of H, which the box phase reads, and c
// replaces f in V_F; H x is formed in operator form (E^T (E x)).  Only instances the assembly left at status 0.
__global__ void __launch_bounds__(256)
mincurv_prox_kernel(int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L, double mu,
                    const double *__restrict__ prox_x, const double *__restrict__ prox_q,
                    const int32_t *__restrict__ status) {
    const int b = blockIdx.x;
    if (status[b] != 0) return;
    const int n = n_pts ? n_pts[b] : n_max;
    double *slab = ws + (size_t)b * L.stride;
    const double *x = prox_x + (size_t)b * n_max, *q = prox_q + (size_t)b * n_max;
    double *HB = slab + L.o_hb, *F = vec(slab, L, V_F), *EX = vec(slab, L, V_EDX), *HX = vec(slab, L, V_T3K);
    double *t0 = vec(slab, L, V_T0), *t1 = vec(slab, L, V_T1), *t2 = vec(slab, L, V_T2), *t3 = vec(slab, L, V_T3);
    double *t4 = vec(slab, L, V_T4), *t5 = vec(slab, L, V_T5);
    for (int i = threadIdx.x; i < n; i += blockDim.x) HB[(size_t)i * HB_PITCH] += mu;
    apply_E(slab, L, n, x, EX, t0, t1, t2, t3, t4, t5);
    apply_Et(slab, L, n, EX, HX, t0, t1, t2, t3, t4, t5);
    for (int i = threadIdx.x; i < n; i += blockDim.x) F[i] = mu * q[i] - (HX[i] + mu * x[i]);
}

}  // namespace mc

extern "C" {

int mc_mincurv_finalize_batch(int B, int n_max, const int32_t *n_pts, const double *alpha, double kappa_bound,
                              double *curv_error_max, double *kappa_lin_max, int32_t *status, void *workspace,
                              size_t workspace_bytes, void *stream) {
    if (!alpha || !curv_error_max || !status) return bad("mc_mincurv_finalize_batch: NULL argument");
    int rc = mc::mincurv_args("mc_mincurv_finalize_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    mc::mincurv_finalize_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace, mc::make_layout(n_max),
                                                                     alpha, kappa_bound, curv_error_max, kappa_lin_max, status);
    return check_cuda("mincurv_finalize_kernel");
}

int mc_mincurv_solve_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                           const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double *alpha,
                           double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                           void *workspace, size_t workspace_bytes, void *stream) {
    return mc_mincurv_solve_batch_ex(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, MC_F_SCALE_DEFAULT,
                                     alpha, curv_error_max, kappa_lin_max, status, iters, 0.0, nullptr, nullptr, workspace,
                                     workspace_bytes, stream);
}

// the projection QP: setup -> prox -> pdip -> finalize -> kappa (with prox_mu) -> finalize
static int mincurv_prox_solve(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                              double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                              double prox_mu, const double *prox_x, const double *prox_q, void *workspace,
                              size_t workspace_bytes, void *stream) {
    if (!reftrack || !normvec || !h || !alpha || !curv_error_max || !status || !prox_q)
        return bad("mc_mincurv_solve_batch_ex: NULL argument");
    if (!(prox_mu > 0.0) || !(prox_mu < INFINITY)) return bad("mc_mincurv_solve_batch_ex: prox_mu must be finite and positive");
    int rc = mc_mincurv_setup_batch_shared(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, nullptr, status,
                                           workspace, workspace_bytes, stream);
    if (rc) return rc;
    mc::mincurv_prox_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace, mc::make_layout(n_max),
                                                                 prox_mu, prox_x, prox_q, status);
    rc = check_cuda("mincurv_prox_kernel");
    if (rc) return rc;
    rc = mc_mincurv_pdip_batch(B, n_max, n_pts, alpha, status, iters, workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc_mincurv_finalize_batch(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, workspace,
                                   workspace_bytes, stream);
    if (rc) return rc;
    rc = mc::mincurv_kappa_phase(B, n_max, n_pts, kappa_bound, prox_mu, alpha, status, iters, workspace, workspace_bytes, stream);
    if (rc) return rc;
    return mc_mincurv_finalize_batch(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, workspace,
                                     workspace_bytes, stream);
}

int mc_mincurv_solve_batch_ex(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                              double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                              double prox_mu, const double *prox_x, const double *prox_q, void *workspace,
                              size_t workspace_bytes, void *stream) {
    if (prox_x)
        return mincurv_prox_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, alpha,
                                  curv_error_max, kappa_lin_max, status, iters, prox_mu, prox_x, prox_q, workspace,
                                  workspace_bytes, stream);
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
        mc::mincurv_sens_export_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace,
                                                                            mc::make_layout(n_max), status, sens, grad_status);
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

}  // extern "C"
