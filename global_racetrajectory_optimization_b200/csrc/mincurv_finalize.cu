// K2c -- post-solve quantities of tph.opt_min_curv (SURVEY.md A.3, call site
// main_globaltraj.py:264-271): the linearised curvature k_ref + E alpha (checked
// against kappa_bound) and the linearisation error curv_error_max, both through the O(N) operator
// form E a = S_y Z (n_y a) - S_x Z (n_x a) (one periodic tridiagonal solve with two right-hand sides).
// LIN: the workspace was assembled about a linearisation point (mincurv_setup.cu): V_XP / V_YP hold its first
// derivatives, which the linearised curvature uses, while the line P + alpha n takes those of the centre line, recomputed
// here from its points and moments.
// KBB: the curvature limit of each instance is kappa_bound_batch[b] (the scalar kappa_bound is not read).  An instance whose
// limit is not finite or not > 0 is refused with status -1 (in the first pass: afterwards its status is negative).  The
// array is the last parameter, so that the scalar instantiations keep their parameter offsets.
#include "capi.cuh"
#include "mincurv_ops.cuh"

namespace mc {

template <bool LIN, bool KBB>
__global__ void __launch_bounds__(256)
mincurv_finalize_kernel(int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                        const double *__restrict__ alpha, double kappa_bound,
                        double *__restrict__ curv_error_max, double *__restrict__ kappa_lin_max,
                        int32_t *__restrict__ status, const double *__restrict__ kappa_bound_batch) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    __shared__ double red[32];
    int st = status[b];
    if constexpr (KBB) {
        kappa_bound = kappa_bound_batch[b];
        if (st >= 0 && !(kappa_bound > 0.0 && kappa_bound < INFINITY)) {
            if (threadIdx.x == 0) status[b] = -1;
            st = -1;
        }
    }
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
    const double *KREF = vec(slab, L, V_KREF), *PX = vec(slab, L, V_PX), *PY = vec(slab, L, V_PY);
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
    // both maxima propagate a NaN as tph's np.amax does (fmax drops it, and the chunked solve confines a NaN of alpha to
    // about 64 points around it, so the maximum over the others would be finite)
    double kmax = 0.0, emax = 0.0;
    bool nan_k = false, nan_e = false;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], h2 = hi * hi;
        const double zx = ZX[i], zy = ZY[i];
        const double klin = KREF[i] + SY[i] * zy - SX[i] * zx;
        kmax = fmax(kmax, fabs(klin));
        nan_k = nan_k || klin != klin;
        const double ddx = h2 * (MX[i] + zx), ddy = h2 * (MY[i] + zy);
        const double xp = XP[i], yp = YP[i];
        double xc = xp, yc = yp;                // first derivatives of the centre line
        if (LIN) {
            xc = (PX[ip1] - PX[i]) - h2 * (2.0 * MX[i] + MX[ip1]) * (1.0 / 6.0);
            yc = (PY[ip1] - PY[i]) - h2 * (2.0 * MY[i] + MY[ip1]) * (1.0 / 6.0);
        }
        const double xpt = xc + (NX[ip1] * al[ip1] - NX[i] * al[i]) - h2 * (2.0 * zx + ZX[ip1]) * (1.0 / 6.0);
        const double ypt = yc + (NY[ip1] * al[ip1] - NY[i] * al[i]) - h2 * (2.0 * zy + ZY[ip1]) * (1.0 / 6.0);
        const double q0 = xp * xp + yp * yp, q1 = xpt * xpt + ypt * ypt;
        const double c0 = (xp * ddy - yp * ddx) / (q0 * sqrt(q0));
        const double c1 = (xpt * ddy - ypt * ddx) / (q1 * sqrt(q1));
        emax = fmax(emax, fabs(c1 - c0));
        nan_e = nan_e || c1 - c0 != c1 - c0;
    }
    kmax = block_reduce<1>(kmax, red);
    emax = block_reduce<1>(emax, red);
    if (__syncthreads_or(nan_k)) kmax = NAN;
    if (__syncthreads_or(nan_e)) emax = NAN;
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

// Second export for the width sensitivities with the curvature rows (K2d', mincurv_ipm.cu), run after the curvature-row
// phase and its finalize pass.  For the instances that phase re-solved (grad_status 4 from the first export) and solved
// (status 0): its final box ratios into sens (over the first export's zeros), the row weights
// sens_rows[b][i] = l3 / s3 + l4 / s4 and n_rows[b] = the count of strong rows (weight > 1).  grad_status[b] becomes
// the final status.  Everything else keeps what the first export wrote, with zero row weights and n_rows 0.
__global__ void __launch_bounds__(256)
mincurv_sens_rows_export_kernel(int n_max, const int32_t *__restrict__ n_pts, double *__restrict__ ws, Layout L,
                                const int32_t *__restrict__ status, double *__restrict__ sens, double *__restrict__ sens_rows,
                                int32_t *__restrict__ n_rows, int32_t *__restrict__ grad_status) {
    const int b = blockIdx.x;
    __shared__ double red[32];
    const int gs = grad_status[b], st = status[b];
    const bool rows = gs == 4 && st == 0;
    const int n = rows ? (n_pts ? n_pts[b] : n_max) : 0;
    double *slab = ws + (size_t)b * L.stride;
    const double *LU = vec(slab, L, V_LU), *LL = vec(slab, L, V_LL), *SU = vec(slab, L, V_SU), *SL = vec(slab, L, V_SL);
    const double *S3 = vec(slab, L, V_S3), *S4 = vec(slab, L, V_S4), *L3 = vec(slab, L, V_L3), *L4 = vec(slab, L, V_L4);
    double *du = sens + (size_t)b * 2 * n_max, *dl = du + n_max, *wr = sens_rows + (size_t)b * n_max;
    double strong = 0.0;
    for (int i = threadIdx.x; i < n_max; i += blockDim.x) {
        const double w = (i < n) ? L3[i] / S3[i] + L4[i] / S4[i] : 0.0;
        wr[i] = w;
        strong += (w > 1.0) ? 1.0 : 0.0;
        if (gs == 4) {
            du[i] = (i < n) ? LU[i] / SU[i] : 0.0;
            dl[i] = (i < n) ? LL[i] / SL[i] : 0.0;
        }
    }
    strong = block_reduce<0>(strong, red);
    if (threadIdx.x == 0) {
        n_rows[b] = (int32_t)strong;
        if (gs == 4) grad_status[b] = st;
    }
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

int mincurv_finalize(int B, int n_max, const int32_t *n_pts, const double *alpha, double kappa_bound, double *curv_error_max,
                     double *kappa_lin_max, int32_t *status, bool lin, const double *kappa_bound_batch, void *workspace,
                     size_t workspace_bytes, void *stream) {
    if (!alpha || !curv_error_max || !status) return bad("mc_mincurv_finalize_batch: NULL argument");
    int rc = mincurv_args("mc_mincurv_finalize_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    auto kernel = kappa_bound_batch ? (lin ? mincurv_finalize_kernel<true, true> : mincurv_finalize_kernel<false, true>)
                                    : (lin ? mincurv_finalize_kernel<true, false> : mincurv_finalize_kernel<false, false>);
    kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace, make_layout(n_max), alpha, kappa_bound,
                                                curv_error_max, kappa_lin_max, status, kappa_bound_batch);
    return check_cuda("mincurv_finalize_kernel");
}

}  // namespace mc

extern "C" {

int mc_mincurv_finalize_batch(int B, int n_max, const int32_t *n_pts, const double *alpha, double kappa_bound,
                              double *curv_error_max, double *kappa_lin_max, int32_t *status, int linearised,
                              const double *kappa_bound_batch, void *workspace, size_t workspace_bytes, void *stream) {
    return mc::mincurv_finalize(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, linearised != 0,
                                kappa_bound_batch, workspace, workspace_bytes, stream);
}

int mc_mincurv_solve_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                           const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double *alpha,
                           double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                           void *workspace, size_t workspace_bytes, void *stream) {
    return mc_mincurv_solve_batch_ex(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, MC_F_SCALE_DEFAULT,
                                     alpha, curv_error_max, kappa_lin_max, status, iters, 0.0, nullptr, nullptr, nullptr,
                                     nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, workspace, workspace_bytes, stream);
}

// the projection QP: setup -> prox -> pdip -> finalize -> kappa (with prox_mu) -> finalize
static int mincurv_prox_solve(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                              double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                              double prox_mu, const double *prox_x, const double *prox_q, const double *lin_alpha,
                              const double *kbb, void *workspace, size_t workspace_bytes, void *stream) {
    if (!reftrack || !normvec || !h || !alpha || !curv_error_max || !status || !prox_q)
        return bad("mc_mincurv_solve_batch_ex: NULL argument");
    if (!(prox_mu > 0.0) || !(prox_mu < INFINITY)) return bad("mc_mincurv_solve_batch_ex: prox_mu must be finite and positive");
    const bool lin = lin_alpha != nullptr;
    int rc = mc::mincurv_setup(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, nullptr, lin_alpha, status,
                               workspace, workspace_bytes, stream);
    if (rc) return rc;
    mc::mincurv_prox_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace, mc::make_layout(n_max),
                                                                 prox_mu, prox_x, prox_q, status);
    rc = check_cuda("mincurv_prox_kernel");
    if (rc) return rc;
    rc = mc_mincurv_pdip_batch(B, n_max, n_pts, alpha, status, iters, workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc::mincurv_finalize(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, lin, kbb,
                              workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc::mincurv_kappa_phase(B, n_max, n_pts, kappa_bound, kbb, prox_mu, alpha, status, iters, workspace, workspace_bytes,
                                 stream);
    if (rc) return rc;
    return mc::mincurv_finalize(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, lin, kbb,
                                workspace, workspace_bytes, stream);
}

// setup -> pdip -> finalize -> (export of the sensitivity data) -> kappa -> finalize -> (export of the curvature-row phase's
// sensitivity data); sens == NULL: no export, sens_rows == NULL: no second export.  Every argument is checked before the
// first launch: the pointers here, f_scale and the sizes by the setup stage.
static int mincurv_solve(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec, const double *h,
                         double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id,
                         double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                         double *sens, int32_t *grad_status, double *sens_rows, int32_t *n_rows, const double *lin_alpha,
                         const double *kbb, void *workspace, size_t workspace_bytes, void *stream) {
    if (!reftrack || !normvec || !h || !alpha || !curv_error_max || !status)
        return bad("mc_mincurv_solve_batch: NULL argument");
    const bool lin = lin_alpha != nullptr;
    int rc = mc::mincurv_setup(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, lin_alpha, status,
                               workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc_mincurv_pdip_batch(B, n_max, n_pts, alpha, status, iters, workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc::mincurv_finalize(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, lin, kbb,
                              workspace, workspace_bytes, stream);
    if (rc) return rc;
    if (sens) {
        // the box phase's final iterate, before the curvature-row phase takes over the status-4 slabs
        mc::mincurv_sens_export_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace,
                                                                            mc::make_layout(n_max), status, sens, grad_status);
        rc = check_cuda("mincurv_sens_export_kernel");
        if (rc) return rc;
    }
    // instances whose box-only optimum violates the curvature rows (status 4) are re-solved with the rows
    rc = mc_mincurv_kappa_batch(B, n_max, n_pts, kappa_bound, alpha, status, iters, kbb, workspace, workspace_bytes, stream);
    if (rc) return rc;
    rc = mc::mincurv_finalize(B, n_max, n_pts, alpha, kappa_bound, curv_error_max, kappa_lin_max, status, lin, kbb,
                              workspace, workspace_bytes, stream);
    if (rc || !sens_rows) return rc;
    mc::mincurv_sens_rows_export_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, (double *)workspace, mc::make_layout(n_max),
                                                                             status, sens, sens_rows, n_rows, grad_status);
    return check_cuda("mincurv_sens_rows_export_kernel");
}

int mc_mincurv_solve_batch_ex(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                              double *alpha, double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters,
                              double prox_mu, const double *prox_x, const double *prox_q, const double *lin_alpha,
                              const double *kappa_bound_batch, const int32_t *centre_id, double *sens, int32_t *grad_status,
                              double *sens_rows, int32_t *n_rows, int dense_below, void *workspace, size_t workspace_bytes,
                              void *stream) {
    if (!sens != !grad_status) return bad("mc_mincurv_solve_batch_ex: sens and grad_status go together");
    if (!sens_rows != !n_rows || (sens_rows && !sens))
        return bad("mc_mincurv_solve_batch_ex: sens_rows and n_rows go together, and with sens");
    if (prox_x && (centre_id || sens)) return bad("mc_mincurv_solve_batch_ex: prox_x takes neither centre_id nor sens");
    if (dense_below != 0) {
        if (dense_below < mc::N_MIN || dense_below > MC_DENSE_N_MAX + 1)
            return bad("mc_mincurv_solve_batch_ex: dense_below must be 0 or in [%d, %d]", mc::N_MIN, MC_DENSE_N_MAX + 1);
        if (prox_x || sens) return bad("mc_mincurv_solve_batch_ex: dense_below takes neither prox_x nor sens");
        if (B <= 0 || n_max <= 0) return bad("mc_mincurv_solve_batch_ex: B <= 0 or n_max <= 0");
        if (!reftrack || !normvec || !h || !alpha || !curv_error_max || !status)
            return bad("mc_mincurv_solve_batch_ex: NULL argument");
        if (!(f_scale > 0.0)) return bad("mc_mincurv_solve_batch_ex: f_scale must be positive");
    }
    if (prox_x)
        return mincurv_prox_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, alpha,
                                  curv_error_max, kappa_lin_max, status, iters, prox_mu, prox_x, prox_q, lin_alpha,
                                  kappa_bound_batch, workspace, workspace_bytes, stream);
    const bool banded = dense_below == 0 || n_max >= mc::N_MIN;
    if (banded) {
        const int rc = mincurv_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, centre_id,
                                     alpha, curv_error_max, kappa_lin_max, status, iters, sens, grad_status, sens_rows, n_rows,
                                     lin_alpha, kappa_bound_batch, workspace, workspace_bytes, stream);
        if (rc || dense_below == 0) return rc;
    }
    // the small tracks: the dense kernel, last on the stream
    return mc::mincurv_dense(B, n_max, dense_below, banded, n_pts, reftrack, normvec, h, kappa_bound, kappa_bound_batch, w_veh,
                             w_veh_batch, f_scale, centre_id, lin_alpha, alpha, curv_error_max, kappa_lin_max, status, iters,
                             stream);
}

int mc_mincurv_solve_batch_shared(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                  const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                  const int32_t *centre_id, double *alpha, double *curv_error_max, double *kappa_lin_max,
                                  int32_t *status, int32_t *iters, void *workspace, size_t workspace_bytes, void *stream) {
    return mincurv_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, centre_id, alpha,
                         curv_error_max, kappa_lin_max, status, iters, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr,
                         workspace, workspace_bytes, stream);
}

int mc_mincurv_solve_batch_sens(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                const double *h, double kappa_bound, double w_veh, const double *w_veh_batch, double f_scale,
                                const int32_t *centre_id, double *alpha, double *curv_error_max, double *kappa_lin_max,
                                int32_t *status, int32_t *iters, double *sens, int32_t *grad_status, double *sens_rows,
                                int32_t *n_rows, void *workspace, size_t workspace_bytes, void *stream) {
    if (!sens || !grad_status) return bad("mc_mincurv_solve_batch_sens: NULL argument");
    if (!sens_rows != !n_rows) return bad("mc_mincurv_solve_batch_sens: sens_rows and n_rows go together");
    return mincurv_solve(B, n_max, n_pts, reftrack, normvec, h, kappa_bound, w_veh, w_veh_batch, f_scale, centre_id, alpha,
                         curv_error_max, kappa_lin_max, status, iters, sens, grad_status, sens_rows, n_rows, nullptr,
                         nullptr, workspace, workspace_bytes, stream);
}

}  // extern "C"
