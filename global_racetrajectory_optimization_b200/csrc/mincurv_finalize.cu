// K2c -- post-solve quantities of tph.opt_min_curv (SURVEY.md A.3, call site
// main_globaltraj.py:264-271): the linearised curvature k_ref + E alpha (checked
// against kappa_bound) and the linearisation error curv_error_max, both through the O(N) operator
// form E a = S_y Z (n_y a) - S_x Z (n_x a) (one periodic tridiagonal solve with two right-hand sides).
#include "mincurv_ws.cuh"

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

void launch_mincurv_sens_export(int B, int n_max, const int32_t *n_pts, double *ws, const Layout &L, const int32_t *status,
                                double *sens, int32_t *grad_status, cudaStream_t stream) {
    mincurv_sens_export_kernel<<<B, 256, 0, stream>>>(n_max, n_pts, ws, L, status, sens, grad_status);
}

void launch_mincurv_finalize(int B, int n_max, const int32_t *n_pts, double *ws, const Layout &L, const double *alpha,
                             double kappa_bound, double *curv_error_max, double *kappa_lin_max, int32_t *status,
                             cudaStream_t stream) {
    mincurv_finalize_kernel<<<B, 256, 0, stream>>>(n_max, n_pts, ws, L, alpha, kappa_bound, curv_error_max,
                                                    kappa_lin_max, status);
}

}  // namespace mc
