// K2e -- the minimum-curvature QP of small closed tracks (3 <= n < dense_below <= MC_DENSE_N_MAX + 1) in one CTA per
// instance, with E and the normal matrix dense in shared memory (DESIGN.md section 3.14).  The banded solver needs
// N_MIN points (its band of half-width 32 and the separator must not wrap onto themselves); below that the whole QP of
// oracle/tph_dense.assemble_min_curv fits on chip, without band truncation:
//   min 1/2 a^T E^T E a + f^T a,  f = f_scale E^T k_ref,   s.t.  lb <= a <= ub,  -kb <= k_ref + E a <= kb
// with E_ij = Z_ij (S_y,i n_y,j - S_x,i n_x,j),  Z = Tri^{-1} 6 D2  (columns by tri_solve2, two per call) and S_x, S_y,
// k_ref, the bounds and the LIN form as in mincurv_setup.cu.  The interior point is the curvature-row phase's Mehrotra
// iteration (mincurv_ipm.cu, K2b') on the box and the 2n rows together from the start: a strictly convex QP whose
// box-only optimum meets the rows has that optimum, so one phase gives what the banded path's two give.  Its normal
// matrix K = E^T (I + W) E + D is formed and Cholesky-factored in shared memory every iteration; the predictor and the
// corrector solve on that one factor.  Stopping rule, iteration cap, step rules and start point are the curvature-row
// phase's, so statuses 2 and 3 mean the same on both paths.  The post-solve quantities are mincurv_finalize.cu's.
// Status 4: the last iterate violates the rows by more than kb * 1e-7 (the finalize criterion; a non-finite iterate counts
// as violating them), however the iteration ended: rows that cannot be met drive their weights l / s up until the
// iteration cap or a non-positive pivot stops it.
// No global workspace: shared memory holds E and K (m x m each, m = min(n_max, dense_below - 1)) and DV vectors of m.
// The same kernel with PROX solves the lap-time refinement's projection QP (mc_mincurv_solve_batch_ex with prox_x and
// prox_dense_below), and mincurv_dense_eval_kernel its post-solve evaluation (mc_mincurv_finalize_batch with
// dense_below), both on the tracks below dense_below; the refinement's metric is the dense adjoint below.
#include "capi.cuh"
#include "mincurv_ws.cuh"

namespace mc {

constexpr int DENSE_THREADS = 256;

// the O(m) vectors in shared memory.  Geometry (kept for the finalize), the QP, the iterates; the assembly's and the
// finalize's scratch lives in the iterate vectors, which are free before the first and after the last iteration.
enum DenseVec : int {
    D_PX = 0, D_PY, D_NX, D_NY, D_H, D_LFW, D_INVD, D_MX, D_MY, D_XP, D_YP, D_SX, D_SY, D_KR,
    D_LB, D_UB, D_F,
    D_AL, D_LU, D_LL, D_SU, D_SL, D_S3, D_S4, D_L3, D_L4, D_KL, D_DX, D_ED, D_RHS, D_DD, D_WK, D_TU, D_TL, D_T3, D_T4,
    D_VV, D_ETV,
    DV
};

__host__ __device__ constexpr size_t dense_smem_bytes(int m) { return (2 * (size_t)m * m + (size_t)DV * m) * sizeof(double); }
static_assert(dense_smem_bytes(MC_DENSE_N_MAX) + 64 * sizeof(double) <= 227 * 1024,
              "E, K and the vectors of the largest dense instance must fit in one CTA's shared memory");

// y = E x (a warp per row)
__device__ __forceinline__ void dense_E(const double *E, int m, int n, const double *x, double *y) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    for (int i = w; i < n; i += DENSE_THREADS / 32) {
        double s = 0.0;
        for (int j = lane; j < n; j += 32) s += E[(size_t)i * m + j] * x[j];
        s = warp_sum(s);
        if (lane == 0) y[i] = s;
    }
    __syncthreads();
}
// y = E^T x (a thread per column)
__device__ __forceinline__ void dense_Et(const double *E, int m, int n, const double *x, double *y) {
    for (int j = threadIdx.x; j < n; j += DENSE_THREADS) {
        double s = 0.0;
        for (int i = 0; i < n; ++i) s += E[(size_t)i * m + j] * x[i];
        y[j] = s;
    }
    __syncthreads();
}

// K = E^T diag(1 + w) E + diag(d) (lower triangle) and its Cholesky factor L L^T in place; false on a non-positive pivot
__device__ bool dense_factor(const double *E, double *K, int m, int n, const double *w, const double *d) {
    for (int idx = threadIdx.x; idx < n * n; idx += DENSE_THREADS) {
        const int i = idx / n, j = idx - i * n;
        if (j > i) continue;
        double s = 0.0;
        for (int k = 0; k < n; ++k) s += E[(size_t)k * m + i] * (1.0 + w[k]) * E[(size_t)k * m + j];
        K[(size_t)i * m + j] = (i == j) ? s + d[i] : s;
    }
    __syncthreads();
    for (int j = 0; j < n; ++j) {
        double *Kj = K + (size_t)j * m;
        const double p = Kj[j];
        if (!(p > 0.0)) return false;          // (every thread reads the same pivot: the exit is uniform)
        const double ljj = sqrt(p), il = 1.0 / ljj;
        for (int i = j + 1 + threadIdx.x; i < n; i += DENSE_THREADS) K[(size_t)i * m + j] *= il;
        __syncthreads();
        if (threadIdx.x == 0) Kj[j] = ljj;
        const int r = n - j - 1;
        for (int idx = threadIdx.x; idx < r * r; idx += DENSE_THREADS) {
            const int i = j + 1 + idx / r, k = j + 1 + idx % r;
            if (k <= i) K[(size_t)i * m + k] -= K[(size_t)i * m + j] * K[(size_t)k * m + j];
        }
        __syncthreads();
    }
    return true;
}

// x = (L L^T)^{-1} r; r is overwritten (x may alias r)
__device__ void dense_solve(const double *L, int m, int n, double *r, double *x) {
    for (int j = 0; j < n; ++j) {               // L y = r
        const double yj = r[j] / L[(size_t)j * m + j];
        for (int i = j + 1 + threadIdx.x; i < n; i += DENSE_THREADS) r[i] -= L[(size_t)i * m + j] * yj;
        __syncthreads();
        if (threadIdx.x == 0) r[j] = yj;
    }
    __syncthreads();
    for (int j = n - 1; j >= 0; --j) {          // L^T x = y
        const double xj = r[j] / L[(size_t)j * m + j];
        for (int i = threadIdx.x; i < j; i += DENSE_THREADS) r[i] -= L[(size_t)j * m + i] * xj;
        __syncthreads();
        if (threadIdx.x == 0) x[j] = xj;
    }
    __syncthreads();
}

__device__ __forceinline__ double d_affine_step(double r) { return (r > 1.0) ? 1.0 / r : 1.0; }
__device__ __forceinline__ double d_damped_step(double eta, double r) { return (eta < r) ? eta / r : 1.0; }

// The QP of one instance in shared memory (mincurv_setup.cu P1-P5): bounds LB / UB, the spline quantities, E, k_ref and
// f = f_scale E^T k_ref; false (every thread alike) when a box is empty (lb > ub: status 1).  LIN: about the line P + la n.
// Called by every thread of the CTA; its scratch lives in the iterate vectors D_AL .. D_L4.
template <bool LIN>
__device__ __forceinline__ bool dense_assemble(double *s_dense, int m, int n, const double *rt, const double *nv,
                                               const double *hb, const double *la, double wv, double f_scale, int &s_flag) {
    double *E = s_dense;
    auto dv = [&](int v) { return s_dense + 2 * (size_t)m * m + (size_t)v * m; };
    double *PX = dv(D_PX), *PY = dv(D_PY), *NX = dv(D_NX), *NY = dv(D_NY), *H = dv(D_H), *LFW = dv(D_LFW);
    double *INVD = dv(D_INVD), *MX = dv(D_MX), *MY = dv(D_MY), *XP = dv(D_XP), *YP = dv(D_YP), *SX = dv(D_SX);
    double *SY = dv(D_SY), *KR = dv(D_KR), *LB = dv(D_LB), *UB = dv(D_UB), *F = dv(D_F);
    double *DG = dv(D_AL), *DFW = dv(D_LU), *DBW = dv(D_LL), *T0 = dv(D_SU), *T1 = dv(D_SL), *Y0 = dv(D_S3);
    double *Y1 = dv(D_S4), *Z0 = dv(D_L3), *Z1 = dv(D_L4);

    // ---- bounds (mincurv_setup.cu P1) ----
    if (threadIdx.x == 0) s_flag = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const int im1 = (i == 0) ? n - 1 : i - 1;
        const double hi = hb[i], him = hb[im1];
        PX[i] = rt[(size_t)i * 4]; PY[i] = rt[(size_t)i * 4 + 1];
        NX[i] = nv[(size_t)i * 2]; NY[i] = nv[(size_t)i * 2 + 1];
        H[i] = hi;
        DG[i] = 2.0 * (him + hi);
        double ub = rt[(size_t)i * 4 + 2] - 0.5 * wv;       // dev_max_right
        double lb = -(rt[(size_t)i * 4 + 3] - 0.5 * wv);    // -dev_max_left
        if (lb > ub) s_flag = 1;
        if (ub - lb < 2.0 * FIX_EPS) { const double mid = 0.5 * (lb + ub); lb = mid - FIX_EPS; ub = mid + FIX_EPS; }
        LB[i] = lb; UB[i] = ub;
    }
    __syncthreads();
    if (s_flag) return false;

    // ---- spline quantities (mincurv_setup.cu P2-P5) ----
    tri_pivots(DG, H, DFW, DBW, n);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], him = H[im1];
        LFW[i] = him / DFW[im1];
        INVD[i] = 1.0 / DFW[i];
        T0[i] = 6.0 * ((PX[ip1] - PX[i]) / hi - (PX[i] - PX[im1]) / him);
        T1[i] = 6.0 * ((PY[ip1] - PY[i]) / hi - (PY[i] - PY[im1]) / him);
    }
    __syncthreads();
    tri_solve2(LFW, INVD, H, T0, T1, Y0, Y1, MX, MY, n);
    if (LIN) {              // moments of the shifted points P + a n, in Z0 / Z1
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
            const double hi = H[i], him = H[im1];
            const double x = PX[i] + la[i] * NX[i], xm = PX[im1] + la[im1] * NX[im1], xp = PX[ip1] + la[ip1] * NX[ip1];
            const double y = PY[i] + la[i] * NY[i], ym = PY[im1] + la[im1] * NY[im1], yp = PY[ip1] + la[ip1] * NY[ip1];
            T0[i] = 6.0 * ((xp - x) / hi - (x - xm) / him);
            T1[i] = 6.0 * ((yp - y) / hi - (y - ym) / him);
        }
        __syncthreads();
        tri_solve2(LFW, INVD, H, T0, T1, Y0, Y1, Z0, Z1, n);
    }
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], h2 = hi * hi;
        double xp, yp;
        if constexpr (LIN) {
            xp = ((PX[ip1] + la[ip1] * NX[ip1]) - (PX[i] + la[i] * NX[i])) - h2 * (2.0 * Z0[i] + Z0[ip1]) * (1.0 / 6.0);
            yp = ((PY[ip1] + la[ip1] * NY[ip1]) - (PY[i] + la[i] * NY[i])) - h2 * (2.0 * Z1[i] + Z1[ip1]) * (1.0 / 6.0);
        } else {
            xp = (PX[ip1] - PX[i]) - h2 * (2.0 * MX[i] + MX[ip1]) * (1.0 / 6.0);
            yp = (PY[ip1] - PY[i]) - h2 * (2.0 * MY[i] + MY[ip1]) * (1.0 / 6.0);
        }
        const double q = xp * xp + yp * yp;
        const double c = 1.0 / (q * sqrt(q));
        const double sy = c * xp * h2, sx = c * yp * h2;
        XP[i] = xp; YP[i] = yp; SX[i] = sx; SY[i] = sy; KR[i] = sy * MY[i] - sx * MX[i];
    }
    __syncthreads();

    // ---- explicit E, two columns of Z = Tri^{-1} 6 D2 per solve ----
    for (int j0 = 0; j0 < n; j0 += 2) {
        const int j1 = (j0 + 1 < n) ? j0 + 1 : j0;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            auto col = [&](int j) {         // 6 D2 e_j
                const int jm1 = (j == 0) ? n - 1 : j - 1, jp1 = (j + 1 == n) ? 0 : j + 1;
                return (i == jm1) ? 6.0 / H[jm1] : (i == jp1) ? 6.0 / H[j] : (i == j) ? -6.0 / H[j] - 6.0 / H[jm1] : 0.0;
            };
            T0[i] = col(j0);
            T1[i] = col(j1);
        }
        __syncthreads();
        tri_solve2(LFW, INVD, H, T0, T1, Y0, Y1, Z0, Z1, n);
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            E[(size_t)i * m + j0] = Z0[i] * (SY[i] * NY[j0] - SX[i] * NX[j0]);
            E[(size_t)i * m + j1] = Z1[i] * (SY[i] * NY[j1] - SX[i] * NX[j1]);
        }
        __syncthreads();
    }
    dense_Et(E, m, n, KR, F);
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) F[i] *= f_scale;
    __syncthreads();
    return true;
}

// The post-solve quantities of mincurv_finalize_kernel at alpha = D_AL, for the QP dense_assemble<LIN> left in s_dense:
// kmax = max |k_ref + E alpha| and emax = curv_error_max (each NaN if any of its terms is, as there), and viol = 1 where
// some point has |k_ref + E alpha| > kb (1 + 1e-7) or a NaN there, else 0.  The iterate vectors D_LU .. D_S4 are scratch.
// Called by every thread of the CTA; the forward kernel and mincurv_dense_eval_kernel share it.
template <bool LIN>
__device__ __forceinline__ void dense_post_solve(double *s_dense, int m, int n, double kb, double *red, double &kmax,
                                                 double &emax, double &viol) {
    auto dv = [&](int v) { return s_dense + 2 * (size_t)m * m + (size_t)v * m; };
    const double *PX = dv(D_PX), *PY = dv(D_PY), *NX = dv(D_NX), *NY = dv(D_NY), *H = dv(D_H), *LFW = dv(D_LFW);
    const double *INVD = dv(D_INVD), *MX = dv(D_MX), *MY = dv(D_MY), *XP = dv(D_XP), *YP = dv(D_YP), *SX = dv(D_SX);
    const double *SY = dv(D_SY), *KR = dv(D_KR), *AL = dv(D_AL);
    double *U0 = dv(D_LU), *U1 = dv(D_LL), *W0 = dv(D_SU), *W1 = dv(D_SL), *ZX = dv(D_S3), *ZY = dv(D_S4);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], him = H[im1];
        const double vx = NX[i] * AL[i], vxm = NX[im1] * AL[im1], vxp = NX[ip1] * AL[ip1];
        const double vy = NY[i] * AL[i], vym = NY[im1] * AL[im1], vyp = NY[ip1] * AL[ip1];
        U0[i] = 6.0 * ((vxp - vx) / hi - (vx - vxm) / him);
        U1[i] = 6.0 * ((vyp - vy) / hi - (vy - vym) / him);
    }
    __syncthreads();
    tri_solve2(LFW, INVD, H, U0, U1, W0, W1, ZX, ZY, n);
    kmax = 0.0; emax = 0.0; viol = 0.0;
    bool nan_k = false, nan_e = false;           // (both maxima propagate a NaN, as in mincurv_finalize_kernel)
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], h2 = hi * hi;
        const double zx = ZX[i], zy = ZY[i];
        const double kl = fabs(KR[i] + SY[i] * zy - SX[i] * zx);
        kmax = fmax(kmax, kl);
        nan_k = nan_k || kl != kl;
        if (!(kl <= kb * (1.0 + 1e-7))) viol = 1.0;         // (a NaN iterate counts as a violation)
        const double ddx = h2 * (MX[i] + zx), ddy = h2 * (MY[i] + zy);
        const double xp = XP[i], yp = YP[i];
        double xc = xp, yc = yp;                // first derivatives of the centre line
        if (LIN) {
            xc = (PX[ip1] - PX[i]) - h2 * (2.0 * MX[i] + MX[ip1]) * (1.0 / 6.0);
            yc = (PY[ip1] - PY[i]) - h2 * (2.0 * MY[i] + MY[ip1]) * (1.0 / 6.0);
        }
        const double xpt = xc + (NX[ip1] * AL[ip1] - NX[i] * AL[i]) - h2 * (2.0 * zx + ZX[ip1]) * (1.0 / 6.0);
        const double ypt = yc + (NY[ip1] * AL[ip1] - NY[i] * AL[i]) - h2 * (2.0 * zy + ZY[ip1]) * (1.0 / 6.0);
        const double q0 = xp * xp + yp * yp, q1 = xpt * xpt + ypt * ypt;
        const double c0 = (xp * ddy - yp * ddx) / (q0 * sqrt(q0));
        const double c1 = (xpt * ddy - ypt * ddx) / (q1 * sqrt(q1));
        emax = fmax(emax, fabs(c1 - c0));
        nan_e = nan_e || c1 - c0 != c1 - c0;
    }
    kmax = block_reduce<1>(kmax, red);
    emax = block_reduce<1>(emax, red);
    viol = block_reduce<1>(viol, red);
    if (__syncthreads_or(nan_k)) kmax = NAN;
    if (__syncthreads_or(nan_e)) emax = NAN;
}

// a follower of centre_id: the banded path's validity rule (its QP is assembled on its own all the same)
__device__ __forceinline__ bool dense_follower_ok(const int32_t *centre_id, const int32_t *n_pts, int n_max, int b, int n) {
    const int o = centre_id[b];
    return !(o < 0 || o >= (int)gridDim.x || centre_id[o] != o || (n_pts ? n_pts[o] : n_max) != n);
}

// banded: the banded stages ran on this batch (they own the status of every instance outside [3, dense_below)); otherwise
// this kernel writes the refusal (status -1) of instances with n < 3 or n > n_max too.
// EXPORT: the row export of mincurv_sens_rows_export_kernel for the instances this kernel writes the status of: the final
// iterate's sens[b] = (lu / su, ll / sl), sens_rows[b] = l3 / s3 + l4 / s4, n_rows[b] = #{weight > 1} and grad_status[b]
// = status[b]; zeros beyond n and wherever the status is not 0.  It is written before the post-solve quantities, which
// take the iterate vectors as scratch.
// PROX: the projection QP of mc_mincurv_solve_batch_ex(prox_x, prox_dense_below), Hessian E^T E + prox_mu I and linear term
// c = prox_mu q - (E^T E + prox_mu I) x (x = prox_x[b], q = prox_q[b]; f_scale does not enter): c replaces f, and prox_mu
// goes on the diagonal of K and, as + prox_mu a, into the gradient, the right-hand sides and the dual residual, as in
// mincurv_pdip_kappa_kernel<true>.  Not with EXPORT.  Without PROX prox_mu, prox_x and prox_q are not read.
template <bool LIN, bool EXPORT, bool PROX>
__global__ void __launch_bounds__(DENSE_THREADS)
mincurv_dense_kernel(int n_max, int m, int dense_below, int banded, const int32_t *__restrict__ n_pts,
                     const double *__restrict__ reftrack, const double *__restrict__ normvec, const double *__restrict__ hin,
                     double kappa_bound, const double *__restrict__ kappa_bound_batch, double w_veh,
                     const double *__restrict__ w_veh_batch, double f_scale, const int32_t *__restrict__ centre_id,
                     const double *__restrict__ lin_alpha, PdipParams prm, double *__restrict__ alpha,
                     double *__restrict__ curv_error_max, double *__restrict__ kappa_lin_max, int32_t *__restrict__ status,
                     int32_t *__restrict__ iters, double *__restrict__ sens, double *__restrict__ sens_rows,
                     int32_t *__restrict__ n_rows, int32_t *__restrict__ grad_status, double prox_mu,
                     const double *__restrict__ prox_x, const double *__restrict__ prox_q) {
    static_assert(!(PROX && EXPORT), "the projection QP has no sensitivity export");
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    __shared__ double red[32];
    __shared__ int s_flag;
    extern __shared__ __align__(16) double s_dense[];
    double *aout = alpha + (size_t)b * n_max;
    double *du = EXPORT ? sens + (size_t)b * 2 * n_max : nullptr, *dl = du + n_max;
    double *wr = EXPORT ? sens_rows + (size_t)b * n_max : nullptr;
    auto export_zeros = [&]() {
        for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) { du[i] = 0.0; dl[i] = 0.0; wr[i] = 0.0; }
        if (threadIdx.x == 0) n_rows[b] = 0;
    };
    // the outputs of a refused instance: those of the banded path (alpha 0 over the whole row, no iterations)
    auto refuse = [&](int st) {
        for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) aout[i] = 0.0;
        if constexpr (EXPORT) export_zeros();
        if (threadIdx.x == 0) {
            status[b] = st;
            curv_error_max[b] = 0.0;
            if (kappa_lin_max) kappa_lin_max[b] = 0.0;
            if (iters) iters[b] = 0;
            if constexpr (EXPORT) grad_status[b] = st;
        }
    };
    const bool owned = n >= 3 && n < dense_below && n <= n_max;
    if (!owned) {
        if (!banded && (n < 3 || n > n_max)) refuse(-1);
        return;
    }
    if (centre_id && centre_id[b] != b && !dense_follower_ok(centre_id, n_pts, n_max, b, n)) { refuse(-1); return; }
    const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
    const double kb = kappa_bound_batch ? kappa_bound_batch[b] : kappa_bound;
    if (!(fabs(wv) < INFINITY) || !(kb > 0.0 && kb < INFINITY)) { refuse(-1); return; }

    double *E = s_dense, *K = s_dense + (size_t)m * m;
    auto dv = [&](int v) { return s_dense + 2 * (size_t)m * m + (size_t)v * m; };
    double *PX = dv(D_PX), *PY = dv(D_PY), *NX = dv(D_NX), *NY = dv(D_NY), *H = dv(D_H), *LFW = dv(D_LFW);
    double *INVD = dv(D_INVD), *MX = dv(D_MX), *MY = dv(D_MY), *XP = dv(D_XP), *YP = dv(D_YP), *SX = dv(D_SX);
    double *SY = dv(D_SY), *KR = dv(D_KR), *LB = dv(D_LB), *UB = dv(D_UB), *F = dv(D_F);
    double *AL = dv(D_AL), *LU = dv(D_LU), *LL = dv(D_LL), *SU = dv(D_SU), *SL = dv(D_SL), *S3 = dv(D_S3);
    double *S4 = dv(D_S4), *L3 = dv(D_L3), *L4 = dv(D_L4), *KL = dv(D_KL), *DX = dv(D_DX), *ED = dv(D_ED);
    double *RHS = dv(D_RHS), *DD = dv(D_DD), *WK = dv(D_WK), *TU = dv(D_TU), *TL = dv(D_TL), *T3 = dv(D_T3);
    double *T4 = dv(D_T4), *VV = dv(D_VV), *ETV = dv(D_ETV);

    const double *rt = reftrack + (size_t)b * n_max * 4;
    const double *nv = normvec + (size_t)b * n_max * 2;
    const double *hb = hin + (size_t)b * n_max;
    const double *la = LIN ? lin_alpha + (size_t)b * n_max : nullptr;

    if (!dense_assemble<LIN>(s_dense, m, n, rt, nv, hb, la, wv, f_scale, s_flag)) { refuse(1); return; }
    const double pmu = PROX ? prox_mu : 0.0;        // (+ pmu a below: only in the PROX instantiations)
    if constexpr (PROX) {       // c = mu q - (H + mu I) x in F (mincurv_prox_kernel); AL, ED and ETV as scratch
        const double *px = prox_x + (size_t)b * n_max, *pq = prox_q + (size_t)b * n_max;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) AL[i] = px[i];
        __syncthreads();
        dense_E(E, m, n, AL, ED);
        dense_Et(E, m, n, ED, ETV);
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) F[i] = pmu * pq[i] - (ETV[i] + pmu * AL[i]);
        __syncthreads();
    }

    // ---- interior point on the box and the curvature rows (the iteration of mincurv_pdip_kappa_kernel) ----
    const double m4 = 4.0 * n;
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) AL[i] = 0.5 * (LB[i] + UB[i]);
    __syncthreads();
    dense_E(E, m, n, AL, ED);
    dense_Et(E, m, n, ED, ETV);
    double gmax = 0.0, fmaxv = 0.0;
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        gmax = fmax(gmax, fabs(PROX ? ETV[i] + pmu * AL[i] + F[i] : ETV[i] + F[i]));
        fmaxv = fmax(fmaxv, fabs(F[i]));
    }
    gmax = block_reduce<1>(gmax, red);
    fmaxv = block_reduce<1>(fmaxv, red);
    const double lam0 = prm.lam0_rel * gmax + 1e-300;
    double musum = 0.0;
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const double gi = PROX ? ETV[i] + pmu * AL[i] + F[i] : ETV[i] + F[i];
        const double lu = fmax(-gi, 0.0) + lam0, ll = fmax(gi, 0.0) + lam0;
        const double a = AL[i], su = UB[i] - a, sl = a - LB[i];
        const double kl = KR[i] + ED[i];
        const double s3 = fmax(kb - kl, 1e-2 * kb), s4 = fmax(kb + kl, 1e-2 * kb);
        LU[i] = lu; LL[i] = ll; SU[i] = su; SL[i] = sl;
        KL[i] = kl; S3[i] = s3; S4[i] = s4; L3[i] = lam0; L4[i] = lam0;
        musum += su * lu + sl * ll + (s3 + s4) * lam0;
    }
    musum = block_reduce<0>(musum, red);
    const double mu0 = musum / m4;
    const double rd_tol = prm.rd_rel * (fmaxv + gmax) + 1e-300;
    double mu = mu0;
    int it = 0, result = 2;
    double rdmax = 1e300, rpmax = 1e300;
    for (it = 0; it < prm.max_iter + 20; ++it) {
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i];
            const double rp3 = kl + s3 - kb, rp4 = -kl + s4 - kb;
            WK[i] = l3 / s3 + l4 / s4;
            DD[i] = PROX ? LU[i] / SU[i] + LL[i] / SL[i] + pmu : LU[i] / SU[i] + LL[i] / SL[i];
            VV[i] = (kl - KR[i]) + l3 * rp3 / s3 - l4 * rp4 / s4;
        }
        __syncthreads();
        dense_Et(E, m, n, VV, ETV);
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) RHS[i] = PROX ? -F[i] - ETV[i] - pmu * AL[i] : -F[i] - ETV[i];
        if (!dense_factor(E, K, m, n, WK, DD)) {
            result = (mu <= 1e-7 * mu0 && rdmax <= 1e3 * rd_tol && rpmax <= 1e-6 * kb) ? 0 : 3;
            break;
        }
        dense_solve(K, m, n, RHS, DX);
        dense_E(E, m, n, DX, ED);
        // ---- affine step lengths and centring ----
        double rp = 0.0, rdl = 0.0, c00 = 0.0, c01 = 0.0, c10 = 0.0, c11 = 0.0;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            const double su = SU[i], sl = SL[i], lu = LU[i], ll = LL[i], dx = DX[i];
            const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = ED[i];
            const double p = dx / su, mm = dx / sl;
            const double ds3 = -(kl + s3 - kb) - ed, ds4 = -(-kl + s4 - kb) + ed;
            const double dlu = lu * (p - 1.0), dll = -ll * (1.0 + mm);
            const double dl3 = -l3 - l3 * ds3 / s3, dl4 = -l4 - l4 * ds4 / s4;
            rp = fmax(rp, fmax(fmax(p, -mm), fmax(-ds3 / s3, -ds4 / s4)));
            rdl = fmax(rdl, fmax(fmax(1.0 - p, 1.0 + mm), fmax(-dl3 / l3, -dl4 / l4)));
            c00 += su * lu + sl * ll + s3 * l3 + s4 * l4;
            c01 += su * dlu + sl * dll + s3 * dl3 + s4 * dl4;
            c10 += dx * (ll - lu) + ds3 * l3 + ds4 * l4;
            c11 += dx * (dll - dlu) + ds3 * dl3 + ds4 * dl4;
        }
        rp = block_reduce<1>(rp, red);
        rdl = block_reduce<1>(rdl, red);
        double ap = d_affine_step(rp), ad = d_affine_step(rdl);
        c00 = block_reduce<0>(c00, red); c01 = block_reduce<0>(c01, red);
        c10 = block_reduce<0>(c10, red); c11 = block_reduce<0>(c11, red);
        const double sigma = (c00 + ad * c01 + ap * c10 + ap * ad * c11) / m4 / mu;
        const double smu = sigma * sigma * sigma * mu;
        // ---- corrector right-hand side ----
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            const double su = SU[i], sl = SL[i], lu = LU[i], ll = LL[i], dx = DX[i], isu = 1.0 / su, isl = 1.0 / sl;
            const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = ED[i];
            const double rp3 = kl + s3 - kb, rp4 = -kl + s4 - kb;
            const double ds3 = -rp3 - ed, ds4 = -rp4 + ed;
            const double dlu = lu * (dx * isu - 1.0), dll = -ll * (1.0 + dx * isl);
            const double dl3 = -l3 - l3 * ds3 / s3, dl4 = -l4 - l4 * ds4 / s4;
            const double tu = smu - su * lu + dx * dlu, tl = smu - sl * ll - dx * dll;
            const double q3 = smu - s3 * l3 - ds3 * dl3, q4 = smu - s4 * l4 - ds4 * dl4;
            TU[i] = tu; TL[i] = tl; T3[i] = q3; T4[i] = q4;
            VV[i] = (kl - KR[i]) + l3 - l4 + (q3 + l3 * rp3) / s3 - (q4 + l4 * rp4) / s4;
            RHS[i] = -(F[i] + lu - ll) - tu * isu + tl * isl;
        }
        __syncthreads();
        dense_Et(E, m, n, VV, ETV);
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) RHS[i] -= PROX ? ETV[i] + pmu * AL[i] : ETV[i];
        __syncthreads();
        dense_solve(K, m, n, RHS, DX);
        dense_E(E, m, n, DX, ED);
        rp = 0.0; rdl = 0.0;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            const double lu = LU[i], ll = LL[i], dx = DX[i], isu = 1.0 / SU[i], isl = 1.0 / SL[i];
            const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = ED[i];
            const double ds3 = -(kl + s3 - kb) - ed, ds4 = -(-kl + s4 - kb) + ed;
            const double dlu = (TU[i] + lu * dx) * isu, dll = (TL[i] - ll * dx) * isl;
            const double dl3 = (T3[i] - l3 * ds3) / s3, dl4 = (T4[i] - l4 * ds4) / s4;
            rp = fmax(rp, fmax(fmax(dx * isu, -dx * isl), fmax(-ds3 / s3, -ds4 / s4)));
            rdl = fmax(rdl, fmax(fmax(-dlu / lu, -dll / ll), fmax(-dl3 / l3, -dl4 / l4)));
        }
        rp = block_reduce<1>(rp, red);
        rdl = block_reduce<1>(rdl, red);
        ap = d_damped_step(prm.eta, rp);
        ad = d_damped_step(prm.eta, rdl);
        double musum2 = 0.0;
        rpmax = 0.0;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            const double su = SU[i], sl = SL[i], lu = LU[i], ll = LL[i], dx = DX[i];
            const double s3 = S3[i], s4 = S4[i], l3 = L3[i], l4 = L4[i], kl = KL[i], ed = ED[i];
            const double ds3 = -(kl + s3 - kb) - ed, ds4 = -(-kl + s4 - kb) + ed;
            const double dlu = (TU[i] + lu * dx) / su, dll = (TL[i] - ll * dx) / sl;
            const double dl3 = (T3[i] - l3 * ds3) / s3, dl4 = (T4[i] - l4 * ds4) / s4;
            const double sun = su - ap * dx, sln = sl + ap * dx, s3n = s3 + ap * ds3, s4n = s4 + ap * ds4;
            const double lun = lu + ad * dlu, lln = ll + ad * dll, l3n = l3 + ad * dl3, l4n = l4 + ad * dl4;
            const double kln = kl + ap * ed;
            AL[i] += ap * dx; SU[i] = sun; SL[i] = sln;
            LU[i] = lun; LL[i] = lln; S3[i] = s3n; S4[i] = s4n; L3[i] = l3n; L4[i] = l4n; KL[i] = kln;
            VV[i] = (kln - KR[i]) + l3n - l4n;
            musum2 += sun * lun + sln * lln + s3n * l3n + s4n * l4n;
            rpmax = fmax(rpmax, fmax(fabs(kln + s3n - kb), fabs(-kln + s4n - kb)));
        }
        mu = block_reduce<0>(musum2, red) / m4;
        rpmax = block_reduce<1>(rpmax, red);
        __syncthreads();
        // dual residual r_d = E^T (kl - k_ref + l3 - l4) (+ mu a) + f + lu - ll
        dense_Et(E, m, n, VV, ETV);
        rdmax = 0.0;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS)
            rdmax = fmax(rdmax, fabs(PROX ? ETV[i] + pmu * AL[i] + F[i] + LU[i] - LL[i] : ETV[i] + F[i] + LU[i] - LL[i]));
        rdmax = block_reduce<1>(rdmax, red);
        if (mu <= prm.mu_rel * mu0 && rdmax <= rd_tol && rpmax <= 1e-8 * kb) { result = 0; ++it; break; }
        if (mu <= 1e-2 * prm.mu_rel * mu0) { result = (rdmax <= 1e3 * rd_tol && rpmax <= 1e-6 * kb) ? 0 : 2; ++it; break; }
    }
    for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) aout[i] = (i < n) ? AL[i] : 0.0;
    if constexpr (EXPORT) {         // (status 4 from the post-solve check zeroes it again below)
        const int ne = (result == 0) ? n : 0;
        double strong = 0.0;
        for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) {
            const double w = (i < ne) ? L3[i] / S3[i] + L4[i] / S4[i] : 0.0;
            du[i] = (i < ne) ? LU[i] / SU[i] : 0.0;
            dl[i] = (i < ne) ? LL[i] / SL[i] : 0.0;
            wr[i] = w;
            strong += (w > 1.0) ? 1.0 : 0.0;
        }
        strong = block_reduce<0>(strong, red);
        if (threadIdx.x == 0) n_rows[b] = (int32_t)strong;
    }

    double kmax, emax, viol;
    dense_post_solve<LIN>(s_dense, m, n, kb, red, kmax, emax, viol);
    if constexpr (EXPORT) {
        if (result == 0 && viol > 0.0) export_zeros();
        if (threadIdx.x == 0) grad_status[b] = (viol > 0.0) ? 4 : result;
    }
    if (threadIdx.x == 0) {
        curv_error_max[b] = emax;
        if (kappa_lin_max) kappa_lin_max[b] = kmax;
        status[b] = (viol > 0.0) ? 4 : result;
        if (iters) iters[b] = it;
    }
}

// A = C C^T in place (lower triangle, row-major with leading dimension lda), every thread of the CTA; false on a
// non-positive pivot
__device__ bool dense_chol(double *A, int lda, int n) {
    for (int j = 0; j < n; ++j) {
        __syncthreads();
        const double p = A[(size_t)j * lda + j];
        if (!(p > 0.0)) return false;          // (every thread reads the same pivot: the exit is uniform)
        const double c = sqrt(p), ic = 1.0 / c;
        __syncthreads();
        if (threadIdx.x == 0) A[(size_t)j * lda + j] = c;
        for (int i = j + 1 + threadIdx.x; i < n; i += DENSE_THREADS) A[(size_t)i * lda + j] *= ic;
        __syncthreads();
        const int r = n - j - 1;
        for (int idx = threadIdx.x; idx < r * r; idx += DENSE_THREADS) {
            const int i = j + 1 + idx / r, k = j + 1 + idx % r;
            if (k <= i) A[(size_t)i * lda + k] -= A[(size_t)i * lda + j] * A[(size_t)k * lda + j];
        }
    }
    __syncthreads();
    return true;
}

// ================================================================================================
// K2e-d -- width sensitivities of the small tracks (DESIGN.md section 3.14): the derivative of K2d' (mincurv_ipm.cu) at the
// dense kernel's final iterate, which is always a curvature-row iterate, without band truncation.  With D = d_u + d_l
// (sens) and the row weights W (sens_rows) of the export:
//   (E^T E + D + E^T W E) v = g,   dL/dub = d_u v,  dL/dlb = d_l v
// split at W = 1 as K2d' does: K = E^T (I + W_weak) E + D by dense_factor, and the ms = n_rows[b] strong rows S
// (ascending) by Woodbury, Sigma = W_S^-1 + E_S K^-1 E_S^T in `schur` (n_rows_cap^2 doubles per instance, column j from
// one solve against row S_j of E), v = K^-1 g - K^-1 E_S^T Sigma^-1 E_S K^-1 g.  The split is needed without truncation
// too: W reaches 1e12 and more, and the late-accept exit returns status 0 at an iterate whose full normal matrix did not
// factor.  The bounds and E are re-assembled as the forward does; the gradients follow the collapsed-box rule of
// mincurv_adjoint_kernel.  One CTA per instance; those with 3 <= n < dense_below, n <= n_max.  banded: the banded
// adjoint ran before on this batch, with these instances held out (grad_status ^ DENSE_HOLD, restored here); otherwise
// this kernel writes the zero gradients of the other instances too.  grad_status 3 (zero gradients): more strong rows
// than n_rows_cap, or a non-positive pivot in K or in Sigma; any other grad_status != 0 is kept, with zero gradients.
__global__ void __launch_bounds__(DENSE_THREADS)
mincurv_dense_adjoint_kernel(int n_max, int m, int dense_below, int banded, const int32_t *__restrict__ n_pts,
                             const double *__restrict__ reftrack, const double *__restrict__ normvec,
                             const double *__restrict__ hin, double w_veh, const double *__restrict__ w_veh_batch,
                             double f_scale, const int32_t *__restrict__ centre_id, const double *__restrict__ sens,
                             const double *__restrict__ sens_rows, const int32_t *__restrict__ n_rows, double *schur,
                             int n_rows_cap, const double *__restrict__ grad_alpha, int32_t *__restrict__ grad_status,
                             double *__restrict__ grad_w_right, double *__restrict__ grad_w_left,
                             double *__restrict__ grad_w_veh) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    __shared__ double red[32];
    __shared__ int s_flag;
    extern __shared__ __align__(16) double s_dense[];
    double *gwr = grad_w_right + (size_t)b * n_max, *gwl = grad_w_left + (size_t)b * n_max;
    const bool owned = n >= 3 && n < dense_below && n <= n_max;
    if (!owned && banded) return;
    int gs = owned ? grad_status[b] : -1;
    if (banded) gs ^= DENSE_HOLD;
    if (owned && centre_id && centre_id[b] != b && !dense_follower_ok(centre_id, n_pts, n_max, b, n)) gs = -1;
    const int ms = owned ? n_rows[b] : 0;
    bool ok = gs == 0 && ms <= n_rows_cap;
    const double *rt = reftrack + (size_t)b * n_max * 4;
    const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
    if (ok) ok = dense_assemble<false>(s_dense, m, n, rt, normvec + (size_t)b * n_max * 2, hin + (size_t)b * n_max, nullptr,
                                       wv, f_scale, s_flag);
    if (ok) {
        double *E = s_dense, *K = s_dense + (size_t)m * m;
        auto dv = [&](int v) { return s_dense + 2 * (size_t)m * m + (size_t)v * m; };
        double *DD = dv(D_DD), *WK = dv(D_WK), *X = dv(D_DX), *Y = dv(D_RHS), *U = dv(D_VV);
        int *S = reinterpret_cast<int *>(dv(D_ETV));        // the strong rows, ascending
        const double *DU = sens + (size_t)b * 2 * n_max, *DL = DU + n_max, *WR = sens_rows + (size_t)b * n_max;
        const double *GA = grad_alpha + (size_t)b * n_max;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
            DD[i] = DU[i] + DL[i];
            WK[i] = (WR[i] <= 1.0) ? WR[i] : 0.0;
            X[i] = GA[i];
        }
        if (warp == 0) {
            int cnt = 0;
            for (int base = 0; base < n; base += 32) {
                const bool st = base + lane < n && WR[base + lane] > 1.0;
                const unsigned bal = __ballot_sync(0xffffffffu, st);
                if (st) S[cnt + __popc(bal & ((1u << lane) - 1u))] = base + lane;
                cnt += __popc(bal);
            }
        }
        __syncthreads();
        ok = dense_factor(E, K, m, n, WK, DD);
        if (ok) dense_solve(K, m, n, X, X);                // K^-1 g
        if (ok && ms > 0) {
            double *Sg = schur + (size_t)b * n_rows_cap * n_rows_cap;      // Sigma, row-major, lower triangle used
            for (int j = 0; j < ms; ++j) {          // column j: E_S K^-1 E_{S_j}^T + e_j / W_{S_j}
                for (int i = threadIdx.x; i < n; i += DENSE_THREADS) Y[i] = E[(size_t)S[j] * m + i];
                __syncthreads();
                dense_solve(K, m, n, Y, Y);
                for (int k = j + warp; k < ms; k += DENSE_THREADS / 32) {
                    double t = 0.0;
                    for (int i = lane; i < n; i += 32) t += E[(size_t)S[k] * m + i] * Y[i];
                    t = warp_sum(t);
                    if (lane == 0) Sg[(size_t)k * n_rows_cap + j] = t + ((k == j) ? 1.0 / WR[S[j]] : 0.0);
                }
                __syncthreads();
            }
            for (int k = warp; k < ms; k += DENSE_THREADS / 32) {       // u = E_S K^-1 g
                double t = 0.0;
                for (int i = lane; i < n; i += 32) t += E[(size_t)S[k] * m + i] * X[i];
                t = warp_sum(t);
                if (lane == 0) U[k] = t;
            }
            ok = dense_chol(Sg, n_rows_cap, ms);
            if (ok) {
                dense_solve(Sg, n_rows_cap, ms, U, U);                 // z = Sigma^-1 u
                for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {  // v = K^-1 g - K^-1 E_S^T z
                    double t = 0.0;
                    for (int k = 0; k < ms; ++k) t += E[(size_t)S[k] * m + i] * U[k];
                    Y[i] = t;
                }
                __syncthreads();
                dense_solve(K, m, n, Y, Y);
                for (int i = threadIdx.x; i < n; i += DENSE_THREADS) X[i] -= Y[i];
                __syncthreads();
            }
        }
        if (ok) {       // the widths (mincurv_setup.cu P1); a collapsed box follows its mid point
            double gv = 0.0;
            for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) {
                double gr = 0.0, gl = 0.0;
                if (i < n) {
                    const double v = X[i], gu = DU[i] * v, glb = DL[i] * v;
                    const double ub = rt[(size_t)i * 4 + 2] - 0.5 * wv, lb = -(rt[(size_t)i * 4 + 3] - 0.5 * wv);
                    if (ub - lb < 2.0 * FIX_EPS) {
                        gr = 0.5 * (gu + glb);
                        gl = -gr;
                    } else {
                        gr = gu;
                        gl = -glb;
                        gv += 0.5 * (glb - gu);
                    }
                }
                gwr[i] = gr;
                gwl[i] = gl;
            }
            gv = block_reduce<0>(gv, red);
            if (threadIdx.x == 0) grad_w_veh[b] = gv;
        }
    }
    if (!ok) {
        for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) { gwr[i] = 0.0; gwl[i] = 0.0; }
        if (threadIdx.x == 0) grad_w_veh[b] = 0.0;
    }
    if (owned && threadIdx.x == 0) grad_status[b] = (gs == 0 && !ok) ? 3 : gs;
}

// held out of the banded adjoint kernels, which factor every instance with grad_status 0 (a track below N_MIN would wrap
// their band onto itself): the instances the dense adjoint takes get grad_status ^ DENSE_HOLD, nonzero whatever it was
__global__ void mincurv_dense_hold_kernel(int B, int n_max, int dense_below, const int32_t *__restrict__ n_pts,
                                          int32_t *__restrict__ grad_status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int n = n_pts ? n_pts[b] : n_max;
    if (n >= 3 && n < dense_below && n <= n_max) grad_status[b] ^= DENSE_HOLD;
}

int mincurv_dense_hold(int B, int n_max, int dense_below, const int32_t *n_pts, int32_t *grad_status, void *stream) {
    mincurv_dense_hold_kernel<<<(B + 255) / 256, 256, 0, (cudaStream_t)stream>>>(B, n_max, dense_below, n_pts, grad_status);
    return check_cuda("mincurv_dense_hold_kernel");
}

int mincurv_dense_adjoint(int B, int n_max, int dense_below, bool banded, const int32_t *n_pts, const double *reftrack,
                          const double *normvec, const double *h, double w_veh, const double *w_veh_batch, double f_scale,
                          const int32_t *centre_id, const double *sens, int32_t *grad_status, const double *grad_alpha,
                          double *grad_w_right, double *grad_w_left, double *grad_w_veh, const double *sens_rows,
                          const int32_t *n_rows, double *schur, int n_rows_cap, void *stream) {
    const int m = n_max < dense_below - 1 ? n_max : dense_below - 1;
    const int smem = (int)dense_smem_bytes(m);
    if (cudaFuncSetAttribute(mincurv_dense_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return check_cuda("mincurv_dense_adjoint_kernel: cudaFuncSetAttribute");
    mincurv_dense_adjoint_kernel<<<B, DENSE_THREADS, smem, (cudaStream_t)stream>>>(
        n_max, m, dense_below, banded ? 1 : 0, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, sens,
        sens_rows, n_rows, schur, n_rows_cap, grad_alpha, grad_status, grad_w_right, grad_w_left, grad_w_veh);
    return check_cuda("mincurv_dense_adjoint_kernel");
}

// ================================================================================================
// K2e-v -- the post-solve quantities at a given alpha (mc_mincurv_finalize_batch with dense_below, for
// raceline_refine.CurvatureProjection.evaluate): those of the finalize stage after the assembly, with its status rules,
// for the instances with 3 <= n < dense_below,
// n <= n_max: status -1 (a vehicle width that is not finite, or a limit that is not finite or not > 0) or 1 (lb > ub) with
// both maxima 0; otherwise kappa_lin_max and curv_error_max of dense_post_solve (NaN-propagating) and status 4 iff
// kappa_lin_max > kb (1 + 1e-7) (a NaN maximum leaves 0), else 0.
template <bool LIN>
__global__ void __launch_bounds__(DENSE_THREADS)
mincurv_dense_eval_kernel(int n_max, int m, int dense_below, const int32_t *__restrict__ n_pts,
                          const double *__restrict__ reftrack, const double *__restrict__ normvec,
                          const double *__restrict__ hin, double kappa_bound, const double *__restrict__ kappa_bound_batch,
                          double w_veh, const double *__restrict__ w_veh_batch, const double *__restrict__ lin_alpha,
                          const double *__restrict__ alpha, double *__restrict__ curv_error_max,
                          double *__restrict__ kappa_lin_max, int32_t *__restrict__ status) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    if (!(n >= 3 && n < dense_below && n <= n_max)) return;
    __shared__ double red[32];
    __shared__ int s_flag;
    extern __shared__ __align__(16) double s_dense[];
    const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
    const double kb = kappa_bound_batch ? kappa_bound_batch[b] : kappa_bound;
    int st = (fabs(wv) < INFINITY && kb > 0.0 && kb < INFINITY) ? 0 : -1;
    if (st == 0 && !dense_assemble<LIN>(s_dense, m, n, reftrack + (size_t)b * n_max * 4, normvec + (size_t)b * n_max * 2,
                                        hin + (size_t)b * n_max, LIN ? lin_alpha + (size_t)b * n_max : nullptr, wv, 1.0,
                                        s_flag))
        st = 1;
    double kmax = 0.0, emax = 0.0, viol;
    if (st == 0) {
        double *AL = s_dense + 2 * (size_t)m * m + (size_t)D_AL * m;
        const double *ab = alpha + (size_t)b * n_max;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) AL[i] = ab[i];
        dense_post_solve<LIN>(s_dense, m, n, kb, red, kmax, emax, viol);
        if (kmax > kb * (1.0 + 1e-7)) st = 4;
    }
    if (threadIdx.x == 0) {
        curv_error_max[b] = emax;
        kappa_lin_max[b] = kmax;
        status[b] = st;
    }
}

// one CTA per instance with dense_smem_bytes(m) of shared memory, m = min(n_max, dense_below - 1)
template <typename Kernel, typename... Args>
static int dense_launch(Kernel kernel, const char *name, int B, int n_max, int dense_below, void *stream, Args... args) {
    const int m = n_max < dense_below - 1 ? n_max : dense_below - 1;
    const int smem = (int)dense_smem_bytes(m);
    // (per launch: the attribute is per device and a process may drive several)
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return check_cuda(name);
    kernel<<<B, DENSE_THREADS, smem, (cudaStream_t)stream>>>(n_max, m, dense_below, args...);
    return check_cuda(name);
}

// the curvature-row phase's parameters (mincurv_kappa_phase)
static PdipParams dense_params() {
    PdipParams prm;
    prm.max_iter = 40;
    prm.mu_rel = 1e-11;
    prm.rd_rel = 1e-8;
    prm.eta = 0.995;
    prm.dx_rel = 0.0;
    prm.lam0_rel = 1e-2;
    return prm;
}

// launched after the banded stages (banded != 0), or alone when n_max < N_MIN
int mincurv_dense(int B, int n_max, int dense_below, bool banded, const int32_t *n_pts, const double *reftrack,
                  const double *normvec, const double *h, double kappa_bound, const double *kappa_bound_batch, double w_veh,
                  const double *w_veh_batch, double f_scale, const int32_t *centre_id, const double *lin_alpha, double *alpha,
                  double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters, double *sens,
                  int32_t *grad_status, double *sens_rows, int32_t *n_rows, void *stream) {
    auto kernel = sens ? (lin_alpha ? mincurv_dense_kernel<true, true, false> : mincurv_dense_kernel<false, true, false>)
                       : (lin_alpha ? mincurv_dense_kernel<true, false, false> : mincurv_dense_kernel<false, false, false>);
    return dense_launch(kernel, "mincurv_dense_kernel", B, n_max, dense_below, stream, banded ? 1 : 0, n_pts, reftrack,
                        normvec, h, kappa_bound, kappa_bound_batch, w_veh, w_veh_batch, f_scale, centre_id, lin_alpha,
                        dense_params(), alpha, curv_error_max, kappa_lin_max, status, iters, sens, sens_rows, n_rows,
                        grad_status, 0.0, (const double *)nullptr, (const double *)nullptr);
}

// the projection QP of mc_mincurv_solve_batch_ex(prox_x, prox_dense_below) on the small tracks alone
int mincurv_dense_prox(int B, int n_max, int dense_below, const int32_t *n_pts, const double *reftrack,
                       const double *normvec, const double *h, double kappa_bound, const double *kappa_bound_batch,
                       double w_veh, const double *w_veh_batch, double prox_mu, const double *prox_x, const double *prox_q,
                       const double *lin_alpha, double *alpha, double *curv_error_max, double *kappa_lin_max,
                       int32_t *status, int32_t *iters, void *stream) {
    auto kernel = lin_alpha ? mincurv_dense_kernel<true, false, true> : mincurv_dense_kernel<false, false, true>;
    return dense_launch(kernel, "mincurv_dense_kernel (prox)", B, n_max, dense_below, stream, 1, n_pts, reftrack, normvec, h,
                        kappa_bound, kappa_bound_batch, w_veh, w_veh_batch, 1.0, (const int32_t *)nullptr, lin_alpha,
                        dense_params(), alpha, curv_error_max, kappa_lin_max, status, iters, (double *)nullptr,
                        (double *)nullptr, (int32_t *)nullptr, (int32_t *)nullptr, prox_mu, prox_x, prox_q);
}

// the post-solve evaluation of mc_mincurv_finalize_batch(dense_below) on the small tracks alone
int mincurv_dense_eval(int B, int n_max, int dense_below, const int32_t *n_pts, const double *reftrack,
                       const double *normvec, const double *h, double kappa_bound, const double *kappa_bound_batch,
                       double w_veh, const double *w_veh_batch, const double *lin_alpha, const double *alpha,
                       double *curv_error_max, double *kappa_lin_max, int32_t *status, void *stream) {
    auto kernel = lin_alpha ? mincurv_dense_eval_kernel<true> : mincurv_dense_eval_kernel<false>;
    return dense_launch(kernel, "mincurv_dense_eval_kernel", B, n_max, dense_below, stream, n_pts, reftrack, normvec, h,
                        kappa_bound, kappa_bound_batch, w_veh, w_veh_batch, lin_alpha, alpha, curv_error_max,
                        kappa_lin_max, status);
}

}  // namespace mc
