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

// banded: the banded stages ran on this batch (they own the status of every instance outside [3, dense_below)); otherwise
// this kernel writes the refusal (status -1) of instances with n < 3 or n > n_max too.
template <bool LIN>
__global__ void __launch_bounds__(DENSE_THREADS)
mincurv_dense_kernel(int n_max, int m, int dense_below, int banded, const int32_t *__restrict__ n_pts,
                     const double *__restrict__ reftrack, const double *__restrict__ normvec, const double *__restrict__ hin,
                     double kappa_bound, const double *__restrict__ kappa_bound_batch, double w_veh,
                     const double *__restrict__ w_veh_batch, double f_scale, const int32_t *__restrict__ centre_id,
                     const double *__restrict__ lin_alpha, PdipParams prm, double *__restrict__ alpha,
                     double *__restrict__ curv_error_max, double *__restrict__ kappa_lin_max, int32_t *__restrict__ status,
                     int32_t *__restrict__ iters) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    __shared__ double red[32];
    __shared__ int s_flag;
    extern __shared__ __align__(16) double s_dense[];
    double *aout = alpha + (size_t)b * n_max;
    // the outputs of a refused instance: those of the banded path (alpha 0 over the whole row, no iterations)
    auto refuse = [&](int st) {
        for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) aout[i] = 0.0;
        if (threadIdx.x == 0) {
            status[b] = st;
            curv_error_max[b] = 0.0;
            if (kappa_lin_max) kappa_lin_max[b] = 0.0;
            if (iters) iters[b] = 0;
        }
    };
    const bool owned = n >= 3 && n < dense_below && n <= n_max;
    if (!owned) {
        if (!banded && (n < 3 || n > n_max)) refuse(-1);
        return;
    }
    if (centre_id && centre_id[b] != b) {       // a follower: the banded path's validity rule; its QP is assembled here
        const int o = centre_id[b];
        if (o < 0 || o >= (int)gridDim.x || centre_id[o] != o || (n_pts ? n_pts[o] : n_max) != n) { refuse(-1); return; }
    }
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
    // assembly scratch (in the iterate vectors)
    double *DG = dv(D_AL), *DFW = dv(D_LU), *DBW = dv(D_LL), *T0 = dv(D_SU), *T1 = dv(D_SL), *Y0 = dv(D_S3);
    double *Y1 = dv(D_S4), *Z0 = dv(D_L3), *Z1 = dv(D_L4);

    const double *rt = reftrack + (size_t)b * n_max * 4;
    const double *nv = normvec + (size_t)b * n_max * 2;
    const double *hb = hin + (size_t)b * n_max;
    const double *la = LIN ? lin_alpha + (size_t)b * n_max : nullptr;

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
    if (s_flag) { refuse(1); return; }

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

    // ---- interior point on the box and the curvature rows (the iteration of mincurv_pdip_kappa_kernel) ----
    const double m4 = 4.0 * n;
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) AL[i] = 0.5 * (LB[i] + UB[i]);
    __syncthreads();
    dense_E(E, m, n, AL, ED);
    dense_Et(E, m, n, ED, ETV);
    double gmax = 0.0, fmaxv = 0.0;
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        gmax = fmax(gmax, fabs(ETV[i] + F[i]));
        fmaxv = fmax(fmaxv, fabs(F[i]));
    }
    gmax = block_reduce<1>(gmax, red);
    fmaxv = block_reduce<1>(fmaxv, red);
    const double lam0 = prm.lam0_rel * gmax + 1e-300;
    double musum = 0.0;
    for (int i = threadIdx.x; i < n; i += DENSE_THREADS) {
        const double gi = ETV[i] + F[i];
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
            DD[i] = LU[i] / SU[i] + LL[i] / SL[i];
            VV[i] = (kl - KR[i]) + l3 * rp3 / s3 - l4 * rp4 / s4;
        }
        __syncthreads();
        dense_Et(E, m, n, VV, ETV);
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) RHS[i] = -F[i] - ETV[i];
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
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) RHS[i] -= ETV[i];
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
        // dual residual r_d = E^T (kl - k_ref + l3 - l4) + f + lu - ll
        dense_Et(E, m, n, VV, ETV);
        rdmax = 0.0;
        for (int i = threadIdx.x; i < n; i += DENSE_THREADS) rdmax = fmax(rdmax, fabs(ETV[i] + F[i] + LU[i] - LL[i]));
        rdmax = block_reduce<1>(rdmax, red);
        if (mu <= prm.mu_rel * mu0 && rdmax <= rd_tol && rpmax <= 1e-8 * kb) { result = 0; ++it; break; }
        if (mu <= 1e-2 * prm.mu_rel * mu0) { result = (rdmax <= 1e3 * rd_tol && rpmax <= 1e-6 * kb) ? 0 : 2; ++it; break; }
    }
    for (int i = threadIdx.x; i < n_max; i += DENSE_THREADS) aout[i] = (i < n) ? AL[i] : 0.0;

    // ---- post-solve quantities (mincurv_finalize_kernel) ----
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
    double kmax = 0.0, emax = 0.0, viol = 0.0;
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
    if (threadIdx.x == 0) {
        curv_error_max[b] = emax;
        if (kappa_lin_max) kappa_lin_max[b] = kmax;
        status[b] = (viol > 0.0) ? 4 : result;
        if (iters) iters[b] = it;
    }
}

// launched after the banded stages (banded != 0), or alone when n_max < N_MIN
int mincurv_dense(int B, int n_max, int dense_below, bool banded, const int32_t *n_pts, const double *reftrack,
                  const double *normvec, const double *h, double kappa_bound, const double *kappa_bound_batch, double w_veh,
                  const double *w_veh_batch, double f_scale, const int32_t *centre_id, const double *lin_alpha, double *alpha,
                  double *curv_error_max, double *kappa_lin_max, int32_t *status, int32_t *iters, void *stream) {
    PdipParams prm;                     // those of the curvature-row phase (mincurv_kappa_phase)
    prm.max_iter = 40;
    prm.mu_rel = 1e-11;
    prm.rd_rel = 1e-8;
    prm.eta = 0.995;
    prm.dx_rel = 0.0;
    prm.lam0_rel = 1e-2;
    const int m = n_max < dense_below - 1 ? n_max : dense_below - 1;
    const int smem = (int)dense_smem_bytes(m);
    auto kernel = lin_alpha ? mincurv_dense_kernel<true> : mincurv_dense_kernel<false>;
    // (per launch: the attribute is per device and a process may drive several)
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return check_cuda("mincurv_dense_kernel: cudaFuncSetAttribute");
    kernel<<<B, DENSE_THREADS, smem, (cudaStream_t)stream>>>(n_max, m, dense_below, banded ? 1 : 0, n_pts, reftrack, normvec,
                                                             h, kappa_bound, kappa_bound_batch, w_veh, w_veh_batch, f_scale,
                                                             centre_id, lin_alpha, prm, alpha, curv_error_max, kappa_lin_max,
                                                             status, iters);
    return check_cuda("mincurv_dense_kernel");
}

}  // namespace mc
