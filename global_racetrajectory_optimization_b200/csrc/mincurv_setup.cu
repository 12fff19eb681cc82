// K2a -- assembly of the minimum-curvature QP in banded form (replaces the dense 4N x 4N inverse and
// the ~10 dense GEMMs of tph.opt_min_curv, call site main_globaltraj.py:264-271).
//
// With the spline moments m = Tri^{-1} 6 D2 p (Tri cyclic tridiagonal, common.cuh) the quantities of
// SURVEY.md A.2/A.3 become O(N) or banded:
//   x', y'       = a1 coefficients of the reference spline          (A_ex_b A^{-1} q)
//   T_c q        = h^2 m                                            (A_ex_c A^{-1} q)
//   T_n{x,y} a   = h^2 Tri^{-1} 6 D2 (n_{x,y} a)   =>  E = S_y Z N_y - S_x Z N_x,  Z = Tri^{-1} 6 D2
//   H = E^T E (half-bandwidth 32 kept),  f = F_SCALE E^T k_ref,  k_ref = S_y m_y - S_x m_x
// The band of H is assembled in O(N b) from the semiseparable structure of Ti = Tri^{-1}
// (Ti[m][c] = Ti[c][c] prod rho+ for m > c, prod rho- for m < c):
//   H[i][j]  = ny_i ny_j A0[i][j] - (ny_i nx_j + nx_i ny_j) A1[i][j] + nx_i nx_j A2[i][j]
//   A_t      = (6 D2)^T B_t (6 D2)                      (9-point stencil, D2 tridiagonal)
//   B_t[c][c'] = sum_m w_t[m] Ti[m][c] Ti[m][c'],        w = (s_y^2, s_x s_y, s_x^2)
//              = Ti[c'][c] (Ti[c'][c'] U_t[c'] + Ti[c][c] V_t[c]) + Mid_t(c, c')          (c < c')
//   U_t[c] = w_t[c] + rho+_{c+1}^2 U_t[c+1],   V_t[c] = w_t[c] + rho-_{c-1}^2 V_t[c-1],
//   Mid_t(c, c'+1) = rho+_{c'+1} (Mid_t(c, c') + w_t[c'] Ti[c'][c] Ti[c'][c'])
// (exact sums over all m -- no truncation of E -- verified against the explicit E^T E in tools/).
// One CTA per QP instance; O(N) vectors and the B / H bands live in the instance's HBM slab.
//
// LIN: linearised about the line P + a n (a = lin_alpha) instead of the centre line P.  The first derivatives x', y'
// (and with them S_x, S_y) are those of the spline through Ps = P + a n, from its moments Ms; k_ref = S_y m_y - S_x m_x
// keeps the centre line's moments, since alpha still enters through E.  Then k_ref + E a is the knot curvature of the
// spline through Ps, and H, f and the curvature rows follow from S_x, S_y, k_ref as about the centre line.
#include "capi.cuh"
#include "mincurv_ops.cuh"

namespace mc {

template <bool LIN>
__global__ void __launch_bounds__(256)
mincurv_setup_kernel(int n_max, const int32_t *__restrict__ n_pts,
                     const double *__restrict__ reftrack, const double *__restrict__ normvec,
                     const double *__restrict__ hin, double w_veh, const double *__restrict__ w_veh_batch, double f_scale,
                     const int32_t *__restrict__ centre_id, double *__restrict__ ws, Layout L, int32_t *__restrict__ status,
                     const double *__restrict__ lin_alpha) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    double *slab = ws + (size_t)b * L.stride;
    __shared__ int s_flag;
    extern __shared__ __align__(16) double s_win[];       // sliding windows + store staging of the B-band recurrence (assemble_hband)
    if (threadIdx.x == 0) s_flag = 0;
    __syncthreads();
    if (n < N_MIN || n > n_max) {
        if (threadIdx.x == 0) status[b] = -1;   // unsupported size (see N_MIN)
        return;
    }
    if (threadIdx.x == 0) *band_owner(slab, L) = b;       // (a follower's is set by mincurv_share_kernel)
    const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
    const bool bad_wv = !(fabs(wv) < INFINITY);           // refused with status -1 (an owner still assembles)
    const double *rt = reftrack + (size_t)b * n_max * 4;
    const double *nv = normvec + (size_t)b * n_max * 2;
    const double *hb = hin + (size_t)b * n_max;

    double *H = vec(slab, L, V_H), *DG = vec(slab, L, V_DIAG), *DFW = vec(slab, L, V_DFW), *DBW = vec(slab, L, V_DBW);
    double *LFW = vec(slab, L, V_LFW), *INVD = vec(slab, L, V_INVD), *TII = vec(slab, L, V_TII);
    double *RHOP = vec(slab, L, V_RHOP), *RHOM = vec(slab, L, V_RHOM);
    double *PX = vec(slab, L, V_PX), *PY = vec(slab, L, V_PY), *NX = vec(slab, L, V_NX), *NY = vec(slab, L, V_NY);
    double *MX = vec(slab, L, V_MX), *MY = vec(slab, L, V_MY), *XP = vec(slab, L, V_XP), *YP = vec(slab, L, V_YP);
    double *SX = vec(slab, L, V_SX), *SY = vec(slab, L, V_SY), *KREF = vec(slab, L, V_KREF);
    double *LB = vec(slab, L, V_LB), *UB = vec(slab, L, V_UB), *F = vec(slab, L, V_F);
    double *T0 = vec(slab, L, V_T0), *T1 = vec(slab, L, V_T1), *T2 = vec(slab, L, V_T2), *T3 = vec(slab, L, V_T3);
    double *T4 = vec(slab, L, V_T4), *T5 = vec(slab, L, V_T5), *IH = vec(slab, L, V_IH);

    // ---- P1: coalesced, vectorised load of the reftrack rows [x, y, w_r, w_l] (32 B per point) ----
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double2 xy = *reinterpret_cast<const double2 *>(rt + (size_t)i * 4);
        const double2 ww = *reinterpret_cast<const double2 *>(rt + (size_t)i * 4 + 2);
        const double2 nn = *reinterpret_cast<const double2 *>(nv + (size_t)i * 2);
        const int im1 = (i == 0) ? n - 1 : i - 1;
        const double hi = hb[i], him = hb[im1];
        PX[i] = xy.x; PY[i] = xy.y; NX[i] = nn.x; NY[i] = nn.y;
        H[i] = hi;
        IH[i] = 1.0 / hi;
        DG[i] = 2.0 * (him + hi);
        double ub = ww.x - 0.5 * wv;          // dev_max_right
        double lb = -(ww.y - 0.5 * wv);       // -dev_max_left
        if (lb > ub) s_flag = 1;              // tph: "Problem not solvable, track might be too small ..."
        if (ub - lb < 2.0 * FIX_EPS) { const double mid = 0.5 * (lb + ub); lb = mid - FIX_EPS; ub = mid + FIX_EPS; }
        LB[i] = lb; UB[i] = ub;
    }
    __syncthreads();
    // Instances that share a centreline (same x, y, normals, spacing: e.g. the width variants of one track) share H, f and
    // k_ref, only the bounds differ: with centre_id the assembly runs once per centreline (the owner, centre_id[b] == b) and
    // mincurv_share_kernel copies its O(N) vectors into the followers' slabs; the band of H stays in the owner's slab.  An
    // owner finishes the assembly even when its own bounds are infeasible (its followers need it).
    const bool follower = centre_id && centre_id[b] != b;
    if (s_flag || bad_wv || follower) {
        if (threadIdx.x == 0) status[b] = bad_wv ? -1 : s_flag ? 1 : 0;
        if (follower || !centre_id) return;
    }
    // ---- P2/P3: periodic LDL^T of the spline system, decay ratios of its inverse ----
    tri_pivots(DG, H, DFW, DBW, n);
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int im1 = (i == 0) ? n - 1 : i - 1;
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], him = H[im1];
        LFW[i] = him / DFW[im1];
        INVD[i] = 1.0 / DFW[i];
        TII[i] = 1.0 / (DFW[i] + DBW[i] - DG[i]);
        RHOP[i] = -him / DBW[i];
        RHOM[i] = -hi / DFW[i];
        T0[i] = 6.0 * ((PX[ip1] - PX[i]) / hi - (PX[i] - PX[im1]) / him);
        T1[i] = 6.0 * ((PY[ip1] - PY[i]) / hi - (PY[i] - PY[im1]) / him);
    }
    __syncthreads();
    // ---- P4: moments of the reference line ----
    tri_solve2(LFW, INVD, H, T0, T1, T2, T3, MX, MY, n);
    // LIN: moments Ms of the shifted points Ps = P + a n, in T4 / T5 (free until the E^T solve below)
    const double *la = LIN ? lin_alpha + (size_t)b * n_max : nullptr;
    if (LIN) {
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int im1 = (i == 0) ? n - 1 : i - 1;
            const int ip1 = (i + 1 == n) ? 0 : i + 1;
            const double hi = H[i], him = H[im1];
            const double x = PX[i] + la[i] * NX[i], xm = PX[im1] + la[im1] * NX[im1], xp = PX[ip1] + la[ip1] * NX[ip1];
            const double y = PY[i] + la[i] * NY[i], ym = PY[im1] + la[im1] * NY[im1], yp = PY[ip1] + la[ip1] * NY[ip1];
            T0[i] = 6.0 * ((xp - x) / hi - (x - xm) / him);
            T1[i] = 6.0 * ((yp - y) / hi - (y - ym) / him);
        }
        __syncthreads();
        tri_solve2(LFW, INVD, H, T0, T1, T2, T3, T4, T5, n);
    }
    // ---- P5: linearisation point; right-hand sides of f = F_SCALE E^T k_ref ----
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], h2 = hi * hi;
        double xp, yp;
        if constexpr (LIN) {                    // first derivatives of the spline through Ps (moments in T4 / T5)
            xp = ((PX[ip1] + la[ip1] * NX[ip1]) - (PX[i] + la[i] * NX[i])) - h2 * (2.0 * T4[i] + T4[ip1]) * (1.0 / 6.0);
            yp = ((PY[ip1] + la[ip1] * NY[ip1]) - (PY[i] + la[i] * NY[i])) - h2 * (2.0 * T5[i] + T5[ip1]) * (1.0 / 6.0);
        } else {
            xp = (PX[ip1] - PX[i]) - h2 * (2.0 * MX[i] + MX[ip1]) * (1.0 / 6.0);
            yp = (PY[ip1] - PY[i]) - h2 * (2.0 * MY[i] + MY[ip1]) * (1.0 / 6.0);
        }
        const double q = xp * xp + yp * yp;
        const double c = 1.0 / (q * sqrt(q));
        const double sy = c * xp * h2, sx = c * yp * h2;
        const double kr = sy * MY[i] - sx * MX[i];
        XP[i] = xp; YP[i] = yp; SX[i] = sx; SY[i] = sy; KREF[i] = kr;
        T0[i] = sx * kr;
        T1[i] = sy * kr;
    }
    __syncthreads();
    // E^T v = N_y Z^T (S_y v) - N_x Z^T (S_x v),  Z^T = 6 D2 Tri^{-1}
    tri_solve2(LFW, INVD, H, T0, T1, T2, T3, T4, T5, n);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], him = H[im1];
        const double zx = 6.0 * ((T4[ip1] - T4[i]) / hi - (T4[i] - T4[im1]) / him);
        const double zy = 6.0 * ((T5[ip1] - T5[i]) / hi - (T5[i] - T5[im1]) / him);
        F[i] = f_scale * (NY[i] * zy - NX[i] * zx);
    }
    __syncthreads();
    assemble_hband(slab, L, n, nullptr, s_win);
    double *HB = slab + L.o_hb;
    for (int i = threadIdx.x; i < n; i += blockDim.x) HB[(size_t)i * HB_PITCH + HBW + 1] = 0.0;
    if (threadIdx.x == 0 && !s_flag && !bad_wv) status[b] = 0;
}

// followers of a shared centreline: copy the vectors the owner assembled (V_H .. V_KREF, V_F, V_IH) and point the
// follower at the owner's band of H.  The band is not copied: the interior-point kernel reads it from the owner's slab,
// so that the instances of one centre line share one copy in L2.  (The curvature-row phase assembles a weighted band in
// the instance's own slab from the copied vectors.)
__global__ void __launch_bounds__(256)
mincurv_share_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, const int32_t *__restrict__ centre_id,
                     double *__restrict__ ws, Layout L, int32_t *__restrict__ status) {
    const int b = blockIdx.x;
    const int o = centre_id[b];
    if (o == b) return;
    const int n = n_pts ? n_pts[b] : n_max;
    if (n < N_MIN || n > n_max) return;                       // (status -1 from the assembly kernel)
    if (o < 0 || o >= B || centre_id[o] != o || (n_pts ? n_pts[o] : n_max) != n) {
        if (threadIdx.x == 0) status[b] = -1;                 // not a valid owner
        return;
    }
    const double *src = ws + (size_t)o * L.stride;
    double *dst = ws + (size_t)b * L.stride;
    const size_t np = (size_t)L.np;
    auto copy = [&](size_t off, size_t count) {               // (all offsets and counts are multiples of 2 doubles)
        const double2 *s2 = reinterpret_cast<const double2 *>(src + off);
        double2 *d2 = reinterpret_cast<double2 *>(dst + off);
        for (size_t i = threadIdx.x; i < count / 2; i += blockDim.x) d2[i] = s2[i];
    };
    copy((size_t)V_H * np, (size_t)(V_KREF - V_H + 1) * np);
    copy((size_t)V_F * np, np);
    copy((size_t)V_IH * np, np);
    if (threadIdx.x == 0) *band_owner(dst, L) = o;
}

int mincurv_setup(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec, const double *h,
                  double w_veh, const double *w_veh_batch, double f_scale, const int32_t *centre_id, const double *lin_alpha,
                  int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    if (!reftrack || !normvec || !h || !status) return bad("mc_mincurv_setup_batch: NULL argument");
    if (!(f_scale > 0.0)) return bad("mc_mincurv_setup_batch: f_scale must be positive");
    int rc = mincurv_args("mc_mincurv_setup_batch", B, n_max, workspace, workspace_bytes);
    if (rc) return rc;
    const Layout L = make_layout(n_max);
    double *ws = (double *)workspace;
    cudaStream_t s = (cudaStream_t)stream;
    constexpr int smem = hband_win_doubles(256) * (int)sizeof(double);      // 49 KB: above the static limit
    // (per launch: the attribute is per device and a process may drive several)
    if (lin_alpha) {
        cudaFuncSetAttribute(mincurv_setup_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        mincurv_setup_kernel<true><<<B, 256, smem, s>>>(n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale,
                                                         centre_id, ws, L, status, lin_alpha);
    } else {
        cudaFuncSetAttribute(mincurv_setup_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        mincurv_setup_kernel<false><<<B, 256, smem, s>>>(n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale,
                                                          centre_id, ws, L, status, nullptr);
    }
    if (centre_id) mincurv_share_kernel<<<B, 256, 0, s>>>(B, n_max, n_pts, centre_id, ws, L, status);
    return check_cuda("mincurv_setup_kernel");
}

}  // namespace mc

extern "C" {

size_t mc_mincurv_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < mc::N_MIN) return 0;
    return mc::mincurv_slabs_bytes(B, n_max) + 256;      // + the work counters of the persistent solver kernels (SCHED_INTS)
}

int mc_mincurv_setup_batch_shared(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                  const double *h, double w_veh, const double *w_veh_batch, double f_scale,
                                  const int32_t *centre_id, int32_t *status, void *workspace, size_t workspace_bytes,
                                  void *stream) {
    return mc::mincurv_setup(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, centre_id, nullptr, status,
                             workspace, workspace_bytes, stream);
}

int mc_mincurv_setup_batch_ex(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                              const double *h, double w_veh, const double *w_veh_batch, double f_scale, int32_t *status,
                              const double *lin_alpha, void *workspace, size_t workspace_bytes, void *stream) {
    return mc::mincurv_setup(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, f_scale, nullptr, lin_alpha, status,
                             workspace, workspace_bytes, stream);
}

int mc_mincurv_setup_batch(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                           const double *h, double w_veh, const double *w_veh_batch, int32_t *status, void *workspace,
                           size_t workspace_bytes, void *stream) {
    return mc_mincurv_setup_batch_ex(B, n_max, n_pts, reftrack, normvec, h, w_veh, w_veh_batch, MC_F_SCALE_DEFAULT, status,
                                     nullptr, workspace, workspace_bytes, stream);
}

}  // extern "C"
