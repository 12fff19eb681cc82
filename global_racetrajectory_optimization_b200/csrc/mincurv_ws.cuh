// Per-instance scratch layout of the minimum-curvature path (all float64, one slab per QP instance).
//
// HBM layout (DESIGN.md section 3): slab b starts at ws + b * stride doubles and holds
//   [NUM_VEC][np]        O(N) vectors (geometry, linearisation, interior-point iterates)
//   [n_max][ZB_PITCH]    bands of B_t = Ti diag(w_t) Ti, t = 0..2  (assembly scratch, mincurv_setup.cu)
//   [np][HB_PITCH]       band of H = E^T E              (row i: H[i][i .. i+32], cyclic; [33] padding)
//   [np][33] + [np][33] + [np]  bordered LDL^T factor of H + D: chain rows [band of (Q - I; L21) | w] per panel of eight
//                        columns, fill rows [G | w], and z = w y of the last forward substitution (mincurv_ipm.cu)
// With shared centre lines a follower's band stays in its owner's slab: V_HBSRC says whose band an instance uses.
#pragma once
#include "capi.cuh"
#include "common.cuh"

namespace mc {

enum Vec : int {
    V_H = 0, V_DIAG, V_DFW, V_DBW, V_LFW, V_INVD, V_TII, V_RHOP, V_RHOM,
    V_PX, V_PY, V_NX, V_NY, V_MX, V_MY, V_XP, V_YP, V_SX, V_SY, V_KREF,
    V_LB, V_UB, V_F,
    V_T0, V_T1, V_T2, V_T3, V_T4, V_T5,
    V_ALPHA, V_LU, V_LL, V_RD, V_RHS, V_DX, V_DXA, V_DD, V_DLU, V_DLL, V_SU, V_SL,   // (DXA: the box phase's affine direction)
    V_ISU, V_ISL, V_HBSRC,                                  // reciprocal slacks (K2b'), band source (band_owner)
    V_S3, V_S4, V_L3, V_L4, V_KL, V_WK, V_EDX, V_T3K, V_T4K, V_VV,   // curvature-row phase (K2b')
    V_IH,                                                   // 1 / h
    NUM_VEC
};

struct Layout {
    int n_max;
    int np;          // padded vector length (multiple of 32, >= n_max + 64)
    size_t o_zb, o_hb, o_tiles, stride;   // in doubles
};

__host__ __device__ inline Layout make_layout(int n_max) {
    Layout L;
    L.n_max = n_max;
    L.np = ((n_max + 31) / 32) * 32 + 64;
    size_t o = (size_t)NUM_VEC * L.np;
    L.o_zb = o;
    o += (size_t)n_max * ZB_PITCH;
    L.o_hb = o;
    o += (size_t)L.np * HB_PITCH;
    L.o_tiles = o;
    o += (size_t)L.np * 67;
    L.stride = (o + 15) & ~(size_t)15;
    return L;
}

// ints behind the slabs (within the 256 bytes there): the work counter of the persistent solver kernels and the schedule
// of the box phase's two launches (mincurv_ipm.cu)
constexpr int SCHED_INTS = 64;
static_assert(SCHED_INTS * sizeof(int) <= 256, "the counters behind the slabs");

// the slabs of B instances; the workspace is these and the 256 bytes of counters behind them (mc_mincurv_workspace_bytes)
static inline size_t mincurv_slabs_bytes(int B, int n_max) { return align256((size_t)B * make_layout(n_max).stride * sizeof(double)); }

// the argument checks every stage of the minimum-curvature path starts with
static inline int mincurv_args(const char *who, int B, int n_max, void *workspace, size_t workspace_bytes) {
    if (B <= 0) return bad("mincurv: B <= 0");
    if (n_max < N_MIN) return bad("mincurv: n_max below the supported minimum (%d points)", N_MIN);
    if (!workspace || workspace_bytes < mincurv_slabs_bytes(B, n_max) + 256) return small_workspace(who);
    return MC_OK;
}

struct PdipParams {
    int max_iter;
    double mu_rel;     // stop when mu <= mu_rel * mu0 ...
    double rd_rel;     // ... and |r_d|_inf <= rd_rel * (|f|_inf + |g0|_inf)
    double eta;        // fraction to the boundary
    double dx_rel;     // ... and the last step moved alpha by <= dx_rel * max(|alpha|_inf, 0.01 m)  (0: not checked)
    double lam0_rel;   // initial multipliers: max(-+g, 0) + lam0_rel * |g|_inf
};

// the curvature-row phase (mincurv_ipm.cu): mc_mincurv_kappa_batch with prox_mu = 0, the projection QP of
// mc_mincurv_solve_batch_ex (Hessian H + prox_mu I) with prox_mu > 0.  Not exported.
__attribute__((visibility("hidden")))
int mincurv_kappa_phase(int B, int n_max, const int32_t *n_pts, double kappa_bound, double prox_mu, double *alpha,
                        int32_t *status, int32_t *iters, void *workspace, size_t workspace_bytes, void *stream);

__device__ __forceinline__ double *vec(double *slab, const Layout &L, int v) { return slab + (size_t)v * L.np; }

// index of the instance whose slab holds this instance's band of H: its own, or with shared centre lines the owner's
// (written by mincurv_setup_kernel / mincurv_share_kernel, read by mincurv_pdip_kernel)
__device__ __forceinline__ int32_t *band_owner(double *slab, const Layout &L) { return reinterpret_cast<int32_t *>(vec(slab, L, V_HBSRC)); }

}  // namespace mc
