// Shared device helpers for the H100 (sm_90a) minimum-curvature path.
//
// Everything on this path is fp64: cond(H) reaches 1e9..1e11 (SURVEY.md section 7), so no tensor-core
// or fp32 shortcut applies.  The one structural idea shared by all kernels is in tri_*():
// the closed-spline system of tph.calc_splines (a 4N x 4N dense solve in the reference, call site
// helper_funcs_glob/src/prep_track.py:48-51) is a *cyclic symmetric tridiagonal*
// system in the spline moments; its inverse decays by >= 2x (typically 3.7x) per off-diagonal, so the
// cyclic solve is computed as the periodic solution of the bi-infinite system: every thread runs the
// LDL^T recurrences over its own chunk after a warm-up of TRI_WARM points (error <= 0.5^56 ~ 1e-17,
// typically 0.268^56), which makes the O(N) recurrences embarrassingly parallel.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

namespace mc {

constexpr int TRI_CHUNK = 8;     // points per thread in the chunked recurrences
constexpr int TRI_WARM = 56;     // warm-up length of the periodic recurrences
constexpr int ZB_PITCH = 108;    // per-point scratch row of the assembly: three B_t bands of 35 entries at pitch 36 (sector-aligned runs)
constexpr int HBW = 32;          // half-bandwidth kept of H = E^T E (truncation error ~1e-10 on alpha)
constexpr int HB_PITCH = 34;     // 33 used, padded so that a row is a multiple of 16 bytes
constexpr int N_MIN = 80;        // smallest supported closed track (band must not wrap onto itself)
constexpr double FIX_EPS = 1e-8; // half-width given to variables whose box has collapsed (lb == ub)

// Kernels that put the track index on blockIdx.y see at most 65535 tracks per launch: launch(b0, nb) is called for
// consecutive chunks of nb <= 65535 tracks starting at track b0, and offsets its pointers by b0.
template <class Launch>
inline void for_grid_y_chunks(int B, Launch &&launch) {
    constexpr int GRID_Y_MAX = 65535;
    for (int b0 = 0; b0 < B; b0 += GRID_Y_MAX) launch(b0, B - b0 < GRID_Y_MAX ? B - b0 : GRID_Y_MAX);
}

__device__ __forceinline__ int wrapi(int i, int n) {
    i %= n;
    return i < 0 ? i + n : i;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// Block-wide reductions (all threads get the result). `red` is a shared array of >= 32 doubles.
template <int OP>  // 0 sum, 1 max, 2 min
__device__ __forceinline__ double block_reduce(double v, double *red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = (OP == 0) ? warp_sum(v) : (OP == 1) ? warp_max(v) : warp_min(v);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    double r = (lane < nw) ? red[lane] : ((OP == 0) ? 0.0 : (OP == 1) ? -INFINITY : INFINITY);
    r = (OP == 0) ? warp_sum(r) : (OP == 1) ? warp_max(r) : warp_min(r);
    return r;
}

// ---------------------------------------------------------------------------------------------
// Periodic symmetric tridiagonal T: T[i][i] = diag[i], T[i][i+1] = T[i+1][i] = off[i] (cyclic).
// Block-cooperative; all arrays may live in global or shared memory; callers __syncthreads() after.
// ---------------------------------------------------------------------------------------------
// forward pivots dfw_i = diag_i - off_{i-1}^2 / dfw_{i-1}, backward pivots dbw_i = diag_i - off_i^2 / dbw_{i+1}
// Each chunk recurrence is split into its warm-up (no stores: unrolled, so that the loads of eight steps are in
// flight together -- rolled, every step paid one memory round trip and these loops were ~45 % of the assembly
// kernel) and the TRI_CHUNK steps that store.
__device__ inline void tri_pivots(const double *diag, const double *off, double *dfw, double *dbw, int n) {
    for (int c0 = threadIdx.x * TRI_CHUNK; c0 < n; c0 += blockDim.x * TRI_CHUNK) {
        const int c1 = min(c0 + TRI_CHUNK, n);
        int i = wrapi(c0 - TRI_WARM, n);
        double prev = diag[i];
#pragma unroll 8
        for (int s = 0; s < TRI_WARM - 1; ++s) {
            const double o = off[i];
            i = (i + 1 == n) ? 0 : i + 1;
            prev = diag[i] - o * o / prev;
        }
        for (int s = c0; s < c1; ++s) {
            const double o = off[i];
            i = (i + 1 == n) ? 0 : i + 1;
            prev = diag[i] - o * o / prev;
            dfw[i] = prev;
        }
        i = wrapi(c1 - 1 + TRI_WARM, n);
        double nxt = diag[i];
#pragma unroll 8
        for (int s = 0; s < TRI_WARM - 1; ++s) {
            i = (i == 0) ? n - 1 : i - 1;
            const double o = off[i];
            nxt = diag[i] - o * o / nxt;
        }
        for (int s = c1 - 1; s >= c0; --s) {
            i = (i == 0) ? n - 1 : i - 1;
            const double o = off[i];
            nxt = diag[i] - o * o / nxt;
            dbw[i] = nxt;
        }
    }
}

// Solve T m = r for two right-hand sides at once.  lfw_i = off_{i-1} / dfw_{i-1}, invd_i = 1 / dfw_i.
// y* are scratch of n doubles each (must not alias r*, m* must not alias y*; m* may alias r*).
__device__ inline void tri_solve2(const double *lfw, const double *invd, const double *off,
                                  const double *rx, const double *ry, double *yx, double *yy,
                                  double *mx, double *my, int n) {
    for (int c0 = threadIdx.x * TRI_CHUNK; c0 < n; c0 += blockDim.x * TRI_CHUNK) {
        const int c1 = min(c0 + TRI_CHUNK, n);
        int i = wrapi(c0 - TRI_WARM, n);
        double px = 0.0, py = 0.0;
#pragma unroll 8
        for (int s = 0; s < TRI_WARM; ++s) {
            const double l = lfw[i];
            px = rx[i] - l * px;
            py = ry[i] - l * py;
            i = (i + 1 == n) ? 0 : i + 1;
        }
        for (int s = c0; s < c1; ++s) {
            const double l = lfw[i];
            px = rx[i] - l * px;
            py = ry[i] - l * py;
            yx[i] = px; yy[i] = py;
            i = (i + 1 == n) ? 0 : i + 1;
        }
    }
    __syncthreads();
    for (int c0 = threadIdx.x * TRI_CHUNK; c0 < n; c0 += blockDim.x * TRI_CHUNK) {
        const int c1 = min(c0 + TRI_CHUNK, n);
        int i = wrapi(c1 - 1 + TRI_WARM, n);
        double nx = 0.0, ny = 0.0;
#pragma unroll 8
        for (int s = 0; s < TRI_WARM; ++s) {
            const double o = off[i], id = invd[i];
            nx = (yx[i] - o * nx) * id;
            ny = (yy[i] - o * ny) * id;
            i = (i == 0) ? n - 1 : i - 1;
        }
        for (int s = c1 - 1; s >= c0; --s) {
            const double o = off[i], id = invd[i];
            nx = (yx[i] - o * nx) * id;
            ny = (yy[i] - o * ny) * id;
            mx[i] = nx; my[i] = ny;
            i = (i == 0) ? n - 1 : i - 1;
        }
    }
    __syncthreads();
}

}  // namespace mc
