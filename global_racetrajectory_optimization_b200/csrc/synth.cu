// Device-side generation of sweep inputs (SURVEY.md section 8d "generate on device from the seed"): the width-jitter
// variants of a set of centre lines that BASELINE.json configs C2 / C4 sweep over (veh_width x w_tr jitter grid,
// main_globaltraj.py:442-496 runs its sweeps the same way: one prepared track, many parameter sets).
// A 256k-track N = 2000 sweep is 16 GB of reftracks: generated here from a few base tracks and one 64-bit seed per
// variant instead of being copied from the host.
//
//   out[v][i][0..1] = base[c][i][0..1]                       c = centre_id[v] (or v % n_base)
//   out[v][i][2+s]  = base[c][i][2+s] * (1 + rel * g_s(i / n)),   g_s(u) = (1/3) sum_{k=0..2} a_k cos(2 pi (k+1) u + p_k)
// with a_k in [-1, 1), p_k in [0, 2 pi) drawn from splitmix64(seed[v], s, k): the same stateless hash is implemented in
// numpy (synth.jitter_widths_hash), so the CPU baseline and the tests see the same variants (cos differs by an ulp).
#include "capi.cuh"
#include "common.cuh"

namespace mc {

__host__ __device__ inline uint64_t splitmix64(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__host__ __device__ inline double u01(uint64_t h) { return (double)(h >> 11) * (1.0 / 9007199254740992.0); }      // [0, 1)

__global__ void __launch_bounds__(256)
jitter_widths_kernel(int V, int n_max, const int32_t *__restrict__ n_pts_base, int n_base, const double *__restrict__ base,
                     const int32_t *__restrict__ centre_id, const int64_t *__restrict__ seed, double rel,
                     double *__restrict__ out, int32_t *__restrict__ n_pts_out) {
    const int v = blockIdx.x;
    if (v >= V) return;
    const int c = centre_id ? centre_id[v] : v % n_base;
    const int n = n_pts_base ? n_pts_base[c] : n_max;
    __shared__ double amp[2][3], ph[2][3];
    if (threadIdx.x < 6) {
        const int s = threadIdx.x / 3, k = threadIdx.x % 3;
        const uint64_t h0 = splitmix64((uint64_t)seed[v] * 6ull + (uint64_t)(2 * (3 * s + k)));
        const uint64_t h1 = splitmix64((uint64_t)seed[v] * 6ull + (uint64_t)(2 * (3 * s + k) + 1) + 0x5851F42D4C957F2Dull);
        amp[s][k] = 2.0 * u01(h0) - 1.0;
        ph[s][k] = 6.283185307179586476925286766559 * u01(h1);
    }
    __syncthreads();
    if (threadIdx.x == 0 && n_pts_out) n_pts_out[v] = n;
    const double *src = base + (size_t)c * n_max * 4;
    double *dst = out + (size_t)v * n_max * 4;
    const double inv_n = 1.0 / (double)n;
    for (int i = threadIdx.x; i < n_max; i += blockDim.x) {
        double2 xy = make_double2(0.0, 0.0), w = make_double2(0.0, 0.0);
        if (i < n) {
            xy = *reinterpret_cast<const double2 *>(src + (size_t)i * 4);
            w = *reinterpret_cast<const double2 *>(src + (size_t)i * 4 + 2);
            const double u = (double)i * inv_n;
            double g0 = 0.0, g1 = 0.0;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const double arg = 6.283185307179586476925286766559 * (double)(k + 1) * u;
                g0 += amp[0][k] * cos(arg + ph[0][k]);
                g1 += amp[1][k] * cos(arg + ph[1][k]);
            }
            w.x *= 1.0 + rel * (g0 * (1.0 / 3.0));
            w.y *= 1.0 + rel * (g1 * (1.0 / 3.0));
        }
        *reinterpret_cast<double2 *>(dst + (size_t)i * 4) = xy;
        *reinterpret_cast<double2 *>(dst + (size_t)i * 4 + 2) = w;
    }
}

// Length of the closed polygon through the points p_i + s_i n_i of every track (s: a per-point shift such as alpha, or a
// width column of the track times +-1; no normals: the points themselves) -- the host sizes re-sampling buffers from it
// (create_raceline / interp_track / iqp_handler capacities) with one small read instead of torch reductions.
__global__ void __launch_bounds__(256)
polygon_length_kernel(int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ pts, int stride,
                      const double *__restrict__ normvec, const double *__restrict__ shift, int shift_stride, double sign,
                      double *__restrict__ length) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    if (n > n_max) {                   // a count beyond the row: length 0 (the re-sampling kernels refuse the track)
        if (threadIdx.x == 0) length[b] = 0.0;
        return;
    }
    __shared__ double red[32];
    double acc = 0.0;
    const double *P = pts + (size_t)b * n_max * stride;
    const double *Nv = normvec ? normvec + (size_t)b * n_max * 2 : nullptr;
    const double *S = shift ? shift + (size_t)b * n_max * shift_stride : nullptr;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int j = (i + 1 == n) ? 0 : i + 1;
        double x0 = P[(size_t)i * stride], y0 = P[(size_t)i * stride + 1], x1 = P[(size_t)j * stride], y1 = P[(size_t)j * stride + 1];
        if (Nv && S) {
            const double s0 = sign * S[(size_t)i * shift_stride], s1 = sign * S[(size_t)j * shift_stride];
            x0 += s0 * Nv[2 * i]; y0 += s0 * Nv[2 * i + 1]; x1 += s1 * Nv[2 * j]; y1 += s1 * Nv[2 * j + 1];
        }
        acc += sqrt((x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0));
    }
    acc = block_reduce<0>(acc, red);
    if (threadIdx.x == 0) length[b] = (n > 1) ? acc : 0.0;
}

}  // namespace mc

extern "C" {

int mc_polygon_length_batch(int B, int n_max, const int32_t *n_pts, const double *pts, int stride, const double *normvec,
                            const double *shift, int shift_stride, double sign, double *length, void *stream) {
    if (B <= 0 || n_max <= 0 || !pts || stride < 2 || !length || ((normvec == nullptr) != (shift == nullptr)) ||
        (shift && shift_stride < 1))
        return bad("mc_polygon_length_batch: bad argument");
    mc::polygon_length_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_pts, pts, stride, normvec, shift, shift_stride,
                                                                   sign, length);
    return check_cuda("polygon_length_kernel");
}

int mc_jitter_widths_batch(int V, int n_max, const int32_t *n_pts_base, int n_base, const double *base,
                           const int32_t *centre_id, const int64_t *seed, double rel, double *out, int32_t *n_pts_out,
                           void *stream) {
    if (V <= 0 || n_max <= 0 || n_base <= 0 || !base || !seed || !out || !(rel >= 0.0) || rel >= 1.0)
        return bad("mc_jitter_widths_batch: bad argument");
    mc::jitter_widths_kernel<<<V, 256, 0, (cudaStream_t)stream>>>(V, n_max, n_pts_base, n_base, base, centre_id, seed, rel, out,
                                                                  n_pts_out);
    return check_cuda("jitter_widths_kernel");
}

}  // extern "C"
