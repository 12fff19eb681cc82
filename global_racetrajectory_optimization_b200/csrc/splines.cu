// K1 / K3 -- closed cubic splines and everything evaluated on them:
//   calc_splines            (tph.calc_splines, call sites helper_funcs_glob/src/prep_track.py:48-51,
//                            main_globaltraj.py:568)                         SURVEY.md A.1
//   create_raceline         (tph.create_raceline incl. calc_spline_lengths / interp_splines,
//                            call site main_globaltraj.py:371-376)           SURVEY.md A.6
//   calc_head_curv_an       (call site main_globaltraj.py:383-387)           SURVEY.md A.7
//   iqp width interpolation (tph.interp_track_widths inside tph.iqp_handler, call site
//                            main_globaltraj.py:273-284)                     SURVEY.md A.5
// The dense 4N x 4N solve of the reference is the periodic tridiagonal moment system of common.cuh.
// One CTA per track; O(N) scratch vectors live in the caller-provided workspace (HBM, L2-resident).
#include "common.cuh"

namespace mc {

enum SVec : int { S_H = 0, S_DG, S_DFW, S_DBW, S_LFW, S_INVD, S_R0, S_R1, S_Y0, S_Y1, S_MX, S_MY, S_PX, S_PY, S_CUM, S_NUM };

__host__ __device__ inline int spl_np(int n_max) { return ((n_max + 31) / 32) * 32 + 32; }
size_t spline_ws_doubles(int n_max) { return (size_t)S_NUM * spl_np(n_max); }

// ---------------------------------------------------------------------------------------------
// Closed spline through (PX, PY) with parameter scales H on EIGHT vectors that live in shared memory whenever the track
// fits (n_max <= ~3400 points): H, PX, PY (inputs) and the five vectors of the periodic tridiagonal moment system
//   h_{i-1} m_{i-1} + 2 (h_{i-1} + h_i) m_i + h_i m_{i+1} = 6 ((p_{i+1} - p_i) / h_i - (p_i - p_{i-1}) / h_{i-1}).
// Tracks of up to 2048 points: PARALLEL CYCLIC REDUCTION, in place -- at stride s every equation eliminates its neighbours
// i - s and i + s with their own equations; the off-diagonal / diagonal ratio is squared by every step (diagonal dominance:
// <= 1/2 to start with), so after six steps (stride 64; five for uniform scales) the couplings are below 1e-17 of the
// diagonal and m = r / b.  All
// threads work on all points in every step (no serial recurrence, one reciprocal per point and step).  Longer tracks use
// the chunked LDL^T recurrences (every thread runs a chunk of TRI_CHUNK points after a warm-up of TRI_WARM points).
// (The first version kept fifteen scratch vectors per track in global memory -- 6.9 % of the HBM roofline; the second
// ran the chunked recurrences for every track: 64 dependent steps with divisions per thread, 3.7 %.)
// ---------------------------------------------------------------------------------------------
constexpr int SPL_SM_VECS = 8;
__host__ __device__ inline size_t spline_smem_bytes(int n_max) { return (size_t)SPL_SM_VECS * spl_np(n_max) * sizeof(double); }
constexpr size_t SPL_SMEM_LIMIT = 220 * 1024;

__device__ __forceinline__ double spl_rcp(double d) {      // 1 / d for a positive normal d (seed + two Newton steps)
    double r;
    asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
    r = fma(r, fma(-d, r, 1.0), r);
    return fma(r, fma(-d, r, 1.0), r);
}

// moments MX, MY (vectors 6, 7) by parallel cyclic reduction; EPT = points per thread (n <= EPT * blockDim.x).
// The equations are kept normalised (diagonal 1): a_i m_{i-s} + m_i + c_i m_{i+s} = r_i, so a step costs one reciprocal.
template <int EPT>
__device__ void spline_moments_pcr(double *sm, int np, int n, int s_end) {
    const double *H = sm, *PX = sm + np, *PY = sm + 2 * np;
    double *A = sm + 3 * np, *C = sm + 5 * np, *RX = sm + 6 * np, *RY = sm + 7 * np;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double hi = H[i], hm = H[im1];
        const double ih = spl_rcp(hi), ihm = spl_rcp(hm), w = 6.0 * spl_rcp(2.0 * (hm + hi));
        const double px = PX[i], py = PY[i];
        A[i] = hm * w * (1.0 / 6.0); C[i] = hi * w * (1.0 / 6.0);
        RX[i] = w * ((PX[ip1] - px) * ih - (px - PX[im1]) * ihm);
        RY[i] = w * ((PY[ip1] - py) * ih - (py - PY[im1]) * ihm);
    }
    __syncthreads();
    for (int s = 1; s < s_end; s <<= 1) {
        double na[EPT], nc[EPT], nx[EPT], ny[EPT];
        const int st = s % n;                                   // (tiny tracks: the stride wraps)
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int i = threadIdx.x + e * blockDim.x;
            if (i < n) {
                int im = i - st; if (im < 0) im += n;
                int ip = i + st; if (ip >= n) ip -= n;
                const double k1 = A[i], k2 = C[i];
                const double w = spl_rcp(fma(-C[im], k1, fma(-A[ip], k2, 1.0)));
                na[e] = -A[im] * k1 * w;
                nc[e] = -C[ip] * k2 * w;
                nx[e] = fma(-RX[im], k1, fma(-RX[ip], k2, RX[i])) * w;
                ny[e] = fma(-RY[im], k1, fma(-RY[ip], k2, RY[i])) * w;
            }
        }
        __syncthreads();
#pragma unroll
        for (int e = 0; e < EPT; ++e) {
            const int i = threadIdx.x + e * blockDim.x;
            if (i < n) { A[i] = na[e]; C[i] = nc[e]; RX[i] = nx[e]; RY[i] = ny[e]; }
        }
        __syncthreads();
    }
}

__device__ void spline_moments_chunked(double *sm, int np, int n) {
    const double *H = sm, *PX = sm + np, *PY = sm + 2 * np;
    double *INVD = sm + 3 * np, *Y0 = sm + 4 * np, *Y1 = sm + 5 * np, *MX = sm + 6 * np, *MY = sm + 7 * np;
    // ---- forward pivots d_i = 2 (h_{i-1} + h_i) - h_{i-1}^2 / d_{i-1}; stored as 1 / d_i ----
    for (int c0 = threadIdx.x * TRI_CHUNK; c0 < n; c0 += blockDim.x * TRI_CHUNK) {
        const int c1 = min(c0 + TRI_CHUNK, n);
        int i = wrapi(c0 - TRI_WARM, n);
        double hm = H[(i == 0) ? n - 1 : i - 1], prev = 2.0 * (hm + H[i]);
        hm = H[i];
#pragma unroll 8
        for (int s = 0; s < TRI_WARM - 1; ++s) {
            i = (i + 1 == n) ? 0 : i + 1;
            const double hi = H[i];
            prev = 2.0 * (hm + hi) - hm * hm / prev;
            hm = hi;
        }
        for (int s = c0; s < c1; ++s) {
            i = (i + 1 == n) ? 0 : i + 1;
            const double hi = H[i];
            prev = 2.0 * (hm + hi) - hm * hm / prev;
            hm = hi;
            INVD[i] = 1.0 / prev;
        }
    }
    __syncthreads();
    // ---- forward substitution y_i = r_i - (h_{i-1} / d_{i-1}) y_{i-1},  r = 6 D2 p ----
    for (int c0 = threadIdx.x * TRI_CHUNK; c0 < n; c0 += blockDim.x * TRI_CHUNK) {
        const int c1 = min(c0 + TRI_CHUNK, n);
        int i = wrapi(c0 - TRI_WARM, n);
        int im = (i == 0) ? n - 1 : i - 1;
        double yx = 0.0, yy = 0.0;
        double hm = H[im], pxm = PX[im], pym = PY[im], pxi = PX[i], pyi = PY[i], idm = INVD[im];
#pragma unroll 4
        for (int s = 0; s < TRI_WARM + TRI_CHUNK; ++s) {
            if (s >= TRI_WARM + (c1 - c0)) break;
            const int ip = (i + 1 == n) ? 0 : i + 1;
            const double hi = H[i], pxp = PX[ip], pyp = PY[ip];
            const double rx = 6.0 * ((pxp - pxi) / hi - (pxi - pxm) / hm), ry = 6.0 * ((pyp - pyi) / hi - (pyi - pym) / hm);
            const double l = hm * idm;
            yx = rx - l * yx;
            yy = ry - l * yy;
            if (s >= TRI_WARM) { Y0[i] = yx; Y1[i] = yy; }
            idm = INVD[i];
            hm = hi; pxm = pxi; pym = pyi; pxi = pxp; pyi = pyp;
            i = ip;
        }
    }
    __syncthreads();
    // ---- backward substitution m_i = (y_i - h_i m_{i+1}) / d_i ----
    for (int c0 = threadIdx.x * TRI_CHUNK; c0 < n; c0 += blockDim.x * TRI_CHUNK) {
        const int c1 = min(c0 + TRI_CHUNK, n);
        int i = wrapi(c1 - 1 + TRI_WARM, n);
        double mx = 0.0, my = 0.0;
#pragma unroll 4
        for (int s = 0; s < TRI_WARM + TRI_CHUNK; ++s) {
            if (s >= TRI_WARM + (c1 - c0)) break;
            const double o = H[i], id = INVD[i];
            mx = (Y0[i] - o * mx) * id;
            my = (Y1[i] - o * my) * id;
            if (s >= TRI_WARM) { MX[i] = mx; MY[i] = my; }
            i = (i == 0) ? n - 1 : i - 1;
        }
    }
    __syncthreads();
}

// uniform: all parameter scales equal (H = 1: create_raceline, calc_splines without distance scaling) -- the couplings start
// at 1/4 of the diagonal and fall to 5e-19 after FIVE steps (0.25 -> 0.071 -> 5.2e-3 -> 2.7e-5 -> 7.3e-10 -> 5.3e-19);
// scaled spacings start anywhere below 1/2 and get the sixth step.
__device__ void closed_spline(double *sm, int np, int n, double *__restrict__ cx, double *__restrict__ cy,
                              double *__restrict__ nvec, bool uniform) {
    const double *H = sm, *PX = sm + np, *PY = sm + 2 * np;
    const double *MX = sm + 6 * np, *MY = sm + 7 * np;
    const int s_end = uniform ? 32 : 64;
    if (n <= 4 * (int)blockDim.x) spline_moments_pcr<4>(sm, np, n, s_end);
    else if (n <= 8 * (int)blockDim.x) spline_moments_pcr<8>(sm, np, n, s_end);
    else spline_moments_chunked(sm, np, n);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double h2 = H[i] * H[i];
        const double ax1 = (PX[ip1] - PX[i]) - h2 * (2.0 * MX[i] + MX[ip1]) * (1.0 / 6.0);
        const double ay1 = (PY[ip1] - PY[i]) - h2 * (2.0 * MY[i] + MY[ip1]) * (1.0 / 6.0);
        if (cx) {
            double4 c;
            c.x = PX[i]; c.y = ax1; c.z = 0.5 * h2 * MX[i]; c.w = h2 * (MX[ip1] - MX[i]) * (1.0 / 6.0);
            *reinterpret_cast<double4 *>(cx + (size_t)i * 4) = c;
            c.x = PY[i]; c.y = ay1; c.z = 0.5 * h2 * MY[i]; c.w = h2 * (MY[ip1] - MY[i]) * (1.0 / 6.0);
            *reinterpret_cast<double4 *>(cy + (size_t)i * 4) = c;
        }
        if (nvec) {
            const double inv = 1.0 / sqrt(ax1 * ax1 + ay1 * ay1);
            *reinterpret_cast<double2 *>(nvec + (size_t)i * 2) = make_double2(ay1 * inv, -ax1 * inv);
        }
    }
    __syncthreads();
}

__global__ void __launch_bounds__(256)
calc_splines_kernel(int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ xy, int xy_stride,
                    const double *__restrict__ el_lengths, int use_dist_scaling,
                    double *__restrict__ coeffs_x, double *__restrict__ coeffs_y, double *__restrict__ normvec,
                    double *__restrict__ h_out, double *__restrict__ ws) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    if (n < 3 || n > n_max) return;
    const int np = spl_np(n_max);
    extern __shared__ __align__(16) double spl_sm[];
    double *sv = (spline_smem_bytes(n_max) <= SPL_SMEM_LIMIT) ? spl_sm : ws + (size_t)b * S_NUM * np;
    double *H = sv, *PX = sv + np, *PY = sv + 2 * np;
    const double *p = xy + (size_t)b * n_max * xy_stride;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int ip1 = (i + 1 == n) ? 0 : i + 1;
        const double2 a = *reinterpret_cast<const double2 *>(p + (size_t)i * xy_stride);
        const double2 c = *reinterpret_cast<const double2 *>(p + (size_t)ip1 * xy_stride);
        PX[i] = a.x; PY[i] = a.y;
        double h = 1.0;
        if (use_dist_scaling) {
            if (el_lengths) h = el_lengths[(size_t)b * n_max + i];
            else { const double dx = c.x - a.x, dy = c.y - a.y; h = sqrt(dx * dx + dy * dy); }
        }
        H[i] = h;
        if (h_out) h_out[(size_t)b * n_max + i] = h;
    }
    __syncthreads();
    closed_spline(sv, np, n, coeffs_x ? coeffs_x + (size_t)b * n_max * 4 : nullptr,
                  coeffs_y ? coeffs_y + (size_t)b * n_max * 4 : nullptr,
                  normvec ? normvec + (size_t)b * n_max * 2 : nullptr, !use_dist_scaling);
}

// ---------------------------------------------------------------------------------------------
// create_raceline (+ optional heading / curvature at the resampled points)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void head_curv(const double4 cx, const double4 cy, double t, double *psi, double *kappa,
                                          double *dkappa) {
    const double xd = cx.y + 2.0 * cx.z * t + 3.0 * cx.w * t * t;
    const double yd = cy.y + 2.0 * cy.z * t + 3.0 * cy.w * t * t;
    const double xdd = 2.0 * cx.z + 6.0 * cx.w * t, ydd = 2.0 * cy.z + 6.0 * cy.w * t;
    if (psi) {
        // tph.normalize_psi: sign(psi) * mod(|psi|, 2 pi), then wrap into [-pi, pi)
        const double PI = 3.14159265358979323846;
        double ps = atan2(yd, xd) - 0.5 * PI;
        const double m = fmod(fabs(ps), 2.0 * PI);
        ps = (ps > 0.0) ? m : ((ps < 0.0) ? -m : 0.0);
        if (ps >= PI) ps -= 2.0 * PI;
        if (ps < -PI) ps += 2.0 * PI;
        *psi = ps;
    }
    const double q = xd * xd + yd * yd;
    if (kappa) *kappa = (xd * ydd - yd * xdd) / (q * sqrt(q));
    if (dkappa) {
        const double xddd = 6.0 * cx.w, yddd = 6.0 * cy.w;
        *dkappa = (q * (xd * yddd - yd * xddd) - 3.0 * (xd * ydd - yd * xdd) * (xd * xdd + yd * ydd)) / (q * q * q);
    }
}

__global__ void __launch_bounds__(256)
create_raceline_kernel(int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ refline, int ref_stride,
                       const double *__restrict__ normvec, const double *__restrict__ alpha, double stepsize,
                       int n_out_max, double *__restrict__ coeffs_x, double *__restrict__ coeffs_y,
                       double *__restrict__ spline_lengths, int32_t *__restrict__ n_out,
                       double *__restrict__ raceline_interp, int32_t *__restrict__ spline_inds,
                       double *__restrict__ t_values, double *__restrict__ s_interp,
                       double *__restrict__ el_lengths_interp, double *__restrict__ psi, double *__restrict__ kappa,
                       double *__restrict__ ws) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    __shared__ double s_part[256];
    if (n < 3 || n > n_max) { if (threadIdx.x == 0) n_out[b] = 0; return; }
    const int np = spl_np(n_max);
    extern __shared__ __align__(16) double spl_sm[];
    double *sv = (spline_smem_bytes(n_max) <= SPL_SMEM_LIMIT) ? spl_sm : ws + (size_t)b * S_NUM * np;
    double *H = sv, *PX = sv + np, *PY = sv + 2 * np, *CUM = sv + 4 * np;      // (CUM takes Y0's place after the spline)
    const double *p = refline + (size_t)b * n_max * ref_stride;
    const double *nv = normvec + (size_t)b * n_max * 2;
    const double *al = alpha + (size_t)b * n_max;
    double *cx = coeffs_x + (size_t)b * n_max * 4, *cy = coeffs_y + (size_t)b * n_max * 4;
    double *sl = spline_lengths + (size_t)b * n_max;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double2 a = *reinterpret_cast<const double2 *>(p + (size_t)i * ref_stride);
        const double2 nn = *reinterpret_cast<const double2 *>(nv + (size_t)i * 2);
        const double av = al[i];
        PX[i] = a.x + av * nn.x;
        PY[i] = a.y + av * nn.y;
        H[i] = 1.0;
    }
    __syncthreads();
    closed_spline(sv, np, n, cx, cy, nullptr, true);
    // spline lengths: polyline through 15 equidistant t samples (tph.calc_spline_lengths, no_interp_points=15)
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double4 a = *reinterpret_cast<const double4 *>(cx + (size_t)i * 4);
        const double4 c = *reinterpret_cast<const double4 *>(cy + (size_t)i * 4);
        double len = 0.0, xprev = a.x, yprev = c.x;
        for (int s = 1; s < 15; ++s) {
            const double t = (s == 14) ? 1.0 : (double)s * (1.0 / 14.0);   // numpy.linspace(0, 1, 15)
            const double t2 = t * t, t3 = t2 * t;
            const double x = a.x + a.y * t + a.z * t2 + a.w * t3;
            const double y = c.x + c.y * t + c.z * t2 + c.w * t3;
            const double dx = x - xprev, dy = y - yprev;
            len += sqrt(dx * dx + dy * dy);
            xprev = x; yprev = y;
        }
        sl[i] = len;
    }
    __syncthreads();
    // inclusive cumulative sum of the lengths (chunk per thread + scan of the chunk sums)
    const int chunk = (n + blockDim.x - 1) / blockDim.x;
    const int c0 = threadIdx.x * chunk, c1 = min(c0 + chunk, n);
    double part = 0.0;
    for (int i = c0; i < c1; ++i) part += sl[i];
    s_part[threadIdx.x] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        double run = 0.0;
        for (int t = 0; t < (int)blockDim.x; ++t) { const double v = s_part[t]; s_part[t] = run; run += v; }
    }
    __syncthreads();
    double run = s_part[threadIdx.x];
    for (int i = c0; i < c1; ++i) { run += sl[i]; CUM[i] = run; }
    __syncthreads();
    const double total = CUM[n - 1];
    const int n_interp = (int)ceil(total / stepsize) + 1;   // incl. the dropped last point
    const int no = n_interp - 1;
    if (no > n_out_max) { if (threadIdx.x == 0) n_out[b] = -no; return; }
    if (threadIdx.x == 0) n_out[b] = no;
    const double dstep = total / (double)(n_interp - 1);     // numpy.linspace step
    double *ri = raceline_interp + (size_t)b * n_out_max * 2;
    int32_t *si = spline_inds + (size_t)b * n_out_max;
    double *tv = t_values + (size_t)b * n_out_max, *ss = s_interp + (size_t)b * n_out_max;
    double *el = el_lengths_interp + (size_t)b * n_out_max;
    for (int i = threadIdx.x; i < n_out_max; i += blockDim.x) {
        if (i >= no) {
            ri[2 * i] = 0.0; ri[2 * i + 1] = 0.0; si[i] = 0; tv[i] = 0.0; ss[i] = 0.0; el[i] = 0.0;
            if (psi) psi[(size_t)b * n_out_max + i] = 0.0;
            if (kappa) kappa[(size_t)b * n_out_max + i] = 0.0;
            continue;
        }
        const double dist = (double)i * dstep;
        // first j with dist < CUM[j]   (np.argmax(dists_interp[i] < dists_cum))
        int lo = 0, hi = n - 1;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (dist < CUM[mid]) hi = mid; else lo = mid + 1;
        }
        const int j = lo;
        const double t = (j > 0) ? (dist - CUM[j - 1]) / sl[j] : dist / sl[0];
        const double4 a = *reinterpret_cast<const double4 *>(cx + (size_t)j * 4);
        const double4 c = *reinterpret_cast<const double4 *>(cy + (size_t)j * 4);
        const double t2 = t * t, t3 = t2 * t;
        ri[2 * i] = a.x + a.y * t + a.z * t2 + a.w * t3;
        ri[2 * i + 1] = c.x + c.y * t + c.z * t2 + c.w * t3;
        si[i] = j; tv[i] = t; ss[i] = dist;
        el[i] = (i + 1 < no) ? ((double)(i + 1) * dstep - dist) : (total - dist);
        if (psi || kappa)
            head_curv(a, c, t, psi ? psi + (size_t)b * n_out_max + i : nullptr,
                      kappa ? kappa + (size_t)b * n_out_max + i : nullptr, nullptr);
    }
}

__global__ void __launch_bounds__(256)
head_curv_kernel(int n_max, const double *__restrict__ coeffs_x, const double *__restrict__ coeffs_y, int n_eval_max,
                 const int32_t *__restrict__ n_eval, const int32_t *__restrict__ ind_spls,
                 const double *__restrict__ t_spls, double *__restrict__ psi, double *__restrict__ kappa,
                 double *__restrict__ dkappa) {
    const int b = blockIdx.y;
    const int ne = n_eval ? n_eval[b] : n_eval_max;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_eval_max) return;
    const size_t o = (size_t)b * n_eval_max + i;
    if (i >= ne) { psi[o] = 0.0; if (kappa) kappa[o] = 0.0; if (dkappa) dkappa[o] = 0.0; return; }
    const int j = ind_spls[o];
    const double4 a = *reinterpret_cast<const double4 *>(coeffs_x + ((size_t)b * n_max + j) * 4);
    const double4 c = *reinterpret_cast<const double4 *>(coeffs_y + ((size_t)b * n_max + j) * 4);
    head_curv(a, c, t_spls[o], psi + o, kappa ? kappa + o : nullptr, dkappa ? dkappa + o : nullptr);
}

// iqp_handler re-linearisation, part 2: widths shifted by alpha, interpolated linearly in t onto the
// re-sampled raceline points; assembles the new reftrack rows [x, y, w_r, w_l].
__global__ void __launch_bounds__(256)
iqp_new_reftrack_kernel(int n_max, const int32_t *__restrict__ n_pts, const int32_t *__restrict__ active,
                        const double *__restrict__ reftrack, const double *__restrict__ normvec,
                        const double *__restrict__ alpha, int n_max_new, const int32_t *__restrict__ n_new,
                        const double *__restrict__ race_xy, const int32_t *__restrict__ inds,
                        const double *__restrict__ tvals, double *__restrict__ reftrack_new,
                        double *__restrict__ normvec_new, int32_t *__restrict__ n_pts_new) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    const double *rt = reftrack + (size_t)b * n_max * 4;
    double *rn = reftrack_new + (size_t)b * n_max_new * 4;
    if (active && !active[b]) {          // finished instance: the driver keeps its result, emit an empty track
        if (threadIdx.x == 0) n_pts_new[b] = 0;
        return;
    }
    const int nn_ = n_new[b];
    if (threadIdx.x == 0) n_pts_new[b] = nn_;
    if (nn_ <= 0) return;
    const double *al = alpha + (size_t)b * n_max;
    const double *rxy = race_xy + (size_t)b * n_max_new * 2;
    const int32_t *si = inds + (size_t)b * n_max_new;
    const double *tv = tvals + (size_t)b * n_max_new;
    for (int i = threadIdx.x; i < n_max_new; i += blockDim.x) {
        double4 row = make_double4(0.0, 0.0, 0.0, 0.0);
        if (i < nn_) {
            const int j = si[i], j1 = (j + 1 == n) ? 0 : j + 1;
            const double t = tv[i];
            const double wr0 = rt[(size_t)j * 4 + 2] - al[j], wr1 = rt[(size_t)j1 * 4 + 2] - al[j1];
            const double wl0 = rt[(size_t)j * 4 + 3] + al[j], wl1 = rt[(size_t)j1 * 4 + 3] + al[j1];
            // np.interp(t, (0, 1), (w0, w1)) = w0 + (w1 - w0) * t
            row = make_double4(rxy[2 * i], rxy[2 * i + 1], wr0 + (wr1 - wr0) * t, wl0 + (wl1 - wl0) * t);
        }
        *reinterpret_cast<double4 *>(rn + (size_t)i * 4) = row;
    }
}

__global__ void scale_alpha_kernel(int n_max, double *__restrict__ alpha, const double *__restrict__ scale_batch,
                                   double scale) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_max) alpha[(size_t)b * n_max + i] *= scale_batch ? scale_batch[b] : scale;
}

// ---------------------------------------------------------------------------------------------
// K3d -- vector-Jacobian product of create_raceline_kernel (DESIGN.md section 3.12).  n_out and every station's segment
// are held at the forward's (read from its outputs, not searched again).  One CTA per track, like the forward:
//   1. station terms: per segment j one thread sums, in station order, the terms of its stations (point, kappa, and
//      t = (i total / no - CUM[j-1]) / sl[j]; every el_i is total / no): the adjoints of the coefficients of j, of
//      sl[j], of CUM[j-1] and a share of the adjoint of total (no atomics);
//   2. lengths: the cumulative sum reversed (a suffix scan, the forward's chunked scan backwards), then the 15-sample
//      polylines back onto the coefficients;
//   3. moments: the coefficients give the adjoint of the moments gm and a direct part of the point adjoint; the moment
//      system m = A^-1 6 D2 p has A = circ(1, 4, 1) and D2 circulant, so they commute and the adjoint of p through m,
//      6 D2 A^-1 gm, is what the forward's own solve (closed_spline: PCR or chunked, shared or global scratch) returns for
//      the input points gm.
// ---------------------------------------------------------------------------------------------
enum CraVec : int { G_SL = 0, G_CUM, G_C0X, G_C1X, G_C2X, G_C3X, G_C0Y, G_C1Y, G_C2Y, G_C3Y, G_NUM };

size_t create_raceline_adjoint_ws_doubles(int n_max) { return (size_t)(S_NUM + G_NUM) * spl_np(n_max); }

struct CraAdjArgs {
    int n_max, n_out_max;
    const int32_t *n_pts, *n_out, *spline_inds;
    const double *normvec, *alpha, *coeffs_x, *coeffs_y, *spline_lengths, *t_values;
    const double *g_raceline, *g_kappa, *g_el;
    double *g_alpha, *g_refline, *g_normvec, *ws;
};

__global__ void __launch_bounds__(256) create_raceline_adjoint_kernel(const CraAdjArgs a) {
    const int b = blockIdx.x;
    const int n = a.n_pts ? a.n_pts[b] : a.n_max;
    const int no = a.n_out[b];
    const size_t row = (size_t)b * a.n_max;
    __shared__ double s_part[256];
    const bool ok = n >= 3 && n <= a.n_max && no > 0 && no <= a.n_out_max;
    for (int i = threadIdx.x + (ok ? n : 0); i < a.n_max; i += blockDim.x) {      // padding / unsupported track: zeros
        a.g_alpha[row + i] = 0.0;
        if (a.g_refline) { a.g_refline[2 * (row + i)] = 0.0; a.g_refline[2 * (row + i) + 1] = 0.0; }
        if (a.g_normvec) { a.g_normvec[2 * (row + i)] = 0.0; a.g_normvec[2 * (row + i) + 1] = 0.0; }
    }
    if (!ok) return;
    const int np = spl_np(a.n_max);
    extern __shared__ __align__(16) double spl_sm[];
    double *sv = (spline_smem_bytes(a.n_max) <= SPL_SMEM_LIMIT) ? spl_sm : a.ws + (size_t)b * (S_NUM + G_NUM) * np;
    double *G = a.ws + (size_t)b * (S_NUM + G_NUM) * np + (size_t)S_NUM * np;
    double *GSL = G + G_SL * np, *GCUM = G + G_CUM * np;
    const double *cx = a.coeffs_x + row * 4, *cy = a.coeffs_y + row * 4, *sl = a.spline_lengths + row;
    const size_t orow = (size_t)b * a.n_out_max;
    const int32_t *si = a.spline_inds + orow;
    const double *tv = a.t_values + orow;
    const double inv_no = 1.0 / (double)no;

    // ---- 1. station terms, one thread per segment ----
    double g_total = 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        int lo = 0, hi = no;                                   // first station of segment j (spline_inds is sorted)
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (si[mid] < j) lo = mid + 1; else hi = mid; }
        const double4 ax = *reinterpret_cast<const double4 *>(cx + (size_t)j * 4);
        const double4 ay = *reinterpret_cast<const double4 *>(cy + (size_t)j * 4);
        const double sj = sl[j];
        double gx[4] = {0.0, 0.0, 0.0, 0.0}, gy[4] = {0.0, 0.0, 0.0, 0.0}, gsl = 0.0, gcum = 0.0;
        for (int i = lo; i < no && si[i] == j; ++i) {
            const double t = tv[i], t2 = t * t, t3 = t2 * t;
            const double gpx = a.g_raceline ? a.g_raceline[2 * (orow + i)] : 0.0;
            const double gpy = a.g_raceline ? a.g_raceline[2 * (orow + i) + 1] : 0.0;
            const double gk = a.g_kappa ? a.g_kappa[orow + i] : 0.0;
            const double xd = ax.y + 2.0 * ax.z * t + 3.0 * ax.w * t2, yd = ay.y + 2.0 * ay.z * t + 3.0 * ay.w * t2;
            const double xdd = 2.0 * ax.z + 6.0 * ax.w * t, ydd = 2.0 * ay.z + 6.0 * ay.w * t;
            double gxd = 0.0, gyd = 0.0, gxdd = 0.0, gydd = 0.0;
            if (gk != 0.0) {                                   // kappa = (xd ydd - yd xdd) / q^1.5
                const double q = xd * xd + yd * yd, q15 = q * sqrt(q);
                const double kap = (xd * ydd - yd * xdd) / q15;
                gxd = gk * (ydd / q15 - 3.0 * kap * xd / q);
                gyd = gk * (-xdd / q15 - 3.0 * kap * yd / q);
                gxdd = -gk * yd / q15;
                gydd = gk * xd / q15;
            }
            gx[0] += gpx; gx[1] += gpx * t + gxd; gx[2] += gpx * t2 + 2.0 * t * gxd + 2.0 * gxdd;
            gx[3] += gpx * t3 + 3.0 * t2 * gxd + 6.0 * t * gxdd;
            gy[0] += gpy; gy[1] += gpy * t + gyd; gy[2] += gpy * t2 + 2.0 * t * gyd + 2.0 * gydd;
            gy[3] += gpy * t3 + 3.0 * t2 * gyd + 6.0 * t * gydd;
            const double gt = gpx * xd + gpy * yd + gxd * xdd + gyd * ydd + 6.0 * (gxdd * ax.w + gydd * ay.w);
            // t = (i total / no - CUM[j-1]) / sl[j];  el_i = total / no
            g_total += gt * (double)i * inv_no / sj + (a.g_el ? a.g_el[orow + i] : 0.0) * inv_no;
            gcum -= gt / sj;
            gsl -= gt * t / sj;
        }
        G[G_C0X * np + j] = gx[0]; G[G_C1X * np + j] = gx[1]; G[G_C2X * np + j] = gx[2]; G[G_C3X * np + j] = gx[3];
        G[G_C0Y * np + j] = gy[0]; G[G_C1Y * np + j] = gy[1]; G[G_C2Y * np + j] = gy[2]; G[G_C3Y * np + j] = gy[3];
        GSL[j] = gsl;
        if (j > 0) GCUM[j - 1] = gcum;
    }
    s_part[threadIdx.x] = g_total;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int t = 0; t < (int)blockDim.x; ++t) s += s_part[t];
        GCUM[n - 1] = s;                                       // total = CUM[n - 1]
    }
    __syncthreads();
    // ---- 2. lengths: GSL[i] += sum_{k >= i} GCUM[k] (chunk per thread + suffix scan of the chunk sums) ----
    const int chunk = (n + blockDim.x - 1) / blockDim.x;
    const int c0 = threadIdx.x * chunk, c1 = min(c0 + chunk, n);
    double part = 0.0;
    for (int i = c0; i < c1; ++i) part += GCUM[i];
    s_part[threadIdx.x] = part;
    __syncthreads();
    if (threadIdx.x == 0) {
        double run = 0.0;
        for (int t = (int)blockDim.x - 1; t >= 0; --t) { const double v = s_part[t]; s_part[t] = run; run += v; }
    }
    __syncthreads();
    double run = s_part[threadIdx.x];
    for (int i = c1 - 1; i >= c0; --i) { run += GCUM[i]; GSL[i] += run; }
    __syncthreads();
    //      the 15-sample polyline of segment i (tph.calc_spline_lengths) onto its coefficients
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const double4 ax = *reinterpret_cast<const double4 *>(cx + (size_t)i * 4);
        const double4 ay = *reinterpret_cast<const double4 *>(cy + (size_t)i * 4);
        const double g = GSL[i];
        double gx[4] = {0.0, 0.0, 0.0, 0.0}, gy[4] = {0.0, 0.0, 0.0, 0.0};
        double xprev = ax.x, yprev = ay.x, tp[4] = {1.0, 0.0, 0.0, 0.0};
        for (int s = 1; s < 15; ++s) {
            const double t = (s == 14) ? 1.0 : (double)s * (1.0 / 14.0);
            const double t2 = t * t, t3 = t2 * t;
            const double x = ax.x + ax.y * t + ax.z * t2 + ax.w * t3;
            const double y = ay.x + ay.y * t + ay.z * t2 + ay.w * t3;
            const double dx = x - xprev, dy = y - yprev, len = sqrt(dx * dx + dy * dy);
            if (len > 0.0) {
                const double ux = g * dx / len, uy = g * dy / len;
                const double tc[4] = {1.0, t, t2, t3};
#pragma unroll
                for (int k = 1; k < 4; ++k) { gx[k] += ux * (tc[k] - tp[k]); gy[k] += uy * (tc[k] - tp[k]); }
            }
            tp[1] = t; tp[2] = t2; tp[3] = t3;
            xprev = x; yprev = y;
        }
        G[G_C1X * np + i] += gx[1]; G[G_C2X * np + i] += gx[2]; G[G_C3X * np + i] += gx[3];
        G[G_C1Y * np + i] += gy[1]; G[G_C2Y * np + i] += gy[2]; G[G_C3Y * np + i] += gy[3];
    }
    __syncthreads();
    // ---- 3. coefficients -> moments (into the points of the spline scratch) and the direct part of the points ----
    //      c0 = p_i, c1 = p_i+1 - p_i - (2 m_i + m_i+1) / 6, c2 = m_i / 2, c3 = (m_i+1 - m_i) / 6
    double *H = sv, *PX = sv + np, *PY = sv + 2 * np;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int im = (i == 0) ? n - 1 : i - 1;
        PX[i] = -G[G_C1X * np + i] / 3.0 + 0.5 * G[G_C2X * np + i] - G[G_C3X * np + i] / 6.0
                - G[G_C1X * np + im] / 6.0 + G[G_C3X * np + im] / 6.0;
        PY[i] = -G[G_C1Y * np + i] / 3.0 + 0.5 * G[G_C2Y * np + i] - G[G_C3Y * np + i] / 6.0
                - G[G_C1Y * np + im] / 6.0 + G[G_C3Y * np + im] / 6.0;
        H[i] = 1.0;
    }
    __syncthreads();
    closed_spline(sv, np, n, nullptr, nullptr, nullptr, true);      // MX, MY = 6 D2 A^-1 gm
    const double *MX = sv + 6 * np, *MY = sv + 7 * np;
    const double *nv = a.normvec + row * 2, *al = a.alpha + row;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const int im = (i == 0) ? n - 1 : i - 1;
        const double gpx = G[G_C0X * np + i] - G[G_C1X * np + i] + G[G_C1X * np + im] + MX[i];
        const double gpy = G[G_C0Y * np + i] - G[G_C1Y * np + i] + G[G_C1Y * np + im] + MY[i];
        const double2 nn = *reinterpret_cast<const double2 *>(nv + (size_t)i * 2);
        a.g_alpha[row + i] = nn.x * gpx + nn.y * gpy;               // P = p + alpha n
        if (a.g_refline) { a.g_refline[2 * (row + i)] = gpx; a.g_refline[2 * (row + i) + 1] = gpy; }
        if (a.g_normvec) { a.g_normvec[2 * (row + i)] = al[i] * gpx; a.g_normvec[2 * (row + i) + 1] = al[i] * gpy; }
    }
}

void launch_create_raceline_adjoint(int B, int n_max, const int32_t *n_pts, const double *normvec, const double *alpha, int n_out_max, const double *cx,
                                    const double *cy, const double *sl, const int32_t *n_out, const int32_t *si,
                                    const double *tv, const double *g_raceline, const double *g_kappa, const double *g_el,
                                    double *g_alpha, double *g_refline, double *g_normvec, double *ws, cudaStream_t stream) {
    CraAdjArgs a;
    a.n_max = n_max; a.n_out_max = n_out_max; a.n_pts = n_pts; a.n_out = n_out;
    a.spline_inds = si; a.normvec = normvec; a.alpha = alpha; a.coeffs_x = cx; a.coeffs_y = cy;
    a.spline_lengths = sl; a.t_values = tv; a.g_raceline = g_raceline; a.g_kappa = g_kappa; a.g_el = g_el;
    a.g_alpha = g_alpha; a.g_refline = g_refline; a.g_normvec = g_normvec; a.ws = ws;
    const size_t sm = spline_smem_bytes(n_max) <= SPL_SMEM_LIMIT ? spline_smem_bytes(n_max) : 0;
    cudaFuncSetAttribute(create_raceline_adjoint_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SPL_SMEM_LIMIT);
    create_raceline_adjoint_kernel<<<B, 256, sm, stream>>>(a);
}

// ---------------------------------------------------------------------------------------------
void launch_calc_splines(int B, int n_max, const int32_t *n_pts, const double *xy, int xy_stride,
                         const double *el_lengths, int use_dist_scaling, double *cx, double *cy, double *nvec,
                         double *h_out, double *ws, cudaStream_t stream) {
    const size_t sm = spline_smem_bytes(n_max) <= SPL_SMEM_LIMIT ? spline_smem_bytes(n_max) : 0;
    cudaFuncSetAttribute(calc_splines_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SPL_SMEM_LIMIT);
    calc_splines_kernel<<<B, 256, sm, stream>>>(n_max, n_pts, xy, xy_stride, el_lengths, use_dist_scaling, cx, cy, nvec,
                                                h_out, ws);
}
void launch_create_raceline(int B, int n_max, const int32_t *n_pts, const double *refline, int ref_stride,
                            const double *normvec, const double *alpha, double stepsize, int n_out_max, double *cx,
                            double *cy, double *sl, int32_t *n_out, double *ri, int32_t *si, double *tv, double *ss,
                            double *el, double *psi, double *kappa, double *ws, cudaStream_t stream) {
    const size_t sm = spline_smem_bytes(n_max) <= SPL_SMEM_LIMIT ? spline_smem_bytes(n_max) : 0;
    cudaFuncSetAttribute(create_raceline_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SPL_SMEM_LIMIT);
    create_raceline_kernel<<<B, 256, sm, stream>>>(n_max, n_pts, refline, ref_stride, normvec, alpha, stepsize, n_out_max,
                                                   cx, cy, sl, n_out, ri, si, tv, ss, el, psi, kappa, ws);
}
void launch_head_curv(int B, int n_max, const double *cx, const double *cy, int n_eval_max, const int32_t *n_eval,
                      const int32_t *ind, const double *t, double *psi, double *kappa, double *dkappa,
                      cudaStream_t stream) {
    for_grid_y_chunks(B, [&](int b0, int nb) {
        const size_t oe = (size_t)b0 * n_eval_max, oc = (size_t)b0 * n_max * 4;
        dim3 grid((n_eval_max + 255) / 256, nb);
        head_curv_kernel<<<grid, 256, 0, stream>>>(n_max, cx + oc, cy + oc, n_eval_max, n_eval ? n_eval + b0 : nullptr, ind + oe,
                                                   t + oe, psi + oe, kappa ? kappa + oe : nullptr, dkappa ? dkappa + oe : nullptr);
    });
}
void launch_iqp_new_reftrack(int B, int n_max, const int32_t *n_pts, const int32_t *active, const double *reftrack,
                             const double *normvec, const double *alpha, int n_max_new, const int32_t *n_new,
                             const double *race_xy, const int32_t *inds, const double *tvals, double *reftrack_new,
                             double *normvec_new, int32_t *n_pts_new, cudaStream_t stream) {
    iqp_new_reftrack_kernel<<<B, 256, 0, stream>>>(n_max, n_pts, active, reftrack, normvec, alpha, n_max_new, n_new,
                                                   race_xy, inds, tvals, reftrack_new, normvec_new, n_pts_new);
}
// ---------------------------------------------------------------------------------------------
// tph.iqp_handler's per-track termination (SURVEY.md A.5) on the device: a track leaves the loop once
// iter >= iters_min and curv_error_max <= curv_error_allowed (or its QP failed, or the iteration cap is reached: status 2);
// its alpha / reftrack / normvectors of THIS iteration are copied into the result buffers and its `active` word is
// cleared, so the host loop needs one small read per outer iteration (counters) instead of masks and gathers.
__global__ void __launch_bounds__(256)
iqp_finish_kernel(int n_max, int n_cap, int it, int iters_min, double curv_error_allowed, int fixed_iters, int limit,
                  int32_t *__restrict__ active, const int32_t *__restrict__ status, const double *__restrict__ curv_err,
                  const int32_t *__restrict__ n_pts, const double *__restrict__ alpha, const double *__restrict__ reftrack,
                  const double *__restrict__ normvec, double *__restrict__ fin_alpha, double *__restrict__ fin_reftrack,
                  double *__restrict__ fin_normvec, int32_t *__restrict__ fin_n_pts, int32_t *__restrict__ fin_iters,
                  int32_t *__restrict__ fin_status, double *__restrict__ fin_curv_err, int32_t *__restrict__ counters) {
    const int b = blockIdx.x;
    if (!active[b]) return;
    const int st = status[b];
    const bool failed = st != 0;
    bool done, capped = false;
    if (fixed_iters > 0) done = (it >= fixed_iters) || failed;
    else {
        const bool conv = (curv_err[b] <= curv_error_allowed) && (it >= iters_min);
        capped = !conv && !failed && it >= limit;
        done = conv || failed || capped;
    }
    if (!done) {
        if (threadIdx.x == 0) atomicAdd(&counters[0], 1);      // still active after this iteration
        return;
    }
    const int n = n_pts ? n_pts[b] : n_max;
    for (int i = threadIdx.x; i < n_cap; i += blockDim.x) {
        const bool in = i < n && i < n_max;
        fin_alpha[(size_t)b * n_cap + i] = in ? alpha[(size_t)b * n_max + i] : 0.0;
        for (int c = 0; c < 4; ++c) fin_reftrack[((size_t)b * n_cap + i) * 4 + c] = in ? reftrack[((size_t)b * n_max + i) * 4 + c] : 0.0;
        for (int c = 0; c < 2; ++c) fin_normvec[((size_t)b * n_cap + i) * 2 + c] = in ? normvec[((size_t)b * n_max + i) * 2 + c] : 0.0;
    }
    if (threadIdx.x == 0) {
        fin_n_pts[b] = n;
        fin_iters[b] = it;
        fin_status[b] = capped ? 2 : st;          // 2: the outer-iteration cap was reached before curv_error_allowed
        fin_curv_err[b] = curv_err[b];
        active[b] = 0;
        atomicAdd(&counters[1], 1);
    }
}
void launch_iqp_finish(int B, int n_max, int n_cap, int it, int iters_min, double curv_error_allowed, int fixed_iters, int limit,
                       int32_t *active, const int32_t *status, const double *curv_err, const int32_t *n_pts, const double *alpha,
                       const double *reftrack, const double *normvec, double *fin_alpha, double *fin_reftrack,
                       double *fin_normvec, int32_t *fin_n_pts, int32_t *fin_iters, int32_t *fin_status, double *fin_curv_err,
                       int32_t *counters, cudaStream_t stream) {
    cudaMemsetAsync(counters, 0, 2 * sizeof(int32_t), stream);
    iqp_finish_kernel<<<B, 256, 0, stream>>>(n_max, n_cap, it, iters_min, curv_error_allowed, fixed_iters, limit, active, status,
                                             curv_err, n_pts, alpha, reftrack, normvec, fin_alpha, fin_reftrack, fin_normvec,
                                             fin_n_pts, fin_iters, fin_status, fin_curv_err, counters);
}

void launch_scale_alpha(int B, int n_max, double *alpha, const double *scale_batch, double scale, cudaStream_t stream) {
    for_grid_y_chunks(B, [&](int b0, int nb) {
        dim3 grid((n_max + 255) / 256, nb);
        scale_alpha_kernel<<<grid, 256, 0, stream>>>(n_max, alpha + (size_t)b0 * n_max, scale_batch ? scale_batch + b0 : nullptr, scale);
    });
}

}  // namespace mc
