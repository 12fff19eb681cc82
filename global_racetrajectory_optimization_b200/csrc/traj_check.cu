// K6 -- the reference's in-tree trajectory back end on the device, batched (SURVEY.md 8f-3/8f-4):
//   interp_track_kernel        helper_funcs_glob/src/interp_track.py:5-49 (also builds the boundary polylines of
//                              check_traj.py:50-64 on the fly when normal vectors are passed)
//   min_bound_dists_kernel     helper_funcs_glob/src/calc_min_bound_dists.py:5-66
//   traj_extrema_kernel        the quantities helper_funcs_glob/src/check_traj.py:74-139 compares with the limits
//   assemble_trajectory_kernel main_globaltraj.py:501-512 (trajectory_opt / traj_race_cl)
// (paths under the reference tree).  calc_min_bound_dists is the only compute-heavy piece: every trajectory point x 4
// vehicle corners against every boundary point (1 m spacing) -- ~22 M distance evaluations per Berlin-sized track, a
// brute-force minimum the reference runs as a Python loop over numpy rows.  One thread per trajectory point keeps its
// four corners in registers; boundary points are staged through shared memory in tiles and read as broadcasts, so the
// kernel is bound by the fp64 pipe (5 DADD/DMUL + 1 min per corner-point pair), not by memory.
#include "capi.cuh"
#include "common.cuh"
#include "traj_check_core.cuh"

namespace mc {

constexpr int IT_THREADS = 256;
constexpr int MB_THREADS = 128;
constexpr int MB_TILE = 512;

// ---- interp_track -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(IT_THREADS) interp_track_kernel(int B, int n_max, const int32_t *n_pts, const double *pts,
                                                                  int stride, const double *normvec, double sign,
                                                                  int width_col, double stepsize, int n_out_max,
                                                                  double *out, int32_t *n_out, double *ws) {
    const int b = blockIdx.x;
    const int n = n_pts ? n_pts[b] : n_max;
    if (n < 2 || n > n_max) {
        if (threadIdx.x == 0) n_out[b] = 0;
        return;
    }
    const double *row = pts + (size_t)b * n_max * stride;
    const double *nrow = normvec ? normvec + (size_t)b * n_max * 2 : nullptr;
    double *dc = ws + (size_t)b * ((size_t)n_max + 1);
    tc::ClosedCol cx{row, (size_t)stride, nrow, 2, row + width_col, (size_t)stride, sign, n};
    tc::ClosedCol cy{row + 1, (size_t)stride, nrow ? nrow + 1 : nullptr, 2, row + width_col, (size_t)stride, sign, n};
    for (int i = threadIdx.x; i < n; i += blockDim.x) dc[i + 1] = tc::closed_el_length(cx, cy, i);
    __syncthreads();
    if (threadIdx.x == 0) {            // numpy.cumsum order (sequential), dists_cum[0] = 0
        double acc = 0.0;
        dc[0] = 0.0;
        for (int i = 1; i <= n; ++i) {
            acc = vp::add(acc, dc[i]);
            dc[i] = acc;
        }
    }
    __syncthreads();
    const double total = dc[n];
    const int num = tc::resample_count(total, stepsize);     // includes the closing point, which is dropped
    const int m = num - 1;
    if (!(total > 0.0) || m > n_out_max) {
        if (threadIdx.x == 0) n_out[b] = (total > 0.0) ? -m : 0;
        return;
    }
    if (threadIdx.x == 0) n_out[b] = m;
    double *orow = out + (size_t)b * n_out_max * 4;
    const bool plain4 = (normvec == nullptr && stride == 4);
    tc::ClosedCol c2{row + 2, (size_t)stride, nullptr, 0, nullptr, 0, 0.0, n};
    tc::ClosedCol c3{row + 3, (size_t)stride, nullptr, 0, nullptr, 0, 0.0, n};
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
        const double d = tc::linspace0(j, num, total);
        orow[4 * (size_t)j] = tc::interp_closed(d, dc, cx);
        orow[4 * (size_t)j + 1] = tc::interp_closed(d, dc, cy);
        orow[4 * (size_t)j + 2] = plain4 ? tc::interp_closed(d, dc, c2) : 0.0;
        orow[4 * (size_t)j + 3] = plain4 ? tc::interp_closed(d, dc, c3) : 0.0;
    }
}

// ---- calc_min_bound_dists -----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MB_THREADS) min_bound_dists_kernel(int n_traj_max, const int32_t *n_traj, const double *xy,
                                                                     const double *psi, int nb_max1, const int32_t *nb1,
                                                                     const double *bound1, int nb_max2, const int32_t *nb2,
                                                                     const double *bound2, int bstride, double length_veh,
                                                                     double width_veh, double *min_dists) {
    __shared__ double sbx[MB_TILE], sby[MB_TILE];
    const int b = blockIdx.y;
    const int nt = n_traj ? n_traj[b] : n_traj_max;
    if ((int)(blockIdx.x * blockDim.x) >= nt) return;              // whole CTA beyond this track's trajectory
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < nt;
    double c[8];
    if (live) {
        const size_t o = (size_t)b * n_traj_max + i;
        tc::vehicle_corners(xy[2 * o], xy[2 * o + 1], psi[o], length_veh, width_veh, c);
    } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) c[k] = 0.0;
    }
    double best = INFINITY;
    for (int side = 0; side < 2; ++side) {
        const double *bd = side == 0 ? bound1 + (size_t)b * nb_max1 * bstride : bound2 + (size_t)b * nb_max2 * bstride;
        int nb = side == 0 ? (nb1 ? nb1[b] : nb_max1) : (nb2 ? nb2[b] : nb_max2);
        if (nb < 0) nb = 0;
        for (int t0 = 0; t0 < nb; t0 += MB_TILE) {
            const int cnt = min(MB_TILE, nb - t0);
            __syncthreads();
            for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
                sbx[k] = bd[(size_t)(t0 + k) * bstride];
                sby[k] = bd[(size_t)(t0 + k) * bstride + 1];
            }
            __syncthreads();
            if (live) {
#pragma unroll 4
                for (int k = 0; k < cnt; ++k) {
                    const double bx = sbx[k], by = sby[k];
                    const double d0 = tc::dist2(bx, by, c[0], c[1]), d1 = tc::dist2(bx, by, c[2], c[3]);
                    const double d2 = tc::dist2(bx, by, c[4], c[5]), d3 = tc::dist2(bx, by, c[6], c[7]);
                    best = fmin(best, fmin(fmin(d0, d1), fmin(d2, d3)));
                }
            }
        }
    }
    // min over sqrt(.) == sqrt(min(.)): sqrt is monotone and correctly rounded
    if (live) min_dists[(size_t)b * n_traj_max + i] = sqrt(best);
}

// ---- extrema tested by check_traj ---------------------------------------------------------------------------------
// extrema[b][0..7] = min(min_dists), max |kappa|, max ay, max ax_wo_drag, min ax_wo_drag, max a_tot, max vx, n points
__global__ void __launch_bounds__(256) traj_extrema_kernel(int n_max, const int32_t *n_traj, const double *kappa,
                                                           const double *vx, const double *ax, const double *min_dists,
                                                           double dragcoeff, double mass_veh, double *extrema) {
    __shared__ double red[32];
    const int b = blockIdx.x;
    const int n = n_traj ? n_traj[b] : n_max;
    const size_t o = (size_t)b * n_max;
    double mn_d = INFINITY, mx_k = -INFINITY, mx_ay = -INFINITY, mx_ax = -INFINITY, mn_ax = INFINITY, mx_at = -INFINITY,
           mx_v = -INFINITY;
    for (int i = threadIdx.x; i < n && i < n_max; i += blockDim.x) {
        const tc::PointChecks q = tc::point_checks(kappa[o + i], vx[o + i], ax[o + i], dragcoeff, mass_veh);
        if (min_dists) mn_d = fmin(mn_d, min_dists[o + i]);
        mx_k = fmax(mx_k, q.kappa_abs);
        mx_ay = fmax(mx_ay, q.ay);
        mx_ax = fmax(mx_ax, q.ax_wo_drag);
        mn_ax = fmin(mn_ax, q.ax_wo_drag);
        mx_at = fmax(mx_at, q.a_tot);
        mx_v = fmax(mx_v, q.v);
    }
    mn_d = block_reduce<2>(mn_d, red);
    mx_k = block_reduce<1>(mx_k, red);
    mx_ay = block_reduce<1>(mx_ay, red);
    mx_ax = block_reduce<1>(mx_ax, red);
    mn_ax = block_reduce<2>(mn_ax, red);
    mx_at = block_reduce<1>(mx_at, red);
    mx_v = block_reduce<1>(mx_v, red);
    if (threadIdx.x == 0) {
        double *e = extrema + (size_t)b * 8;
        e[0] = mn_d; e[1] = mx_k; e[2] = mx_ay; e[3] = mx_ax; e[4] = mn_ax; e[5] = mx_at; e[6] = mx_v; e[7] = (double)n;
    }
}

// ---- trajectory_opt / traj_race_cl --------------------------------------------------------------------------------
// traj[b][j][0..6] = s, x, y, psi, kappa, vx, ax for j < n; row n = row 0 with s = sum(spline_lengths) (closed race
// trajectory); rows beyond stay untouched.
__global__ void __launch_bounds__(256) assemble_trajectory_kernel(int n_max, const int32_t *n_traj, const double *s,
                                                                  const double *xy, const double *psi, const double *kappa,
                                                                  const double *vx, const double *ax, int n_spl_max,
                                                                  const int32_t *n_spl, const double *spline_lengths,
                                                                  double *traj) {
    const int b = blockIdx.x;
    const int n = n_traj ? n_traj[b] : n_max;
    if (n <= 0 || n > n_max) return;
    const size_t o = (size_t)b * n_max;
    double *t = traj + (size_t)b * ((size_t)n_max + 1) * 7;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        double *r = t + (size_t)j * 7;
        r[0] = s[o + j]; r[1] = xy[2 * (o + j)]; r[2] = xy[2 * (o + j) + 1]; r[3] = psi[o + j]; r[4] = kappa[o + j];
        r[5] = vx[o + j]; r[6] = ax[o + j];
    }
    if (threadIdx.x == 0) {
        const int ns = n_spl ? n_spl[b] : n_spl_max;
        double total = 0.0;
        for (int i = 0; i < ns; ++i) total += spline_lengths[(size_t)b * n_spl_max + i];
        double *r = t + (size_t)n * 7;
        r[0] = total; r[1] = xy[2 * o]; r[2] = xy[2 * o + 1]; r[3] = psi[o]; r[4] = kappa[o]; r[5] = vx[o]; r[6] = ax[o];
    }
}

// ---- tph.check_normals_crossing (prep_track.py:57-59) -------------------------------------------------------------
// crossing[b] = 1 if any two normals within `horizon` points of each other cross inside the track (0 otherwise)
__global__ void __launch_bounds__(128) normals_crossing_kernel(int n_max, const int32_t *n_pts, const double *track,
                                                               const double *normvec, int horizon, int32_t *crossing) {
    const int b = blockIdx.y;
    const int n = n_pts ? n_pts[b] : n_max;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (n <= horizon || n > n_max || i >= n) return;
    if (tc::normals_cross_point(i, n, horizon, track + (size_t)b * n_max * 4, normvec + (size_t)b * n_max * 2))
        atomicOr(crossing + b, 1);
}

}  // namespace mc

extern "C" {

size_t mc_interp_track_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < 2) return 0;
    return align256((size_t)B * ((size_t)n_max + 1) * sizeof(double));
}

int mc_interp_track_batch(int B, int n_max, const int32_t *n_pts, const double *pts, int stride, const double *normvec,
                          double normal_sign, int width_col, double stepsize_approx, int n_out_max, double *out,
                          int32_t *n_out, void *workspace, size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_max < 2 || !pts || (stride != 2 && stride != 4) || !(stepsize_approx > 0.0) || n_out_max <= 0 || !out ||
        !n_out || (normvec && (stride != 4 || (width_col != 2 && width_col != 3))))
        return bad("mc_interp_track_batch: bad argument");
    if (!workspace || workspace_bytes < mc_interp_track_workspace_bytes(B, n_max))
        return small_workspace("mc_interp_track_batch");
    mc::interp_track_kernel<<<B, mc::IT_THREADS, 0, (cudaStream_t)stream>>>(B, n_max, n_pts, pts, stride, normvec, normal_sign,
                                                                            normvec ? width_col : 2, stepsize_approx, n_out_max,
                                                                            out, n_out, (double *)workspace);
    return check_cuda("interp_track_kernel");
}

int mc_min_bound_dists_batch(int B, int n_traj_max, const int32_t *n_traj, const double *xy, const double *psi, int nb1_max,
                             const int32_t *nb1, const double *bound1, int nb2_max, const int32_t *nb2, const double *bound2,
                             int bound_stride, double length_veh, double width_veh, double *min_dists, void *stream) {
    if (B <= 0 || n_traj_max <= 0 || !xy || !psi || !bound1 || !bound2 || nb1_max <= 0 || nb2_max <= 0 ||
        bound_stride < 2 || !min_dists)
        return bad("mc_min_bound_dists_batch: bad argument");
    mc::for_grid_y_chunks(B, [&](int b0, int nb) {
        const size_t ot = (size_t)b0 * n_traj_max;
        dim3 grid((n_traj_max + mc::MB_THREADS - 1) / mc::MB_THREADS, nb);
        mc::min_bound_dists_kernel<<<grid, mc::MB_THREADS, 0, (cudaStream_t)stream>>>(
            n_traj_max, n_traj ? n_traj + b0 : nullptr, xy + 2 * ot, psi + ot, nb1_max, nb1 ? nb1 + b0 : nullptr,
            bound1 + (size_t)b0 * nb1_max * bound_stride, nb2_max, nb2 ? nb2 + b0 : nullptr,
            bound2 + (size_t)b0 * nb2_max * bound_stride, bound_stride, length_veh, width_veh, min_dists + ot);
    });
    return check_cuda("min_bound_dists_kernel");
}

int mc_traj_extrema_batch(int B, int n_max, const int32_t *n_traj, const double *kappa, const double *vx, const double *ax,
                          const double *min_dists, double dragcoeff, double mass_veh, double *extrema, void *stream) {
    if (B <= 0 || n_max <= 0 || !kappa || !vx || !ax || !extrema || !(mass_veh > 0.0))
        return bad("mc_traj_extrema_batch: bad argument");
    mc::traj_extrema_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_traj, kappa, vx, ax, min_dists, dragcoeff, mass_veh,
                                                                 extrema);
    return check_cuda("traj_extrema_kernel");
}

int mc_assemble_trajectory_batch(int B, int n_max, const int32_t *n_traj, const double *s, const double *xy,
                                 const double *psi, const double *kappa, const double *vx, const double *ax, int n_spl_max,
                                 const int32_t *n_spl, const double *spline_lengths, double *traj, void *stream) {
    if (B <= 0 || n_max <= 0 || !s || !xy || !psi || !kappa || !vx || !ax || n_spl_max <= 0 || !spline_lengths || !traj)
        return bad("mc_assemble_trajectory_batch: bad argument");
    mc::assemble_trajectory_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_max, n_traj, s, xy, psi, kappa, vx, ax, n_spl_max,
                                                                        n_spl, spline_lengths, traj);
    return check_cuda("assemble_trajectory_kernel");
}

int mc_check_normals_crossing_batch(int B, int n_max, const int32_t *n_pts, const double *track, const double *normvec,
                                    int horizon, int32_t *crossing, void *stream) {
    if (B <= 0 || n_max < 3 || !track || !normvec || horizon < 1 || !crossing)
        return bad("mc_check_normals_crossing_batch: bad argument");
    cudaMemsetAsync(crossing, 0, (size_t)B * sizeof(int32_t), (cudaStream_t)stream);
    mc::for_grid_y_chunks(B, [&](int b0, int nb) {
        dim3 grid((n_max + 127) / 128, nb);
        mc::normals_crossing_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(n_max, n_pts ? n_pts + b0 : nullptr,
                                                                            track + (size_t)b0 * n_max * 4,
                                                                            normvec + (size_t)b0 * n_max * 2, horizon,
                                                                            crossing + b0);
    });
    return check_cuda("normals_crossing_kernel");
}

}  // extern "C"
