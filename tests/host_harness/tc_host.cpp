// TEST INFRASTRUCTURE: the statements of csrc/traj_check_core.cuh (arithmetic of the K6 kernels) run on the host in the
// same order as the kernels run them, for comparison with the fixtures produced by the reference's own helpers
// (tests/golden/refback_*.npz).  Built by tests/test_refback_host.py with g++; never part of libmincurv_b200.so.
#include <cmath>
#include <vector>
#include "../../global_racetrajectory_optimization_b200/csrc/traj_check_core.cuh"

using namespace mc::tc;

// interp_track_kernel, one track
extern "C" int tc_host_interp_track(int n, const double *pts, int stride, const double *normvec, double sign, int width_col,
                                    double stepsize, int n_out_max, double *out) {
    std::vector<double> dc(n + 1);
    ClosedCol cx{pts, (size_t)stride, normvec, 2, pts + width_col, (size_t)stride, sign, n};
    ClosedCol cy{pts + 1, (size_t)stride, normvec ? normvec + 1 : nullptr, 2, pts + width_col, (size_t)stride, sign, n};
    for (int i = 0; i < n; ++i) dc[i + 1] = closed_el_length(cx, cy, i);
    double acc = 0.0;
    dc[0] = 0.0;
    for (int i = 1; i <= n; ++i) { acc = add(acc, dc[i]); dc[i] = acc; }
    const double total = dc[n];
    const int num = resample_count(total, stepsize);
    const int m = num - 1;
    if (!(total > 0.0 && total < (double)INFINITY)) return 0;
    if (m > n_out_max) return -m;
    const bool plain4 = (normvec == nullptr && stride == 4);
    ClosedCol c2{pts + 2, (size_t)stride, nullptr, 0, nullptr, 0, 0.0, n};
    ClosedCol c3{pts + 3, (size_t)stride, nullptr, 0, nullptr, 0, 0.0, n};
    for (int j = 0; j < m; ++j) {
        const double d = linspace0(j, num, total);
        out[4 * j] = interp_closed(d, dc.data(), cx);
        out[4 * j + 1] = interp_closed(d, dc.data(), cy);
        out[4 * j + 2] = plain4 ? interp_closed(d, dc.data(), c2) : 0.0;
        out[4 * j + 3] = plain4 ? interp_closed(d, dc.data(), c3) : 0.0;
    }
    return m;
}

// min_bound_dists_kernel, one track (the kernel's NaN-propagating form; on finite data it takes fmin, which gives the
// same bits).  nearest (may be NULL): per trajectory point, side * 2^20 + index within the side of the boundary point that
// decides the minimum (the first one on a tie), -1 if none.
extern "C" void tc_host_min_bound_dists(int nt, const double *xy, const double *psi, int nb1, const double *b1, int nb2,
                                        const double *b2, int bstride, double length_veh, double width_veh, double *out,
                                        int *nearest) {
    for (int i = 0; i < nt; ++i) {
        double c[8];
        vehicle_corners(xy[2 * i], xy[2 * i + 1], psi[i], length_veh, width_veh, c);
        double best = INFINITY;
        int arg = -1;
        for (int side = 0; side < 2; ++side) {
            const double *bd = side ? b2 : b1;
            const int nb = side ? nb2 : nb1;
            for (int k = 0; k < nb; ++k) {
                const double bx = bd[(size_t)k * bstride], by = bd[(size_t)k * bstride + 1];
                const double d0 = dist2(bx, by, c[0], c[1]), d1 = dist2(bx, by, c[2], c[3]);
                const double d2 = dist2(bx, by, c[4], c[5]), d3 = dist2(bx, by, c[6], c[7]);
                const double m = nan_min(nan_min(d0, d1), nan_min(d2, d3));
                if (best == best && (m != m || m < best)) arg = (side << 20) + k;
                best = nan_min(best, m);
            }
        }
        out[i] = sqrt(best);
        if (nearest) nearest[i] = arg;
    }
}

// traj_extrema_kernel, one track
extern "C" void tc_host_extrema(int n, const double *kappa, const double *vx, const double *ax, const double *min_dists,
                                double dragcoeff, double mass_veh, double *e) {
    double mn_d = INFINITY, mx_k = -INFINITY, mx_ay = -INFINITY, mx_ax = -INFINITY, mn_ax = INFINITY, mx_at = -INFINITY,
           mx_v = -INFINITY;
    for (int i = 0; i < n; ++i) {
        const PointChecks q = point_checks(kappa[i], vx[i], ax[i], dragcoeff, mass_veh);
        if (min_dists) mn_d = nan_min(mn_d, min_dists[i]);
        mx_k = nan_max(mx_k, q.kappa_abs); mx_ay = fmax(mx_ay, q.ay); mx_ax = fmax(mx_ax, q.ax_wo_drag);
        mn_ax = fmin(mn_ax, q.ax_wo_drag); mx_at = fmax(mx_at, q.a_tot); mx_v = fmax(mx_v, q.v);
    }
    e[0] = mn_d; e[1] = mx_k; e[2] = mx_ay; e[3] = mx_ax; e[4] = mn_ax; e[5] = mx_at; e[6] = mx_v; e[7] = (double)n;
}

// interp_track coverage: the number of stations that land exactly on a cumulative distance (interp_closed's dc[j] == d)
extern "C" int tc_host_interp_exact_hits(int n, const double *pts, int stride, double stepsize) {
    std::vector<double> dc(n + 1);
    ClosedCol cx{pts, (size_t)stride, nullptr, 0, nullptr, 0, 0.0, n};
    ClosedCol cy{pts + 1, (size_t)stride, nullptr, 0, nullptr, 0, 0.0, n};
    for (int i = 0; i < n; ++i) dc[i + 1] = closed_el_length(cx, cy, i);
    double acc = 0.0;
    dc[0] = 0.0;
    for (int i = 1; i <= n; ++i) { acc = add(acc, dc[i]); dc[i] = acc; }
    const int num = resample_count(dc[n], stepsize), m = num - 1;
    int hits = 0;
    for (int j = 0; j < m; ++j) {
        const double d = linspace0(j, num, dc[n]);
        if (d >= dc[n] || d < dc[0]) continue;
        hits += dc[find_span(d, dc.data(), n + 1)] == d;
    }
    return hits;
}

// normals_cross coverage, one pair: bit 0 = rows swapped by the pivot search, bit 1 = collinear (|cross| <= 1e-8),
// bits 2..5 = which of (-w1l <= l1, l1 <= w1r, -w2l <= l2, l2 <= w2r) held with equality, bit 6 = the result
extern "C" int tc_host_normals_cross_info(const double *p, const double *n1, const double *q, const double *n2) {
    const double cross = sub(mul(n1[0], n2[1]), mul(n1[1], n2[0]));
    if (fabs(cross) <= 1e-8) return 2;
    double a00 = n1[0], a01 = -n2[0], a10 = n1[1], a11 = -n2[1], c0 = sub(q[0], p[0]), c1 = sub(q[1], p[1]);
    int info = 0;
    if (fabs(a10) > fabs(a00)) {
        double t = a00; a00 = a10; a10 = t;
        t = a01; a01 = a11; a11 = t;
        t = c0; c0 = c1; c1 = t;
        info |= 1;
    }
    const double l = mul(a10, 1.0 / a00), u11 = sub(a11, mul(l, a01)), y1 = sub(c1, mul(l, c0));
    const double l2 = y1 / u11, l1 = sub(c0, mul(a01, l2)) / a00;
    info |= (-p[3] == l1) << 2 | (l1 == p[2]) << 3 | (-q[3] == l2) << 4 | (l2 == q[2]) << 5;
    const bool r = normals_cross(p[0], p[1], n1[0], n1[1], p[2], p[3], q[0], q[1], n2[0], n2[1], q[2], q[3]);
    return info | (int)r << 6;
}

// normals_crossing_kernel, one track
extern "C" int tc_host_normals_crossing(int n, const double *track, const double *nrm, int horizon) {
    for (int i = 0; i < n; ++i)
        if (normals_cross_point(i, n, horizon, track, nrm)) return 1;
    return 0;
}
