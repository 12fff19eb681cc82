// K7 -- tph.spline_approximation + prep_track's min-width inflation on the device (SURVEY.md 8f-2; call sites
// helper_funcs_glob/src/prep_track.py:39-45 and :89-98): the one stage between a raw track file and the
// minimum-curvature path.  One CTA per raw track; every statement of tph.spline_approximation is kept
//   linear pre-interpolation to stepsize_prep -> smoothing spline through the closed point set (chord-length parameter,
//   s = s_reg) -> curve length from 4 samples per metre -> re-sampling at ~stepsize_reg -> closest curve point of every
//   original point (tph: fmin) -> side of the centre line -> new widths -> linear interpolation of the widths
// except the smoothing spline itself: tph calls scipy's splprep (FITPACK's adaptive-knot fpclos, whose result is defined
// only up to its own 1e-3 tolerance on s); here it is the periodic cubic smoothing spline of Reinsch with the SAME
// residual budget sum |p_i - f(u_i)|^2 = s over x and y together (one smoothing parameter, like splprep) and every data
// point a knot: (R + lam Q^T Q) gamma = Q^T p, f = p - lam Q gamma, a cyclic pentadiagonal SPD system solved in O(n) per
// trial lam.  oracle/tph_prep.py states the same algorithm in dense numpy (checked to 1e-8 in tests/test_gpu_prep.py, which
// also reports the distance to the scipy/FITPACK route: decimetres at sharp corners, centimetres on the real circuits).
#include "capi.cuh"
#include "common.cuh"

namespace mc {

constexpr int PT_VECS = 22;       // per-track scratch vectors of n_int_max doubles (and six of n_raw_max + 1)

struct PtSpline {                 // the fitted curve: knots u (period 1), values f, second derivatives g
    const double *u, *fx, *fy, *gx, *gy;
    int n;
};
__device__ inline void pt_eval(const PtSpline &s, double t, double *x, double *y, double *dx, double *dy, double *ddx, double *ddy) {
    // segment j with u[j] <= t < u[j+1] (u[n] = 1)
    int lo = 0, hi = s.n;                          // invariant: u[lo] <= t
    while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s.u[mid] <= t) lo = mid; else hi = mid; }
    const int j = lo, jp = (j + 1 == s.n) ? 0 : j + 1;
    const double u1 = (j + 1 == s.n) ? 1.0 : s.u[j + 1];
    const double h = u1 - s.u[j], a = (u1 - t) / h, b = (t - s.u[j]) / h;
    const double ca = (a * a * a - a) * h * h / 6.0, cb = (b * b * b - b) * h * h / 6.0;
    *x = a * s.fx[j] + b * s.fx[jp] + ca * s.gx[j] + cb * s.gx[jp];
    *y = a * s.fy[j] + b * s.fy[jp] + ca * s.gy[j] + cb * s.gy[jp];
    if (dx) {
        const double da = -(3.0 * a * a - 1.0) * h / 6.0, db = (3.0 * b * b - 1.0) * h / 6.0;
        *dx = (s.fx[jp] - s.fx[j]) / h + da * s.gx[j] + db * s.gx[jp];
        *dy = (s.fy[jp] - s.fy[j]) / h + da * s.gy[j] + db * s.gy[jp];
        *ddx = a * s.gx[j] + b * s.gx[jp];
        *ddy = a * s.gy[j] + b * s.gy[jp];
    }
}

// cyclic pentadiagonal SPD solve (a0 diagonal, a1 / a2 first / second off-diagonals, indices mod n) for two right-hand
// sides, by a bordered LDL^T: chain 0..n-3, separator = the last two nodes.  Sequential: run by ONE thread.
__device__ void penta_cyclic_solve2(int n, const double *a0, const double *a1, const double *a2, const double *bx, const double *by,
                                    double *d, double *l1, double *l2, double *g0, double *g1, double *x, double *y) {
    // (recurrence state is carried in registers: the loads of an iteration never depend on the previous iteration's stores,
    //  so the unrolled loops keep several of them in flight)
    const int m = n - 2;
    double dm2 = a0[0];
    d[0] = dm2; l1[0] = 0.0; l2[0] = 0.0;
    double l1m1 = a1[0] / dm2;
    double dm1 = a0[1] - l1m1 * l1m1 * dm2;
    l1[1] = l1m1; l2[1] = 0.0; d[1] = dm1;
#pragma unroll 4
    for (int k = 2; k < m; ++k) {
        const double l2k = a2[k - 2] / dm2;
        const double l1k = (a1[k - 1] - l2k * l1m1 * dm2) / dm1;
        const double dk = a0[k] - l1k * l1k * dm1 - l2k * l2k * dm2;
        l2[k] = l2k; l1[k] = l1k; d[k] = dk;
        dm2 = dm1; dm1 = dk; l1m1 = l1k;
    }
    // Y = A[sep, chain]: node m couples to m-2 (a2), m-1 (a1) and across the wrap to 0 (a2[m]); node m+1 to m-1 (a2) and to 0 (a1), 1 (a2)
    double s00 = a0[m], s01 = a1[m], s11 = a0[m + 1];
    {
        double p0 = 0.0, p1 = 0.0, pp0 = 0.0, pp1 = 0.0;        // g[k-1], g[k-2]
#pragma unroll 4
        for (int k = 0; k < m; ++k) {
            double y0 = 0.0, y1 = 0.0;
            if (k == m - 2) y0 += a2[m - 2];
            if (k == m - 1) { y0 += a1[m - 1]; y1 += a2[m - 1]; }
            if (k == 0) { y0 += a2[m]; y1 += a1[m + 1]; }
            if (k == 1) y1 += a2[m + 1];
            const double c1 = l1[k], c2 = l2[k];
            const double v0 = y0 - p0 * c1 - pp0 * c2, v1 = y1 - p1 * c1 - pp1 * c2;
            g0[k] = v0; g1[k] = v1;
            const double w = 1.0 / d[k];
            s00 -= v0 * v0 * w; s01 -= v0 * v1 * w; s11 -= v1 * v1 * w;
            pp0 = p0; pp1 = p1; p0 = v0; p1 = v1;
        }
    }
    const double det = s00 * s11 - s01 * s01;
    for (int r = 0; r < 2; ++r) {
        const double *b = r ? by : bx;
        double *xx = r ? y : x;
        double b0 = b[m], b1 = b[m + 1];
        {
            double p = 0.0, pp = 0.0;
#pragma unroll 4
            for (int k = 0; k < m; ++k) {            // forward (result in xx)
                const double v = b[k] - l1[k] * p - l2[k] * pp;
                xx[k] = v;
                const double z = v / d[k];
                b0 -= g0[k] * z; b1 -= g1[k] * z;
                pp = p; p = v;
            }
        }
        const double xs0 = (s11 * b0 - s01 * b1) / det, xs1 = (s00 * b1 - s01 * b0) / det;
        xx[m] = xs0; xx[m + 1] = xs1;
        double n1 = 0.0, n2 = 0.0, c1 = 0.0, c2a = 0.0, c2b = 0.0;      // x[k+1], x[k+2]; l1[k+1], l2[k+2] (as seen from k), l2[k+1]
#pragma unroll 4
        for (int k = m - 1; k >= 0; --k) {
            const double v = (xx[k] - g0[k] * xs0 - g1[k] * xs1) / d[k] - c1 * n1 - c2a * n2;
            xx[k] = v;
            n2 = n1; n1 = v;
            c2a = c2b;               // l2[k+1] becomes the l2[(k-1)+2] of the next step
            c1 = l1[k]; c2b = l2[k];
        }
    }
}

__global__ void __launch_bounds__(256)
prep_track_kernel(int n_raw_max, const int32_t *__restrict__ n_raw_b, const double *__restrict__ raw, double s_reg,
                  double stepsize_prep, double stepsize_reg, double min_width, int n_int_max, int n_out_max,
                  double *__restrict__ out, int32_t *__restrict__ n_out, double *__restrict__ lam_out, double *__restrict__ ws) {
    const int b = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const int nr = n_raw_b ? n_raw_b[b] : n_raw_max;
    const double *tr = raw + (size_t)b * n_raw_max * 4;
    double *w = ws + (size_t)b * ((size_t)PT_VECS * n_int_max + (size_t)6 * (n_raw_max + 1));
    double *px = w, *py = px + n_int_max, *u = py + n_int_max, *h = u + n_int_max;
    double *q0 = h + n_int_max, *q1 = q0 + n_int_max, *q2 = q1 + n_int_max, *r0 = q2 + n_int_max, *r1 = r0 + n_int_max;
    double *a0 = r1 + n_int_max, *a1 = a0 + n_int_max, *a2 = a1 + n_int_max, *bx = a2 + n_int_max, *by = bx + n_int_max;
    double *dd = by + n_int_max, *l1 = dd + n_int_max, *l2 = l1 + n_int_max, *g0 = l2 + n_int_max, *g1 = g0 + n_int_max;
    double *gx = g1 + n_int_max, *gy = gx + n_int_max, *fx = gy + n_int_max;      // (fy re-uses bx after the fit)
    double *dist = fx + n_int_max;                        // [nr + 1] cumulative chord length of the closed raw track
    double *tcl = dist + (n_raw_max + 1), *wr = tcl + (n_raw_max + 1), *wl = wr + (n_raw_max + 1);
    double *pcx = wl + (n_raw_max + 1), *pcy = pcx + (n_raw_max + 1);
    __shared__ double red[32];
    __shared__ double sh_val[4];
    __shared__ int sh_n[4];
    // n_out[b] (include/mincurv_b200.h): >= 0 points, -(points needed) for a capacity, -MC_PREP_REFUSED - reason for a
    // track refused.  Every refusal is decided from values all threads share, before anything is written to the row.
    if (tid == 0) { n_out[b] = 0; if (lam_out) lam_out[b] = 0.0; }
    if (nr == 0) return;                                    // an inactive slot
    if (nr < 0 || nr > n_raw_max) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_N_RAW; return; }
    if (nr < 5) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_TOO_FEW; return; }
    // ---- 1. cumulative chord length of the closed raw polygon (numpy.cumsum order) ----
    if (tid == 0) {
        double acc = 0.0;
        bool finite = true;
        dist[0] = 0.0;
        for (int i = 0; i < nr; ++i) {
            const int j = (i + 1 == nr) ? 0 : i + 1;
            const double ex = tr[4 * j] - tr[4 * i], ey = tr[4 * j + 1] - tr[4 * i + 1];
            acc += sqrt(ex * ex + ey * ey);
            dist[i + 1] = acc;
            finite = finite && isfinite(tr[4 * i + 2]) && isfinite(tr[4 * i + 3]);
        }
        // (a non-finite coordinate makes the length inf or NaN; the counts are compared in double before the conversions)
        if (!finite || !isfinite(acc)) sh_n[0] = -MC_PREP_REFUSED - MC_PREP_R_NONFINITE;
        else if (!(ceil(acc / stepsize_prep) + 1.0 < (double)MC_PREP_REFUSED) || !(ceil(acc) * 4.0 < (double)MC_PREP_REFUSED))
            sh_n[0] = -MC_PREP_REFUSED - MC_PREP_R_COUNT;
        else sh_n[0] = (int)ceil(acc / stepsize_prep) + 1;     // points of the interpolated closed track
        sh_val[0] = acc;
    }
    __syncthreads();
    const int ni_cl = sh_n[0];
    const double Lraw = sh_val[0];
    const int n = ni_cl - 1;                                // periodic data points
    if (ni_cl < 0) { if (tid == 0) n_out[b] = ni_cl; return; }
    if (n < 5) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_TOO_FEW; return; }
    if (ni_cl > n_int_max) { if (tid == 0) n_out[b] = -ni_cl; return; }
    // ---- 2. linear pre-interpolation (numpy.linspace / numpy.interp statements) ----
    for (int i = tid; i < ni_cl; i += nt) {
        const double di = (i == ni_cl - 1) ? Lraw : i * (Lraw / (double)(ni_cl - 1));
        int lo = 0, hi = nr;
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (dist[mid] <= di) lo = mid; else hi = mid; }
        const int j = lo, jp = (j + 1 == nr) ? 0 : j + 1;
        const double t = (dist[j + 1] > dist[j]) ? (di - dist[j]) / (dist[j + 1] - dist[j]) : 0.0;
        double x = tr[4 * j] + t * (tr[4 * jp] - tr[4 * j]), y = tr[4 * j + 1] + t * (tr[4 * jp + 1] - tr[4 * j + 1]);
        if (i == ni_cl - 1) { x = tr[0]; y = tr[1]; }
        px[i] = x; py[i] = y;
    }
    __syncthreads();
    // ---- 3. chord-length parameter of the data points, normalised to [0, 1] (splprep's default u) ----
    if (tid == 0) {
        double acc = 0.0;
        u[0] = 0.0;
        for (int i = 0; i < n; ++i) {
            const double ex = px[i + 1] - px[i], ey = py[i + 1] - py[i];
            acc += sqrt(ex * ex + ey * ey);
            if (i + 1 < n) u[i + 1] = acc;
        }
        sh_val[1] = acc;
    }
    __syncthreads();
    const double Lu = sh_val[1];
    for (int i = tid; i < n; i += nt) if (i > 0) u[i] /= Lu;
    __syncthreads();
    for (int i = tid; i < n; i += nt) h[i] = ((i + 1 == n) ? 1.0 : u[i + 1]) - u[i];
    __syncthreads();
    for (int i = tid; i < n; i += nt) {
        const int im = (i == 0) ? n - 1 : i - 1, ip = (i + 1 == n) ? 0 : i + 1;
        const double ih = 1.0 / h[i], ihm = 1.0 / h[im], ihp = 1.0 / h[ip];
        q0[i] = ihm * ihm + (ih + ihm) * (ih + ihm) + ih * ih;
        q1[i] = -ih * (ih + ihm) - ih * (ihp + ih);
        q2[i] = ih * ihp;
        r0[i] = (h[im] + h[i]) / 3.0;
        r1[i] = h[i] / 6.0;
        bx[i] = (px[ip] - px[i]) * ih - (px[i] - px[im]) * ihm;       // Q^T p
        by[i] = (py[ip] - py[i]) * ih - (py[i] - py[im]) * ihm;
    }
    __syncthreads();
    // ---- 4. smoothing parameter: F(lam) = |lam Q gamma|^2 = s, F increasing; bracket by factors of 16, then the Illinois
    //         variant of regula falsi on log F over log lam ----
    double lo_l = 1e-12, hi_l = 1.0, f_lo = 0.0, f_hi = 0.0, lam = 1.0, F_last = 0.0;
    bool have_lo = false, have_hi = false, reached = false;  // reached: the loop ended on its tolerance with a finite F
    int side = 0;
    for (int iter = 0; iter < 200; ++iter) {
        if (!have_hi) lam = hi_l;
        else if (!have_lo) lam = lo_l;
        else {
            const double xl = log(lo_l), xh = log(hi_l), yl = log(f_lo / s_reg), yh = log(f_hi / s_reg);
            double xm = (xl * yh - xh * yl) / (yh - yl);
            if (!(xm > xl && xm < xh)) xm = 0.5 * (xl + xh);
            lam = exp(xm);
        }
        for (int i = tid; i < n; i += nt) { a0[i] = r0[i] + lam * q0[i]; a1[i] = r1[i] + lam * q1[i]; a2[i] = lam * q2[i]; }
        __syncthreads();
        if (tid == 0) penta_cyclic_solve2(n, a0, a1, a2, bx, by, dd, l1, l2, g0, g1, gx, gy);
        __syncthreads();
        double acc = 0.0;
        for (int i = tid; i < n; i += nt) {
            const int im = (i == 0) ? n - 1 : i - 1, ip = (i + 1 == n) ? 0 : i + 1;
            const double rx = lam * ((gx[ip] - gx[i]) / h[i] - (gx[i] - gx[im]) / h[im]);
            const double ry = lam * ((gy[ip] - gy[i]) / h[i] - (gy[i] - gy[im]) / h[im]);
            acc += rx * rx + ry * ry;
        }
        const double F = block_reduce<0>(acc, red);
        __syncthreads();
        F_last = F;
        if (!have_hi) {
            if (F >= s_reg) { have_hi = true; f_hi = F; }
            else { lo_l = hi_l; f_lo = F; have_lo = true; hi_l *= 16.0; if (hi_l > 1e30) break; }
            continue;
        }
        if (!have_lo) {
            if (F <= s_reg) { have_lo = true; f_lo = F; }
            else { hi_l = lo_l; f_hi = F; lo_l /= 16.0; if (lo_l < 1e-300) break; }
            continue;
        }
        if (fabs(F - s_reg) <= 1e-13 * s_reg || hi_l / lo_l < 1.0 + 4e-16) { reached = isfinite(F); break; }
        if (F < s_reg) { lo_l = lam; f_lo = F; if (side == -1) f_hi = s_reg + 0.5 * (f_hi - s_reg); side = -1; }
        else { hi_l = lam; f_hi = F; if (side == 1) f_lo = s_reg - 0.5 * (s_reg - f_lo); side = 1; }
    }
    if (tid == 0 && lam_out) lam_out[b] = lam;
    // s_reg >= F(inf) (the residual of the best constant) ends the bracket at lam > 1e30, and a bracket below 1e-300 ends
    // it too: the budget is not reached and the curve would not be the one asked for.  At the iteration cap (rounding in
    // F can keep the loop from its 1e-13 tolerance under heavy smoothing) the budget counts as reached within 1e-6 s_reg.
    if (!reached && have_lo && have_hi && isfinite(F_last) && fabs(F_last - s_reg) <= 1e-6 * s_reg) reached = true;
    if (!reached) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_BUDGET; return; }
    // fitted values f = p - lam Q gamma (fy takes the place of bx)
    double *fy = bx;
    __syncthreads();
    for (int i = tid; i < n; i += nt) {
        const int im = (i == 0) ? n - 1 : i - 1, ip = (i + 1 == n) ? 0 : i + 1;
        fx[i] = px[i] - lam * ((gx[ip] - gx[i]) / h[i] - (gx[i] - gx[im]) / h[im]);
        a0[i] = py[i] - lam * ((gy[ip] - gy[i]) / h[i] - (gy[i] - gy[im]) / h[im]);
    }
    __syncthreads();
    for (int i = tid; i < n; i += nt) fy[i] = a0[i];
    __syncthreads();
    const PtSpline sp{u, fx, fy, gx, gy, n};
    // ---- 5. curve length from ceil(L_raw) * 4 samples ----
    const int n_len = (int)ceil(Lraw) * 4;
    double acc = 0.0;
    for (int i = tid; i + 1 < n_len; i += nt) {
        const double t0 = (double)i / (double)(n_len - 1), t1 = (i + 2 == n_len) ? 1.0 : (double)(i + 1) / (double)(n_len - 1);
        double x0, y0, x1, y1;
        pt_eval(sp, fmin(t0, 1.0 - 1e-16), &x0, &y0, nullptr, nullptr, nullptr, nullptr);
        if (i + 2 == n_len) { x1 = fx[0]; y1 = fy[0]; }
        else pt_eval(sp, t1, &x1, &y1, nullptr, nullptr, nullptr, nullptr);
        acc += sqrt((x1 - x0) * (x1 - x0) + (y1 - y0) * (y1 - y0));
    }
    const double Lsm = block_reduce<0>(acc, red);
    if (!isfinite(Lsm)) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_NONFINITE; return; }
    if (!(ceil(Lsm / stepsize_reg) < (double)MC_PREP_REFUSED)) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_COUNT; return; }
    const int n_reg_cl = (int)ceil(Lsm / stepsize_reg) + 1, n_reg = n_reg_cl - 1;
    if (n_reg < 3) { if (tid == 0) n_out[b] = -MC_PREP_REFUSED - MC_PREP_R_FEW_OUT; return; }
    if (n_reg > n_out_max) { if (tid == 0) n_out[b] = -n_reg; return; }
    // ---- 6. closest curve point of every point of the closed raw track (tph: fmin from the chord-length guess) ----
    for (int i = tid; i <= nr; i += nt) {
        const int ii = (i == nr) ? 0 : i;
        const double qx = tr[4 * ii], qy = tr[4 * ii + 1];
        const double t0 = dist[i] / Lraw, span = 4.0 * stepsize_prep / Lraw;
        double best = 1e300, tb = t0;
        for (int c = 0; c <= 32; ++c) {                     // coarse scan of +-4 pre-interpolation steps
            const double tc = t0 - span + (2.0 * span) * c / 32.0;
            double tw = tc - floor(tc), x, y;
            pt_eval(sp, tw, &x, &y, nullptr, nullptr, nullptr, nullptr);
            const double d2 = (x - qx) * (x - qx) + (y - qy) * (y - qy);
            if (d2 < best) { best = d2; tb = tc; }
        }
        double lo = tb - span / 16.0, hi = tb + span / 16.0, t = tb;
        for (int it = 0; it < 60; ++it) {                   // safeguarded Newton on d/dt |f(t) - q|^2
            double tw = t - floor(t), x, y, dx, dy, ddx, ddy;
            pt_eval(sp, tw, &x, &y, &dx, &dy, &ddx, &ddy);
            const double gdt = (x - qx) * dx + (y - qy) * dy, hdt = dx * dx + dy * dy + (x - qx) * ddx + (y - qy) * ddy;
            if (gdt > 0.0) hi = t; else lo = t;
            double tn = (hdt > 0.0) ? t - gdt / hdt : 0.5 * (lo + hi);
            if (!(tn > lo && tn < hi)) tn = 0.5 * (lo + hi);
            if (fabs(tn - t) <= 1e-15) { t = tn; break; }
            t = tn;
        }
        double tw = t - floor(t), x, y;
        pt_eval(sp, tw, &x, &y, nullptr, nullptr, nullptr, nullptr);
        tcl[i] = (i == 0) ? 0.0 : (i == nr) ? 1.0 : t;
        pcx[i] = x; pcy[i] = y;
        wr[i] = sqrt((x - qx) * (x - qx) + (y - qy) * (y - qy));     // distance (the side is applied below)
    }
    __syncthreads();
    for (int i = tid; i <= nr; i += nt) {
        // side of the closest point relative to the raw segment i -> i + 1 (the closing entry re-uses the first side)
        const int i0 = (i == nr) ? 0 : i, i1 = (i0 + 1 == nr) ? 0 : i0 + 1;
        const double cr = (tr[4 * i1] - tr[4 * i0]) * (pcy[i0] - tr[4 * i0 + 1]) - (tr[4 * i1 + 1] - tr[4 * i0 + 1]) * (pcx[i0] - tr[4 * i0]);
        const double sgn = (cr > 0.0) ? 1.0 : (cr < 0.0) ? -1.0 : 0.0;
        const double dst = wr[i];
        wl[i] = tr[4 * i0 + 3] - sgn * dst;
        wr[i] = tr[4 * i0 + 2] + sgn * dst;
    }
    __syncthreads();
    // ---- 7. re-sampled centre line + widths (numpy.interp over the closest-point parameters), min-width inflation ----
    double *o = out + (size_t)b * n_out_max * 4;
    for (int i = tid; i < n_reg; i += nt) {
        const double tq = (double)i / (double)(n_reg_cl - 1);
        double x, y;
        pt_eval(sp, tq, &x, &y, nullptr, nullptr, nullptr, nullptr);
        int lo = 0, hi = nr;                                // tcl[lo] <= tq < tcl[hi]
        while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (tcl[mid] <= tq) lo = mid; else hi = mid; }
        const double den = tcl[lo + 1] - tcl[lo], f = (den > 0.0) ? (tq - tcl[lo]) / den : 0.0;
        double w_r = wr[lo] + f * (wr[lo + 1] - wr[lo]), w_l = wl[lo] + f * (wl[lo + 1] - wl[lo]);
        if (min_width > 0.0 && w_r + w_l < min_width) { const double add = 0.5 * (min_width - (w_r + w_l)); w_r += add; w_l += add; }
        o[4 * i] = x; o[4 * i + 1] = y; o[4 * i + 2] = w_r; o[4 * i + 3] = w_l;
    }
    for (int i = n_reg + tid; i < n_out_max; i += nt) { o[4 * i] = 0.0; o[4 * i + 1] = 0.0; o[4 * i + 2] = 0.0; o[4 * i + 3] = 0.0; }
    if (tid == 0) n_out[b] = n_reg;
}

}  // namespace mc

extern "C" {

size_t mc_prep_track_workspace_bytes(int B, int n_raw_max, int n_int_max) {
    if (B <= 0 || n_raw_max < 5 || n_int_max < 6) return 0;
    return align256((size_t)B * ((size_t)mc::PT_VECS * n_int_max + (size_t)6 * (n_raw_max + 1)) * sizeof(double));
}

int mc_prep_track_batch(int B, int n_raw_max, const int32_t *n_raw, const double *track, int k_reg, double s_reg,
                        double stepsize_prep, double stepsize_reg, double min_width, int n_int_max, int n_out_max,
                        double *reftrack_interp, int32_t *n_out, double *smoothing_lambda, void *workspace,
                        size_t workspace_bytes, void *stream) {
    if (B <= 0 || n_raw_max < 5 || !track || !(s_reg > 0.0) || !(stepsize_prep > 0.0) || !(stepsize_reg > 0.0) || n_int_max < 6 ||
        n_out_max < 4 || !reftrack_interp || !n_out)
        return bad("mc_prep_track_batch: bad argument");
    if (k_reg != 3) return bad("mc_prep_track_batch: only cubic splines (k_reg = 3, the reference's setting) are implemented");
    if (!workspace || workspace_bytes < mc_prep_track_workspace_bytes(B, n_raw_max, n_int_max))
        return small_workspace("mc_prep_track_batch");
    mc::prep_track_kernel<<<B, 256, 0, (cudaStream_t)stream>>>(n_raw_max, n_raw, track, s_reg, stepsize_prep, stepsize_reg,
                                                               min_width, n_int_max, n_out_max, reftrack_interp, n_out,
                                                               smoothing_lambda, (double *)workspace);
    return check_cuda("prep_track_kernel");
}

}  // extern "C"
