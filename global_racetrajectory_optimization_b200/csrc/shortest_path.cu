// K4 -- tph.opt_shortest_path (call site main_globaltraj.py:286-290, SURVEY.md A.4):
//   min 1/2 a^T H a + f^T a,  -dev_max_left <= a <= dev_max_right,
//   H cyclic tridiagonal (diag 4 |n_i|^2, off-diag -2 n_i.n_{i+1}),  f_i = 2 n_i.(2 p_i - p_{i+1} - p_{i-1}).
// The same Mehrotra primal-dual interior-point iteration as K2b, but M = H + D is cyclic tridiagonal,
// so each instance costs O(N) per iteration: the second "H form" of the QP path is HBM-streaming work.
// Mapping: one THREAD per QP instance, all per-instance vectors interleaved over the batch
// (element i of instance b at [i * B + b]) so that every pass is a fully coalesced stream; the cyclic
// system is solved by the Thomas recurrences + Sherman-Morrison (gamma = -diag_0, T = M + |gamma| w w^T
// stays SPD).  Large batches (BASELINE config 5: 32k instances) fill the machine.
#include "common.cuh"
#include "../../include/mincurv_b200.h"

namespace mc {

enum SpVec : int { SP_LB = 0, SP_UB, SP_F, SP_OFF, SP_DG, SP_AL, SP_LU, SP_LL, SP_RD, SP_X, SP_CP, SP_MI, SP_Q, SP_TU, SP_TL, SP_DD, SP_RHS, SP_SU, SP_SL, SP_NUM };

size_t shortest_path_ws_doubles(int n_max) { return (size_t)SP_NUM * n_max; }

struct SpView {
    double *base; size_t B; size_t nB;   // nB = n_max * B
    int b;
    __device__ __forceinline__ double &operator()(int v, int i) const { return base[(size_t)v * nB + (size_t)i * B + b]; }
};

// Solve M x = rhs with M = tridiag(off, dg + dd, off) cyclic.  If `refactor`, (re)build cp, mi, q.
__device__ inline void cyc_solve(const SpView &w, int n, bool refactor) {
    const double d0 = w(SP_DG, 0) + w(SP_DD, 0);
    const double gamma = -d0;
    const double cN = w(SP_OFF, n - 1);          // corner M[n-1][0] = M[0][n-1]
    // forward elimination of T = M - u v^T,  u = (gamma, 0, .., cN), v = (1, 0, .., cN / gamma)
    double cp_prev = 0.0, xp = 0.0, qp = 0.0;
    for (int i = 0; i < n; ++i) {
        double mi, cp;
        const double offm = (i > 0) ? w(SP_OFF, i - 1) : 0.0;
        if (refactor) {
            double dg = w(SP_DG, i) + w(SP_DD, i);
            if (i == 0) dg -= gamma;
            if (i == n - 1) dg -= cN * cN / gamma;
            mi = 1.0 / (dg - offm * cp_prev);
            cp = ((i < n - 1) ? w(SP_OFF, i) : 0.0) * mi;
            w(SP_MI, i) = mi; w(SP_CP, i) = cp;
            const double ui = (i == 0) ? gamma : ((i == n - 1) ? cN : 0.0);
            qp = (ui - offm * qp) * mi;
            w(SP_Q, i) = qp;
        } else {
            mi = w(SP_MI, i); cp = w(SP_CP, i);
        }
        xp = (w(SP_RHS, i) - offm * xp) * mi;
        w(SP_X, i) = xp;
        cp_prev = cp;
    }
    // back substitution
    double xn = w(SP_X, n - 1), qn = refactor ? w(SP_Q, n - 1) : 0.0;
    for (int i = n - 2; i >= 0; --i) {
        const double cp = w(SP_CP, i);
        xn = w(SP_X, i) - cp * xn;
        w(SP_X, i) = xn;
        if (refactor) { qn = w(SP_Q, i) - cp * qn; w(SP_Q, i) = qn; }
    }
    // Sherman-Morrison correction  x = y - q (v.y) / (1 + v.q)
    const double vy = w(SP_X, 0) + cN / gamma * w(SP_X, n - 1);
    const double vq = w(SP_Q, 0) + cN / gamma * w(SP_Q, n - 1);
    const double fac = vy / (1.0 + vq);
    for (int i = 0; i < n; ++i) w(SP_X, i) -= fac * w(SP_Q, i);
}

__global__ void __launch_bounds__(128)
shortest_path_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ reftrack,
                     const double *__restrict__ normvec, double w_veh, const double *__restrict__ w_veh_batch,
                     double *__restrict__ alpha, int32_t *__restrict__ status, int32_t *__restrict__ iters,
                     double *__restrict__ ws) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int n = n_pts ? n_pts[b] : n_max;
    double *aout = alpha + (size_t)b * n_max;
    if (n < 3 || n > n_max) {
        for (int i = 0; i < n_max; ++i) aout[i] = 0.0;
        status[b] = -1;
        if (iters) iters[b] = 0;
        return;
    }
    SpView w{ws, (size_t)B, (size_t)n_max * B, b};
    const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
    const double *rt = reftrack + (size_t)b * n_max * 4;
    const double *nv = normvec + (size_t)b * n_max * 2;
    // ---- assembly (tph clamps both bounds to >= 0.001) ----
    double gmax = 0.0;
    for (int i = 0; i < n; ++i) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double nx = nv[2 * i], ny = nv[2 * i + 1], nxp = nv[2 * ip1], nyp = nv[2 * ip1 + 1];
        const double px = rt[4 * i], py = rt[4 * i + 1];
        double dr = rt[4 * i + 2] - 0.5 * wv, dl = rt[4 * i + 3] - 0.5 * wv;
        if (dr < 0.001) dr = 0.001;
        if (dl < 0.001) dl = 0.001;
        const double fi = 2.0 * (nx * (2.0 * px - rt[4 * ip1] - rt[4 * im1]) + ny * (2.0 * py - rt[4 * ip1 + 1] - rt[4 * im1 + 1]));
        w(SP_UB, i) = dr; w(SP_LB, i) = -dl; w(SP_F, i) = fi;
        w(SP_DG, i) = 4.0 * (nx * nx + ny * ny);
        w(SP_OFF, i) = -2.0 * (nx * nxp + ny * nyp);
        w(SP_AL, i) = 0.5 * (dr - dl);
    }
    // gradient at the box centre
    double fmaxv = 0.0;
    for (int i = 0; i < n; ++i) {
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double g = w(SP_DG, i) * w(SP_AL, i) + w(SP_OFF, i) * w(SP_AL, ip1) + w(SP_OFF, im1) * w(SP_AL, im1) + w(SP_F, i);
        w(SP_RD, i) = g;
        gmax = fmax(gmax, fabs(g));
        fmaxv = fmax(fmaxv, fabs(w(SP_F, i)));
    }
    const double lam0 = 1e-2 * gmax + 1e-300;
    double musum = 0.0;
    for (int i = 0; i < n; ++i) {
        const double g = w(SP_RD, i);
        const double lu = fmax(-g, 0.0) + lam0, ll = fmax(g, 0.0) + lam0;
        w(SP_LU, i) = lu; w(SP_LL, i) = ll; w(SP_RD, i) = g + lu - ll;
        const double a = w(SP_AL, i);
        const double su = w(SP_UB, i) - a, sl = a - w(SP_LB, i);
        w(SP_SU, i) = su; w(SP_SL, i) = sl;
        musum += su * lu + sl * ll;
    }
    const double mu0 = musum / (2.0 * n);
    const double rd_tol = 1e-8 * (fmaxv + gmax) + 1e-300;
    double mu = mu0;
    int it = 0, result = MC_STATUS_MAXITER;
    for (it = 0; it < 50; ++it) {
        for (int i = 0; i < n; ++i) {
            const double su = w(SP_SU, i), sl = w(SP_SL, i), lu = w(SP_LU, i), ll = w(SP_LL, i);
            w(SP_DD, i) = lu / su + ll / sl;
            w(SP_RHS, i) = -w(SP_RD, i) + lu - ll;
        }
        cyc_solve(w, n, true);
        double ap = 1.0, ad = 1.0;
        for (int i = 0; i < n; ++i) {
            const double su = w(SP_SU, i), sl = w(SP_SL, i), lu = w(SP_LU, i), ll = w(SP_LL, i);
            const double dx = w(SP_X, i);
            const double dlu = -lu + lu * dx / su, dll = -ll - ll * dx / sl;
            if (dx > 0.0) ap = fmin(ap, su / dx);
            if (dx < 0.0) ap = fmin(ap, -sl / dx);
            if (dlu < 0.0) ad = fmin(ad, -lu / dlu);
            if (dll < 0.0) ad = fmin(ad, -ll / dll);
        }
        double mua = 0.0;
        for (int i = 0; i < n; ++i) {
            const double su = w(SP_SU, i), sl = w(SP_SL, i), lu = w(SP_LU, i), ll = w(SP_LL, i);
            const double dx = w(SP_X, i);
            const double dlu = -lu + lu * dx / su, dll = -ll - ll * dx / sl;
            mua += (su - ap * dx) * (lu + ad * dlu) + (sl + ap * dx) * (ll + ad * dll);
        }
        mua /= (2.0 * n);
        double sigma = mua / mu;
        sigma = sigma * sigma * sigma;
        const double smu = sigma * mu;
        for (int i = 0; i < n; ++i) {
            const double su = w(SP_SU, i), sl = w(SP_SL, i), lu = w(SP_LU, i), ll = w(SP_LL, i);
            const double dx = w(SP_X, i);
            const double dlu = -lu + lu * dx / su, dll = -ll - ll * dx / sl;
            const double tu = smu - su * lu + dx * dlu, tl = smu - sl * ll - dx * dll;
            w(SP_TU, i) = tu; w(SP_TL, i) = tl;
            w(SP_RHS, i) = -w(SP_RD, i) - tu / su + tl / sl;
        }
        cyc_solve(w, n, false);
        ap = 1e300; ad = 1e300;
        for (int i = 0; i < n; ++i) {
            const double su = w(SP_SU, i), sl = w(SP_SL, i), lu = w(SP_LU, i), ll = w(SP_LL, i);
            const double dx = w(SP_X, i);
            const double dlu = (w(SP_TU, i) + lu * dx) / su, dll = (w(SP_TL, i) - ll * dx) / sl;
            if (dx > 0.0) ap = fmin(ap, su / dx);
            if (dx < 0.0) ap = fmin(ap, -sl / dx);
            if (dlu < 0.0) ad = fmin(ad, -lu / dlu);
            if (dll < 0.0) ad = fmin(ad, -ll / dll);
        }
        ap = fmin(1.0, 0.995 * ap);
        ad = fmin(1.0, 0.995 * ad);
        double musum2 = 0.0, rdmax = 0.0;
        for (int i = 0; i < n; ++i) {
            const double su = w(SP_SU, i), sl = w(SP_SL, i), lu = w(SP_LU, i), ll = w(SP_LL, i);
            const double dx = w(SP_X, i);
            const double dlu = (w(SP_TU, i) + lu * dx) / su, dll = (w(SP_TL, i) - ll * dx) / sl;
            const double an = w(SP_AL, i) + ap * dx, lun = lu + ad * dlu, lln = ll + ad * dll;
            const double sun = su - ap * dx, sln = sl + ap * dx;
            const double rdn = w(SP_RD, i) + ap * (w(SP_RHS, i) - w(SP_DD, i) * dx) + ad * (dlu - dll);
            w(SP_AL, i) = an; w(SP_LU, i) = lun; w(SP_LL, i) = lln; w(SP_RD, i) = rdn; w(SP_SU, i) = sun; w(SP_SL, i) = sln;
            musum2 += sun * lun + sln * lln;
            rdmax = fmax(rdmax, fabs(rdn));
        }
        mu = musum2 / (2.0 * n);
        if (mu <= 1e-11 * mu0 && rdmax <= rd_tol) { result = MC_STATUS_OK; ++it; break; }
        if (mu <= 1e-15 * mu0) { result = (rdmax <= 1e3 * rd_tol) ? MC_STATUS_OK : MC_STATUS_MAXITER; ++it; break; }
        if (!(mu == mu)) { result = MC_STATUS_BREAKDOWN; break; }
    }
    for (int i = 0; i < n_max; ++i) aout[i] = (i < n) ? w(SP_AL, i) : 0.0;
    status[b] = result;
    if (iters) iters[b] = it;
}

int launch_shortest_path(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                         double w_veh, const double *w_veh_batch, double *alpha, int32_t *status, int32_t *iters,
                         double *ws, cudaStream_t stream) {
    const int threads = 128;
    shortest_path_kernel<<<(B + threads - 1) / threads, threads, 0, stream>>>(B, n_max, n_pts, reftrack, normvec, w_veh,
                                                                             w_veh_batch, alpha, status, iters, ws);
    return 0;
}

// ---- sensitivities (csrc/shortest_path_sens.h, DESIGN.md section 3.11) ----
// Run right after shortest_path_kernel on the same workspace: the final iterate's lu / su and ll / sl, the diagonal D of
// M = H + D that the backward pass factorises, and grad_status = status.
__global__ void __launch_bounds__(128)
shortest_path_sens_export_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, const int32_t *__restrict__ status,
                                 const double *__restrict__ ws, double *__restrict__ sens, int32_t *__restrict__ grad_status) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int n = n_pts ? n_pts[b] : n_max;
    const int st = status[b];
    const bool ok = st == MC_STATUS_OK && n >= 3 && n <= n_max;
    const SpView w{const_cast<double *>(ws), (size_t)B, (size_t)n_max * B, b};
    double *du = sens + (size_t)b * 2 * n_max, *dl = du + n_max;
#pragma unroll 1
    for (int i = 0; i < n_max; ++i) {
        const bool in = ok && i < n;
        du[i] = in ? w(SP_LU, i) / w(SP_SU, i) : 0.0;
        dl[i] = in ? w(SP_LL, i) / w(SP_SL, i) : 0.0;
    }
    grad_status[b] = st;
}

// Vector-Jacobian product of alpha: v = (H + D)^-1 grad_alpha by the forward's cyclic solve, then the gradients with
// respect to f, H, and the bounds, chained to the centre line, the normals and the widths (DESIGN.md section 3.11).
__global__ void __launch_bounds__(128)
shortest_path_adjoint_kernel(int B, int n_max, const int32_t *__restrict__ n_pts, const double *__restrict__ reftrack,
                             const double *__restrict__ normvec, double w_veh, const double *__restrict__ w_veh_batch,
                             const double *__restrict__ alpha, const double *__restrict__ sens, int32_t *__restrict__ grad_status,
                             const double *__restrict__ grad_alpha, double *__restrict__ grad_reftrack,
                             double *__restrict__ grad_normvec, double *__restrict__ grad_w_veh, double *__restrict__ ws) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int n = n_pts ? n_pts[b] : n_max;
    double *grt = grad_reftrack + (size_t)b * n_max * 4;
    double *gnv = grad_normvec ? grad_normvec + (size_t)b * n_max * 2 : nullptr;
    const bool sized = n >= 3 && n <= n_max;
    bool ok = sized && grad_status[b] == MC_STATUS_OK;
    const SpView w{ws, (size_t)B, (size_t)n_max * B, b};
    const double *rt = reftrack + (size_t)b * n_max * 4;
    const double *nv = normvec + (size_t)b * n_max * 2;
    const double *a = alpha + (size_t)b * n_max;
    const double *du = sens + (size_t)b * 2 * n_max, *dl = du + n_max;
    if (ok) {
        const double *g = grad_alpha + (size_t)b * n_max;
        for (int i = 0; i < n; ++i) {
            const int ip1 = (i + 1 == n) ? 0 : i + 1;
            const double nx = nv[2 * i], ny = nv[2 * i + 1];
            w(SP_DG, i) = 4.0 * (nx * nx + ny * ny);
            w(SP_OFF, i) = -2.0 * (nx * nv[2 * ip1] + ny * nv[2 * ip1 + 1]);
            w(SP_DD, i) = du[i] + dl[i];
            w(SP_RHS, i) = g[i];
        }
        cyc_solve(w, n, true);
        for (int i = 0; i < n; ++i) ok = ok && isfinite(w(SP_X, i));
        if (!ok) grad_status[b] = MC_STATUS_BREAKDOWN;
    }
    if (!sized) grad_status[b] = -1;
    const double wv = w_veh_batch ? w_veh_batch[b] : w_veh;
    double gwv = 0.0;
    for (int i = 0; i < n_max; ++i) {
        if (!ok || i >= n) {
            grt[4 * i] = grt[4 * i + 1] = grt[4 * i + 2] = grt[4 * i + 3] = 0.0;
            if (gnv) gnv[2 * i] = gnv[2 * i + 1] = 0.0;
            continue;
        }
        const int im1 = (i == 0) ? n - 1 : i - 1, ip1 = (i + 1 == n) ? 0 : i + 1;
        const double v = w(SP_X, i), vm = w(SP_X, im1), vp = w(SP_X, ip1);
        const double nx = nv[2 * i], ny = nv[2 * i + 1];
        const double nxm = nv[2 * im1], nym = nv[2 * im1 + 1], nxp = nv[2 * ip1], nyp = nv[2 * ip1 + 1];
        // dL/df_i = -v_i  ->  the centre line (f_j = 2 n_j.(2 p_j - p_{j+1} - p_{j-1}))
        grt[4 * i] = -(4.0 * nx * v - 2.0 * nxm * vm - 2.0 * nxp * vp);
        grt[4 * i + 1] = -(4.0 * ny * v - 2.0 * nym * vm - 2.0 * nyp * vp);
        // dL/dub = d_u v, dL/dlb = d_l v; a clamped bound (the forward's test dr < 0.001) does not move with the widths
        const double dr = rt[4 * i + 2] - 0.5 * wv, dlw = rt[4 * i + 3] - 0.5 * wv;
        const double gub = (dr < 0.001) ? 0.0 : du[i] * v, glb = (dlw < 0.001) ? 0.0 : dl[i] * v;
        grt[4 * i + 2] = gub;
        grt[4 * i + 3] = -glb;
        gwv += 0.5 * (glb - gub);
        if (gnv) {
            // dL/dH_ii = -v_i a_i, dL/dH_{i,i+1} = -(v_i a_{i+1} + v_{i+1} a_i) (both symmetric entries), dL/df_i = -v_i
            const double ai = a[i];
            const double gd = -v * ai, go = -(v * a[ip1] + vp * ai), gom = -(vm * ai + v * a[im1]);
            const double cx = 2.0 * rt[4 * i] - rt[4 * ip1] - rt[4 * im1], cy = 2.0 * rt[4 * i + 1] - rt[4 * ip1 + 1] - rt[4 * im1 + 1];
            gnv[2 * i] = 8.0 * nx * gd - 2.0 * nxp * go - 2.0 * nxm * gom - 2.0 * cx * v;
            gnv[2 * i + 1] = 8.0 * ny * gd - 2.0 * nyp * go - 2.0 * nym * gom - 2.0 * cy * v;
        }
    }
    if (grad_w_veh) grad_w_veh[b] = ok ? gwv : 0.0;
}

void launch_shortest_path_sens_export(int B, int n_max, const int32_t *n_pts, const int32_t *status, const double *ws,
                                      double *sens, int32_t *grad_status, cudaStream_t stream) {
    const int threads = 128;
    shortest_path_sens_export_kernel<<<(B + threads - 1) / threads, threads, 0, stream>>>(B, n_max, n_pts, status, ws, sens,
                                                                                         grad_status);
}

void launch_shortest_path_adjoint(int B, int n_max, const int32_t *n_pts, const double *reftrack, const double *normvec,
                                  double w_veh, const double *w_veh_batch, const double *alpha, const double *sens,
                                  int32_t *grad_status, const double *grad_alpha, double *grad_reftrack, double *grad_normvec,
                                  double *grad_w_veh, double *ws, cudaStream_t stream) {
    const int threads = 128;
    shortest_path_adjoint_kernel<<<(B + threads - 1) / threads, threads, 0, stream>>>(
        B, n_max, n_pts, reftrack, normvec, w_veh, w_veh_batch, alpha, sens, grad_status, grad_alpha, grad_reftrack,
        grad_normvec, grad_w_veh, ws);
}

}  // namespace mc
