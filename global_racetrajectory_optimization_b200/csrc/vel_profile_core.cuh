// K5 core -- per-profile arithmetic of tph.calc_vel_profile / calc_ax_profile / calc_t_profile (closed tracks, ggv
// branch), the stage that follows the raceline in the reference (call sites main_globaltraj.py:400-421
// and the lap-time matrix sweep :442-496; SURVEY.md 8f-1).
//
// One profile = one (track, variant) pair: the track supplies kappa / el_lengths (/ mu), the variant a ggv scale and a
// top speed (the two axes of the reference's lap-time matrix).  The forward/backward solver is a nonlinear recurrence
// along the lap, so a profile is sequential; profiles are independent, so one THREAD runs one profile and every
// per-profile array is addressed through a stride (stride = number of profiles on the device: element i of profile p at
// [i * P + p], every pass a coalesced stream -- the layout of K4, shortest_path.cu).
//
// The functions are __host__ __device__ and free of CUDA-only constructs so that tests/ can compile this header with
// g++ and run the identical statements on the CPU against the numpy oracle (tests/host_harness/); the product only ever
// calls them from vel_profile_kernel.  Arithmetic mirrors tph statement by statement (operation order, no fused
// multiply-add: the products/sums that tph evaluates separately go through __dmul_rn/__dadd_rn).
#pragma once
#include <math.h>
#include <stddef.h>

#if defined(__CUDACC__)
#define VP_HD __host__ __device__ __forceinline__
#else
#define VP_HD inline
#endif

namespace mc {
namespace vp {

// tph (as recalled) keeps vx_profile_double[no_points:] after the backward pass over the doubled lap, i.e. the half the
// backward pass visits first.  Cannot be confirmed offline (parity unpinned); oracle/tph_velprofile.py carries the same
// switch (DECEL_LAP_SLICE_UPPER).  It is a RUN-TIME parameter (Params::decel_slice_upper, C-ABI mc_vel_profile_batch_ex):
// 0 => the backward pass runs both laps and keeps the second one.  VP_DECEL_SLICE_UPPER is only the default
// (tools/pin_against_tph.py reports which value the real package implies).
#ifndef VP_DECEL_SLICE_UPPER
#define VP_DECEL_SLICE_UPPER 1
#endif

constexpr int VP_UNROLL = 4;             // elements per block of the streaming loops (loads first, then arithmetic)
constexpr int VP_STATUS_OK = 0;
constexpr int VP_STATUS_NONFINITE = 3;   // NaN/inf lap time (tph would raise a math domain error or return NaN)

VP_HD double mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
VP_HD double add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
VP_HD double sub(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}

struct Tables {
    const double *gv, *gax, *gay;   // ggv diagram columns v, ax_max, ay_max (n_ggv rows)
    int n_ggv;
    const double *mv, *ma;          // ax_max_machines columns v, ax_max_machines (n_mach rows)
    int n_mach;
};

struct Params {
    double dyn_model_exp, drag_coeff, m_veh;
    int filt_window;                // <= 1: no moving-average filter (tph: filt_window=None)
    int decel_slice_upper = VP_DECEL_SLICE_UPPER;   // which half of the doubled lap the backward pass keeps (see above)
};

struct Strided {
    double *p;
    size_t s;
    VP_HD double &operator[](int i) const { return p[(size_t)i * s]; }
};

// numpy.interp(x, xp, fp * s) for a scalar x (xp increasing): clamped outside the table, exact at the knots.
// `hint`: segment found by the previous call of the same caller (speeds change slowly along a lap, so the search is
// skipped almost always); any value in [0, n - 2] is valid, the result does not depend on it.
VP_HD int find_segment(double x, const double *xp, int n, int &hint) {     // requires xp[0] <= x < xp[n - 1]
    int lo = hint;
    if (xp[lo] <= x && x < xp[lo + 1]) return lo;
    lo = 0;
    int hi = n - 1;                               // xp[lo] <= x < xp[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (xp[mid] <= x) lo = mid; else hi = mid;
    }
    hint = lo;
    return lo;
}

VP_HD double interp(double x, const double *xp, const double *fp, int n, double s, int &hint) {
    if (x != x) return x;
    if (x >= xp[n - 1]) return mul(fp[n - 1], s);
    if (x < xp[0]) return mul(fp[0], s);
    const int lo = find_segment(x, xp, n, hint);
    const double f0 = mul(fp[lo], s);
    if (xp[lo] == x) return f0;
    const double f1 = mul(fp[lo + 1], s);
    const double slope = sub(f1, f0) / sub(xp[lo + 1], xp[lo]);
    return add(mul(slope, sub(x, xp[lo])), f0);
}

// Both columns of the ggv diagram at one speed: numpy.interp(x, xp, fa * s), numpy.interp(x, xp, fb * s) with one
// search of xp (the two interpolations of calc_ax_poss share their abscissa).
VP_HD void interp2(double x, const double *xp, const double *fa, const double *fb, int n, double s, double &oa,
                   double &ob, int &hint) {
    if (x != x) { oa = x; ob = x; return; }
    if (x >= xp[n - 1]) { oa = mul(fa[n - 1], s); ob = mul(fb[n - 1], s); return; }
    if (x < xp[0]) { oa = mul(fa[0], s); ob = mul(fb[0], s); return; }
    const int lo = find_segment(x, xp, n, hint);
    const double a0 = mul(fa[lo], s), b0 = mul(fb[lo], s), x0 = xp[lo];
    if (x0 == x) { oa = a0; ob = b0; return; }
    const double a1 = mul(fa[lo + 1], s), b1 = mul(fb[lo + 1], s);
    const double dx = sub(xp[lo + 1], x0), t = sub(x, x0);
    oa = add(mul(sub(a1, a0) / dx, t), a0);
    ob = add(mul(sub(b1, b0) / dx, t), b0);
}

// tph.calc_vel_profile.calc_ax_poss: usable longitudinal acceleration at one point.
// accel_forw == true: forward acceleration (machine limit applies, drag opposes);
// false: "decel_backw", the deceleration pass walked backwards (drag helps).
struct Hints { int g, m; };   // last segments of the ggv / machine tables
VP_HD double ax_poss(double vx, double radius, double mu, bool has_mu, bool accel_forw, const Tables &tb, double s,
                     const Params &pr, Hints &h) {
    double ax_max_tires, ay_max_tires;
    interp2(vx, tb.gv, tb.gax, tb.gay, tb.n_ggv, s, ax_max_tires, ay_max_tires, h.g);
    if (has_mu) {
        ax_max_tires = mul(mu, ax_max_tires);
        ay_max_tires = mul(mu, ay_max_tires);
    }
    const double v2 = mul(vx, vx);
    const double ay_used = v2 / radius;
    const double q = ay_used / ay_max_tires;
    const bool lin = (pr.dyn_model_exp == 1.0);
    const double radicand = sub(1.0, lin ? q : pow(q, pr.dyn_model_exp));
    double ax_avail;
    if (radicand > 0.0)
        ax_avail = mul(ax_max_tires, lin ? radicand : pow(radicand, 1.0 / pr.dyn_model_exp));
    else
        ax_avail = 0.0;
    if (accel_forw) {
        const double ax_mach = interp(vx, tb.mv, tb.ma, tb.n_mach, 1.0, h.m);
        if (ax_mach < ax_avail) ax_avail = ax_mach;      // python min(a, b): b if b < a else a
    }
    const double ax_drag = mul(-v2, pr.drag_coeff) / pr.m_veh;
    return accel_forw ? add(ax_avail, ax_drag) : sub(ax_avail, ax_drag);
}

// sqrt(v^2 + 2 a el)
VP_HD double v_next(double v, double a, double el) { return sqrt(add(mul(v, v), mul(mul(2.0, a), el))); }

// Tape policy of profile_thread that records nothing (the forward kernel); TapeRecorder below records what the adjoint
// needs.  The hooks see the values of the forward statements and never change them.
struct NoTape {
    VP_HD void initial(int, int, double, double, double, double, const Tables &, double) const {}
    VP_HD void fwd(int, double, int) const {}
    VP_HD void bwd(int, double, int) const {}
};

// Branch codes of one step of the forward / backward pass (the low byte; the adjoint adds the table segments above it)
constexpr int VP_BR_ACTIVE = 1;     // the step computed a reachable speed
constexpr int VP_BR_TAKEN = 2;      // ... and it won the min against the initial profile
constexpr int VP_BR_LEAVE = 4;      // ... and it exceeded v_max (the phase ends)
constexpr int VP_BR_VTMP = 8;       // backward pass: the one-step correction vtmp won the min against vpn
constexpr int VP_BR_CLAMP = 16;     // set by the adjoint: the radicand of an ax_poss call was clamped to 0
constexpr int VP_BR_MACH = 32;      // set by the adjoint: the machine limit won against the tyre limit
constexpr int VP_BR_CLAMP2 = 64;    // set by the adjoint: the radicand of the correction step's ax_poss was clamped

// One closed-track profile.  kappa/el/mu: this profile's track rows (contiguous, n entries; mu may be null).
// R, EL, MU, V, W: scratch vectors of n entries each (MU unused without mu, W unused without filter).
// vx_out/ax_out [n], t_out [n + 1] may each be null; *laptime always written.  Returns the status code.
// tp: the tape policy (NoTape: the forward alone).
template <class Tape = NoTape>
VP_HD int profile_thread(int n, const double *kappa, const double *el, const double *mu, double scale, double v_max,
                         const Tables &tb, const Params &pr, Strided R, Strided EL, Strided MU, Strided V, Strided W,
                         double *vx_out, double *ax_out, double *t_out, double *laptime, const Tape &tp = Tape()) {
    const bool has_mu = (mu != nullptr);
    // radii = |1 / kappa| (inf where kappa == 0); private coalesced copies of the track rows.
    // All streaming loops below are blocked by VP_UNROLL with the loads of a block issued before its arithmetic
    // (memory-level parallelism: a thread otherwise exposes one L2/HBM round trip per element).
    double mu_sum = 0.0;
    for (int i = 0; i < n; i += VP_UNROLL) {
        double k[VP_UNROLL], e[VP_UNROLL], m[VP_UNROLL];
#pragma unroll
        for (int u = 0; u < VP_UNROLL; ++u)
            if (i + u < n) {
                k[u] = kappa[i + u];
                e[u] = el[i + u];
                m[u] = has_mu ? mu[i + u] : 1.0;
            }
#pragma unroll
        for (int u = 0; u < VP_UNROLL; ++u)
            if (i + u < n) {
                R[i + u] = (k[u] != 0.0) ? fabs(1.0 / k[u]) : (double)INFINITY;
                EL[i + u] = e[u];
                if (has_mu) {
                    MU[i + u] = m[u];
                    mu_sum += m[u];
                }
            }
    }
    const double mu_mean = has_mu ? mu_sum / (double)n : 1.0;

    // ---- initial profile from the lateral limit: v = sqrt(ay_max(v) r), iterated until it moves by < 0.5 % ----------
    double ay_min = mul(tb.gay[0], scale);
    for (int k = 1; k < tb.n_ggv; ++k) {
        const double a = mul(tb.gay[k], scale);
        if (a < ay_min) ay_min = a;
    }
    const double ay_global = mul(mu_mean, ay_min);
    Hints hints{0, 0};
    // first estimate and first fixed-point sweep fused (V is written once instead of twice)
    for (int it = 0; it < 100; ++it) {
        double dmax = 0.0;
        bool any_nan = false;
        for (int i = 0; i < n; i += VP_UNROLL) {
            double vp[VP_UNROLL], r[VP_UNROLL], m[VP_UNROLL];
#pragma unroll
            for (int u = 0; u < VP_UNROLL; ++u)
                if (i + u < n) {
                    r[u] = R[i + u];
                    vp[u] = (it == 0) ? sqrt(mul(ay_global, r[u])) : (double)V[i + u];
                    m[u] = has_mu ? (double)MU[i + u] : 1.0;
                }
#pragma unroll
            for (int u = 0; u < VP_UNROLL; ++u)
                if (i + u < n) {
                    double ay = interp(vp[u], tb.gv, tb.gay, tb.n_ggv, scale, hints.g);
                    if (has_mu) ay = mul(m[u], ay);
                    const double vn = sqrt(mul(ay, r[u]));
                    V[i + u] = vn;
                    tp.initial(it, i + u, r[u], vp[u], ay, vn, tb, scale);
                    const double d = fabs(sub(vn / vp[u], 1.0));
                    if (d != d) any_nan = true;
                    else if (d > dmax) dmax = d;
                }
        }
        if (!any_nan && dmax < 0.005) break;
    }
    // The cut to the top speed (vx_profile[vx_profile > v_max] = v_max) is applied where the forward pass reads the
    // estimate: every index is read (and cut) before the pass stores to it, and it stores to all of them.
#define VP_CLIP(x) (((x) > v_max) ? v_max : (x))

    // ---- forward (acceleration) pass over the doubled lap; the second lap is kept -----------------------------------
    // Sequential form of tph's phase list: a phase starts where the INITIAL profile begins to rise, runs while the
    // reachable speed stays <= v_max, and hands over seamlessly when it reaches the next phase start.
    // Software pipeline: the loads of step j + 1 are issued before the dependent arithmetic of step j (their
    // addresses do not depend on the recurrence; index i1(j + 1) is never the one step j stores to).
    {
        bool active = false;
        const int J = 2 * n - 1;
        double cur = VP_CLIP((double)V[0]), prev0 = cur, dprev = 0.0;
        double nxt0_n = VP_CLIP((double)V[1]), r_n = R[0], e_n = EL[0], m_n = has_mu ? (double)MU[0] : 1.0;
        for (int j = 0; j < J; ++j) {
            const int i1 = (j + 1 < n) ? j + 1 : j + 1 - n;
            const double nxt0 = nxt0_n, r = r_n, e = e_n, m = m_n;
            if (j + 1 < J) {
                const int i0n = (j + 1 < n) ? j + 1 : j + 1 - n;
                const int i1n = (j + 2 < n) ? j + 2 : j + 2 - n;
                nxt0_n = VP_CLIP((double)V[i1n]);                 // every index is read before its (only) store
                r_n = R[i0n];
                e_n = EL[i0n];
                if (has_mu) m_n = MU[i0n];
            }
            const double dj = sub(nxt0, prev0);
            if (dj > 0.0 && (j == 0 || !(dprev > 0.0))) active = true;
            double nxt = nxt0;
            int code = 0;
            if (active) {
                const double a = ax_poss(cur, r, m, has_mu, true, tb, scale, pr, hints);
                const double vpn = v_next(cur, a, e);
                if (vpn < nxt0) nxt = vpn;
                if (vpn > v_max) active = false;
                code = VP_BR_ACTIVE | (vpn < nxt0 ? VP_BR_TAKEN : 0) | (vpn > v_max ? VP_BR_LEAVE : 0);
            }
            tp.fwd(j, cur, code);
            if (j + 1 >= n) V[i1] = nxt;
            cur = nxt;
            prev0 = nxt0;
            dprev = dj;
        }
    }
#undef VP_CLIP

    // ---- backward (deceleration) pass: the same scan on the flipped doubled lap (V, V) ------------------------------
    // flipped index j <-> original index 2n-1-j; tph flips radii, el_lengths and mu with it (el_lengths one-to-one, so
    // the step from original point m to m-1 uses el[m], as in tph).  Point i1 of step j is point i0 of step j + 1, so
    // each step loads one new point, one step ahead.
    {
        const bool slice_upper = pr.decel_slice_upper != 0;
        const int j_end = slice_upper ? n - 1 : 2 * n - 1;
        bool active = false;
        double cur = V[n - 1], prev0 = cur, dprev = 0.0;
        double r0 = R[n - 1], e0 = EL[n - 1], m0 = has_mu ? (double)MU[n - 1] : 1.0;
        const int i1_first = n - 2;
        double v1_n = V[i1_first], r1_n = R[i1_first], e1_n = EL[i1_first], m1_n = has_mu ? (double)MU[i1_first] : 1.0;
        for (int j = 0; j < j_end; ++j) {
            const int i1 = (j + 1 < n) ? n - 2 - j : 2 * n - 2 - j;
            const double nxt0 = v1_n, r1 = r1_n, e1 = e1_n, m1 = m1_n;
            if (j + 1 < j_end) {
                const int i1n = (j + 2 < n) ? n - 3 - j : 2 * n - 3 - j;
                v1_n = V[i1n];
                r1_n = R[i1n];
                e1_n = EL[i1n];
                if (has_mu) m1_n = MU[i1n];
            }
            const double dj = sub(nxt0, prev0);
            if (dj > 0.0 && (j == 0 || !(dprev > 0.0))) active = true;
            double nxt = nxt0;
            int code = 0;
            if (active) {
                const double a = ax_poss(cur, r0, m0, has_mu, false, tb, scale, pr, hints);
                double vpn = v_next(cur, a, e0);
                // the acceleration found at this point need not be feasible at the next one: one correction step
                const double a2 = ax_poss(vpn, r1, m1, has_mu, false, tb, scale, pr, hints);
                const double vtmp = v_next(cur, a2, e0);
                code = VP_BR_ACTIVE | (vtmp < vpn ? VP_BR_VTMP : 0);
                if (vtmp < vpn) vpn = vtmp;
                if (vpn < nxt0) nxt = vpn;
                if (vpn > v_max) active = false;
                code |= (vpn < nxt0 ? VP_BR_TAKEN : 0) | (vpn > v_max ? VP_BR_LEAVE : 0);
            }
            tp.bwd(j, cur, code);
            if (slice_upper || j + 1 >= n) V[i1] = nxt;
            cur = nxt;
            prev0 = nxt0;
            dprev = dj;
            r0 = r1;
            e0 = e1;
            m0 = m1;
        }
    }

    // ---- optional cyclic moving average (tph.conv_filt, closed) ------------------------------------------------------
    const bool filt = pr.filt_window > 1;
    if (filt) {
        const int h = (pr.filt_window - 1) / 2;
        const double wgt = 1.0 / (double)pr.filt_window;
        for (int i = 0; i < n; ++i) {
            double acc = 0.0;
            for (int k = -h; k <= h; ++k) {
                int m = (i + k) % n;
                if (m < 0) m += n;
                acc = add(acc, mul(V[m], wgt));
            }
            W[i] = acc;
        }
    }
    const Strided F = filt ? W : V;

    // ---- calc_ax_profile on the closed profile and calc_t_profile ----------------------------------------------------
    double t = 0.0;
    if (t_out) t_out[0] = 0.0;
    for (int i = 0; i < n; ++i) {
        const double v = F[i];
        const double vn = F[(i + 1 < n) ? i + 1 : 0];
        const double e = EL[i];
        const double ax = sub(mul(vn, vn), mul(v, v)) / mul(2.0, e);
        double ts;
        if (ax != 0.0)
            ts = add(-v, sqrt(add(mul(v, v), mul(mul(2.0, ax), e)))) / ax;
        else
            ts = e / v;
        t = add(t, ts);
        if (vx_out) vx_out[i] = v;
        if (ax_out) ax_out[i] = ax;
        if (t_out) t_out[i + 1] = t;
    }
    *laptime = t;
    return (t == t && fabs(t) < (double)INFINITY) ? VP_STATUS_OK : VP_STATUS_NONFINITE;
}

// ================================================================================================================
// K5d -- vector-Jacobian product of profile_thread (mu == nullptr) with respect to kappa and el (DESIGN.md section 3.12).
// The function differentiated is the one the forward evaluates with every discrete decision frozen as it took it: the
// active flags, the winner of every min, the radicand clamp, the table segments, the v_max clip and the number of
// fixed-point iterations of the initial profile.
// ================================================================================================================

// d/dx of numpy.interp(x, xp, fp * s) on the segment interp takes (the right-hand one at a knot), 0 where interp clamps.
// *seg: that segment, -1 where clamped.
VP_HD double interp_slope(double x, const double *xp, const double *fp, int n, double s, int *seg) {
    if (!(x >= xp[0]) || x >= xp[n - 1]) {
        *seg = -1;
        return 0.0;
    }
    int h = 0;
    const int lo = find_segment(x, xp, n, h);
    *seg = lo;
    return sub(mul(fp[lo + 1], s), mul(fp[lo], s)) / sub(xp[lo + 1], xp[lo]);
}

// What profile_thread<TapeRecorder> leaves for the reverse walk, interleaved like the forward's scratch vectors:
//   V0 [n]      the initial profile (before the v_max clip)
//   D  [n]      dV0/dr, carried in forward mode through the fixed-point iterations (pointwise: one scalar per point)
//   CF, CB [2n] the carried speed `cur` before every step of the forward / backward pass
//   KF, KB [2n] the branch code of every step (VP_BR_*; the reverse walk adds the table segments in bits 8..23)
//   iters [1]   index of the last fixed-point iteration
// keep_codes: the reverse walk writes the codes with the table segments back into KF / KB (for tests that compare the
// decisions at +-delta; the kernel does not)
struct TapeRecorder {
    Strided V0, D, CF, CB, KF, KB, iters;
    bool keep_codes;
    VP_HD void initial(int it, int i, double r, double vp, double ay, double vn, const Tables &tb, double scale) const {
        V0[i] = vn;
        if (i == 0) iters[0] = it;
        if (!(r < (double)INFINITY)) {           // kappa == 0: V0 = inf is clipped, nothing flows back
            D[i] = 0.0;
            return;
        }
        const double dvp = (it == 0) ? vp / (2.0 * r) : (double)D[i];     // it == 0: vp = sqrt(ay_global r)
        int seg;
        const double say = interp_slope(vp, tb.gv, tb.gay, tb.n_ggv, scale, &seg);
        D[i] = (say * dvp * r + ay) / (2.0 * vn);                          // vn = sqrt(ay(vp) r)
    }
    VP_HD void fwd(int j, double cur, int code) const { CF[j] = cur; KF[j] = code; }
    VP_HD void bwd(int j, double cur, int code) const { CB[j] = cur; KB[j] = code; }
};

// Partial derivatives of ax_poss (no mu) at (vx, radius): da/dvx, da/dradius.  Returns the frozen decisions of the call
// as a code: VP_BR_CLAMP, VP_BR_MACH, the ggv segment + 1 in bits 8..15 and (accel_forw) the machine segment + 1 in
// bits 16..23.
VP_HD int ax_poss_lin(double vx, double radius, bool accel_forw, const Tables &tb, double s, const Params &pr,
                      double &da_dv, double &da_dr) {
    int hint = 0, seg_g, seg_m = -1;
    double ax_t, ay_t;
    interp2(vx, tb.gv, tb.gax, tb.gay, tb.n_ggv, s, ax_t, ay_t, hint);
    const double sax = interp_slope(vx, tb.gv, tb.gax, tb.n_ggv, s, &seg_g);
    const double say = interp_slope(vx, tb.gv, tb.gay, tb.n_ggv, s, &seg_g);
    const double q = mul(vx, vx) / radius / ay_t;
    const double dq_dv = (2.0 * vx / radius - q * say) / ay_t, dq_dr = -q / radius;
    const double p = pr.dyn_model_exp;
    const bool lin = (p == 1.0);
    const double radicand = sub(1.0, lin ? q : pow(q, p));
    int code = 0;
    double avail = 0.0, dav_dv = 0.0, dav_dr = 0.0;
    if (radicand > 0.0) {
        if (lin) {
            avail = mul(ax_t, radicand);
            dav_dv = sax * radicand - ax_t * dq_dv;
            dav_dr = -ax_t * dq_dr;
        } else {
            const double rp = pow(radicand, 1.0 / p);
            avail = mul(ax_t, rp);
            // d rp = rp / (p radicand) d radicand,  d radicand = -p q^(p - 1) dq
            const double drp_dq = (q > 0.0) ? -rp / radicand * pow(q, p - 1.0) : 0.0;
            dav_dv = sax * rp + ax_t * drp_dq * dq_dv;
            dav_dr = ax_t * drp_dq * dq_dr;
        }
    } else {
        code |= VP_BR_CLAMP;
    }
    if (accel_forw) {
        int hm = 0;
        const double ax_mach = interp(vx, tb.mv, tb.ma, tb.n_mach, 1.0, hm);
        const double sm = interp_slope(vx, tb.mv, tb.ma, tb.n_mach, 1.0, &seg_m);
        if (ax_mach < avail) {
            code |= VP_BR_MACH;
            dav_dv = sm;
            dav_dr = 0.0;
        }
    }
    const double ddrag = 2.0 * vx * pr.drag_coeff / pr.m_veh;        // |d ax_drag / dvx|
    da_dv = accel_forw ? dav_dv - ddrag : dav_dv + ddrag;
    da_dr = dav_dr;
    return code | ((seg_g + 1) & 0xff) << 8 | ((seg_m + 1) & 0xff) << 16;
}

// Reverse walk of profile_thread<TapeRecorder> (mu == nullptr, so MU is not touched).  Runs the forward again with the
// recorder, then walks its stages backwards: t / ax, filter, backward pass, forward pass, initial profile, r = |1 / kappa|.
// Upstream: g_lap (d L / d laptime) and g_vx [n] (d L / d vx, may be null).  Writes g_kappa [n] and g_el [n] (either may
// be null).  GV, GR, GE: scratch vectors of n entries (adjoints of the speeds, the radii and the lengths).
// Returns the forward's status, or VP_STATUS_NONFINITE for a non-finite gradient; the gradients are zero unless it is 0.
VP_HD int profile_adjoint_thread(int n, const double *kappa, const double *el, double scale, double v_max, const Tables &tb,
                                 const Params &pr, Strided R, Strided EL, Strided V, Strided W, const TapeRecorder &tp,
                                 Strided GV, Strided GR, Strided GE, double g_lap, const double *g_vx, double *g_kappa,
                                 double *g_el, double *laptime) {
    int st = profile_thread(n, kappa, el, nullptr, scale, v_max, tb, pr, R, EL, GR, V, W, nullptr, nullptr, nullptr,
                            laptime, tp);
    const bool filt = pr.filt_window > 1;
    const Strided F = filt ? W : V;
    if (st == VP_STATUS_OK) {
        // ---- t / ax: laptime = sum_i 2 e_i / (v_i + v_i+1), the closed form of calc_t_profile's step times --------
        for (int i = 0; i < n; ++i) {
            GV[i] = g_vx ? g_vx[i] : 0.0;
            GR[i] = 0.0;
            GE[i] = 0.0;
        }
        for (int i = 0; i < n; ++i) {
            const int i1 = (i + 1 < n) ? i + 1 : 0;
            const double s = F[i] + F[i1];
            const double dv = -2.0 * EL[i] / (s * s) * g_lap;
            GV[i] += dv;
            GV[i1] += dv;
            GE[i] += 2.0 / s * g_lap;
        }
        // ---- the cyclic moving average is symmetric: its transpose is itself ------------------------------------
        if (filt) {
            const int h = (pr.filt_window - 1) / 2;
            const double wgt = 1.0 / (double)pr.filt_window;
            for (int i = 0; i < n; ++i) W[i] = GV[i];
            for (int i = 0; i < n; ++i) {
                double acc = 0.0;
                for (int k = -h; k <= h; ++k) {
                    int m = (i + k) % n;
                    if (m < 0) m += n;
                    acc += W[m] * wgt;
                }
                GV[i] = acc;
            }
        }
        // ---- backward pass, steps in reverse.  GV holds the adjoint of the stored speeds (seeds); a step that stored
        // consumes its seed on the first visit, every step passes what the initial speed nxt0 receives into GV[i1].
        {
            const bool slice_upper = pr.decel_slice_upper != 0;
            const int j_end = slice_upper ? n - 1 : 2 * n - 1;
            double gc = 0.0;                                  // adjoint of cur after step j
            for (int j = j_end - 1; j >= 0; --j) {
                const int i1 = (j + 1 < n) ? n - 2 - j : 2 * n - 2 - j;
                const int i0 = (j < n) ? n - 1 - j : 2 * n - 1 - j;
                const bool stored = slice_upper || j + 1 >= n;
                const double g = gc + (stored ? (double)GV[i1] : 0.0);
                int code = (int)tp.KB[j];
                if ((code & VP_BR_ACTIVE) && (code & VP_BR_TAKEN)) {
                    const double cur = tp.CB[j], r0 = R[i0], e0 = EL[i0];
                    Hints hh{0, 0};
                    double da_dv, da_dr;
                    code |= ax_poss_lin(cur, r0, false, tb, scale, pr, da_dv, da_dr) & 0xff3f;
                    const double a = ax_poss(cur, r0, 1.0, false, false, tb, scale, pr, hh);
                    const double vpn = v_next(cur, a, e0);
                    double dc = (cur + e0 * da_dv) / vpn, dr0 = e0 * da_dr / vpn, de0 = a / vpn, dr1 = 0.0;
                    if (code & VP_BR_VTMP) {                     // vtmp = v_next(cur, ax_poss(vpn, r1), e0)
                        const double r1 = R[i1];
                        double db_dv, db_dr;
                        const int c2 = ax_poss_lin(vpn, r1, false, tb, scale, pr, db_dv, db_dr);
                        code |= ((c2 & VP_BR_CLAMP) ? VP_BR_CLAMP2 : 0) | (c2 & 0xff00) << 8;
                        const double a2 = ax_poss(vpn, r1, 1.0, false, false, tb, scale, pr, hh);
                        const double vt = v_next(cur, a2, e0);
                        dc = (cur + e0 * db_dv * dc) / vt;
                        dr0 = e0 * db_dv * dr0 / vt;
                        de0 = (a2 + e0 * db_dv * de0) / vt;
                        dr1 = e0 * db_dr / vt;
                        GR[i1] += g * dr1;
                    }
                    gc = g * dc;
                    GR[i0] += g * dr0;
                    GE[i0] += g * de0;
                    if (stored) GV[i1] = 0.0;
                } else {
                    gc = 0.0;
                    if (stored) GV[i1] = g; else GV[i1] += g;
                }
                if (tp.keep_codes) tp.KB[j] = code;
            }
            GV[n - 1] += gc;                                  // cur of step 0 is V[n - 1]
        }
        // ---- forward pass, steps in reverse (the same bookkeeping; GV becomes the adjoint of the clipped V0) ------
        {
            double gc = 0.0;
            for (int j = 2 * n - 2; j >= 0; --j) {
                const int i1 = (j + 1 < n) ? j + 1 : j + 1 - n;
                const int i0 = (j < n) ? j : j - n;
                const bool stored = j + 1 >= n;
                const double g = gc + (stored ? (double)GV[i1] : 0.0);
                int code = (int)tp.KF[j];
                if ((code & VP_BR_ACTIVE) && (code & VP_BR_TAKEN)) {
                    const double cur = tp.CF[j], r = R[i0], e = EL[i0];
                    Hints hh{0, 0};
                    double da_dv, da_dr;
                    code |= ax_poss_lin(cur, r, true, tb, scale, pr, da_dv, da_dr);
                    const double a = ax_poss(cur, r, 1.0, false, true, tb, scale, pr, hh);
                    const double vpn = v_next(cur, a, e);
                    gc = g * (cur + e * da_dv) / vpn;
                    GR[i0] += g * e * da_dr / vpn;
                    GE[i0] += g * a / vpn;
                    if (stored) GV[i1] = 0.0;
                } else {
                    gc = 0.0;
                    if (stored) GV[i1] = g; else GV[i1] += g;
                }
                if (tp.keep_codes) tp.KF[j] = code;
            }
            GV[0] += gc;                                      // cur of step 0 is the clipped V0[0]
        }
        // ---- initial profile (V0 > v_max was clipped: no dependence), then r = |1 / kappa| ------------------------
        bool finite = true;
        for (int i = 0; i < n; ++i) {
            const double k = kappa[i];
            const double v0 = tp.V0[i];
            const double gr = GR[i] + ((v0 > v_max) ? 0.0 : GV[i] * tp.D[i]);
            const double gk = (k != 0.0) ? gr * (k > 0.0 ? -1.0 : 1.0) / (k * k) : 0.0;
            const double ge = GE[i];
            if (!(fabs(gk) < (double)INFINITY && fabs(ge) < (double)INFINITY)) finite = false;
            GR[i] = gk;
        }
        if (!finite) st = VP_STATUS_NONFINITE;
    }
    for (int i = 0; i < n; ++i) {
        if (g_kappa) g_kappa[i] = (st == VP_STATUS_OK) ? (double)GR[i] : 0.0;
        if (g_el) g_el[i] = (st == VP_STATUS_OK) ? (double)GE[i] : 0.0;
    }
    return st;
}

// tph.calc_ax_profile / tph.calc_t_profile on given profiles (stand-alone forms of the two stages above).
// vx: >= n + 1 entries when ax_in is null (ax is derived from vx[0..n], eq_length_output=False), else >= n.
VP_HD void ax_t_thread(int n, const double *vx, const double *el, const double *ax_in, double t_start, double *ax_out,
                       double *t_out) {
    double t = 0.0;                         // t_profile = insert(cumsum(t_steps), 0, 0.0) + t_start
    if (t_out) t_out[0] = add(0.0, t_start);
    for (int i = 0; i < n; ++i) {
        const double v = vx[i];
        const double e = el[i];
        const double ax = ax_in ? ax_in[i] : sub(mul(vx[i + 1], vx[i + 1]), mul(v, v)) / mul(2.0, e);
        if (ax_out) ax_out[i] = ax;
        if (t_out) {
            double ts;
            if (ax != 0.0)
                ts = add(-v, sqrt(add(mul(v, v), mul(mul(2.0, ax), e)))) / ax;
            else
                ts = e / v;
            t = add(t, ts);
            t_out[i + 1] = add(t, t_start);
        }
    }
}

}  // namespace vp
}  // namespace mc
