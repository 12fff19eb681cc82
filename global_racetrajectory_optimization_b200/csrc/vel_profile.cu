// K5 -- tph.calc_vel_profile + calc_ax_profile + calc_t_profile for batches of closed racelines and batches of
// (ggv scale, top speed) variants per raceline: the velocity-profile stage after the minimum-curvature path and the
// reference's lap-time matrix sweep (main_globaltraj.py:400-421, :442-496; SURVEY.md 8f-1).
//
// Mapping: one thread per profile p = track * V + variant (vel_profile_core.cuh has the arithmetic).  The variants of
// a track are neighbouring threads, so their reads of kappa / el_lengths hit the same sectors (broadcast); all
// multi-pass state lives in the workspace interleaved over the P profiles ([vector][i][p]: coalesced streams).
// The ggv / machine tables (a few dozen rows) are staged in shared memory once per CTA.
// Bound: latency of the sequential fp64 recurrences (div/sqrt chains), hidden by P >> resident threads; the
// streaming traffic is 5 workspace vectors x a handful of passes.
#include "common.cuh"
#include "vel_profile_core.cuh"
#include "../../include/mincurv_b200.h"

namespace mc {

constexpr int VP_TAB_MAX = 256;      // rows of the ggv / ax_max_machines tables held in shared memory
constexpr int VP_VECS = 5;           // R, EL, MU, V, W

size_t vel_profile_ws_doubles(int n_max) { return (size_t)VP_VECS * n_max; }

struct VpArgs {
    int B, V, n_max;
    const int32_t *n_pts;
    const double *kappa, *el, *mu;
    const double *ggv_scale, *v_max_batch;
    double v_max;
    int n_ggv, n_mach;
    const double *ggv, *mach;
    vp::Params pr;
    double *vx, *ax, *t, *laptime;
    int32_t *status;
    double *ws;
};

__global__ void __launch_bounds__(128, 5) vel_profile_kernel(const VpArgs a) {
    __shared__ double s_tab[5 * VP_TAB_MAX];
    double *gv = s_tab, *gax = s_tab + VP_TAB_MAX, *gay = s_tab + 2 * VP_TAB_MAX;
    double *mv = s_tab + 3 * VP_TAB_MAX, *ma = s_tab + 4 * VP_TAB_MAX;
    for (int k = threadIdx.x; k < a.n_ggv; k += blockDim.x) {
        gv[k] = a.ggv[3 * k];
        gax[k] = a.ggv[3 * k + 1];
        gay[k] = a.ggv[3 * k + 2];
    }
    for (int k = threadIdx.x; k < a.n_mach; k += blockDim.x) {
        mv[k] = a.mach[2 * k];
        ma[k] = a.mach[2 * k + 1];
    }
    __syncthreads();
    const size_t P = (size_t)a.B * a.V;
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int b = (int)(p / a.V), v = (int)(p - (size_t)b * a.V);
    const int n = a.n_pts ? a.n_pts[b] : a.n_max;
    if (n < 2 || n > a.n_max) {          // inactive / invalid track: no profile
        a.laptime[p] = 0.0;
        // n == 0: an inactive slot (ok); n < 0: the producer reported an overflow (create_raceline's -needed) -- never a lap time
        if (a.status) a.status[p] = (n == 0) ? vp::VP_STATUS_OK : MC_STATUS_BREAKDOWN;
        return;
    }
    vp::Tables tb{gv, gax, gay, a.n_ggv, mv, ma, a.n_mach};
    const size_t vec = (size_t)a.n_max * P;
    vp::Strided R{a.ws + p, P}, EL{a.ws + vec + p, P}, MU{a.ws + 2 * vec + p, P}, V{a.ws + 3 * vec + p, P},
        W{a.ws + 4 * vec + p, P};
    const size_t row = (size_t)b * a.n_max;
    const double scale = a.ggv_scale ? a.ggv_scale[v] : 1.0;
    const double v_max = a.v_max_batch ? a.v_max_batch[v] : a.v_max;
    double lap;
    const int st = vp::profile_thread(n, a.kappa + row, a.el + row, a.mu ? a.mu + row : nullptr, scale, v_max, tb, a.pr,
                                      R, EL, MU, V, W, a.vx ? a.vx + p * a.n_max : nullptr,
                                      a.ax ? a.ax + p * a.n_max : nullptr, a.t ? a.t + p * ((size_t)a.n_max + 1) : nullptr,
                                      &lap);
    a.laptime[p] = lap;
    if (a.status) a.status[p] = st;
}

int launch_vel_profile(int B, int V, int n_max, const int32_t *n_pts, const double *kappa, const double *el,
                       const double *mu, const double *ggv_scale, const double *v_max_batch, double v_max, int n_ggv,
                       const double *ggv, int n_mach, const double *mach, double dyn_model_exp, double drag_coeff,
                       double m_veh, int filt_window, int decel_slice_upper, double *vx, double *ax, double *t, double *laptime,
                       int32_t *status, double *ws, cudaStream_t stream) {
    if (n_ggv > VP_TAB_MAX || n_mach > VP_TAB_MAX) return -1;
    VpArgs a;
    a.B = B; a.V = V; a.n_max = n_max; a.n_pts = n_pts; a.kappa = kappa; a.el = el; a.mu = mu;
    a.ggv_scale = ggv_scale; a.v_max_batch = v_max_batch; a.v_max = v_max; a.n_ggv = n_ggv; a.n_mach = n_mach;
    a.ggv = ggv; a.mach = mach;
    a.pr.dyn_model_exp = dyn_model_exp; a.pr.drag_coeff = drag_coeff; a.pr.m_veh = m_veh; a.pr.filt_window = filt_window;
    a.pr.decel_slice_upper = decel_slice_upper;
    a.vx = vx; a.ax = ax; a.t = t; a.laptime = laptime; a.status = status; a.ws = ws;
    const size_t P = (size_t)B * V;
    const int threads = 128;
    vel_profile_kernel<<<(unsigned)((P + threads - 1) / threads), threads, 0, stream>>>(a);
    return 0;
}

// ------------------------------------------------------------------------------------------------
// K5d -- the adjoint of K5 for V = 1 (vel_profile_core.cuh: profile_adjoint_thread).  One thread per profile, like K5;
// the forward is run again with the tape recorder, so the entry takes the forward's inputs only.  Workspace per profile:
// the 9 vectors R, EL, V, W, V0, D, GV, GR, GE, the 4 step tapes CF, CB, KF, KB of 2 n_max entries and one scalar,
// interleaved over the profiles ([vector][i][p]) like K5's.
constexpr int VPA_VECS = 17;         // in units of n_max entries

size_t vel_profile_adjoint_ws_doubles(int n_max) { return (size_t)VPA_VECS * n_max + 1; }

struct VpAdjArgs {
    int B, n_max;
    const int32_t *n_pts;
    const double *kappa, *el;
    double v_max;
    int n_ggv, n_mach;
    const double *ggv, *mach;
    vp::Params pr;
    const double *g_lap, *g_vx;
    double *g_kappa, *g_el;
    int32_t *grad_status;
    double *ws;
};

__global__ void __launch_bounds__(128) vel_profile_adjoint_kernel(const VpAdjArgs a) {
    __shared__ double s_tab[5 * VP_TAB_MAX];
    double *gv = s_tab, *gax = s_tab + VP_TAB_MAX, *gay = s_tab + 2 * VP_TAB_MAX;
    double *mv = s_tab + 3 * VP_TAB_MAX, *ma = s_tab + 4 * VP_TAB_MAX;
    for (int k = threadIdx.x; k < a.n_ggv; k += blockDim.x) {
        gv[k] = a.ggv[3 * k];
        gax[k] = a.ggv[3 * k + 1];
        gay[k] = a.ggv[3 * k + 2];
    }
    for (int k = threadIdx.x; k < a.n_mach; k += blockDim.x) {
        mv[k] = a.mach[2 * k];
        ma[k] = a.mach[2 * k + 1];
    }
    __syncthreads();
    const size_t P = (size_t)a.B;
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int n = a.n_pts ? a.n_pts[p] : a.n_max;
    const size_t row = p * a.n_max;
    const bool active = n >= 2 && n <= a.n_max;
    int st = (n == 0) ? vp::VP_STATUS_OK : MC_STATUS_BREAKDOWN;          // an inactive slot: K5's status, zeros
    if (active) {
        vp::Tables tb{gv, gax, gay, a.n_ggv, mv, ma, a.n_mach};
        const size_t vec = (size_t)a.n_max * P;
        auto at = [&](int k) { return vp::Strided{a.ws + k * vec + p, P}; };
        const vp::TapeRecorder tp{at(4), at(5), at(9), at(11), at(13), at(15), vp::Strided{a.ws + VPA_VECS * vec + p, P}, false};
        double lap;
        st = vp::profile_adjoint_thread(n, a.kappa + row, a.el + row, 1.0, a.v_max, tb, a.pr, at(0), at(1), at(2), at(3), tp,
                                        at(6), at(7), at(8), a.g_lap ? a.g_lap[p] : 0.0, a.g_vx ? a.g_vx + row : nullptr,
                                        a.g_kappa ? a.g_kappa + row : nullptr, a.g_el ? a.g_el + row : nullptr, &lap);
    }
    for (int i = active ? n : 0; i < a.n_max; ++i) {
        if (a.g_kappa) a.g_kappa[row + i] = 0.0;
        if (a.g_el) a.g_el[row + i] = 0.0;
    }
    a.grad_status[p] = st;
}

int launch_vel_profile_adjoint(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el, double v_max,
                               int n_ggv, const double *ggv, int n_mach, const double *mach, double dyn_model_exp,
                               double drag_coeff, double m_veh, int filt_window, int decel_slice_upper, const double *g_lap,
                               const double *g_vx, double *g_kappa, double *g_el, int32_t *grad_status, double *ws,
                               cudaStream_t stream) {
    if (n_ggv > VP_TAB_MAX || n_mach > VP_TAB_MAX) return -1;
    VpAdjArgs a;
    a.B = B; a.n_max = n_max; a.n_pts = n_pts; a.kappa = kappa; a.el = el; a.v_max = v_max;
    a.n_ggv = n_ggv; a.n_mach = n_mach; a.ggv = ggv; a.mach = mach;
    a.pr.dyn_model_exp = dyn_model_exp; a.pr.drag_coeff = drag_coeff; a.pr.m_veh = m_veh; a.pr.filt_window = filt_window;
    a.pr.decel_slice_upper = decel_slice_upper;
    a.g_lap = g_lap; a.g_vx = g_vx; a.g_kappa = g_kappa; a.g_el = g_el; a.grad_status = grad_status; a.ws = ws;
    const int threads = 128;
    vel_profile_adjoint_kernel<<<(unsigned)((B + threads - 1) / threads), threads, 0, stream>>>(a);
    return 0;
}

// stand-alone calc_ax_profile / calc_t_profile: one thread per profile, rows contiguous
__global__ void __launch_bounds__(128) ax_t_profile_kernel(int P, int n_max, const int32_t *n_pts, const double *vx,
                                                           int vx_pitch, const double *el, const double *ax_in,
                                                           double t_start, double *ax_out, double *t_out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int n = n_pts ? n_pts[p] : n_max;
    if (n <= 0 || n > n_max) return;
    vp::ax_t_thread(n, vx + (size_t)p * vx_pitch, el + (size_t)p * n_max, ax_in ? ax_in + (size_t)p * n_max : nullptr,
                    t_start, ax_out ? ax_out + (size_t)p * n_max : nullptr,
                    t_out ? t_out + (size_t)p * (n_max + 1) : nullptr);
}

void launch_ax_t_profile(int P, int n_max, const int32_t *n_pts, const double *vx, int vx_pitch, const double *el,
                         const double *ax_in, double t_start, double *ax_out, double *t_out, cudaStream_t stream) {
    const int threads = 128;
    ax_t_profile_kernel<<<(P + threads - 1) / threads, threads, 0, stream>>>(P, n_max, n_pts, vx, vx_pitch, el, ax_in,
                                                                            t_start, ax_out, t_out);
}

}  // namespace mc
