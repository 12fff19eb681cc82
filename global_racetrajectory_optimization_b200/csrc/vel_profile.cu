// K5 -- tph.calc_vel_profile + calc_ax_profile + calc_t_profile for batches of closed racelines and batches of
// (ggv scale, top speed) variants per raceline: the velocity-profile stage after the minimum-curvature path and the
// reference's lap-time matrix sweep (main_globaltraj.py:400-421, :442-496; SURVEY.md 8f-1).
//
// Mapping: one thread per profile p = track * V + variant (vel_profile_core.cuh has the arithmetic).  The variants of
// a track are neighbouring threads, so their reads of kappa / el_lengths hit the same sectors (broadcast); all
// multi-pass state lives in the workspace interleaved over the P profiles ([vector][i][p]: coalesced streams).
// The ggv / machine tables (a few dozen rows) are staged in shared memory once per CTA.  With a vehicle per track (the
// *_veh kernels) a CTA's profiles may belong to several vehicles, so each thread reads its vehicle's rows in place from
// global memory through the read-only path instead (vp::VehTables); the arithmetic is the same template.
// Bound: latency of the sequential fp64 recurrences (div/sqrt chains), hidden by P >> resident threads; the
// streaming traffic is 5 workspace vectors x a handful of passes.
#include "capi.cuh"
#include "common.cuh"
#include "vel_profile_core.cuh"

namespace mc {

constexpr int VP_TAB_MAX = 256;      // rows of the ggv / ax_max_machines tables held in shared memory
constexpr int VP_VECS = 5;           // R, EL, MU, V, W

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

// Vehicle mode: n_veh vehicles; vehicle k has ggv rows [veh_rows[2k], veh_rows[2k + 2]) and machine rows
// [veh_rows[2k + 1], veh_rows[2k + 3]) of the packed tables (n_ggv / n_mach rows in all), and v_max, drag_coeff, m_veh
// in veh_par[3k .. 3k + 2]; track b drives vehicle veh_id[b].
struct VpVehicles {
    int n_veh;
    const int32_t *veh_id, *veh_rows;
    const double *veh_par;
};

// Track b's vehicle: its tables tb, pr with its drag_coeff and m_veh, and its top speed (unless the variants give one).
// false where veh_id[b] is out of range or the vehicle's rows or scalars are invalid: the track is refused.
__device__ __forceinline__ bool vehicle_of(const VpVehicles &vh, int b, int n_ggv, const double *ggv, int n_mach,
                                           const double *mach, bool own_v_max, vp::VehTables &tb, vp::Params &pr,
                                           double &v_max) {
    const int k = __ldg(vh.veh_id + b);
    if (k < 0 || k >= vh.n_veh) return false;
    const int g0 = __ldg(vh.veh_rows + 2 * k), m0 = __ldg(vh.veh_rows + 2 * k + 1);
    const int ng = __ldg(vh.veh_rows + 2 * k + 2) - g0, nm = __ldg(vh.veh_rows + 2 * k + 3) - m0;
    const double *par = vh.veh_par + 3 * k;
    const double vm = __ldg(par), drag = __ldg(par + 1), mass = __ldg(par + 2);
    if (g0 < 0 || m0 < 0 || ng < 1 || nm < 1 || ng > VP_TAB_MAX || nm > VP_TAB_MAX || g0 + ng > n_ggv ||
        m0 + nm > n_mach || !(mass > 0.0) || (own_v_max && !(vm > 0.0)))
        return false;
    tb = vp::row_tables(ggv, g0, ng, mach, m0, nm);
    pr.drag_coeff = drag;
    pr.m_veh = mass;
    v_max = vm;
    return true;
}

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
    // inactive / invalid track: no profile.  A track shorter than the half-width of the moving-average window is refused
    // too: tph's cyclic conv_filt returns a profile of the wrong length there (the kernel would average over more than one
    // lap).
    if (n < 2 || n > a.n_max || (a.pr.filt_window > 1 && (a.pr.filt_window - 1) / 2 > n)) {
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

// K5 with a vehicle per track: the tables and scalars of vehicle veh_id[b] (vehicle_of); a refused track gets lap
// time 0 and status VP_STATUS_BAD_VEHICLE.
__global__ void __launch_bounds__(128, 5) vel_profile_veh_kernel(const VpArgs a, const VpVehicles vh) {
    const size_t P = (size_t)a.B * a.V;
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int b = (int)(p / a.V), v = (int)(p - (size_t)b * a.V);
    const int n = a.n_pts ? a.n_pts[b] : a.n_max;
    if (n < 2 || n > a.n_max || (a.pr.filt_window > 1 && (a.pr.filt_window - 1) / 2 > n)) {     // as K5
        a.laptime[p] = 0.0;
        if (a.status) a.status[p] = (n == 0) ? vp::VP_STATUS_OK : MC_STATUS_BREAKDOWN;
        return;
    }
    vp::VehTables tb;
    vp::Params pr = a.pr;
    double v_max;
    if (!vehicle_of(vh, b, a.n_ggv, a.ggv, a.n_mach, a.mach, !a.v_max_batch, tb, pr, v_max)) {
        a.laptime[p] = 0.0;
        if (a.status) a.status[p] = vp::VP_STATUS_BAD_VEHICLE;
        return;
    }
    const size_t vec = (size_t)a.n_max * P;
    vp::Strided R{a.ws + p, P}, EL{a.ws + vec + p, P}, MU{a.ws + 2 * vec + p, P}, V{a.ws + 3 * vec + p, P},
        W{a.ws + 4 * vec + p, P};
    const size_t row = (size_t)b * a.n_max;
    const double scale = a.ggv_scale ? a.ggv_scale[v] : 1.0;
    if (a.v_max_batch) v_max = a.v_max_batch[v];
    double lap;
    const int st = vp::profile_thread(n, a.kappa + row, a.el + row, a.mu ? a.mu + row : nullptr, scale, v_max, tb, pr,
                                      R, EL, MU, V, W, a.vx ? a.vx + p * a.n_max : nullptr,
                                      a.ax ? a.ax + p * a.n_max : nullptr, a.t ? a.t + p * ((size_t)a.n_max + 1) : nullptr,
                                      &lap);
    a.laptime[p] = lap;
    if (a.status) a.status[p] = st;
}

// ------------------------------------------------------------------------------------------------
// K5d -- the adjoint of K5 (vel_profile_core.cuh: profile_adjoint_thread) over P = B * V profiles, profile p = track * V +
// variant as in K5.  One thread per profile, like K5; the forward is run again with the tape recorder, so the entries take
// the forward's inputs only.  Workspace per profile: the 9 vectors R, EL, V, W, V0, D, GV, GR, GE, the 4 step tapes CF,
// CB, KF, KB of 2 n_max entries and one scalar, interleaved over the profiles ([vector][i][p]) like K5's.
// V = 1: each thread writes its track's gradient rows.  V > 1: each thread leaves its profile's dL/dkappa, dL/del in its
// GR / GE vectors and vel_profile_adjoint_sum_kernel adds a track's V of them in variant order (no atomics: a track's
// gradient does not depend on the batch it is in).
constexpr int VPA_VECS = 17;         // in units of n_max entries
constexpr int VPA_GR = 7, VPA_GE = 8;

struct VpAdjArgs {
    int B, V, n_max;
    const int32_t *n_pts;
    const double *kappa, *el;
    const double *ggv_scale, *v_max_batch;
    double v_max;
    int n_ggv, n_mach;
    const double *ggv, *mach;
    vp::Params pr;
    const double *g_lap, *g_vx;      // [P], [P][n_max]
    double *g_kappa, *g_el;          // [B][n_max]
    int32_t *grad_status;            // [P]
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
    const size_t P = (size_t)a.B * a.V;
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int b = (int)(p / a.V), v = (int)(p - (size_t)b * a.V);
    const int n = a.n_pts ? a.n_pts[b] : a.n_max;
    const size_t row = (size_t)b * a.n_max;
    const bool active = n >= 2 && n <= a.n_max && !(a.pr.filt_window > 1 && (a.pr.filt_window - 1) / 2 > n);   // as K5
    double *g_kappa = (a.V == 1 && a.g_kappa) ? a.g_kappa + row : nullptr;
    double *g_el = (a.V == 1 && a.g_el) ? a.g_el + row : nullptr;
    int st = (n == 0) ? vp::VP_STATUS_OK : MC_STATUS_BREAKDOWN;          // an inactive slot: K5's status, zeros
    if (active) {
        vp::Tables tb{gv, gax, gay, a.n_ggv, mv, ma, a.n_mach};
        const size_t vec = (size_t)a.n_max * P;
        auto at = [&](int k) { return vp::Strided{a.ws + k * vec + p, P}; };
        const vp::TapeRecorder tp{at(4), at(5), at(9), at(11), at(13), at(15), vp::Strided{a.ws + VPA_VECS * vec + p, P}, false};
        const double scale = a.ggv_scale ? a.ggv_scale[v] : 1.0;
        const double v_max = a.v_max_batch ? a.v_max_batch[v] : a.v_max;
        double lap;
        st = vp::profile_adjoint_thread(n, a.kappa + row, a.el + row, scale, v_max, tb, a.pr, at(0), at(1), at(2), at(3), tp,
                                        at(6), at(VPA_GR), at(VPA_GE), a.g_lap ? a.g_lap[p] : 0.0,
                                        a.g_vx ? a.g_vx + p * a.n_max : nullptr, g_kappa, g_el, &lap);
    }
    for (int i = active ? n : 0; i < a.n_max; ++i) {
        if (g_kappa) g_kappa[i] = 0.0;
        if (g_el) g_el[i] = 0.0;
    }
    a.grad_status[p] = st;
}

// K5d with a vehicle per track (as vel_profile_veh_kernel); a refused track gets zero gradients and grad_status
// VP_STATUS_BAD_VEHICLE.
__global__ void __launch_bounds__(128) vel_profile_adjoint_veh_kernel(const VpAdjArgs a, const VpVehicles vh) {
    const size_t P = (size_t)a.B * a.V;
    const size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const int b = (int)(p / a.V), v = (int)(p - (size_t)b * a.V);
    const int n = a.n_pts ? a.n_pts[b] : a.n_max;
    const size_t row = (size_t)b * a.n_max;
    bool active = n >= 2 && n <= a.n_max && !(a.pr.filt_window > 1 && (a.pr.filt_window - 1) / 2 > n);   // as K5
    double *g_kappa = (a.V == 1 && a.g_kappa) ? a.g_kappa + row : nullptr;
    double *g_el = (a.V == 1 && a.g_el) ? a.g_el + row : nullptr;
    int st = (n == 0) ? vp::VP_STATUS_OK : MC_STATUS_BREAKDOWN;
    vp::VehTables tb;
    vp::Params pr = a.pr;
    double v_max;
    if (active && !vehicle_of(vh, b, a.n_ggv, a.ggv, a.n_mach, a.mach, !a.v_max_batch, tb, pr, v_max)) {
        active = false;
        st = vp::VP_STATUS_BAD_VEHICLE;
    }
    if (active) {
        const size_t vec = (size_t)a.n_max * P;
        auto at = [&](int k) { return vp::Strided{a.ws + k * vec + p, P}; };
        const vp::TapeRecorder tp{at(4), at(5), at(9), at(11), at(13), at(15), vp::Strided{a.ws + VPA_VECS * vec + p, P}, false};
        const double scale = a.ggv_scale ? a.ggv_scale[v] : 1.0;
        if (a.v_max_batch) v_max = a.v_max_batch[v];
        double lap;
        st = vp::profile_adjoint_thread(n, a.kappa + row, a.el + row, scale, v_max, tb, pr, at(0), at(1), at(2), at(3), tp,
                                        at(6), at(VPA_GR), at(VPA_GE), a.g_lap ? a.g_lap[p] : 0.0,
                                        a.g_vx ? a.g_vx + p * a.n_max : nullptr, g_kappa, g_el, &lap);
    }
    for (int i = active ? n : 0; i < a.n_max; ++i) {
        if (g_kappa) g_kappa[i] = 0.0;
        if (g_el) g_el[i] = 0.0;
    }
    a.grad_status[p] = st;
}

// V > 1: g_kappa / g_el [b][i] = the sum over v = 0 .. V - 1 of profile b * V + v's GR / GE [i], skipping the profiles
// whose grad_status is not 0 (their gradient is zero); zeros beyond n_pts[b] and for an inactive track.  One thread per
// (track, point).
__global__ void __launch_bounds__(128) vel_profile_adjoint_sum_kernel(const VpAdjArgs a) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)a.B * a.n_max) return;
    const int b = (int)(idx / a.n_max), i = (int)(idx - (size_t)b * a.n_max);
    const int n = a.n_pts ? a.n_pts[b] : a.n_max;
    const size_t P = (size_t)a.B * a.V, vec = (size_t)a.n_max * P;
    const double *gr = a.ws + VPA_GR * vec + (size_t)i * P, *ge = a.ws + VPA_GE * vec + (size_t)i * P;
    double sk = 0.0, se = 0.0;
    if (n >= 2 && n <= a.n_max && i < n) {
        for (size_t p = (size_t)b * a.V; p < (size_t)(b + 1) * a.V; ++p) {
            if (a.grad_status[p] != vp::VP_STATUS_OK) continue;
            sk += gr[p];
            se += ge[p];
        }
    }
    if (a.g_kappa) a.g_kappa[idx] = sk;
    if (a.g_el) a.g_el[idx] = se;
}

// Vehicle mode of the entries (n_ggv == MC_VP_VEHICLES): desc is a host mc_vp_vehicles.  Fills vh and replaces the
// table arguments by the packed tables it names; false for a NULL or incomplete descriptor.
static bool read_vehicles(const double *desc, VpVehicles &vh, int &n_ggv, const double *&ggv, int &n_mach,
                          const double *&mach) {
    if (!desc) return false;
    const mc_vp_vehicles &d = *reinterpret_cast<const mc_vp_vehicles *>(desc);
    if (d.n_veh < 1 || !d.veh_id || !d.veh_rows || !d.veh_par) return false;
    vh = VpVehicles{d.n_veh, d.veh_id, d.veh_rows, d.veh_par};
    n_ggv = d.n_ggv;
    ggv = d.ggv;
    n_mach = d.n_mach;
    mach = d.ax_max_machines;
    return true;
}

// The launch of both adjoint entries (a.V = 1 for mc_vel_profile_adjoint_batch); vh.veh_id != NULL: a vehicle per track.
static int launch_vel_profile_adjoint(const VpAdjArgs &a, const VpVehicles &vh, cudaStream_t stream) {
    const size_t P = (size_t)a.B * a.V;
    const int threads = 128;
    const unsigned blocks = (unsigned)((P + threads - 1) / threads);
    if (vh.veh_id)
        vel_profile_adjoint_veh_kernel<<<blocks, threads, 0, stream>>>(a, vh);
    else
        vel_profile_adjoint_kernel<<<blocks, threads, 0, stream>>>(a);
    const int rc = check_cuda(vh.veh_id ? "vel_profile_adjoint_veh_kernel" : "vel_profile_adjoint_kernel");
    if (rc != MC_OK || a.V == 1 || (!a.g_kappa && !a.g_el)) return rc;
    const size_t E = (size_t)a.B * a.n_max;
    vel_profile_adjoint_sum_kernel<<<(unsigned)((E + threads - 1) / threads), threads, 0, stream>>>(a);
    return check_cuda("vel_profile_adjoint_sum_kernel");
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

}  // namespace mc

extern "C" {

size_t mc_vel_profile_workspace_bytes(int B, int V, int n_max) {
    if (B <= 0 || V <= 0 || n_max < 2) return 0;
    return align256((size_t)B * V * mc::VP_VECS * n_max * sizeof(double));
}

int mc_vel_profile_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                         const double *mu, int V, const double *ggv_scale, const double *v_max_batch, double v_max,
                         int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines, double dyn_model_exp,
                         double drag_coeff, double m_veh, int filt_window, double *vx, double *ax, double *t,
                         double *laptime, int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    return mc_vel_profile_batch_ex(B, n_max, n_pts, kappa, el_lengths, mu, V, ggv_scale, v_max_batch, v_max, n_ggv, ggv, n_mach,
                                   ax_max_machines, dyn_model_exp, drag_coeff, m_veh, filt_window, MC_VP_DECEL_SLICE_UPPER_DEFAULT,
                                   vx, ax, t, laptime, status, nullptr, nullptr, nullptr, nullptr, workspace, workspace_bytes,
                                   stream);
}

int mc_vel_profile_batch_ex(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                            const double *mu, int V, const double *ggv_scale, const double *v_max_batch, double v_max,
                            int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines, double dyn_model_exp,
                            double drag_coeff, double m_veh, int filt_window, int decel_slice_upper, double *vx, double *ax,
                            double *t, double *laptime, int32_t *status, const double *grad_laptime, double *grad_kappa,
                            double *grad_el_lengths, int32_t *grad_status, void *workspace, size_t workspace_bytes,
                            void *stream) {
    const bool adjoint = grad_laptime != nullptr;
    // vehicle mode: the tables come from the descriptor; the scalar v_max / drag_coeff / m_veh are not used (each
    // vehicle has its own, checked by the kernel)
    mc::VpVehicles vh{};
    const bool veh = n_ggv == MC_VP_VEHICLES;
    if (veh && !mc::read_vehicles(ggv, vh, n_ggv, ggv, n_mach, ax_max_machines))
        return bad("mc_vel_profile_batch: bad mc_vp_vehicles");
    if (B <= 0 || V <= 0 || n_max < 2 || !kappa || !el_lengths || !ggv || !ax_max_machines || (!laptime && !adjoint) ||
        n_ggv < 1 || n_mach < 1 || (!veh && !(m_veh > 0.0)) || !(dyn_model_exp > 0.0) ||
        (!veh && !v_max_batch && !(v_max > 0.0)))
        return bad("mc_vel_profile_batch: bad argument");
    if (adjoint && (mu || !grad_status))
        return bad("mc_vel_profile_batch: the adjoint takes no mu and needs grad_status");
    if (filt_window > 1 && (filt_window % 2 == 0 || filt_window >= n_max))
        return bad("mc_vel_profile_batch: filt_window must be odd (tph: 'Window width of moving average filter must be odd!')");
    if ((size_t)B * V > (size_t)0x7fffffff - 256) return bad("mc_vel_profile_batch: too many profiles in one call");
    if (!workspace || workspace_bytes < (adjoint ? mc_vel_profile_adjoint_workspace_bytes(B * V, n_max)
                                                 : mc_vel_profile_workspace_bytes(B, V, n_max)))
        return small_workspace("mc_vel_profile_batch");
    if (!veh && (n_ggv > mc::VP_TAB_MAX || n_mach > mc::VP_TAB_MAX))
        return bad("mc_vel_profile_batch: ggv / ax_max_machines tables are limited to 256 rows");
    mc::vp::Params pr;
    pr.dyn_model_exp = dyn_model_exp; pr.drag_coeff = drag_coeff; pr.m_veh = m_veh; pr.filt_window = filt_window;
    pr.decel_slice_upper = decel_slice_upper != 0;
    if (adjoint) {
        mc::VpAdjArgs a;
        a.B = B; a.V = V; a.n_max = n_max; a.n_pts = n_pts; a.kappa = kappa; a.el = el_lengths;
        a.ggv_scale = ggv_scale; a.v_max_batch = v_max_batch; a.v_max = v_max;
        a.n_ggv = n_ggv; a.n_mach = n_mach; a.ggv = ggv; a.mach = ax_max_machines; a.pr = pr;
        a.g_lap = grad_laptime; a.g_vx = nullptr; a.g_kappa = grad_kappa; a.g_el = grad_el_lengths;
        a.grad_status = grad_status; a.ws = (double *)workspace;
        return mc::launch_vel_profile_adjoint(a, vh, (cudaStream_t)stream);
    }
    mc::VpArgs a;
    a.B = B; a.V = V; a.n_max = n_max; a.n_pts = n_pts; a.kappa = kappa; a.el = el_lengths; a.mu = mu;
    a.ggv_scale = ggv_scale; a.v_max_batch = v_max_batch; a.v_max = v_max; a.n_ggv = n_ggv; a.n_mach = n_mach;
    a.ggv = ggv; a.mach = ax_max_machines; a.pr = pr;
    a.vx = vx; a.ax = ax; a.t = t; a.laptime = laptime; a.status = status; a.ws = (double *)workspace;
    const size_t P = (size_t)B * V;
    const int threads = 128;
    const unsigned blocks = (unsigned)((P + threads - 1) / threads);
    if (veh) {
        mc::vel_profile_veh_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(a, vh);
        return check_cuda("vel_profile_veh_kernel");
    }
    mc::vel_profile_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(a);
    return check_cuda("vel_profile_kernel");
}

size_t mc_vel_profile_adjoint_workspace_bytes(int B, int n_max) {
    if (B <= 0 || n_max < 2) return 0;
    return align256((size_t)B * ((size_t)mc::VPA_VECS * n_max + 1) * sizeof(double));
}

int mc_vel_profile_adjoint_batch(int B, int n_max, const int32_t *n_pts, const double *kappa, const double *el_lengths,
                                 double v_max, int n_ggv, const double *ggv, int n_mach, const double *ax_max_machines,
                                 double dyn_model_exp, double drag_coeff, double m_veh, int filt_window,
                                 int decel_slice_upper, const double *grad_laptime, const double *grad_vx,
                                 double *grad_kappa, double *grad_el_lengths, int32_t *grad_status,
                                 void *workspace, size_t workspace_bytes, void *stream) {
    mc::VpVehicles vh{};
    const bool veh = n_ggv == MC_VP_VEHICLES;
    if (veh && !mc::read_vehicles(ggv, vh, n_ggv, ggv, n_mach, ax_max_machines))
        return bad("mc_vel_profile_adjoint_batch: bad mc_vp_vehicles");
    if (B <= 0 || n_max < 2 || !kappa || !el_lengths || !ggv || !ax_max_machines || !grad_status || n_ggv < 1 ||
        n_mach < 1 || (!veh && !(m_veh > 0.0)) || !(dyn_model_exp > 0.0) || (!veh && !(v_max > 0.0)))
        return bad("mc_vel_profile_adjoint_batch: bad argument");
    if (filt_window > 1 && (filt_window % 2 == 0 || filt_window >= n_max))
        return bad("mc_vel_profile_adjoint_batch: filt_window must be odd and smaller than n_max");
    if ((size_t)B > (size_t)0x7fffffff - 256) return bad("mc_vel_profile_adjoint_batch: too many profiles in one call");
    if (!workspace || workspace_bytes < mc_vel_profile_adjoint_workspace_bytes(B, n_max))
        return small_workspace("mc_vel_profile_adjoint_batch");
    if (!veh && (n_ggv > mc::VP_TAB_MAX || n_mach > mc::VP_TAB_MAX))
        return bad("mc_vel_profile_adjoint_batch: ggv / ax_max_machines tables are limited to 256 rows");
    mc::VpAdjArgs a;
    a.B = B; a.V = 1; a.n_max = n_max; a.n_pts = n_pts; a.kappa = kappa; a.el = el_lengths;
    a.ggv_scale = nullptr; a.v_max_batch = nullptr; a.v_max = v_max;
    a.n_ggv = n_ggv; a.n_mach = n_mach; a.ggv = ggv; a.mach = ax_max_machines;
    a.pr.dyn_model_exp = dyn_model_exp; a.pr.drag_coeff = drag_coeff; a.pr.m_veh = m_veh; a.pr.filt_window = filt_window;
    a.pr.decel_slice_upper = decel_slice_upper != 0;
    a.g_lap = grad_laptime; a.g_vx = grad_vx; a.g_kappa = grad_kappa; a.g_el = grad_el_lengths; a.grad_status = grad_status;
    a.ws = (double *)workspace;
    return mc::launch_vel_profile_adjoint(a, vh, (cudaStream_t)stream);
}

int mc_calc_ax_t_profile_batch(int P, int n_max, const int32_t *n_pts, const double *vx, int vx_pitch,
                               const double *el_lengths, const double *ax_in, double t_start, double *ax_out,
                               double *t_out, void *stream) {
    if (P <= 0 || n_max < 1 || !vx || !el_lengths || (!ax_out && !t_out) || vx_pitch < n_max + (ax_in ? 0 : 1))
        return bad("mc_calc_ax_t_profile_batch: bad argument");
    const int threads = 128;
    mc::ax_t_profile_kernel<<<(P + threads - 1) / threads, threads, 0, (cudaStream_t)stream>>>(P, n_max, n_pts, vx, vx_pitch,
                                                                                              el_lengths, ax_in, t_start,
                                                                                              ax_out, t_out);
    return check_cuda("ax_t_profile_kernel");
}

}  // extern "C"
