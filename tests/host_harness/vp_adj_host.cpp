// TEST INFRASTRUCTURE: runs the velocity-profile adjoint of csrc/vel_profile_core.cuh (the arithmetic of
// vel_profile_adjoint_kernel) on the host, so that the CPU test-suite can check it against central differences of the
// host forward without a GPU.  Exposes the tape's branch codes, so that a test can assert that a finite difference kept
// every discrete decision of the forward.  Built by tests/test_lap_time_grad_host.py with g++ into a temporary
// directory; never part of libmincurv_b200.so.
#include <vector>
#include "../../global_racetrajectory_optimization_b200/csrc/vel_profile_core.cuh"

using namespace mc::vp;

// codes: [4n] -- the forward pass's codes (2n entries, the last unused), then the backward pass's (2n); iters: [1]
extern "C" int vp_adj_host(int n, const double *kappa, const double *el, double scale, double v_max, int n_ggv,
                           const double *ggv, int n_mach, const double *mach, double dyn_model_exp, double drag_coeff,
                           double m_veh, int filt_window, int decel_slice_upper, int stride, double g_lap,
                           const double *g_vx, double *g_kappa, double *g_el, double *laptime, int *codes, int *iters) {
    std::vector<double> gv(n_ggv), gax(n_ggv), gay(n_ggv), mv(n_mach), ma(n_mach);
    for (int k = 0; k < n_ggv; ++k) { gv[k] = ggv[3 * k]; gax[k] = ggv[3 * k + 1]; gay[k] = ggv[3 * k + 2]; }
    for (int k = 0; k < n_mach; ++k) { mv[k] = mach[2 * k]; ma[k] = mach[2 * k + 1]; }
    Tables tb{gv.data(), gax.data(), gay.data(), n_ggv, mv.data(), ma.data(), n_mach};
    Params pr{dyn_model_exp, drag_coeff, m_veh, filt_window, decel_slice_upper};
    // the kernel's addressing: vector k of the profile at ws + k * n * stride + p, element stride `stride`
    const size_t P = (size_t)stride, p = (size_t)(stride - 1), vec = (size_t)n * P;
    std::vector<double> ws(17 * vec + P, -777.0);
    auto at = [&](int k) { return Strided{ws.data() + k * vec + p, P}; };
    TapeRecorder tp{at(4), at(5), at(9), at(11), at(13), at(15), Strided{ws.data() + 17 * vec + p, P}, true};
    for (int j = 0; j < 2 * n; ++j) { tp.KF[j] = 0.0; tp.KB[j] = 0.0; }
    const int st = profile_adjoint_thread(n, kappa, el, scale, v_max, tb, pr, at(0), at(1), at(2), at(3), tp, at(6), at(7),
                                          at(8), g_lap, g_vx, g_kappa, g_el, laptime);
    for (int j = 0; j < 2 * n; ++j) {
        codes[j] = (int)tp.KF[j];
        codes[2 * n + j] = (int)tp.KB[j];
    }
    *iters = (int)tp.iters[0];
    return st;
}
