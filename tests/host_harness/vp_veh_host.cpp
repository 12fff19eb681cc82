// TEST INFRASTRUCTURE: runs the statements of csrc/vel_profile_core.cuh with the tables the vehicle kernels use
// (VehTables: one vehicle's rows read in place from packed row-major tables, stride 3 / 2) on the host, so that the CPU
// test-suite can show them bit-identical to the shared-table form of vp_host.cpp / vp_adj_host.cpp.  Built by
// tests/test_velprofile_vehicles_host.py with g++ into a temporary directory; never part of libmincurv_b200.so.
#include <vector>
#include "../../global_racetrajectory_optimization_b200/csrc/vel_profile_core.cuh"

using namespace mc::vp;

// ggv [.][3] / mach [.][2]: packed tables; this vehicle has rows g0 .. g0 + n_ggv - 1 and m0 .. m0 + n_mach - 1
extern "C" int vp_veh_profile(int n, const double *kappa, const double *el, const double *mu, double scale, double v_max,
                              const double *ggv, int g0, int n_ggv, const double *mach, int m0, int n_mach,
                              double dyn_model_exp, double drag_coeff, double m_veh, int filt_window, int decel_slice_upper,
                              int stride, double *vx, double *ax, double *t, double *laptime) {
    const VehTables tb = row_tables(ggv, g0, n_ggv, mach, m0, n_mach);
    const Params pr{dyn_model_exp, drag_coeff, m_veh, filt_window, decel_slice_upper};
    const size_t P = (size_t)stride, p = (size_t)(stride - 1), vec = (size_t)n * P;
    std::vector<double> ws(5 * vec, -777.0);
    Strided R{ws.data() + p, P}, EL{ws.data() + vec + p, P}, MU{ws.data() + 2 * vec + p, P}, V{ws.data() + 3 * vec + p, P},
        W{ws.data() + 4 * vec + p, P};
    return profile_thread(n, kappa, el, mu, scale, v_max, tb, pr, R, EL, MU, V, W, vx, ax, t, laptime);
}

// as vp_adj_host, with the tables of vp_veh_profile
extern "C" int vp_veh_adjoint(int n, const double *kappa, const double *el, double scale, double v_max, const double *ggv,
                              int g0, int n_ggv, const double *mach, int m0, int n_mach, double dyn_model_exp,
                              double drag_coeff, double m_veh, int filt_window, int decel_slice_upper, int stride,
                              double g_lap, const double *g_vx, double *g_kappa, double *g_el, double *laptime, int *codes,
                              int *iters) {
    const VehTables tb = row_tables(ggv, g0, n_ggv, mach, m0, n_mach);
    const Params pr{dyn_model_exp, drag_coeff, m_veh, filt_window, decel_slice_upper};
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
