"""Host build of the velocity-profile stage and its adjoint (csrc/vel_profile_core.cuh compiled with g++ through
tests/host_harness/vp_host.cpp and vp_adj_host.cpp): the reference of the device adjoint (vel_profile_adjoint_kernel
runs the same statements) and the forward whose central differences check it.  Test infrastructure, not product code."""
import ctypes
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DP = ctypes.POINTER(ctypes.c_double)
IP = ctypes.POINTER(ctypes.c_int)


def _p(a, t=DP):
    return a.ctypes.data_as(t) if a is not None else None


class Harness:
    """harness.forward / harness.adjoint for both readings of decel_slice_upper (one build each: the forward harness takes
    the reading as a compile-time default)."""

    def __init__(self, tmpdir):
        cxx = shutil.which("g++")
        if cxx is None:
            raise RuntimeError("g++ not available")
        src = [os.path.join(ROOT, "tests", "host_harness", f) for f in ("vp_host.cpp", "vp_adj_host.cpp")]
        self.libs = {}
        for upper in (0, 1):
            so = os.path.join(str(tmpdir), f"libvp_adj_{upper}.so")
            subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-std=c++17",
                                   f"-DVP_DECEL_SLICE_UPPER={upper}", "-o", so, *src])
            lib = ctypes.CDLL(so)
            lib.vp_host_profile.restype = ctypes.c_int
            lib.vp_host_profile.argtypes = [ctypes.c_int, DP, DP, DP, ctypes.c_double, ctypes.c_double, ctypes.c_int, DP,
                                            ctypes.c_int, DP, ctypes.c_double, ctypes.c_double, ctypes.c_double,
                                            ctypes.c_int, ctypes.c_int, DP, DP, DP, DP]
            lib.vp_adj_host.restype = ctypes.c_int
            lib.vp_adj_host.argtypes = [ctypes.c_int, DP, DP, ctypes.c_double, ctypes.c_double, ctypes.c_int, DP,
                                        ctypes.c_int, DP, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_int,
                                        ctypes.c_int, ctypes.c_int, ctypes.c_double, DP, DP, DP, DP, IP, IP]
            self.libs[upper] = lib

    def forward(self, kappa, el, ggv, mach, v_max, exp=1.0, filt=0, upper=1, drag_coeff=0.75, m_veh=1200.0):
        """(status, vx [n], laptime) of profile_thread."""
        n = kappa.size
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        ggv, mach = np.ascontiguousarray(ggv, dtype=float), np.ascontiguousarray(mach, dtype=float)
        vx, ax, t, lap = np.zeros(n), np.zeros(n), np.zeros(n + 1), np.zeros(1)
        st = self.libs[int(upper)].vp_host_profile(n, _p(kappa), _p(el), None, 1.0, float(v_max), ggv.shape[0], _p(ggv),
                                                   mach.shape[0], _p(mach), float(exp), drag_coeff, m_veh, int(filt), 1,
                                                   _p(vx), _p(ax), _p(t), _p(lap))
        return st, vx, float(lap[0])

    def profile(self, kappa, el, ggv, mach, v_max, scale=1.0, exp=1.0, filt=0, mu=None, upper=1, drag_coeff=0.75,
                m_veh=1200.0, stride=1):
        """dict(status, vx [n], ax [n], t [n + 1], laptime) of profile_thread, with a ggv scale and per-point mu."""
        n = kappa.size
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        ggv, mach = np.ascontiguousarray(ggv, dtype=float), np.ascontiguousarray(mach, dtype=float)
        mu = None if mu is None else np.ascontiguousarray(mu, dtype=float)
        vx, ax, t, lap = np.zeros(n), np.zeros(n), np.zeros(n + 1), np.zeros(1)
        st = self.libs[int(upper)].vp_host_profile(n, _p(kappa), _p(el), _p(mu), float(scale), float(v_max), ggv.shape[0],
                                                   _p(ggv), mach.shape[0], _p(mach), float(exp), drag_coeff, m_veh, int(filt),
                                                   int(stride), _p(vx), _p(ax), _p(t), _p(lap))
        return dict(status=st, vx=vx, ax=ax, t=t, laptime=float(lap[0]))

    def adjoint(self, kappa, el, ggv, mach, v_max, g_lap, g_vx=None, exp=1.0, filt=0, upper=1, drag_coeff=0.75,
                m_veh=1200.0, stride=1):
        """dict(status, g_kappa, g_el, laptime, codes [4n] (forward pass, then backward pass), iters) of
        profile_adjoint_thread."""
        n = kappa.size
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        ggv, mach = np.ascontiguousarray(ggv, dtype=float), np.ascontiguousarray(mach, dtype=float)
        g_vx = None if g_vx is None else np.ascontiguousarray(g_vx, dtype=float)
        gk, ge, lap = np.zeros(n), np.zeros(n), np.zeros(1)
        codes, iters = np.zeros(4 * n, dtype=np.int32), np.zeros(1, dtype=np.int32)
        st = self.libs[int(upper)].vp_adj_host(n, _p(kappa), _p(el), 1.0, float(v_max), ggv.shape[0], _p(ggv),
                                               mach.shape[0], _p(mach), float(exp), drag_coeff, m_veh, int(filt), int(upper),
                                               int(stride), float(g_lap), _p(g_vx), _p(gk), _p(ge), _p(lap), _p(codes, IP),
                                               _p(iters, IP))
        return dict(status=st, g_kappa=gk, g_el=ge, laptime=float(lap[0]), codes=codes, iters=int(iters[0]))
