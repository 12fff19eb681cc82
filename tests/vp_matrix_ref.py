"""Host build of the velocity profile and its adjoint for any cell of the lap-time matrix: tests/vp_adj_ref.py's Harness
with the ggv scale as an argument (the host functions take it; vp_adj_ref passes 1), and the matrix adjoint the device
computes, summed over the cells in variant order.  Test infrastructure, not product code."""
import numpy as np

from vp_adj_ref import Harness, IP, _p


class MatrixHarness(Harness):
    def forward(self, kappa, el, ggv, mach, v_max, exp=1.0, filt=0, upper=1, drag_coeff=0.75, m_veh=1200.0, scale=1.0):
        """(status, vx [n], laptime) of profile_thread for one cell (ggv scale, top speed v_max)."""
        n = kappa.size
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        ggv, mach = np.ascontiguousarray(ggv, dtype=float), np.ascontiguousarray(mach, dtype=float)
        vx, ax, t, lap = np.zeros(n), np.zeros(n), np.zeros(n + 1), np.zeros(1)
        st = self.libs[int(upper)].vp_host_profile(n, _p(kappa), _p(el), None, float(scale), float(v_max), ggv.shape[0],
                                                   _p(ggv), mach.shape[0], _p(mach), float(exp), drag_coeff, m_veh,
                                                   int(filt), 1, _p(vx), _p(ax), _p(t), _p(lap))
        return st, vx, float(lap[0])

    def adjoint(self, kappa, el, ggv, mach, v_max, g_lap, g_vx=None, exp=1.0, filt=0, upper=1, drag_coeff=0.75,
                m_veh=1200.0, stride=1, scale=1.0):
        """dict(status, g_kappa, g_el, laptime, codes [4n], iters) of profile_adjoint_thread for one cell."""
        n = kappa.size
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        ggv, mach = np.ascontiguousarray(ggv, dtype=float), np.ascontiguousarray(mach, dtype=float)
        g_vx = None if g_vx is None else np.ascontiguousarray(g_vx, dtype=float)
        gk, ge, lap = np.zeros(n), np.zeros(n), np.zeros(1)
        codes, iters = np.zeros(4 * n, dtype=np.int32), np.zeros(1, dtype=np.int32)
        st = self.libs[int(upper)].vp_adj_host(n, _p(kappa), _p(el), float(scale), float(v_max), ggv.shape[0], _p(ggv),
                                               mach.shape[0], _p(mach), float(exp), drag_coeff, m_veh, int(filt),
                                               int(upper), int(stride), float(g_lap), _p(g_vx), _p(gk), _p(ge), _p(lap),
                                               _p(codes, IP), _p(iters, IP))
        return dict(status=st, g_kappa=gk, g_el=ge, laptime=float(lap[0]), codes=codes, iters=int(iters[0]))

    def matrix_adjoint(self, kappa, el, ggv, mach, ggv_scales, top_speeds, g_lap, **kw):
        """The gradient of sum(g_lap * laptime matrix) [len(top_speeds), len(ggv_scales)] for one track:
        dict(g_kappa, g_el, status [T, S], laptime [T, S], cells: the per-cell adjoint dicts in variant order).  The sum
        runs over the cells in the device's order (top speed major) and skips cells whose status is not 0."""
        g_lap = np.asarray(g_lap, dtype=float).reshape(len(top_speeds), len(ggv_scales))
        gk, ge = np.zeros(kappa.size), np.zeros(kappa.size)
        cells = []
        for t, vm in enumerate(top_speeds):
            for s, sc in enumerate(ggv_scales):
                a = self.adjoint(kappa, el, ggv, mach, vm, float(g_lap[t, s]), scale=sc, **kw)
                if a["status"] == 0:
                    gk += a["g_kappa"]
                    ge += a["g_el"]
                cells.append(a)
        shape = (len(top_speeds), len(ggv_scales))
        return dict(g_kappa=gk, g_el=ge, cells=cells, status=np.array([c["status"] for c in cells]).reshape(shape),
                    laptime=np.array([c["laptime"] for c in cells]).reshape(shape))
