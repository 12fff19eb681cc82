"""CPU tests of the velocity profile with a vehicle per track (batch.Vehicles, the vehicles= / veh_id= keywords, the
trailing MC_OPTIONAL2 group of mc_vel_profile_batch_ex and mc_vel_profile_adjoint_batch).

1. The core with the tables the vehicle kernels read (VehTables: one vehicle's rows in place in packed row-major tables,
   tests/host_harness/vp_veh_host.cpp) is bit-identical to the shared-table form (tests/vp_adj_ref.py) on every lap and
   vehicle table of tests/vp_cases.py, forward and adjoint.
2. Vehicles checks and packs its tables on the host, with tph's messages.
3. Every wrapper passes the vehicle arguments in the order of the signature table (tests/fake_lib.py).
4. The header's parsed signatures with and without the trailing group, and the exported symbol count."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import vp_cases as C
from fake_lib import fake  # noqa: F401  (the fixture)
from vp_adj_ref import DP, IP, ROOT, Harness, _p
from global_racetrajectory_optimization_b200 import _lib, batch as B_, build as _build, raceline_refine as R

CASES = C.cases()


# ---- 1. the in-place table accessor against the shared-table form -------------------------------------------------------
class VehHarness:
    def __init__(self, tmpdir):
        cxx = shutil.which("g++")
        if cxx is None:
            pytest.skip("g++ not available")
        so = os.path.join(str(tmpdir), "libvp_veh.so")
        subprocess.check_call([cxx, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-x", "c++", "-std=c++17", "-o", so,
                               os.path.join(ROOT, "tests", "host_harness", "vp_veh_host.cpp")])
        self.lib = ctypes.CDLL(so)
        I, D = ctypes.c_int, ctypes.c_double
        self.lib.vp_veh_profile.restype = I
        self.lib.vp_veh_profile.argtypes = [I, DP, DP, DP, D, D, DP, I, I, DP, I, I, D, D, D, I, I, I, DP, DP, DP, DP]
        self.lib.vp_veh_adjoint.restype = I
        self.lib.vp_veh_adjoint.argtypes = [I, DP, DP, D, D, DP, I, I, DP, I, I, D, D, D, I, I, I, D, DP, DP, DP, DP, IP,
                                            IP]

    @staticmethod
    def _packed(ggv, mach):
        """The case's tables behind another vehicle's rows (as Vehicles packs them): (ggv, g0, mach, m0)."""
        g = np.ascontiguousarray(np.vstack((C.ggv_table(3), ggv)), dtype=float)
        m = np.ascontiguousarray(np.vstack((C.mach_table(5), mach)), dtype=float)
        return g, 3, m, 5

    def profile(self, kappa, el, ggv, mach, v_max, scale=1.0, exp=1.0, filt=0, mu=None, upper=1, drag_coeff=0.75,
                m_veh=1200.0, stride=2):
        n = kappa.size
        g, g0, m, m0 = self._packed(ggv, mach)
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        mu = None if mu is None else np.ascontiguousarray(mu, dtype=float)
        vx, ax, t, lap = np.zeros(n), np.zeros(n), np.zeros(n + 1), np.zeros(1)
        st = self.lib.vp_veh_profile(n, _p(kappa), _p(el), _p(mu), float(scale), float(v_max), _p(g), g0, ggv.shape[0],
                                     _p(m), m0, mach.shape[0], float(exp), drag_coeff, m_veh, int(filt), int(upper),
                                     int(stride), _p(vx), _p(ax), _p(t), _p(lap))
        return dict(status=st, vx=vx, ax=ax, t=t, laptime=float(lap[0]))

    def adjoint(self, kappa, el, ggv, mach, v_max, g_lap, g_vx=None, exp=1.0, filt=0, upper=1, drag_coeff=0.75,
                m_veh=1200.0, stride=2):
        n = kappa.size
        g, g0, m, m0 = self._packed(ggv, mach)
        kappa, el = np.ascontiguousarray(kappa, dtype=float), np.ascontiguousarray(el, dtype=float)
        g_vx = None if g_vx is None else np.ascontiguousarray(g_vx, dtype=float)
        gk, ge, lap = np.zeros(n), np.zeros(n), np.zeros(1)
        codes, iters = np.zeros(4 * n, dtype=np.int32), np.zeros(1, dtype=np.int32)
        st = self.lib.vp_veh_adjoint(n, _p(kappa), _p(el), 1.0, float(v_max), _p(g), g0, ggv.shape[0], _p(m), m0,
                                     mach.shape[0], float(exp), drag_coeff, m_veh, int(filt), int(upper), int(stride),
                                     float(g_lap), _p(g_vx), _p(gk), _p(ge), _p(lap), _p(codes, IP), _p(iters, IP))
        return dict(status=st, g_kappa=gk, g_el=ge, laptime=float(lap[0]), codes=codes, iters=int(iters[0]))


@pytest.fixture(scope="module")
def harnesses(tmp_path_factory):
    d = tmp_path_factory.mktemp("vp_veh_host")
    return Harness(d), VehHarness(d)


def _same(a, b, keys):
    for k in keys:
        assert np.array_equal(a[k], b[k]), k


@pytest.mark.parametrize("upper", [1, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_in_place_tables_match_the_shared_tables_forward(harnesses, name, upper):
    shared, veh = harnesses
    c = CASES[name]
    rng = np.random.default_rng(len(name))
    mu = 0.75 + 0.4 * rng.random(c["kappa"].size)
    for kw in (dict(), dict(exp=1.5), dict(exp=2.0, filt=3), dict(filt=7), dict(mu=mu, scale=0.6),
               dict(drag_coeff=1.1, m_veh=800.0, v_max=0.8 * c["v_max"])):
        kw = dict(dict(v_max=c["v_max"]), **kw)
        a = shared.profile(c["kappa"], c["el"], c["ggv"], c["mach"], upper=upper, **kw)
        b = veh.profile(c["kappa"], c["el"], c["ggv"], c["mach"], upper=upper, **kw)
        assert a["status"] == 0
        _same(a, b, ("status", "vx", "ax", "t", "laptime"))


@pytest.mark.parametrize("upper", [1, 0])
@pytest.mark.parametrize("name", sorted(CASES))
def test_in_place_tables_match_the_shared_tables_adjoint(harnesses, name, upper):
    shared, veh = harnesses
    c = CASES[name]
    g_vx = np.linspace(-0.3, 0.2, c["kappa"].size)
    for kw in (dict(), dict(exp=1.5), dict(filt=5, g_vx=g_vx), dict(drag_coeff=1.1, m_veh=800.0)):
        a = shared.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, upper=upper, **kw)
        b = veh.adjoint(c["kappa"], c["el"], c["ggv"], c["mach"], c["v_max"], 1.0, upper=upper, **kw)
        assert a["status"] == 0
        _same(a, b, ("status", "g_kappa", "g_el", "laptime", "codes", "iters"))


# ---- 2. Vehicles ---------------------------------------------------------------------------------------------------------
def _three():
    g = [C.ggv_table(18), C.ggv_table(2, v1=60.0), C.ggv_table(1, v1=80.0)]
    m = [C.mach_table(18), C.mach_table(3, v1=65.0), C.mach_table(1, v1=80.0)]
    return g, m, [70.0, 55.0, 50.0], [0.75, 0.9, 1.1], [1200.0, 900.0, 750.0]


def test_vehicles_pack_their_rows_back_to_back():
    g, m, vm, dc, mv = _three()
    veh = B_.Vehicles(g, m, vm, dc, mv, device="cpu")
    assert veh.n_veh == 3 and veh.device == torch.device("cpu")
    assert torch.equal(veh.ggv, torch.tensor(np.vstack(g))) and torch.equal(veh.ax_max_machines, torch.tensor(np.vstack(m)))
    assert veh.rows.dtype == torch.int32 and veh.rows.tolist() == [[0, 0], [18, 18], [20, 21], [21, 22]]
    assert veh.par.tolist() == [[70.0, 0.75, 1200.0], [55.0, 0.9, 900.0], [50.0, 1.1, 750.0]]
    one = B_.Vehicles([g[0]], [m[0]], 70.0, 0.75, 1200.0, device="cpu")       # numbers stand for every vehicle
    assert one.par.tolist() == [[70.0, 0.75, 1200.0]]
    tens = B_.Vehicles(g, m, torch.tensor(vm), np.array(dc), tuple(mv), device="cpu")
    assert torch.equal(tens.par, veh.par)


@pytest.mark.parametrize("change, err, match", [
    (dict(ggv=torch.zeros((2, 3))), TypeError, "one table per vehicle"),
    (dict(ggv=[]), ValueError, "one table per vehicle"),
    (dict(ax_max_machines=[C.mach_table(18)]), ValueError, "one table per vehicle"),
    (dict(v_max=[70.0, 55.0]), ValueError, "v_max needs one value per vehicle"),
    (dict(m_veh=[1200.0, 0.0, 750.0]), ValueError, r"m_veh\[1\] must be > 0"),
    (dict(m_veh=[1200.0, 900.0, -1.0]), ValueError, r"m_veh\[2\] must be > 0"),
    (dict(v_max=[70.0, 0.0, 50.0]), ValueError, r"v_max\[1\] must be"),
    (dict(ggv=[C.ggv_table(18), np.zeros((2, 2)), C.ggv_table(1, v1=80.0)]), RuntimeError,
     r"ggv diagram must consist of the three columns \[vx, ax_max, ay_max\]!"),
    (dict(ax_max_machines=[C.mach_table(18), np.zeros((3, 3)), C.mach_table(1, v1=80.0)]), RuntimeError,
     r"ax_max_machines must consist of the two columns \[vx, ax_max_machines\]!"),
    (dict(ggv=[C.ggv_table(257), C.ggv_table(2, v1=60.0), C.ggv_table(1, v1=80.0)]), ValueError, "at most 256 rows"),
    (dict(ax_max_machines=[C.mach_table(18), C.mach_table(300, v1=65.0), C.mach_table(1, v1=80.0)]), ValueError,
     "at most 256 rows"),
    (dict(ggv=[C.ggv_table(18), np.zeros((0, 3)), C.ggv_table(1, v1=80.0)]), ValueError, "vehicle 1 has an empty table"),
    (dict(v_max=[70.0, 61.0, 50.0]), RuntimeError,
     r"ggv has to cover the entire velocity range of the car \(i.e. >= v_max\)!"),
    (dict(v_max=[70.0, 55.0, 81.0]), RuntimeError,
     r"ax_max_machines has to cover the entire velocity range of the car \(i.e. >= v_max\)!"),
])
def test_vehicles_refusals(change, err, match):
    g, m, vm, dc, mv = _three()
    kw = dict(dict(ggv=g, ax_max_machines=m, v_max=vm, drag_coeff=dc, m_veh=mv), **change)
    with pytest.raises(err, match=match):
        B_.Vehicles(device="cpu", **kw)


def test_veh_id_forms_and_refusals():
    veh = B_.Vehicles(*_three(), device="cpu")
    assert veh.veh_id(None, 3, "cpu").tolist() == [0, 1, 2]
    assert veh.veh_id([2, 0, 1, 1], 4, "cpu").dtype == torch.int32
    assert veh.veh_id(np.array([2, 2]), 2, "cpu").tolist() == [2, 2]
    with pytest.raises(ValueError, match="veh_id is required unless there is one vehicle per track"):
        veh.veh_id(None, 4, "cpu")
    with pytest.raises(ValueError, match=r"veh_id must be in 0 \.\. 2"):
        veh.veh_id([0, 3], 2, "cpu")
    with pytest.raises(ValueError, match=r"veh_id must be in 0 \.\. 2"):
        veh.veh_id(torch.tensor([-1, 0]), 2, "cpu")
    with pytest.raises(ValueError, match="one integer per track"):
        veh.veh_id([0.0, 1.0], 2, "cpu")
    with pytest.raises(ValueError, match="one integer per track"):
        veh.veh_id([0, 1, 2], 2, "cpu")


# ---- 3. the wrappers against the signature table ------------------------------------------------------------------------
B, N = 5, 60


def _tracks():
    return torch.rand((B, N), dtype=torch.float64), torch.ones((B, N), dtype=torch.float64)


@pytest.fixture()
def fake_t(fake, monkeypatch):
    """fake, with tensors passed to the stand-in as they are (not as pointers), so that their values can be checked."""
    monkeypatch.setattr(B_, "_ptr", lambda t: t)
    return fake


def _veh_calls(fake, entry):
    return [a for name, a in fake.calls if name == entry]


NGGV = {"mc_vel_profile_batch_ex": 10, "mc_vel_profile_adjoint_batch": 6}        # index of n_ggv in each entry


def _desc(entry, a):
    """The mc_vp_vehicles a call of entry passed in place of ggv (n_ggv = MC_VP_VEHICLES, then NULL machine table)."""
    k = NGGV[entry]
    assert a[k] == B_.VP_VEHICLES == -1 and a[k + 2] == 0 and a[k + 3] is None
    return a[k + 1]._obj


def _check_vehicles(fake, entry, veh, ids, calls=None):
    """Every call of entry passes the descriptor of veh with the chunk's rows of veh_id, and 0 for the scalar drag and
    mass; the chunks cover the tracks in order."""
    calls = _veh_calls(fake, entry) if calls is None else calls
    assert calls
    got = []
    for a in calls:
        d = _desc(entry, a)
        assert (d.n_veh, d.n_ggv, d.n_mach) == (veh.n_veh, 21, 22)
        assert (d.ggv, d.ax_max_machines) == (veh.ggv.data_ptr(), veh.ax_max_machines.data_ptr())
        assert (d.veh_rows, d.veh_par) == (veh.rows.data_ptr(), veh.par.data_ptr())
        vid = d.tensors[1]
        assert d.tensors[0] is veh and vid.dtype == torch.int32
        s = (d.veh_id - vid.data_ptr()) // 4
        got += vid[s:s + a[0]].tolist()
        k = NGGV[entry]
        assert a[k + 5] == 0.0 and a[k + 6] == 0.0                               # drag_coeff, m_veh: not used
    assert got == [int(i) for i in ids]
    return calls


def test_vel_profile_batch_and_diff_pass_the_vehicles(fake_t):
    veh = B_.Vehicles(*_three(), device="cpu")
    kap, el = _tracks()
    ids = [2, 0, 1, 1, 0]
    res = B_.vel_profile_batch(kap, el, vehicles=veh, veh_id=ids)
    assert res["laptime"].shape == (B, 1)
    for a in _check_vehicles(fake_t, "mc_vel_profile_batch_ex", veh, ids):
        assert a[6] == 1 and a[7] is None and a[8] is None                     # V = 1 at the vehicles' own v_max
    fake_t.calls.clear()
    kg = kap.clone().requires_grad_()
    B_.vel_profile_diff(kg, el, vehicles=veh, veh_id=torch.tensor(ids), max_chunk=2)["laptime"].sum().backward()
    assert kg.grad.shape == (B, N)
    calls = _check_vehicles(fake_t, "mc_vel_profile_adjoint_batch", veh, ids)
    assert [a[0] for a in calls] == [2, 2, 1]                                  # max_chunk
    assert all(a[5] == 0.0 for a in calls)                                     # v_max: not used


def test_lap_time_matrices_pass_the_vehicles(fake_t):
    veh = B_.Vehicles(*_three(), device="cpu")
    kap, el = _tracks()
    ids = [1, 1, 0, 2, 0]
    ltm = B_.lap_time_matrix_batch(kap, el, ggv_scales=[0.5, 1.0], top_speeds=[30.0, 40.0, 50.0], vehicles=veh,
                                   veh_id=ids)
    assert ltm.shape == (B, 3, 2)
    for a in _check_vehicles(fake_t, "mc_vel_profile_batch_ex", veh, ids):
        assert a[6] == 6 and a[7].tolist() == [0.5, 1.0] * 3 and a[8].tolist() == [30.0] * 2 + [40.0] * 2 + [50.0] * 2
    fake_t.calls.clear()
    own = B_.lap_time_matrix_batch(kap, el, ggv_scales=[0.5, 0.8, 1.0], vehicles=veh, veh_id=ids)
    assert own.shape == (B, 1, 3)
    for a in _check_vehicles(fake_t, "mc_vel_profile_batch_ex", veh, ids):
        assert a[6] == 3 and a[8] is None                                      # each cell at its vehicle's v_max
    fake_t.calls.clear()
    kg = kap.clone().requires_grad_()
    out = B_.lap_time_matrix_diff(kg, el, ggv_scales=[0.5, 1.0], top_speeds=[30.0, 40.0], vehicles=veh, veh_id=ids)
    out["laptime"].sum().backward()
    assert out["laptime"].shape == (B, 2, 2) and kg.grad.shape == (B, N)
    calls = [a for a in _veh_calls(fake_t, "mc_vel_profile_batch_ex") if a[24] is not None]       # the adjoint launches
    _check_vehicles(fake_t, "mc_vel_profile_batch_ex", veh, ids, calls)


def test_vehicle_keywords_refuse_mixed_and_missing_arguments(fake_t):
    g, m, vm, dc, mv = _three()
    veh = B_.Vehicles(g, m, vm, dc, mv, device="cpu")
    kap, el = _tracks()
    both = "with vehicles= the ggv, ax_max_machines, v_max, drag_coeff and m_veh arguments must be None"
    for kw in (dict(ggv=g[0]), dict(ax_max_machines=m[0]), dict(v_max=70.0), dict(drag_coeff=0.75), dict(m_veh=1.0)):
        with pytest.raises(ValueError, match=both):
            B_.vel_profile_batch(kap, el, vehicles=veh, veh_id=[0] * B, **kw)
    with pytest.raises(ValueError, match=both):
        B_.vel_profile_diff(kap, el, g[0], vehicles=veh, veh_id=[0] * B)
    with pytest.raises(ValueError, match=both):
        B_.lap_time_matrix_batch(kap, el, g[0], m[0], [1.0], [40.0], vehicles=veh, veh_id=[0] * B)
    with pytest.raises(ValueError, match="veh_id is required"):
        B_.vel_profile_batch(kap, el, vehicles=veh)
    with pytest.raises(ValueError, match="veh_id needs vehicles="):
        B_.vel_profile_batch(kap, el, g[0], m[0], 70.0, 0.75, 1200.0, veh_id=[0] * B)
    with pytest.raises(TypeError, match="must be a batch.Vehicles"):
        B_.vel_profile_batch(kap, el, vehicles=object(), veh_id=[0] * B)
    with pytest.raises(TypeError, match="needs ggv, ax_max_machines, v_max, drag_coeff and m_veh"):
        B_.vel_profile_batch(kap, el, g[0], m[0], 70.0)
    with pytest.raises(TypeError, match="needs ggv_scales and top_speeds"):
        B_.lap_time_matrix_batch(kap, el, g[0], m[0], [1.0], None, 0.75, 1200.0)
    with pytest.raises(RuntimeError, match=r"ggv has to cover the entire velocity range"):     # 61 > vehicle 1's 60
        B_.vel_profile_batch(kap, el, v_max=[61.0], ggv_scales=[1.0], vehicles=veh, veh_id=[0] * B)
    with pytest.raises(ValueError, match="one entry per variant"):
        B_.vel_profile_batch(kap, el, v_max=[40.0, 50.0], ggv_scales=[1.0, 0.9, 0.8], vehicles=veh, veh_id=[0] * B)
    with pytest.raises(ValueError, match=r"veh_id must be in 0 \.\. 2"):
        B_.vel_profile_batch(kap, el, vehicles=veh, veh_id=[0, 1, 2, 3, 0])
    assert not fake_t.calls or all(not n.startswith("mc_vel_profile_batch") for n, _ in fake_t.calls)
    one = B_.Vehicles(g, m, vm, dc, mv, device="cpu")
    B_.vel_profile_batch(kap[:3], el[:3], vehicles=one)                        # K == B: track b drives vehicle b
    d = _desc("mc_vel_profile_batch_ex", _veh_calls(fake_t, "mc_vel_profile_batch_ex")[0])
    assert d.tensors[1].tolist() == [0, 1, 2]


def test_lap_time_objective_passes_the_vehicles_through(fake_t):
    veh = B_.Vehicles(*_three(), device="cpu")
    rt = torch.rand((3, 40, 4), dtype=torch.float64) + 3.0
    obj = R.LapTime(rt, torch.rand((3, 40, 2), dtype=torch.float64), None, 2.0,
                    dict(vehicles=veh, veh_id=[2, 2, 0], dyn_model_exp=1.0, filt_window=None))
    assert obj.vp["vehicles"] is veh and obj.vp["veh_id"].tolist() == [2, 2, 0] and "ggv" not in obj.vp
    obj.n_out_max = 60
    obj(torch.zeros((3, 40), dtype=torch.float64), torch.ones(3, dtype=torch.bool), False)
    d = _desc("mc_vel_profile_batch_ex", _veh_calls(fake_t, "mc_vel_profile_batch_ex")[-1])
    assert d.tensors[0] is veh and d.tensors[1].data_ptr() == obj.vp["veh_id"].data_ptr()   # no copy of veh_id per call
    with pytest.raises(ValueError, match="with vehicles= the ggv"):
        R.refine_raceline_batch(rt, torch.rand((3, 40, 2), dtype=torch.float64), torch.zeros((3, 40), dtype=torch.float64),
                                2.0, C.ggv_table(18), vehicles=veh, veh_id=[0, 1, 2])
    with pytest.raises(TypeError, match="needs ggv, ax_max_machines, v_max, drag_coeff and m_veh"):
        R.refine_raceline_batch(rt, torch.rand((3, 40, 2), dtype=torch.float64), torch.zeros((3, 40), dtype=torch.float64),
                                2.0, C.ggv_table(18))


# ---- 4. the header -------------------------------------------------------------------------------------------------------
def test_the_entries_keep_their_signatures_and_the_library_its_47_symbols():
    assert len(_lib.EXPORTED_SYMBOLS) == 47 and len(set(_lib.EXPORTED_SYMBOLS)) == 47
    assert "mc_vp_vehicles" not in _lib.EXPORTED_SYMBOLS
    assert len(_lib._SIGS["mc_vel_profile_batch_ex"][1]) == 31 and len(_lib._SIGS["mc_vel_profile_adjoint_batch"][1]) == 23
    assert len(_lib._SIGS["mc_vel_profile_batch"][1]) == 26
    for entry in ("mc_vel_profile_batch", "mc_vel_profile_batch_ex", "mc_vel_profile_adjoint_batch"):
        assert entry not in _lib._OPTIONAL and entry not in _lib._OPTIONAL2


def test_the_descriptor_is_read_from_the_header(tmp_path):
    assert B_.VP_VEHICLES == -1
    assert [(n, t) for n, t in B_._VpVehiclesDesc._fields_] == (
        [(n, ctypes.c_int) for n in ("n_veh", "n_ggv", "n_mach")]
        + [(n, ctypes.c_void_p) for n in ("ggv", "ax_max_machines", "veh_rows", "veh_par", "veh_id")])
    h = tmp_path / "s.h"
    h.write_text("/* c */\n#define MC_X (-7)\n#define MC_Y 12\ntypedef struct {\n    int a, *b;  // note\n"
                 "    const double *c, d;\n    size_t e;\n} mc_s;\nint mc_f(int n);\n")
    S = _lib.header_struct(str(h), "mc_s")
    assert S._fields_ == [("a", ctypes.c_int), ("b", ctypes.c_void_p), ("c", ctypes.c_void_p), ("d", ctypes.c_double),
                          ("e", ctypes.c_size_t)]
    assert _lib.header_define(str(h), "MC_X") == -7 and _lib.header_define(str(h), "MC_Y") == 12
    assert _lib.header_signatures(str(h)) == {"mc_f": (ctypes.c_int, [ctypes.c_int])}
    with pytest.raises(_lib.MinCurvLibError, match="no typedef struct mc_t"):
        _lib.header_struct(str(h), "mc_t")
    with pytest.raises(_lib.MinCurvLibError, match="no #define MC_Z"):
        _lib.header_define(str(h), "MC_Z")


def test_the_entries_check_the_descriptor_without_gpu():
    """Vehicle mode is validated on the host before any CUDA call: a NULL or incomplete descriptor gives -1, a complete
    one gets as far as the workspace check (-3); the scalar v_max, drag_coeff and m_veh are not checked."""
    lib = _lib.load()
    d = ctypes.c_void_p(4096)

    def desc(**kw):
        f = dict(n_veh=2, n_ggv=4, n_mach=4, ggv=4096, ax_max_machines=4096, veh_rows=4096, veh_par=4096, veh_id=4096)
        f.update(kw)
        return ctypes.byref(B_._VpVehiclesDesc(**f))

    def ex(g, **kw):
        a = dict(B=2, n_max=100, n_pts=None, k=d, el=d, mu=None, V=1, scale=None, vmb=None, v_max=0.0, n_ggv=-1, ggv=g,
                 n_mach=0, mach=None, exp=1.0, cd=0.0, m=0.0, fw=0, dsu=1, vx=None, ax=None, t=None, lap=d, st=None,
                 gl=None, gk=None, ge=None, gs=None, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_vel_profile_batch_ex(*a.values())

    def adj(g):
        return lib.mc_vel_profile_adjoint_batch(2, 100, None, d, d, 0.0, -1, g, 0, None, 1.0, 0.0, 0.0, 0, 1, d, None, d,
                                                d, d, None, 0, None)
    for call in (ex, adj):
        assert call(None) == -1 and b"mc_vp_vehicles" in lib.mc_last_error()
        for bad in (dict(n_veh=0), dict(veh_id=0), dict(veh_rows=0), dict(veh_par=0)):
            assert call(desc(**bad)) == -1, (call.__name__, bad)
        for bad in (dict(n_ggv=0), dict(n_mach=0), dict(ggv=0), dict(ax_max_machines=0)):
            assert call(desc(**bad)) == -1 and b"bad argument" in lib.mc_last_error(), (call.__name__, bad)
        assert call(desc()) == -3 and b"workspace too small" in lib.mc_last_error()
        assert call(desc(n_ggv=300, n_mach=600)) == -3                           # 256 rows per vehicle, not in all
    assert ex(desc(), mach=d, n_mach=3, v_max=70.0, cd=0.75, m=1200.0) == -3     # (the table arguments are replaced)
