"""CPU tests (-m "not gpu") of the lap-time sensitivities of the velocity profile (DESIGN.md section 3.12):

* the adjoint the CUDA kernel runs (csrc/vel_profile_core.cuh: profile_adjoint_thread), compiled for the host by
  tests/vp_adj_ref.py, against central differences of the host forward, with the tape's branch codes asserted unchanged
  at +-delta (the derivative is that of the forward with its discrete decisions frozen);
* the argument validation of the C entries without a GPU, and that the library exports and load() binds them;
* the host logic of batch.vel_profile_diff against the recording stand-in of the library (fake_lib.py)."""
import ctypes

import numpy as np
import pytest
import torch

from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_
from vp_adj_ref import Harness

# (relative perturbation of every kappa / el, bound on |central difference - adjoint| / |directional derivative|): the
# first delta at which no branch code changes is used.  Measured on these cases: <= 2.3e-6 at 1e-5, <= 3.1e-6 at 1e-6
# (the kinks of the radicand clamp ties below lie inside +-delta)
DELTAS = [(1e-5, 2e-5), (1e-6, 2e-5), (1e-7, 1e-4)]
# The radicand clamp is compared without: where a phase starts, the carried speed is the lateral limit itself, so q = 1
# up to rounding at every delta and along every perturbation (dq = 0 there); which side it rounds to is a tie.
CODE_MASK = ~(16 | 64)
GGV_SPEED = np.array([[0.0, 14.0, 15.0], [20.0, 13.0, 14.0], [40.0, 12.5, 13.0], [60.0, 11.0, 12.0], [90.0, 10.0, 11.0]])
MACH_LOW = np.array([[0.0, 4.0], [30.0, 3.0], [90.0, 1.5]])


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    try:
        return Harness(tmp_path_factory.mktemp("vp_adj"))
    except RuntimeError as e:
        pytest.skip(str(e))


def _case(golden, name):
    v = golden("velprofile")
    ggv, mach = v["ggv"], v["ax_max_machines"]
    return dict(
        flat=dict(ggv=ggv, mach=mach, v_max=70.0),
        speed_dependent_ggv=dict(ggv=GGV_SPEED, mach=mach, v_max=70.0),
        machine_limit=dict(ggv=ggv, mach=MACH_LOW, v_max=70.0),
        exp_1_5=dict(ggv=GGV_SPEED, mach=mach, v_max=70.0, exp=1.5),
        filt_5=dict(ggv=ggv, mach=mach, v_max=70.0, filt=5),
        first_lap_reading=dict(ggv=ggv, mach=mach, v_max=70.0, upper=0),
        at_v_max=dict(ggv=ggv, mach=mach, v_max=30.0),
    )[name]


def _seam(harness, kw, k, el, where):
    """k, el rolled so that the start/finish line lies inside an acceleration phase (where = 1) or a braking zone (-1)."""
    _, vx, _ = harness.forward(k, el, **kw)
    dv = np.roll(vx, -1) - vx
    i = int(np.argmax(dv * where))
    assert dv[i] * where > 0.0
    return np.roll(k, -i), np.roll(el, -i)


CASES = ["flat", "speed_dependent_ggv", "machine_limit", "exp_1_5", "filt_5", "first_lap_reading", "at_v_max"]


@pytest.mark.parametrize("seam", [0, 1, -1])
@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("name", ["handling", "synth333"])
def test_host_adjoint_matches_central_differences_with_frozen_branches(golden, harness, name, case, seam):
    g = golden(name)
    kw = _case(golden, case)
    k, el = g["rl_kappa"].copy(), g["rl_el_lengths"].copy()
    k[20:45] = 0.0                                         # a straight: r = inf, V0 = inf (clipped)
    if seam:
        k, el = _seam(harness, kw, k, el, seam)
    n = k.size
    rng = np.random.default_rng(3)
    g_lap, g_vx = 1.0, 0.01 * rng.standard_normal(n)
    a = harness.adjoint(k, el, g_lap=g_lap, g_vx=g_vx, stride=3, **kw)
    assert a["status"] == 0
    st, vx, lap = harness.forward(k, el, **kw)
    assert st == 0 and a["laptime"] == lap                 # the recording forward is the forward
    assert np.all(a["g_kappa"][k == 0.0] == 0.0) and np.count_nonzero(k == 0.0) == 25
    codes = a["codes"]
    if case == "speed_dependent_ggv":
        assert a["iters"] == 99                            # (kappa == 0: inf / inf never settles the 0.5 % test)
    if case == "machine_limit":
        assert np.any(codes[:2 * n] & 32)
    if case == "at_v_max":
        assert np.any(codes[:2 * n] & 4) and vx.max() <= 30.0

    def loss(kk, ee):
        s, v, t = harness.forward(kk, ee, **kw)
        return g_lap * t + g_vx @ v

    def frozen(delta, dk, de):
        for sgn in (1.0, -1.0):
            b = harness.adjoint(k + sgn * delta * dk, el + sgn * delta * de, g_lap=g_lap, g_vx=g_vx, **kw)
            if not (np.array_equal(b["codes"] & CODE_MASK, codes & CODE_MASK) and b["iters"] == a["iters"]):
                return False
        return True

    for which in ("kappa", "el"):
        u = rng.uniform(-1.0, 1.0, n)
        dk, de = (k * u, 0.0 * el) if which == "kappa" else (0.0 * k, el * u)
        # the largest delta that keeps every decision (speeds can sit on a table knot, q on 1: ties in the forward)
        delta, tol = next(((d, t) for d, t in DELTAS if frozen(d, dk, de)), (None, None))
        assert delta is not None, which
        fd = (loss(k + delta * dk, el + delta * de) - loss(k - delta * dk, el - delta * de)) / (2.0 * delta)
        an = a["g_kappa"] @ dk + a["g_el"] @ de
        assert abs(fd - an) <= tol * abs(an), (which, delta, fd, an)


def test_host_adjoint_with_a_converging_fixed_point_matches_central_differences(golden, harness):
    """No straight: the initial profile's fixed point settles after a few sweeps of a speed-dependent ggv, and the
    iteration count is held at +-delta like every other decision."""
    g = golden("synth333")
    k, el = g["rl_kappa"], g["rl_el_lengths"]
    kw = dict(ggv=GGV_SPEED, mach=golden("velprofile")["ax_max_machines"], v_max=70.0)
    a = harness.adjoint(k, el, g_lap=1.0, **kw)
    assert a["status"] == 0 and 1 <= a["iters"] < 20
    u = np.random.default_rng(9).uniform(-1.0, 1.0, k.size)
    for dk, de in ((k * u, 0.0 * el), (0.0 * k, el * u)):
        for d, tol in DELTAS:
            bs = [harness.adjoint(k + s * d * dk, el + s * d * de, g_lap=1.0, **kw) for s in (1.0, -1.0)]
            if all(np.array_equal(b["codes"] & CODE_MASK, a["codes"] & CODE_MASK) and b["iters"] == a["iters"] for b in bs):
                break
        else:
            raise AssertionError("no delta keeps the decisions")
        fd = (harness.forward(k + d * dk, el + d * de, **kw)[2] - harness.forward(k - d * dk, el - d * de, **kw)[2]) / (2 * d)
        an = a["g_kappa"] @ dk + a["g_el"] @ de
        assert abs(fd - an) <= tol * abs(an), (d, fd, an)


def test_host_adjoint_of_a_non_finite_lap_time_is_zero(golden, harness):
    v, g = golden("velprofile"), golden("handling")
    el = g["rl_el_lengths"].copy()
    el[7] = np.nan
    a = harness.adjoint(g["rl_kappa"], el, v["ggv"], v["ax_max_machines"], 70.0, g_lap=1.0)
    assert a["status"] == 3 and not a["g_kappa"].any() and not a["g_el"].any()


def test_host_adjoint_is_linear_in_the_upstream_gradient_and_independent_of_the_stride(golden, harness):
    v, g = golden("velprofile"), golden("synth333")
    k, el = g["rl_kappa"], g["rl_el_lengths"]
    gv = np.random.default_rng(1).standard_normal(k.size)
    one = harness.adjoint(k, el, v["ggv"], v["ax_max_machines"], 70.0, g_lap=1.0)
    two = harness.adjoint(k, el, v["ggv"], v["ax_max_machines"], 70.0, g_lap=0.0, g_vx=gv, stride=5)
    both = harness.adjoint(k, el, v["ggv"], v["ax_max_machines"], 70.0, g_lap=1.0, g_vx=gv, stride=2)
    scale = np.abs(both["g_kappa"]).max()
    assert np.abs(one["g_kappa"] + two["g_kappa"] - both["g_kappa"]).max() <= 1e-12 * scale
    assert np.array_equal(one["g_el"], harness.adjoint(k, el, v["ggv"], v["ax_max_machines"], 70.0, g_lap=1.0,
                                                       stride=7)["g_el"])


# ------------------------------------------------------------------------------------------------
def test_lap_time_entries_are_exported_and_bound():
    lib = _lib.load()
    assert {"mc_vel_profile_adjoint_workspace_bytes", "mc_vel_profile_adjoint_batch",
            "mc_create_raceline_adjoint_workspace_bytes", "mc_create_raceline_adjoint_batch"} <= set(_lib.EXPORTED_SYMBOLS)
    assert set(_lib._SIGS) == set(_lib.EXPORTED_SYMBOLS)
    for name, (res, args) in _lib._SIGS.items():
        fn = getattr(lib, name)
        assert fn.restype == res and list(fn.argtypes) == args, name


def test_vel_profile_adjoint_validates_its_arguments_without_gpu():
    lib = _lib.load()
    d = ctypes.c_void_p(4096)
    assert lib.mc_vel_profile_adjoint_workspace_bytes(0, 100) == 0
    assert lib.mc_vel_profile_adjoint_workspace_bytes(2, 100) >= 2 * (17 * 100 + 1) * 8

    def adjoint(**kw):
        a = dict(B=1, n_max=100, n_pts=None, k=d, el=d, v_max=70.0, n_ggv=2, ggv=d, n_mach=2, mach=d, exp=1.0, cd=0.75,
                 m=1200.0, fw=0, dsu=1, gl=d, gvx=None, gk=d, ge=d, gs=d, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_vel_profile_adjoint_batch(*a.values())

    assert adjoint() == -3 and b"workspace too small" in lib.mc_last_error()
    assert adjoint(ws=d, wsb=lib.mc_vel_profile_adjoint_workspace_bytes(1, 100) - 8) == -3
    for bad in (dict(B=0), dict(n_max=1), dict(k=None), dict(el=None), dict(ggv=None), dict(mach=None), dict(gs=None),
                dict(n_ggv=0), dict(m=0.0), dict(exp=0.0), dict(v_max=0.0), dict(fw=4), dict(fw=101)):
        assert adjoint(**bad) == -1, bad


# ------------------------------------------------------------------------------------------------
def test_vel_profile_diff_calls_forward_and_adjoint_with_their_declared_arity(fake):
    B, n = 5, 200
    ggv = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
    mach = np.array([[0.0, 5.0], [80.0, 5.0]])
    kap = (torch.rand((B, n), dtype=torch.float64) * 0.02).requires_grad_()
    el = (torch.ones((B, n), dtype=torch.float64) * 2.0).requires_grad_()
    npts = torch.full((B,), n, dtype=torch.int32)
    res = B_.vel_profile_diff(kap, el, ggv, mach, 70.0, 0.75, 1200.0, filt_window=5, n_pts=npts, decel_slice_upper=0)
    assert set(res) == {"laptime", "vx", "ax", "t", "status", "grad_status"}
    assert res["laptime"].shape == (B,) and res["vx"].shape == (B, n) and res["t"].shape == (B, n + 1)
    assert res["laptime"].requires_grad and res["vx"].requires_grad
    assert not res["ax"].requires_grad and not res["status"].requires_grad and not res["grad_status"].requires_grad
    fwd = [a for name, a in fake.calls if name == "mc_vel_profile_batch_ex"]
    assert len(fwd) == 3 and fwd[0][6] == 1                           # V = 1, chunks of 2
    res["laptime"].sum().backward()
    assert kap.grad.shape == (B, n) and el.grad.shape == (B, n)
    bwd = [a for name, a in fake.calls if name == "mc_vel_profile_adjoint_batch"]
    assert [a[0] for a in bwd] == [2, 2, 1]                           # chunked like the forward
    a = bwd[0]
    assert a[5] == 70.0 and a[13] == 5 and a[14] == 0                 # v_max, filt_window, decel_slice_upper
    assert a[15] is not None and a[16] is None                        # grad_laptime only: vx received no gradient
    assert a[17] is not None and a[18] is not None
    # a constant el_lengths: its gradient is not asked for
    fake.calls.clear()
    k2 = kap.detach().clone().requires_grad_()
    r2 = B_.vel_profile_diff(k2, el.detach(), ggv, mach, 70.0, 0.75, 1200.0, n_pts=npts)
    (r2["vx"] * 2.0).sum().backward()
    a = [a for name, a in fake.calls if name == "mc_vel_profile_adjoint_batch"][0]
    assert a[15] is None and a[16] is not None and a[17] is not None and a[18] is None and a[13] == 0
    assert k2.grad.shape == (B, n)


def test_vel_profile_diff_checks_its_arguments(fake):
    kap, el = torch.zeros((2, 50), dtype=torch.float64), torch.ones((2, 50), dtype=torch.float64)
    ggv = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
    mach = np.array([[0.0, 5.0], [80.0, 5.0]])
    with pytest.raises(ValueError, match="one number"):
        B_.vel_profile_diff(kap, el, ggv, mach, [70.0, 60.0], 0.75, 1200.0)
    with pytest.raises(RuntimeError, match="must be odd"):
        B_.vel_profile_diff(kap, el, ggv, mach, 70.0, 0.75, 1200.0, filt_window=4)
    with pytest.raises(RuntimeError, match="entire velocity range"):
        B_.vel_profile_diff(kap, el, ggv, mach, 90.0, 0.75, 1200.0)
    with pytest.raises(RuntimeError, match="three columns"):
        B_.vel_profile_diff(kap, el, ggv[:, :2], mach, 70.0, 0.75, 1200.0)


def test_create_raceline_diff_calls_forward_and_adjoint_with_their_declared_arity(fake):
    B, n = 5, 120
    rt = (torch.rand((B, n, 4), dtype=torch.float64) + 3.0).requires_grad_()
    nv = torch.rand((B, n, 2), dtype=torch.float64).requires_grad_()
    al = torch.zeros((B, n), dtype=torch.float64).requires_grad_()
    npts = torch.full((B,), n, dtype=torch.int32)
    rl = B_.create_raceline_diff(rt, nv, al, 2.0, n_pts=npts, n_out_max=300)
    assert set(rl) == {"raceline_interp", "kappa", "el_lengths_interp", "coeffs_x", "coeffs_y", "spline_lengths", "n_out",
                       "spline_inds", "t_values", "s_interp", "psi"}
    assert rl["kappa"].requires_grad and rl["raceline_interp"].requires_grad and rl["el_lengths_interp"].requires_grad
    assert not rl["psi"].requires_grad and not rl["coeffs_x"].requires_grad
    # (the stand-in writes nothing: n_out stays 0, so only strict=False lets the gradient through -- as zeros)
    with pytest.raises(_lib.MinCurvLibError, match="n_out <= 0"):
        rl["kappa"].sum().backward()
    fake.calls.clear()
    rl = B_.create_raceline_diff(rt, nv, al, 2.0, n_pts=npts, n_out_max=300, strict=False)
    (rl["kappa"].sum() + rl["el_lengths_interp"].sum()).backward()
    assert rt.grad.shape == (B, n, 4) and not rt.grad[:, :, 2:].any() and nv.grad.shape == (B, n, 2) and al.grad.shape == (B, n)
    bwd = [a for name, a in fake.calls if name == "mc_create_raceline_adjoint_batch"]
    assert [a[0] for a in bwd] == [2, 2, 1] and bwd[0][5] == 300                # chunks of 2, n_out_max
    assert bwd[0][12] is None and bwd[0][13] is not None and bwd[0][14] is not None   # no raceline gradient
    assert all(x is not None for x in bwd[0][15:18])
    fake.calls.clear()
    al2 = al.detach().clone().requires_grad_()
    B_.create_raceline_diff(rt.detach(), nv.detach(), al2, 2.0, n_out_max=300, strict=False)["raceline_interp"].sum().backward()
    a = [a for name, a in fake.calls if name == "mc_create_raceline_adjoint_batch"][0]
    assert a[12] is not None and a[16] is None and a[17] is None and al2.grad.shape == (B, n)


def test_create_raceline_adjoint_validates_its_arguments_without_gpu():
    lib = _lib.load()
    d = ctypes.c_void_p(4096)

    def adjoint(**kw):
        a = dict(B=1, n_max=100, n_pts=None, nv=d, al=d, n_out_max=50, cx=d, cy=d, sl=d, n_out=d, si=d, tv=d, gri=None,
                 gk=d, gel=None, ga=d, gref=None, gnv=None, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_create_raceline_adjoint_batch(*a.values())

    assert adjoint() == -3 and b"workspace too small" in lib.mc_last_error()
    for bad in (dict(B=0), dict(n_max=2), dict(n_out_max=0), dict(nv=None), dict(al=None), dict(cx=None), dict(sl=None),
                dict(n_out=None), dict(si=None), dict(tv=None), dict(ga=None)):
        assert adjoint(**bad) == -1, bad
