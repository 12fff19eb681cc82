"""CPU tests (-m "not gpu") of the lap-time matrix's sensitivities (batch.lap_time_matrix_diff, the V > 1 form of
vel_profile_adjoint_kernel; DESIGN.md section 3.12):

* the adjoint the kernel runs for one cell (csrc/vel_profile_core.cuh: profile_adjoint_thread with a ggv scale and a
  top speed), compiled for the host by tests/vp_matrix_ref.py, against central differences of the host forward with the
  tape's branch codes held at +-delta, at ggv scales 0.6, 1.0, 1.3 and top speeds that bind and that do not;
* the argument validation of mc_vel_profile_batch_ex's adjoint mode without a GPU;
* the host logic of batch.lap_time_matrix_diff against the recording stand-in of the library (fake_lib.py)."""
import ctypes

import numpy as np
import pytest
import torch

from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_
from vp_matrix_ref import MatrixHarness

# the protocol of test_lap_time_grad_host.py: the first delta at which no branch code changes, and the bound on
# |central difference - adjoint| / |directional derivative| there
DELTAS = [(1e-5, 2e-5), (1e-6, 2e-5), (1e-7, 1e-4)]
CODE_MASK = ~(16 | 64)          # the radicand clamp ties where a phase starts (see test_lap_time_grad_host.py)
VP_BR_LEAVE = 4                 # a step of a pass exceeded v_max: the top speed binds
VEH = dict(drag_coeff=0.75, m_veh=1200.0)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    try:
        return MatrixHarness(tmp_path_factory.mktemp("vp_matrix"))
    except RuntimeError as e:
        pytest.skip(str(e))


def _seam(harness, kw, k, el, where):
    """k, el rolled so that the start/finish line lies inside an acceleration phase (where = 1) or a braking zone (-1)."""
    _, vx, _ = harness.forward(k, el, **kw)
    dv = np.roll(vx, -1) - vx
    i = int(np.argmax(dv * where))
    assert dv[i] * where > 0.0
    return np.roll(k, -i), np.roll(el, -i)


@pytest.mark.parametrize("seam", [0, 1, -1])
@pytest.mark.parametrize("v_max", [30.0, 70.0])
@pytest.mark.parametrize("scale", [0.6, 1.0, 1.3])
@pytest.mark.parametrize("name", ["handling", "synth333"])
def test_host_cell_adjoint_matches_central_differences_with_frozen_branches(golden, harness, name, scale, v_max, seam):
    v, g = golden("velprofile"), golden(name)
    kw = dict(ggv=v["ggv"], mach=v["ax_max_machines"], v_max=v_max, scale=scale, **VEH)
    k, el = g["rl_kappa"].copy(), g["rl_el_lengths"].copy()
    k[20:45] = 0.0                                         # a straight: r = inf, V0 = inf (clipped)
    if seam:
        k, el = _seam(harness, kw, k, el, seam)
    n = k.size
    a = harness.adjoint(k, el, g_lap=1.0, **kw)
    st, vx, lap = harness.forward(k, el, **kw)
    assert a["status"] == 0 and st == 0 and a["laptime"] == lap
    # the top speed binds in a pass at 30 m/s and nowhere at 70 m/s
    assert bool(np.any(a["codes"] & VP_BR_LEAVE)) == (v_max == 30.0) and vx.max() <= v_max
    if scale != 1.0:                                       # the scale reaches the lap time
        assert harness.forward(k, el, **dict(kw, scale=1.0))[2] != lap
    rng = np.random.default_rng(5)

    def frozen(delta, dk, de):
        for sgn in (1.0, -1.0):
            b = harness.adjoint(k + sgn * delta * dk, el + sgn * delta * de, g_lap=1.0, **kw)
            if not (np.array_equal(b["codes"] & CODE_MASK, a["codes"] & CODE_MASK) and b["iters"] == a["iters"]):
                return False
        return True

    for which in ("kappa", "el"):
        u = rng.uniform(-1.0, 1.0, n)
        dk, de = (k * u, 0.0 * el) if which == "kappa" else (0.0 * k, el * u)
        delta, tol = next(((d, t) for d, t in DELTAS if frozen(d, dk, de)), (None, None))
        assert delta is not None, which
        fd = (harness.forward(k + delta * dk, el + delta * de, **kw)[2]
              - harness.forward(k - delta * dk, el - delta * de, **kw)[2]) / (2.0 * delta)
        an = a["g_kappa"] @ dk + a["g_el"] @ de
        assert abs(fd - an) <= tol * abs(an), (which, delta, fd, an)


# ------------------------------------------------------------------------------------------------
def _ex(lib, **kw):
    d = ctypes.c_void_p(4096)
    a = dict(B=2, n_max=100, n_pts=None, k=d, el=d, mu=None, V=3, scale=d, vmb=d, v_max=0.0, n_ggv=2, ggv=d, n_mach=2, mach=d,
             exp=1.0, cd=0.75, m=1200.0, fw=0, dsu=1, vx=None, ax=None, t=None, lap=None, st=None, gl=d, gk=d, ge=d, gs=d,
             ws=None, wsb=0, stream=None)
    a.update(kw)
    return lib.mc_vel_profile_batch_ex(*a.values())


def test_the_extended_ex_entry_validates_its_adjoint_arguments_without_gpu():
    lib = _lib.load()
    assert len(_lib._SIGS["mc_vel_profile_batch_ex"][1]) == 31
    d = ctypes.c_void_p(4096)
    adj = lib.mc_vel_profile_adjoint_workspace_bytes(2 * 3, 100)
    fwd = lib.mc_vel_profile_workspace_bytes(2, 3, 100)
    assert fwd < adj
    # the adjoint mode needs no forward outputs: with a too small workspace it gets as far as the size check
    assert _ex(lib) == -3 and b"workspace too small" in lib.mc_last_error()
    assert _ex(lib, ws=d, wsb=fwd) == -3                                     # the forward's workspace is not enough
    assert _ex(lib, ws=d, wsb=adj - 8) == -3
    assert _ex(lib, mu=d) == -1 and b"mu" in lib.mc_last_error()            # no mu in the adjoint
    assert _ex(lib, gs=None) == -1 and b"grad_status" in lib.mc_last_error()
    for bad in (dict(B=0), dict(V=0), dict(n_max=1), dict(k=None), dict(el=None), dict(ggv=None), dict(mach=None),
                dict(n_ggv=0), dict(m=0.0), dict(exp=0.0), dict(vmb=None), dict(fw=4), dict(fw=101), dict(n_ggv=257)):
        assert _ex(lib, ws=d, wsb=adj, **bad) == -1, bad
    # without seeds the call is the forward: it needs laptime, and the forward's workspace suffices
    assert _ex(lib, gl=None) == -1
    assert _ex(lib, gl=None, lap=d, wsb=fwd - 8, ws=d) == -3


# ------------------------------------------------------------------------------------------------
GGV = np.array([[0.0, 12.0, 12.0], [80.0, 12.0, 12.0]])
MACH = np.array([[0.0, 5.0], [80.0, 5.0]])


def _doubles(ptr, count):
    return list((ctypes.c_double * count).from_address(ptr.value))


def test_lap_time_matrix_diff_calls_ex_forward_and_backward_with_its_declared_arity(fake):
    B, n = 5, 200
    scales, speeds = [0.5, 0.75, 1.0], [30.0, 40.0]
    V = 6
    kap = (torch.rand((B, n), dtype=torch.float64) * 0.02).requires_grad_()
    el = (torch.ones((B, n), dtype=torch.float64) * 2.0).requires_grad_()
    npts = torch.full((B,), n, dtype=torch.int32)
    res = B_.lap_time_matrix_diff(kap, el, GGV, MACH, scales, speeds, 0.75, 1200.0, filt_window=5, n_pts=npts,
                                  decel_slice_upper=0)
    assert set(res) == {"laptime", "status", "grad_status"}
    assert all(res[k].shape == (B, 2, 3) for k in res)
    assert res["laptime"].requires_grad and not res["status"].requires_grad and not res["grad_status"].requires_grad
    fwd = [a for name, a in fake.calls if name == "mc_vel_profile_batch_ex"]
    assert [a[0] for a in fwd] == [2, 2, 1] and all(a[6] == V for a in fwd)             # chunks of 2 tracks, V = T * S
    assert all(x is None for x in fwd[0][24:28])                                        # no seeds: the forward
    # the variant order of lap_time_matrix_batch (v = top-speed index * S + scale index), read while autograd holds it
    assert _doubles(fwd[0][7], V) == [0.5, 0.75, 1.0] * 2 and _doubles(fwd[0][8], V) == [30.0] * 3 + [40.0] * 3
    fake.calls.clear()
    w = torch.arange(1.0, B * V + 1.0, dtype=torch.float64).reshape(B, 2, 3)
    (res["laptime"] * w).sum().backward()
    assert kap.grad.shape == (B, n) and el.grad.shape == (B, n)
    bwd = [a for name, a in fake.calls if name == "mc_vel_profile_batch_ex"]
    assert [a[0] for a in bwd] == [2, 2, 1] and all(a[6] == V for a in bwd)             # chunked like the forward
    a = bwd[0]
    assert a[5] is None and a[17] == 5 and a[18] == 0                                   # no mu, filt_window, dsu
    assert all(x is None for x in a[19:24])                                             # no forward outputs
    assert all(x is not None for x in a[24:28])                                         # seeds, both gradients, status
    assert a[7].value == fwd[0][7].value and a[8].value == fwd[0][8].value            # the forward's variants
    # per-track rows: the seeds and grad_status of chunk 2 start 2 tracks (2 V cells) after chunk 1's
    assert bwd[1][24].value - a[24].value == 2 * V * 8 and bwd[1][27].value - a[27].value == 2 * V * 4
    assert bwd[1][25].value - a[25].value == 2 * n * 8
    ws = [x for name, x in fake.calls if name == "mc_vel_profile_adjoint_workspace_bytes"]
    assert ws[-1] == (2 * V, n)                                                         # the tape of a chunk's profiles
    # a constant el_lengths: its gradient is not asked for
    fake.calls.clear()
    k2 = kap.detach().clone().requires_grad_()
    B_.lap_time_matrix_diff(k2, el.detach(), GGV, MACH, scales, speeds, 0.75, 1200.0)["laptime"].sum().backward()
    a = [a for name, a in fake.calls if name == "mc_vel_profile_batch_ex"][-1]
    assert a[24] is not None and a[25] is not None and a[26] is None and a[27] is not None and a[17] == 0
    assert k2.grad.shape == (B, n)


def test_lap_time_matrix_diff_without_a_differentiable_input_and_its_checks(fake):
    kap, el = torch.zeros((2, 50), dtype=torch.float64), torch.ones((2, 50), dtype=torch.float64)
    res = B_.lap_time_matrix_diff(kap, el, GGV, MACH, [1.0], [30.0, 40.0], 0.75, 1200.0)
    assert res["laptime"].shape == (2, 2, 1) and not res["laptime"].requires_grad
    with pytest.raises(RuntimeError, match="must be odd"):
        B_.lap_time_matrix_diff(kap, el, GGV, MACH, [1.0], [30.0], 0.75, 1200.0, filt_window=4)
    with pytest.raises(RuntimeError, match="entire velocity range"):
        B_.lap_time_matrix_diff(kap, el, GGV, MACH, [1.0], [30.0, 90.0], 0.75, 1200.0)
    with pytest.raises(RuntimeError, match="three columns"):
        B_.lap_time_matrix_diff(kap, el, GGV[:, :2], MACH, [1.0], [30.0], 0.75, 1200.0)
