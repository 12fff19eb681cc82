"""CPU tests (-m "not gpu") of the shortest-path sensitivities: the oracle's exact active-set VJP (tests/sp_sens.py) against
central finite differences of the oracle's own Goldfarb-Idnani solves, the argument validation of the two C entries
without a GPU, and the host logic of batch.opt_shortest_path_diff against the recording stand-in of the library
(fake_lib.py)."""
import ctypes
import glob
import os
import re

import numpy as np
import pytest
import torch

import sp_sens as S
from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_, build

DELTA = 1e-6
FD_TOL = 1e-6           # measured: <= 5e-8 of max |gradient| on these fixtures


def _grads(ref):
    """kind -> (column getter of an input perturbation, gradient [n]) for the six per-point input kinds."""
    g, gn = ref["grad_reftrack"], ref["grad_normvec"]
    return {"x": ("rt", 0, g[:, 0]), "y": ("rt", 1, g[:, 1]), "w_right": ("rt", 2, g[:, 2]), "w_left": ("rt", 3, g[:, 3]),
            "normal_x": ("nv", 0, gn[:, 0]), "normal_y": ("nv", 1, gn[:, 1])}


@pytest.mark.parametrize("name", ["synth128", "handling", "berlin500_jitter_b"])
def test_oracle_vjp_matches_central_differences_of_the_qp(golden, name):
    g = golden(name)
    rt, nv, wv = g["reftrack"], g["normvec"], float(g["w_veh"])
    n = rt.shape[0]
    rng = np.random.default_rng(17)
    gbar = rng.standard_normal(n)
    ref = S.vjp(rt, nv, wv, gbar)
    assert not S.degenerate(ref, np.abs(ref["f"]).max()).any()
    kinds = _grads(ref)

    def loss(key=None, col=None, d=None, dv=0.0):
        r, v = rt.copy(), nv.copy()
        if key is not None:
            (r if key == "rt" else v)[:, col] += d
        return gbar @ S.solve(r, v, wv + dv)

    def fd(key=None, col=None, d=None, dv=0.0):
        return (loss(key, col, None if d is None else DELTA * d, DELTA * dv)
                - loss(key, col, None if d is None else -DELTA * d, -DELTA * dv)) / (2.0 * DELTA)

    # every kind along a random direction over all points, and w_veh
    for kind, (key, col, grad) in kinds.items():
        d = rng.uniform(-1.0, 1.0, n)
        assert abs(fd(key, col, d) - grad @ d) <= FD_TOL * np.abs(grad).sum(), kind
    assert abs(fd(dv=1.0) - ref["grad_w_veh"]) <= FD_TOL * abs(ref["grad_w_veh"])
    # single coordinates at a point on each bound and a free point
    free = ~(ref["at_ub"] | ref["at_lb"])
    picks = [int(np.flatnonzero(m)[0]) for m in (ref["at_ub"], ref["at_lb"], free) if m.any()]
    for i in picks:
        e = np.zeros(n)
        e[i] = 1.0
        for kind, (key, col, grad) in kinds.items():
            assert abs(fd(key, col, e) - grad[i]) <= FD_TOL * np.abs(grad).max(), (kind, i)
    # the clamped bounds: their widths have no influence; the other width of the point does
    clamped = np.flatnonzero(ref["clamped_r"] | ref["clamped_l"])
    assert clamped.size == (3 if name == "berlin500_jitter_b" else 0)
    for i in clamped:
        e = np.zeros(n)
        e[i] = 1.0
        for kind, mask in (("w_right", ref["clamped_r"]), ("w_left", ref["clamped_l"])):
            key, col, grad = kinds[kind]
            got = fd(key, col, e)
            if mask[i]:
                assert got == 0.0 and grad[i] == 0.0, (kind, i)
            else:
                assert abs(got - grad[i]) <= FD_TOL * np.abs(grad).max(), (kind, i)
    # an inactive bound has no influence
    assert np.all(ref["grad_reftrack"][free, 2:] == 0.0)


def test_sensitivity_entries_validate_their_arguments_without_gpu():
    lib = _lib.load()
    d = ctypes.c_void_p(4096)

    def solve(**kw):
        a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, wv=2.0, wvb=None, alpha=d, st=d, it=None, sens=d, gs=d, ws=None,
                 wsb=0, stream=None)
        a.update(kw)
        return lib.mc_shortest_path_solve_batch_sens(*a.values())

    def adjoint(**kw):
        a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, wv=2.0, wvb=None, alpha=d, sens=d, gs=d, ga=d, grt=d, gnv=None,
                 gwv=None, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_shortest_path_adjoint_batch(*a.values())

    small = lib.mc_shortest_path_workspace_bytes(1, 100) - 8
    for call in (solve, adjoint):
        assert call() == -3 and b"workspace too small" in lib.mc_last_error()
        assert call(ws=d, wsb=small) == -3
        assert call(n_max=2) == -1
        assert call(B=0) == -1
        assert call(sens=None) == -1
        assert call(gs=None) == -1
        assert call(rt=None) == -1 and call(nv=None) == -1 and call(alpha=None) == -1
    assert solve(st=None) == -1
    assert adjoint(ga=None) == -1 and adjoint(grt=None) == -1


def test_opt_shortest_path_diff_calls_both_entries_with_their_declared_arity(fake):
    B, n = 5, 120
    rt = (torch.rand((B, n, 4), dtype=torch.float64) + 3.0).requires_grad_()
    nv = torch.rand((B, n, 2), dtype=torch.float64).requires_grad_()
    wv = torch.full((B,), 2.0, dtype=torch.float64, requires_grad=True)
    res = B_.opt_shortest_path_diff(rt, nv, wv, n_pts=torch.full((B,), n, dtype=torch.int32))
    assert set(res) == {"alpha", "status", "iters", "grad_status"}
    assert res["alpha"].requires_grad and not res["status"].requires_grad
    (res["alpha"] * 2.0).sum().backward()
    assert rt.grad.shape == (B, n, 4) and nv.grad.shape == (B, n, 2) and wv.grad.shape == (B,)
    calls = {name: a for name, a in fake.calls}
    sens_entries = {"mc_shortest_path_solve_batch_sens", "mc_shortest_path_adjoint_batch"}
    assert sens_entries <= set(_lib.EXPORTED_SYMBOLS)
    assert sens_entries <= set(calls)
    fwd, bwd = calls["mc_shortest_path_solve_batch_sens"], calls["mc_shortest_path_adjoint_batch"]
    assert fwd[0] == bwd[0] == B                                       # one unchunked call each way
    assert bwd[12] is not None and bwd[13] is not None                 # grad_normvec, grad_w_veh
    # constants: no optional output is asked for, and the gradient reaches only what requires it
    fake.calls.clear()
    rt2 = rt.detach().clone().requires_grad_()
    B_.opt_shortest_path_diff(rt2, nv.detach(), 2.0)["alpha"].sum().backward()
    bwd = [a for name, a in fake.calls if name == "mc_shortest_path_adjoint_batch"][0]
    assert bwd[12] is None and bwd[13] is None and rt2.grad.shape == (B, n, 4)
    fake.calls.clear()
    nv2 = nv.detach().clone().requires_grad_()
    B_.opt_shortest_path_diff(rt.detach(), nv2, torch.full((B,), 2.0, dtype=torch.float64))["alpha"].sum().backward()
    bwd = [a for name, a in fake.calls if name == "mc_shortest_path_adjoint_batch"][0]
    assert bwd[12] is not None and bwd[13] is None and nv2.grad.shape == (B, n, 2)
    with pytest.raises(RuntimeError, match="same as normvectors"):
        B_.opt_shortest_path_diff(rt, nv[:, :-1], 2.0)


def _kernel_sources():
    return {os.path.basename(p): _lib._c_source(p) for p in sorted(glob.glob(os.path.join(build.CSRC, "*.cu")))}


def test_the_kernel_files_define_each_header_entry_once():
    """Every entry point is defined once, in the extern "C" block of the kernel file that launches its kernels, and the
    defined set is the one the public header declares (the table load() binds); no header of the kernels declares one."""
    where = {}
    for name, src in _kernel_sources().items():
        for block in src.split('extern "C" {')[1:]:
            for sym in re.findall(r"^\w[\w \t*]*?\b(mc_\w+)\s*\([^)]*\)\s*\{", block, flags=re.M):
                where.setdefault(sym, []).append(name)
    assert {sym: files for sym, files in where.items() if len(files) != 1} == {}
    assert sorted(where) == sorted(_lib.EXPORTED_SYMBOLS)
    kernel_headers = glob.glob(os.path.join(build.CSRC, "*.h")) + glob.glob(os.path.join(build.CSRC, "*.cuh"))
    assert kernel_headers
    for path in kernel_headers:
        assert not re.findall(r"\bmc_\w+\s*\(", _lib._c_source(path)), path


def test_no_source_declares_a_function_it_does_not_define():
    """A prototype in a .cu file of a function defined in another one is never compared with its definition by the
    compiler (a drifted type shows only when the library is loaded, swapped arguments of one type never): calls between
    the sources go through the mc_ entries of the public header."""
    prototype = re.compile(r"^[A-Za-z_][\w \t*&:<>,]*?\b(\w+)\s*\([^;{}]*\)\s*;", re.M)
    definition = re.compile(r"\b(\w+)\s*\([^;{}]*\)\s*(?:const\s*)?\{")
    undefined = {}
    for name, src in _kernel_sources().items():
        declared = set(prototype.findall(src)) - {"static_assert"}
        missing = sorted(declared - set(definition.findall(src)))
        if missing:
            undefined[name] = missing
    assert undefined == {}
