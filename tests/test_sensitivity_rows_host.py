"""CPU tests (-m "not gpu") of the width sensitivities with the curvature rows: the oracle's exact active-set VJP with
rows (tests/qp_sens_rows.py) against central finite differences of the oracle's own Goldfarb-Idnani solves, the argument
validation of the two C entries without a GPU, and the wiring of batch.opt_min_curv_diff(curvature_rows=...) against
the recording stand-in of the library (fake_lib.py)."""
import ctypes

import numpy as np
import pytest
import torch

import qp_sens_rows as QR
from fake_lib import fake, FakeLib  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_


@pytest.mark.parametrize("name", ["synth160_kappa", "synth333_kappa"])
def test_oracle_vjp_with_rows_matches_central_differences_of_the_qp(golden, name):
    g = golden(name)
    rt, wv, kb = g["reftrack"], float(g["w_veh"]), float(g["kappa_bound"])
    d = QR.qp_data(rt, g["normvec"], kb, wv)
    n = rt.shape[0]
    rng = np.random.default_rng(21)
    gbar = rng.standard_normal(n)
    ref = QR.width_vjp_rows(d, rt, wv, kb, gbar)
    assert (ref["row_hi"] | ref["row_lo"]).any() and (ref["at_ub"] | ref["at_lb"]).any()
    assert np.allclose(ref["alpha"], g["alpha_mincurv"], rtol=0, atol=1e-6)
    delta = 1e-6

    def loss(rt_, wv_):
        out = QR.width_vjp_rows(d, rt_, wv_, kb, gbar)
        # the perturbation keeps the active set: the solution is affine in the bounds on it
        for k in ("at_ub", "at_lb", "row_hi", "row_lo"):
            assert np.array_equal(out[k], ref[k]), k
        return gbar @ out["alpha"]

    for k in range(3):
        dw = rng.uniform(-1.0, 1.0, (n, 2))
        dv = rng.uniform(-1.0, 1.0)
        rp, rm = rt.copy(), rt.copy()
        rp[:, 2:] += delta * dw
        rm[:, 2:] -= delta * dw
        fd = (loss(rp, wv + delta * dv) - loss(rm, wv - delta * dv)) / (2 * delta)
        ad = ref["grad_w_right"] @ dw[:, 0] + ref["grad_w_left"] @ dw[:, 1] + ref["grad_w_veh"] * dv
        assert abs(fd - ad) <= 1e-6 * abs(ad), (k, fd, ad)
    # single coordinates: a bound active together with a row, if there is one, else the first active bound
    box = ref["at_ub"] | ref["at_lb"]
    both = np.flatnonzero(box & (ref["row_hi"] | ref["row_lo"]))
    i = int(both[0]) if both.size else int(np.flatnonzero(box)[0])
    for col, key in ((2, "grad_w_right"), (3, "grad_w_left")):
        rp, rm = rt.copy(), rt.copy()
        rp[i, col] += delta
        rm[i, col] -= delta
        fd = (loss(rp, wv) - loss(rm, wv)) / (2 * delta)
        assert abs(fd - ref[key][i]) <= 1e-6 * np.abs(ref[key]).max(), (i, key)
    # an inactive bound has no influence
    free = np.flatnonzero(~box)
    assert np.all(ref["grad_w_right"][free] == 0.0) and np.all(ref["grad_w_left"][free] == 0.0)


def test_curvature_row_arguments_are_validated_without_gpu():
    """The full signatures with the curvature-row arguments: they pass the checks together and are refused apart; a call
    that leaves them out (the signature before they were added) is the call with NULL / 0."""
    lib = _lib.load()
    d = ctypes.c_void_p(4096)

    def solve(**kw):
        a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, h=d, kb=0.12, wv=2.0, wvb=None, fs=2.0, cid=None, alpha=d, cerr=d,
                 kmax=None, st=d, it=None, sens=d, gs=d, srows=None, nrows=None, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_mincurv_solve_batch_sens(*a.values())

    def adjoint(**kw):
        a = dict(B=1, n_max=100, n_pts=None, rt=d, nv=d, h=d, wv=2.0, wvb=None, fs=2.0, cid=None, sens=d, gs=d, ga=d, gwr=d,
                 gwl=d, gwv=d, srows=None, nrows=None, schur=None, cap=0, ws=None, wsb=0, stream=None)
        a.update(kw)
        return lib.mc_mincurv_adjoint_batch(*a.values())

    for call in (solve, adjoint):
        assert call() == -3 and b"workspace too small" in lib.mc_last_error()
        assert call(srows=d, nrows=d, schur=d) == -3                  # the row export passes the checks
        assert call(srows=d, nrows=d, schur=d, n_max=10) == -1
    assert solve(srows=d) == -1 and b"go together" in lib.mc_last_error()
    assert solve(nrows=d) == -1
    assert adjoint(srows=d, nrows=d) == -1 and b"schur" in lib.mc_last_error()
    assert adjoint(srows=d, schur=d) == -1
    assert adjoint(srows=d, nrows=d, schur=d, cap=-1) == -1 and b"n_rows_cap" in lib.mc_last_error()
    # the binding's short form: the same checks, in the same order, as the call with NULL / 0
    assert _lib._OPTIONAL == {"mc_mincurv_solve_batch_sens": (18, 2), "mc_mincurv_adjoint_batch": (16, 4)}
    short = [1, 100, None, d, d, d, 2.0, None, 2.0, None, d, d, d, d, d, d]
    assert lib.mc_mincurv_adjoint_batch(*short, None, 0, None) == -3
    assert lib.mc_mincurv_adjoint_batch(*short[:10], None, *short[11:], None, 0, None) == -1
    with pytest.raises(TypeError):
        lib.mc_mincurv_adjoint_batch(*short, None, None, 0, None)          # neither form


def test_optional_parameters_are_parsed_from_the_header(tmp_path):
    h = tmp_path / "opt.h"
    h.write_text("#define MC_OPTIONAL\nint mc_a(int n, MC_OPTIONAL double *x, MC_OPTIONAL int k, void *stream);\n"
                 "int mc_b(int n);\n")
    assert _lib.optional_parameters(str(h)) == {"mc_a": (1, 2)}
    assert _lib.header_signatures(str(h))["mc_a"] == (ctypes.c_int, [ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                                                       ctypes.c_void_p])
    h.write_text("int mc_a(MC_OPTIONAL double *x, int n, MC_OPTIONAL int k);\n")
    with pytest.raises(_lib.MinCurvLibError, match="consecutive"):
        _lib.optional_parameters(str(h))


@pytest.fixture()
def rowfake(fake, monkeypatch):
    """The stand-in with n_rows = [0, 3, 7, 0, 2, ...] written by the forward (per chunk, in the order of the batch)."""
    real = FakeLib.__getattr__
    fake.n_rows = [0, 3, 7, 0, 2, 5, 1]

    def patched(self, name):
        fn = real(self, name)
        if name == "mc_mincurv_solve_batch_sens":
            def fwd(*a):
                fn(*a)
                if a[19] is not None:
                    k = sum(c[1][0] for c in self.calls[:-1] if c[0] == name)
                    (ctypes.c_int32 * a[0]).from_address(a[19].value)[:] = self.n_rows[k:k + a[0]]
                return 0
            return fwd
        return fn
    monkeypatch.setattr(FakeLib, "__getattr__", patched)
    return fake


def _diff(B=7, n=120, **kw):
    centre = torch.rand((B, n, 2), dtype=torch.float64)
    widths = (torch.rand((B, n, 2), dtype=torch.float64) + 3.0).requires_grad_()
    nv, h = torch.rand((B, n, 2), dtype=torch.float64), torch.ones((B, n), dtype=torch.float64)
    res = B_.opt_min_curv_diff(centre, widths, nv, h, 0.02, 2.0, **kw)
    res["alpha"].sum().backward()
    return widths


@pytest.mark.parametrize("flag", [False, True])
def test_curvature_rows_wiring(rowfake, flag):
    """Off: both entries get NULL for every curvature-row argument (and capacity 0).  On: the forward gets sens_rows
    [chunk, n_max] and n_rows [chunk]; the backward gets them back row for row, with one Schur buffer of at least
    cap^2 doubles per instance of its chunk, cap = max(n_rows) over the whole batch."""
    B, n = 7, 120
    widths = _diff(B, n, curvature_rows=flag)
    assert widths.grad.shape == (B, n, 2)
    fwd = [c[1] for c in rowfake.calls if c[0] == "mc_mincurv_solve_batch_sens"]
    bwd = [c[1] for c in rowfake.calls if c[0] == "mc_mincurv_adjoint_batch"]
    assert [a[0] for a in fwd] == [3, 3, 1] and [a[0] for a in bwd] == [3, 3, 1]    # the stand-in's chunks: B // 2
    if not flag:
        assert all(a[18] is None and a[19] is None for a in fwd)
        assert all(a[16] is None and a[17] is None and a[18] is None and a[19] == 0 for a in bwd)
        return
    cap = max(rowfake.n_rows)
    for f, b in zip(fwd, bwd):
        assert f[18] is not None and f[19] is not None
        assert b[16].value == f[18].value and b[17].value == f[19].value       # the forward's export, same rows
        assert b[18] is not None and b[19] == cap
    assert len({b[18].value for b in bwd}) == 1                                   # one buffer, reused by every chunk
    for b in bwd:                                                                 # consecutive rows of one export
        assert b[16].value - bwd[0][16].value == 8 * n * sum(x[0] for x in bwd[:bwd.index(b)])


def test_curvature_rows_schur_buffer_size(rowfake, monkeypatch):
    """The Schur buffer holds cap^2 doubles for every instance of the backward's chunk."""
    seen = []
    real_empty = torch.empty

    def spy(*a, **k):
        t = real_empty(*a, **k)
        seen.append(tuple(t.shape))
        return t
    monkeypatch.setattr(torch, "empty", lambda *a, **k: spy(*a, **k).zero_())
    _diff(7, 120, curvature_rows=True)
    cap = max(rowfake.n_rows)
    assert (3, cap * cap) in seen
