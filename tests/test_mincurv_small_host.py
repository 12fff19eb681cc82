"""CPU tests (-m "not gpu") of the dense small-track solver's interface: the MC_OPTIONAL4 parameter of
mc_mincurv_solve_batch_ex as the binding reads it and its short forms, the argument checks of the real library before any
CUDA call, the launches of opt_min_curv_batch / iqp_batch / globaltraj_batch with and without small_tracks against the
recording stand-in of the library, and the oracle statuses the GPU tests rely on."""
import ctypes

import numpy as np
import pytest
import torch

from fake_lib import fake  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_, globaltraj, synth
from oracle import tph_dense as T


def test_the_dense_parameter_is_parsed_from_the_header():
    assert _lib._OPTIONAL4 == {"mc_mincurv_solve_batch_ex": (25, 1)}
    assert _lib._SIGS["mc_mincurv_solve_batch_ex"][1][25] is ctypes.c_int
    assert B_.N_DENSE_MAX == _lib.header_define(_lib._build.HEADER, "MC_DENSE_N_MAX") >= 96


def _ex(d, B=1, n_max=100, tail=()):
    head = [B, n_max, None, d, d, d]
    return head + [0.12, 2.0, None, 2.0, d, d, None, d, None, 0.0, None, None, None] + list(tail)


def test_the_real_library_refuses_before_any_cuda_call():
    lib = _lib.load()
    d = ctypes.c_void_p(4096)
    none6 = [None] * 6
    # every short form still binds: without the dense group, without it and the MC_OPTIONAL3 group
    assert lib.mc_mincurv_solve_batch_ex(*_ex(d), None, 0, None) == -3
    assert lib.mc_mincurv_solve_batch_ex(*_ex(d, tail=none6), None, 0, None) == -3
    assert lib.mc_mincurv_solve_batch_ex(*_ex(d, tail=none6 + [0]), None, 0, None) == -3
    for bad in (1, 79, B_.N_DENSE_MAX + 2, -80):
        assert lib.mc_mincurv_solve_batch_ex(*_ex(d, tail=none6 + [bad]), None, 0, None) == -1
        assert b"dense_below" in lib.mc_last_error()
    ex = _ex(d, tail=none6 + [B_.N_MIN])
    prox = list(ex)
    prox[16], prox[17] = d, d                       # prox_x, prox_q
    assert lib.mc_mincurv_solve_batch_ex(*prox, None, 0, None) == -1
    sens = _ex(d, tail=[None, None, d, d, None, None, B_.N_MIN])
    assert lib.mc_mincurv_solve_batch_ex(*sens, None, 0, None) == -1
    # n_max below N_MIN: refused without the dense solver, as before; with it, a NULL input is still refused
    assert lib.mc_mincurv_solve_batch_ex(*_ex(d, n_max=60, tail=none6 + [0]), None, 0, None) == -1
    no_rt = _ex(d, n_max=60, tail=none6 + [B_.N_MIN])
    no_rt[3] = None
    assert lib.mc_mincurv_solve_batch_ex(*no_rt, None, 0, None) == -1


def _qp(B=4, n=100):
    g = torch.Generator().manual_seed(1)
    return (torch.rand((B, n, 4), dtype=torch.float64, generator=g), torch.rand((B, n, 2), dtype=torch.float64, generator=g),
            torch.ones((B, n), dtype=torch.float64))


def _mincurv_calls(fake):
    return [(c[0], c[1]) for c in fake.calls if c[0].startswith("mc_mincurv") and not c[0].endswith("_bytes")]


@pytest.mark.parametrize("n", [100, 60])
def test_small_tracks_go_through_the_extended_entry(fake, n):
    rt, nv, h = _qp(n=n)
    kb_t = torch.full((4,), 0.12, dtype=torch.float64)
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, small_tracks=True)
    B_.opt_min_curv_batch(rt, nv, h, kb_t, torch.full((4,), 2.0, dtype=torch.float64), small_tracks=True,
                          centre_id=torch.tensor([0, 0, 2, 2]))
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, small_tracks=True, lin_alpha=torch.zeros((4, n), dtype=torch.float64))
    calls = _mincurv_calls(fake)
    assert [c[0] for c in calls] == ["mc_mincurv_solve_batch_ex"] * 6        # (two chunks each)
    for _, a in calls:
        assert a[25] == B_.N_MIN and a[16] is None and a[21] is None
    assert calls[0][1][6] == 0.12 and calls[0][1][19] is None                 # the scalar limit
    assert calls[2][1][19] is not None and calls[2][1][20] is not None        # the [B] limit, the chunk's centre ids
    assert calls[4][1][18] is not None                                        # lin_alpha
    fake.calls.clear()
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, small_tracks=True, _dense_below=B_.N_DENSE_MAX + 1)
    assert all(a[25] == B_.N_DENSE_MAX + 1 for _, a in _mincurv_calls(fake))


def test_without_the_flag_nothing_changes(fake):
    rt, nv, h = _qp()
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0)
    B_.opt_min_curv_batch(rt, nv, h, torch.full((4,), 0.12, dtype=torch.float64), 2.0)
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, lin_alpha=torch.zeros((4, 100), dtype=torch.float64))
    assert [c[0] for c in _mincurv_calls(fake)] == ["mc_mincurv_solve_batch_shared"] * 2 + ["mc_mincurv_solve_batch_ex"] * 4
    assert all(a[25] == 0 for name, a in _mincurv_calls(fake) if name == "mc_mincurv_solve_batch_ex")
    rt, nv, h = _qp(n=60)
    with pytest.raises(NotImplementedError):
        B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0)


def test_iqp_and_globaltraj_pass_the_flag_on(fake, monkeypatch):
    seen = []
    real = B_.opt_min_curv_batch
    monkeypatch.setattr(B_, "opt_min_curv_batch", lambda *a, **k: seen.append(k.get("small_tracks")) or real(*a, **k))
    rt, nv, h = _qp(n=60)
    rt[:, :, 2:] += 5.0
    B_.iqp_batch(rt, nv, h, 0.12, 2.0, 3.0, fixed_iters=2, small_tracks=True)
    assert seen == [True, True]
    seen.clear()
    pars = globaltraj.default_pars()
    for opt_type, want in (("mincurv", [True]), ("mincurv_iqp", [True])):
        globaltraj.globaltraj_batch(rt, opt_type, pars, np.array([[0.0, 5.0, 6.0], [80.0, 4.0, 7.0]]),
                                    np.array([[0.0, 8.0], [80.0, 3.0]]), small_tracks=True)
        assert seen[:len(want)] == want, opt_type
        seen.clear()


def test_the_refinement_projection_passes_no_dense_solver(fake):
    from global_racetrajectory_optimization_b200 import raceline_refine as Rf
    rt, nv, h = _qp()
    proj = Rf.CurvatureProjection(rt, nv, None, 2.0, 0.12, 10.0)
    fake.calls.clear()
    x = torch.zeros((4, 100), dtype=torch.float64)
    proj(x, x, torch.ones(4, dtype=torch.bool))
    ex = [a for name, a in fake.calls if name == "mc_mincurv_solve_batch_ex"]
    assert ex and all(a[25] == 0 and a[16] is not None for a in ex)


def _closed(rt):
    return np.vstack((rt[:, :2], rt[0, :2]))


@pytest.mark.parametrize("n,kb,want", [(3, 0.12, RuntimeError), (5, 0.12, ValueError), (8, 0.12, ValueError),
                                       (16, 0.12, None), (40, 0.12, None), (79, 0.12, None), (40, 0.03, ValueError)])
def test_the_oracle_statuses_the_gpu_tests_rely_on(n, kb, want):
    rt = synth.make_track(1, n)
    _, _, A, nv = T.calc_splines(_closed(rt))
    if want is None:
        T.opt_min_curv(rt, nv, A, kb, 2.0)
    else:
        with pytest.raises(want):
            T.opt_min_curv(rt, nv, A, kb, 2.0)
