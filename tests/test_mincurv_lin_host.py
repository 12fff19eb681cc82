"""CPU tests (-m "not gpu") of the linearisation point of the minimum-curvature QP: the MC_OPTIONAL2 parameters of the
C-ABI as the binding reads them, the short forms of each call without a GPU, the wiring of
opt_min_curv_batch(lin_alpha=...) and of the refinement's rounds against the recording stand-in of the library, and
the dense QP about a line (lin_ref.py) against the oracle's assembly and the knot curvature."""
import ctypes

import numpy as np
import pytest
import torch

import lin_ref
from fake_lib import fake, FakeLib  # noqa: F401  (the fixture)
from global_racetrajectory_optimization_b200 import _lib, batch as B_


def test_the_linearisation_parameters_are_parsed_from_the_header(tmp_path):
    assert _lib._OPTIONAL2 == {"mc_mincurv_solve_batch_ex": (18, 1), "mc_mincurv_setup_batch_ex": (10, 1), "mc_mincurv_finalize_batch": (8, 1),
                               "mc_mincurv_adjoint_batch": (20, 1)}
    assert len(_lib.EXPORTED_SYMBOLS) == 47
    h = tmp_path / "opt.h"
    h.write_text("#define MC_OPTIONAL\n#define MC_OPTIONAL2\n"
                 "int mc_a(int n, MC_OPTIONAL double *x, MC_OPTIONAL2 int k, void *stream);\n")
    assert _lib.optional_parameters(str(h)) == {"mc_a": (1, 1)}
    assert _lib.optional_parameters(str(h), "MC_OPTIONAL2") == {"mc_a": (2, 1)}
    assert _lib.header_signatures(str(h))["mc_a"][1] == [ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]


def test_short_forms_without_gpu():
    """Each entry taken with and without its linearisation parameter (and for the adjoint without its MC_OPTIONAL ones as
    well) passes the same argument checks: an undersized workspace gives -3, a NULL input -1."""
    lib = _lib.load()
    d = ctypes.c_void_p(4096)
    head = [1, 100, None, d, d, d]
    setup = head + [2.0, None, 2.0, d]
    for lin in ([], [None], [d]):
        assert lib.mc_mincurv_setup_batch_ex(*setup, *lin, None, 0, None) == -3
        assert lib.mc_mincurv_setup_batch_ex(*head[:3], None, *head[4:], 2.0, None, 2.0, d, *lin, None, 0, None) == -1
        assert lib.mc_mincurv_solve_batch_ex(*head, 0.12, 2.0, None, 2.0, d, d, None, d, None, 0.0, None, None, *lin,
                                             None, 0, None) == -3
    for lin in ([], [0], [1]):
        assert lib.mc_mincurv_finalize_batch(1, 100, None, d, 0.12, d, None, d, *lin, None, 0, None) == -3
    adj = head + [2.0, None, 2.0, None, d, d, d, d, d, d]
    for tail in ([], [None, None, None, 0], [None, None, None, 0, None], [None, None, None, 0, d]):
        assert lib.mc_mincurv_adjoint_batch(*adj, *tail, None, 0, None) == -3


def test_opt_min_curv_batch_passes_the_linearisation_point(fake):
    B, n = 4, 100
    rt = torch.rand((B, n, 4), dtype=torch.float64)
    nv = torch.rand((B, n, 2), dtype=torch.float64)
    h = torch.ones((B, n), dtype=torch.float64)
    la = torch.rand((B, n), dtype=torch.float64)
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0)
    B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, lin_alpha=la)
    names = [name for name, _ in fake.calls if name.startswith("mc_mincurv_solve")]
    assert names == ["mc_mincurv_solve_batch_shared"] * 2 + ["mc_mincurv_solve_batch_ex"] * 2    # chunks of two
    for k, a in enumerate(a for name, a in fake.calls if name == "mc_mincurv_solve_batch_ex"):
        assert a[15] == 0.0 and a[16] is None and a[17] is None
        assert a[18].value == la[2 * k:2 * k + 2].data_ptr()
    # with shared centre lines a follower is solved about its owner's row (and the shared entry is not used)
    fake.calls.clear()
    out = B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, lin_alpha=la, centre_id=torch.tensor([0, 0, 2, 5]))
    rows = [a[18].value for name, a in fake.calls if name == "mc_mincurv_solve_batch_ex"]
    assert [name for name, _ in fake.calls if name.startswith("mc_mincurv_solve")] == ["mc_mincurv_solve_batch_ex"] * 2
    assert out["status"].tolist() == [0, 0, 0, -1]                      # instance 3's owner is out of range
    assert len(rows) == 2
    with pytest.raises(ValueError, match="lin_alpha"):
        B_.opt_min_curv_batch(rt, nv, h, 0.12, 2.0, lin_alpha=la[:, :50])


def test_dense_qp_about_a_line(golden):
    """The dense QP about a = 0 is the oracle's assembly exactly; about a line its rows are the knot curvature of the
    spline through P + a n at alpha = a, and k_ref + E alpha matches lin_ref.linearised_curvature everywhere."""
    g = golden("synth128")
    rt, nvec, wv = g["reftrack"], g["normvec"], float(g["w_veh"])
    ref = lin_ref.dense_qp_about(rt, nvec, None, 0.12, wv)
    zero = lin_ref.dense_qp_about(rt, nvec, np.zeros(rt.shape[0]), 0.12, wv)
    for k in ("H", "f", "E", "k_ref", "G", "h"):
        assert np.array_equal(zero[k], ref[k]), k
    p = rt[:, :2]
    el = np.linalg.norm(np.roll(p, -1, axis=0) - p, axis=1)
    h = el / el.mean()
    a = 0.5 * g["alpha_mincurv"]
    d = lin_ref.dense_qp_about(rt, nvec, a, 0.12, wv)
    k_true = lin_ref.knot_curvature(p + a[:, None] * nvec, h)
    assert np.allclose(d["k_ref"] + d["E"] @ a, k_true, rtol=0, atol=1e-9 * np.abs(k_true).max())
    assert np.allclose(lin_ref.linearised_curvature(p, nvec, h, a, a), k_true, rtol=0, atol=1e-12)
    v = np.random.default_rng(3).standard_normal(p.shape[0]) * 0.1
    assert np.allclose(d["k_ref"] + d["E"] @ (a + v), lin_ref.linearised_curvature(p, nvec, h, a, a + v), rtol=0,
                       atol=1e-9 * np.abs(k_true).max())


def test_refinement_rounds(fake, monkeypatch):
    """relinearise: each round's projection and metric are built about the round's start (the previous round's result),
    spg starts there; tracks leave when curv_error_max <= curv_error_allowed, at round relinearise, or with
    NO_PROJECTION (keeping the previous result) when the round-start projection fails; rounds, iters and evals as
    documented.  relinearise without kappa_bound is refused."""
    from global_racetrajectory_optimization_b200 import raceline_refine as R
    B, n = 4, 100
    rt = torch.rand((B, n, 4), dtype=torch.float64) + torch.tensor([0.0, 0.0, 5.0, 5.0], dtype=torch.float64)
    nv = torch.rand((B, n, 2), dtype=torch.float64)
    veh = dict(ggv=np.ones((2, 3)), ax_max_machines=np.ones((2, 2)), v_max=70.0, drag_coeff=0.75, m_veh=1200.0)
    with pytest.raises(ValueError, match="kappa_bound"):
        R.refine_raceline_batch(rt, nv, torch.zeros((B, n), dtype=torch.float64), 2.0, relinearise=2, **veh)
    starts, lins = [], []
    ce_of_round = {0: [0.5, 0.005, 0.5, 0.5], 1: [0.5, 0.5, 0.002, 0.5], 2: [0.5, 0.5, 0.5, 0.5], 3: [0.5, 0.5, 0.5, 0.5]}

    def spg(fun, x0, lb, ub, active, metric=None, project=None, **kw):
        r = len(starts)
        starts.append((x0.clone(), active.clone()))
        lins.append((None if project.lin is None else project.lin.clone(),
                     None if metric.lin is None else metric.lin[::2].clone()))
        fail = active & (torch.arange(B) == 3) & (r == 2)              # track 3: round 2's start projection fails
        ok = active & ~fail
        i32 = lambda v: torch.where(ok, v, 0).to(torch.int32)         # noqa: E731
        return dict(x=torch.where(ok[:, None], x0 + 1.0, x0), f=torch.full((B,), 10.0 - r, dtype=torch.float64),
                    f0=torch.full((B,), 10.0, dtype=torch.float64),
                    status=torch.where(fail, R.NO_PROJECTION, torch.where(ok, R.ITER_CAP, R.INACTIVE)).to(torch.int32),
                    iters=i32(3), evals=i32(5), pg_norm=torch.zeros(B, dtype=torch.float64),
                    projection_failures=fail.to(torch.int32))

    def evaluate(self, x, mask):
        ce = torch.tensor(ce_of_round[len(starts) - 1], dtype=torch.float64)
        return torch.full((B,), 0.1, dtype=torch.float64), ce

    monkeypatch.setattr(R, "spg", spg)
    monkeypatch.setattr(R.CurvatureProjection, "evaluate", evaluate)
    res = R.refine_raceline_batch(rt, nv, torch.zeros((B, n), dtype=torch.float64), 2.0, metric_length=10.0,
                                  kappa_bound=0.12, relinearise=3, **veh)
    assert len(starts) == 4                                            # track 0 runs to round relinearise
    assert lins[0] == (None, None)
    assert starts[1][1].tolist() == [True, False, True, True]          # track 1 met curv_error_allowed in round 0
    assert starts[2][1].tolist() == [True, False, False, True]         # track 2 in round 1
    assert starts[3][1].tolist() == [True, False, False, False]        # track 3's projection failed in round 2
    for r in (1, 2, 3):
        x0, _ = starts[r]
        assert torch.equal(lins[r][0], x0) and torch.equal(lins[r][1], x0)
    assert torch.equal(starts[1][0][0], torch.full((n,), 1.0, dtype=torch.float64))
    assert res["rounds"].tolist() == [3, 0, 1, 1]
    assert res["status"].tolist() == [R.ITER_CAP, R.ITER_CAP, R.ITER_CAP, R.NO_PROJECTION]
    assert res["alpha"][:, 0].tolist() == [4.0, 1.0, 2.0, 2.0]             # track 3 keeps round 1's result
    assert res["iters"].tolist() == [12, 3, 6, 6] and res["evals"].tolist() == [20, 5, 10, 10]
    assert res["projection_failures"].tolist() == [0, 0, 0, 1]
    assert res["curv_error_max"].tolist() == [0.5, 0.005, 0.002, 0.5]
    # relinearise = 0: one spg call, rounds 0
    starts.clear()
    res0 = R.refine_raceline_batch(rt, nv, torch.zeros((B, n), dtype=torch.float64), 2.0, metric_length=10.0,
                                   kappa_bound=0.12, **veh)
    assert len(starts) == 1 and res0["rounds"].tolist() == [0] * B
