"""CPU tests (-m "not gpu") of tests/raceline_ref.py, the torch restatement of create_raceline that is the reference of
its device adjoint: its values against oracle/tph_dense.create_raceline and the rl_* golden keys, and its autograd against
central differences at the station count and station segments held (both asserted unchanged at +-delta)."""
import numpy as np
import pytest
import torch

import raceline_ref as R
from oracle import tph_dense as T

DELTA = 1e-6
FD_TOL = 1e-6           # relative to |directional derivative|


def _inputs(g):
    t = lambda a: torch.tensor(np.asarray(a, dtype=float))
    return t(g["reftrack"][:, :2]), t(g["normvec"]), t(g["alpha_mincurv"])


@pytest.mark.parametrize("name", ["synth333", "handling", "berlin"])
def test_reference_values_match_the_oracle_and_the_golden_keys(golden, name):
    g = golden(name)
    p, nv, al = _inputs(g)
    r = R.create_raceline(p, nv, al, 2.0)
    o = T.create_raceline(g["reftrack"][:, :2], g["normvec"], g["alpha_mincurv"], 2.0)
    assert r["no"] == g["rl_spline_inds"].size == o[4].size
    assert np.array_equal(r["spline_inds"].numpy(), g["rl_spline_inds"])
    for got, want in ((r["raceline"], g["rl_raceline_interp"]), (r["coeffs_x"], g["rl_coeffs_x"]),
                      (r["spline_lengths"], g["rl_spline_lengths"]), (r["t"], g["rl_t_values"]),
                      (r["kappa"], g["rl_kappa"]), (r["el_lengths"], g["rl_el_lengths"])):
        want = np.asarray(want)
        assert np.abs(got.numpy() - want).max() <= 1e-8 * max(np.abs(want).max(), 1.0)


@pytest.mark.parametrize("name", ["synth333", "handling"])
def test_reference_autograd_matches_central_differences(golden, name):
    g = golden(name)
    p, nv, al = _inputs(g)
    r0 = R.create_raceline(p, nv, al, 2.0)
    no, seg = r0["no"], r0["spline_inds"]
    rng = np.random.default_rng(4)
    wr = torch.tensor(rng.standard_normal((no, 2)))
    wk, we = torch.tensor(rng.standard_normal(no)), torch.tensor(rng.standard_normal(no))

    def loss(pp, vv, aa):
        r = R.create_raceline(pp, vv, aa, 2.0, no=no, seg=seg)
        return (r["raceline"] * wr).sum() + 100.0 * (r["kappa"] * wk).sum() + (r["el_lengths"] * we).sum()

    xs = [x.clone().requires_grad_() for x in (p, nv, al)]
    grads = torch.autograd.grad(loss(*xs), xs)
    for k in range(3):
        d = torch.tensor(rng.uniform(-1.0, 1.0, tuple(xs[k].shape)))
        plus = [x.detach().clone() for x in xs]
        minus = [x.detach().clone() for x in xs]
        plus[k] += DELTA * d
        minus[k] -= DELTA * d
        for q in (plus, minus):       # the held station count and segments are the forward's own at +-delta
            r = R.create_raceline(*q, 2.0)
            assert r["no"] == no and torch.equal(r["spline_inds"], seg)
        fd = (float(loss(*plus)) - float(loss(*minus))) / (2.0 * DELTA)
        an = float((grads[k] * d).sum())
        assert abs(fd - an) <= FD_TOL * abs(an), (k, fd, an)
