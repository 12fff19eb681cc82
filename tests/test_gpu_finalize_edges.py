"""GPU tests (-m gpu) of the minimum-curvature post-solve kernels of csrc/mincurv_finalize.cu against the long-double
replay of tests/finalize_ref.py, per point and at the precision the decisions are made.

mincurv_finalize_kernel (K2c) runs after mc_mincurv_setup_batch_ex with a chosen alpha and chosen statuses; the slab is
then read back.  The kernel leaves Z (n_x alpha) and Z (n_y alpha) in V_T4 / V_T5, so these are checked at every point,
and kappa_lin_max and curv_error_max against the replay on the slab's own vectors (finalize_ref.from_slab):
  shapes   every n from 80 to 129 in one ragged launch with NaN padding; 2047, 2048, 2049, 4095, 4097 and 10 000 (one
           thread runs several 2048-point sweeps of the chunked solve); the 14 fixtures, 1:5 and 1:20 spacing and
           collapsed boxes;
  alpha    0, the QP solution, the box limits, ten times the QP solution (a large linearisation error) and a bump at the
           wrap (so that the maxima are taken at i = 0 and n - 1);
  LIN      about lin_alpha = alpha (no error) and about another line; followers of shared centre lines; kappa_lin_max
           and n_pts NULL;
  status   the status-4 decision ulp by ulp around its threshold, scalar and per-instance; every (status, limit) pair of
           the per-instance refusals in the middle of a batch; NaN and inf in alpha (both maxima NaN, as tph's np.amax).
The full solves: both finalize passes of a mixed curvature-row batch against the replay at the alpha they saw; the
sensitivity exports bit for bit against the final slab; the projection QP's H + mu I and linear term.
Every measured error is printed next to its bound (pytest -s)."""
import numpy as np
import pytest

import finalize_ref as F
import mincurv_ref as R

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402

# Bounds, about ten times the values measured on an H100 80GB HBM3 (700 W power limit) over the cases below, against the
# long-double replay on the device's own slab vectors:
#   z: max |Z_dev - Z_ref| / max |Z_ref| per instance: 1.6e-14 (N104, the QP alpha);
#   kmax: |kappa_lin_max - ref| / ref: 7.8e-15 (synth2000 about alpha);
#   emax: |curv_error_max - ref| / max(ref, 1e-3 kappa_lin_max): 1.1e-13 (synth2000 at ten times the QP alpha).  c1 - c0
#   is the difference of two curvatures of size kappa_lin_max, so its rounding is relative to that, not to itself.
# 1:20 spacing: Z = Tri^-1 6 D2 (n alpha) divides the differences of alpha by the short steps, and kappa_lin = k_ref +
# S_y z_y - S_x z_x adds S z of the long steps, which is up to 20^2 larger: z 1.3e-13, kmax 6.6e-14 there.
# The projection's V_F: 3.5e-16.
TOL = dict(z=2e-13, kmax=1e-13, emax=1e-12)
TOL_1_20 = dict(z=1.5e-12, kmax=7e-13, emax=1e-12)
PROX_TOL = 5e-15       # V_F of the projection QP against long double, max |diff| / max |ref|
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a, dtype=torch.float64):
    return torch.tensor(np.asarray(a), dtype=dtype, device=DEV)


def _closed(rt):
    return np.vstack((rt[:, :2], rt[:1, :2]))


def track(rt, name=""):
    _, _, nv = R.periodic_spline(_closed(rt))
    return dict(rt=rt, nv=nv, h=np.linalg.norm(np.diff(_closed(rt), axis=0), axis=1), name=name)


def _pack(tracks, rows, n_max=None, pad=np.nan):
    """[B, n_max, ...] arrays of the tracks' rt, nv, h and of rows (per-track [n] arrays), padding pad."""
    n = [t["rt"].shape[0] for t in tracks]
    n_max = n_max or max(n)
    rt, nv, h = np.full((len(n), n_max, 4), pad), np.full((len(n), n_max, 2), pad), np.full((len(n), n_max), pad)
    out = [np.full((len(n), n_max), pad) for _ in rows]
    for b, t in enumerate(tracks):
        rt[b, :n[b]], nv[b, :n[b]], h[b, :n[b]] = t["rt"], t["nv"], t["h"]
        for o, r in zip(out, rows):
            if r[b] is not None:
                o[b, :n[b]] = r[b]
    return n, n_max, rt, nv, h, out


def _slab(ws, b, n, n_max):
    lay = B_.mincurv_slab_layout(n_max)
    s = ws[b * lay["stride"]:(b + 1) * lay["stride"]]
    v = {nm: s[i * lay["np"]:i * lay["np"] + n].copy() for i, nm in enumerate(B_.SLAB_VECTORS)}
    v["HB"] = s[lay["o_hb"]:lay["o_hb"] + lay["np"] * B_.HB_PITCH].reshape(-1, B_.HB_PITCH)[:n, :33].copy()
    return v


def _ws(B, n_max):
    return torch.zeros(_lib.load().mc_mincurv_workspace_bytes(B, n_max), dtype=torch.uint8, device=DEV)


def _read(ws):
    torch.cuda.synchronize()
    return ws.view(torch.float64).cpu().numpy()


def finalize(tracks, alphas, statuses=None, kb=0.2, kbb=None, lins=None, n_max=None, npts=True, klin=True,
             centre_id=None):
    """setup (about lins[b], or the centre line) -> statuses overwritten -> mc_mincurv_finalize_batch; dict of numpy
    status, cerr, klin and slab (per instance: the slab vectors)."""
    lin = lins is not None
    n, n_max, rt, nv, h, (al, la) = _pack(tracks, [alphas, lins if lin else [None] * len(tracks)], n_max)
    B = len(n)
    ws = _ws(B, n_max)
    st = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    np_ = _dev(n, torch.int32) if npts else None
    if centre_id is None:
        B_._call("mc_mincurv_setup_batch_ex", B, n_max, np_, _dev(rt), _dev(nv), _dev(h), 2.0, None, B_.F_SCALE, st,
                 _dev(la) if lin else None, ws=ws)
    else:
        B_._call("mc_mincurv_setup_batch_shared", B, n_max, np_, _dev(rt), _dev(nv), _dev(h), 2.0, None, B_.F_SCALE,
                 _dev(centre_id, torch.int32), st, ws=ws)
    setup_status = st.cpu().numpy()
    if statuses is not None:
        st.copy_(_dev(statuses, torch.int32))
    cerr = torch.full((B,), -1.0, dtype=torch.float64, device=DEV)
    kl = torch.full((B,), -1.0, dtype=torch.float64, device=DEV) if klin else None
    B_._call("mc_mincurv_finalize_batch", B, n_max, np_, _dev(al), float(kb), cerr, kl, st, int(lin),
             None if kbb is None else _dev(kbb), ws=ws)
    torch.cuda.synchronize()
    w = _read(ws)
    return dict(status=st.cpu().numpy(), setup_status=setup_status, cerr=cerr.cpu().numpy(),
                klin=None if kl is None else kl.cpu().numpy(), slab=[_slab(w, b, n[b], n_max) for b in range(B)])


def _errors(res, b, alpha, lin=False):
    """(errors dict, replay) of instance b of a finalize result against from_slab on its own slab"""
    v = res["slab"][b]
    r = F.from_slab(v, alpha, lin=lin)
    zx, zy = np.asarray(r["zx"], np.float64), np.asarray(r["zy"], np.float64)
    ez = max(np.abs(v["T4"] - zx).max() / max(np.abs(zx).max(), 1e-300),
             np.abs(v["T5"] - zy).max() / max(np.abs(zy).max(), 1e-300))
    km, em = float(r["kmax"]), float(r["emax"])
    ek = abs(res["klin"][b] - km) / km if res["klin"] is not None else 0.0
    ee = abs(res["cerr"][b] - em) / max(em, 1e-3 * km)
    return dict(z=float(ez), kmax=float(ek), emax=float(ee)), r


class Worst:
    def __init__(self, what):
        self.what, self.w, self.bad = what, {}, []

    def add(self, name, e, tol):
        for k, x in e.items():
            if x > self.w.get(k, (-1.0, ""))[0]:
                self.w[k] = (x, name)
            if not x <= tol[k]:
                self.bad.append((name, k, x, tol[k]))

    def report(self, tol):
        print(f"{self.what}: " + ", ".join(f"{k} {x:.2e} ({nm}; bound {tol[k]:.0e})" for k, (x, nm) in self.w.items()))
        assert not self.bad, self.bad


def _alphas(t, qp):
    """named alpha of one track: 0, the QP solution, the box limits, 10x the QP solution, a bump at the wrap"""
    n = t["rt"].shape[0]
    ub, lb = t["rt"][:, 2] - 1.0, -(t["rt"][:, 3] - 1.0)
    i = np.arange(n)
    d = np.minimum(i, n - i)
    return dict(zero=np.zeros(n), qp=qp, box=np.where((i // 7) % 2 == 0, ub, lb), large=10.0 * qp,
                wrap=np.where(d < 5, 3.0 * np.cos(0.3 * d), 0.0))


def _qp(tracks, kb=10.0):
    n, n_max, rt, nv, h, _ = _pack(tracks, [], pad=0.0)
    h[h == 0.0] = 1.0
    out = B_.opt_min_curv_batch(_dev(rt), _dev(nv), _dev(h), kb, 2.0, n_pts=_dev(n, torch.int32))
    a = out["alpha"].cpu().numpy()
    assert (out["status"].cpu().numpy() == 0).all()
    return [a[b, :n[b]] for b in range(len(tracks))]


def _sweep(tracks, what, tol_of=lambda t: TOL, n_max=None):
    qps = _qp(tracks)
    worst = Worst(what)
    for kind in ("zero", "qp", "box", "large", "wrap"):
        als = [_alphas(t, q)[kind] for t, q in zip(tracks, qps)]
        res = finalize(tracks, als, n_max=n_max)
        for b, (t, a) in enumerate(zip(tracks, als)):
            assert res["status"][b] == res["setup_status"][b] == 0 or (kind != "zero" and res["status"][b] == 4)
            e, r = _errors(res, b, a)
            assert res["status"][b] == F.status_after(0, res["klin"][b], 0.2)[0]
            worst.add(f"{t['name']} {kind}", e, tol_of(t))
    worst.report(tol_of(tracks[-1]))


def test_every_n_from_80_to_129_in_a_ragged_launch():
    tracks = [track(synth.make_track(300 + n, n), f"N{n}") for n in range(80, 130)]
    _sweep(tracks, "N 80..129 (n_max 129, NaN padding)")


@pytest.mark.parametrize("n", [2047, 2048, 2049, 4095, 4097, 10000])
def test_long_tracks(n):
    _sweep([track(synth.make_track(17, n), f"N{n}")], f"N{n}")


GOLDEN = ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth1000", "synth128",
          "synth160_kappa", "synth200", "synth2000", "synth333", "synth333_kappa", "synth500", "synth500_narrow"]


def test_fixtures_spacing_and_collapsed_boxes(golden):
    tracks = [track(golden(nm)["reftrack"], nm) for nm in GOLDEN]
    tracks += [track(R.uneven_track(260, 5.0, 1), "spacing 1:5"), track(R.uneven_track(300, 20.0, 2), "spacing 1:20")]
    col = synth.make_track(2, 240, amp=0.1)
    for i in (5, 77, 78, 239):
        col[i, 3] = 2.0 - col[i, 2]
    tracks.append(track(col, "collapsed"))
    _sweep(tracks, "fixtures", tol_of=lambda t: TOL_1_20 if "1:20" in t["name"] else TOL)


def test_linearised_about_alpha_and_about_another_line(golden):
    names = ["handling", "synth160_kappa", "berlin", "synth2000"]
    tracks = [track(golden(nm)["reftrack"], nm) for nm in names] + [track(R.uneven_track(300, 20.0, 2), "spacing 1:20")]
    qps = _qp(tracks)
    worst = Worst("LIN")
    for about in ("alpha", "other"):
        lins = qps if about == "alpha" else [0.5 * q + 0.2 for q in qps]
        res = finalize(tracks, qps, lins=lins)
        for b, t in enumerate(tracks):
            e, r = _errors(res, b, qps[b], lin=True)
            worst.add(f"{t['name']} about {about}", e, TOL_1_20 if "1:20" in t["name"] else TOL)
            if about == "alpha":
                print(f"{t['name']} about alpha: curv_error_max {res['cerr'][b]:.2e} (replay {float(r['emax']):.2e}), "
                      f"kappa_lin_max {res['klin'][b]:.4g}")
                assert res["cerr"][b] <= 1e-12 * res["klin"][b]
    worst.report(TOL)
    # lin_alpha = 0 is the centre-line call bit for bit, and the LIN branch recomputes the centre line's derivatives
    a = finalize(tracks, qps, lins=[np.zeros_like(q) for q in qps])
    c = finalize(tracks, qps)
    for k in ("status", "cerr", "klin"):
        assert np.array_equal(a[k], c[k]), k


def test_followers_null_outputs_and_null_n_pts():
    base = synth.make_track(5, 300)
    wide, narrow = base.copy(), base.copy()
    narrow[:, 2:] *= 0.5
    tracks = [track(x, nm) for x, nm in ((wide, "owner"), (narrow, "follower"), (narrow, "owner 2"), (wide, "follower 2"))]
    qp = _qp(tracks[:1])[0]
    als = [qp, 0.5 * qp, -qp, 2.0 * qp]
    lone = finalize(tracks, als)
    shared = finalize(tracks, als, centre_id=[0, 0, 2, 2])
    nul = finalize(tracks, als, klin=False)
    nonp = finalize(tracks, als, npts=False)
    for k in ("status", "cerr", "klin"):
        assert np.array_equal(lone[k], shared[k]) and np.array_equal(lone[k], nonp[k]), k
    assert np.array_equal(lone["status"], nul["status"]) and np.array_equal(lone["cerr"], nul["cerr"])
    for b in range(4):
        for v in ("T4", "T5"):
            assert np.array_equal(lone["slab"][b][v], shared["slab"][b][v]), (b, v)
    # with LIN, through the full solve: followers against their unshared solves
    rt = np.stack([t["rt"] for t in tracks])
    nv, h = np.stack([t["nv"] for t in tracks]), np.stack([t["h"] for t in tracks])
    lin = _dev(np.stack([0.5 * qp] * 4))
    for la in (None, lin):
        s = B_.opt_min_curv_batch(_dev(rt), _dev(nv), _dev(h), 0.05, 2.0, lin_alpha=la,
                                  centre_id=_dev([0, 0, 2, 2], torch.int32))
        u = B_.opt_min_curv_batch(_dev(rt), _dev(nv), _dev(h), 0.05, 2.0, lin_alpha=la)
        for k in ("alpha", "curv_error_max", "kappa_lin_max", "status", "iters"):
            assert torch.equal(s[k], u[k]), (la is None, k)


def test_status_4_decision_ulp_by_ulp():
    tracks = [track(synth.make_track(7, 150), "N150"), track(synth.make_track(8, 4097), "N4097")]
    qps = _qp(tracks)
    for t, q in zip(tracks, qps):
        K = float(finalize([t], [q], kb=1e3)["klin"][0])
        kb0 = K / (1.0 + 1e-7)
        up, dn = [kb0], [kb0]
        for _ in range(3):
            up.append(float(np.nextafter(up[-1], np.inf)))
            dn.append(float(np.nextafter(dn[-1], -np.inf)))
        kbs = sorted(set(up + dn))
        want = [4 if K > kb * (1.0 + 1e-7) else 0 for kb in kbs]
        assert 0 in want and 4 in want, (K, kbs)
        scalar = [int(finalize([t], [q], kb=kb)["status"][0]) for kb in kbs]
        batch = finalize([t] * len(kbs), [q] * len(kbs), kbb=kbs)
        assert np.all(batch["klin"] == K)
        print(f"{t['name']}: K {K!r}, kb around K / (1 + 1e-7): predicted {want}, scalar {scalar}, "
              f"per-instance {batch['status'].tolist()}")
        assert scalar == want and batch["status"].tolist() == want


KB_BAD = [0.0, -0.0, -1.0, np.nan, np.inf, -np.inf, 5e-324, 1e300]
STATUSES = [0, 1, 2, 3, 4, -1, -2]          # (-2: any other negative status is kept as it is)


def test_per_instance_refusals_in_the_middle_of_a_batch():
    t = track(synth.make_track(9, 120), "N120")
    q = _qp([t])[0]
    good = 0.05
    pairs = [(kb, st) for kb in KB_BAD for st in STATUSES]
    kbs, sts = [good], [0]
    for kb, st in pairs:
        kbs += [kb, good]
        sts += [st, 0]
    res = finalize([t] * len(kbs), [q] * len(kbs), statuses=sts, kbb=kbs)
    lone = finalize([t], [q], kb=good)
    K = float(finalize([t], [q], kb=1e3)["klin"][0])
    for b in range(0, len(kbs), 2):
        assert res["status"][b] == lone["status"][0] and res["cerr"][b] == lone["cerr"][0] \
            and res["klin"][b] == lone["klin"][0], b
        assert np.array_equal(res["slab"][b]["T4"], lone["slab"][0]["T4"])
    for j, (kb, st) in enumerate(pairs):
        b = 2 * j + 1
        want, zeroed = F.status_after(st, K, kb, kbb=True)
        got = (int(res["status"][b]), float(res["cerr"][b]), float(res["klin"][b]))
        if zeroed:
            assert got == (want, 0.0, 0.0), (kb, st, got)
        else:
            assert got[0] == want and got[2] == K and got[1] == lone["cerr"][0], (kb, st, got)
    print(f"{len(pairs)} (limit, status) pairs: statuses as status_after, neighbours bit for bit their lone run")


@pytest.mark.parametrize("n", [100, 4097])
@pytest.mark.parametrize("bad", [np.nan, np.inf])
def test_non_finite_alpha_gives_nan_maxima(n, bad):
    t = track(synth.make_track(10, n), f"N{n}")
    q = _qp([t])[0]
    a = q.copy()
    a[n // 2] = bad
    res = finalize([t, t, t], [q, a, q], statuses=[0, 0, 2], kbb=[0.05, 0.05, 0.05])
    r = F.from_slab(res["slab"][1], a)
    print(f"N{n} alpha[{n // 2}] = {bad}: kappa_lin_max {res['klin'][1]}, curv_error_max {res['cerr'][1]}, "
          f"status {res['status'][1]} (replay {float(r['kmax'])}, {float(r['emax'])})")
    assert np.isnan(r["kmax"]) and np.isnan(r["emax"])
    assert np.isnan(res["klin"][1]) and np.isnan(res["cerr"][1])
    assert res["status"][1] == F.status_after(0, np.nan, 0.05, kbb=True)[0] == 0
    assert np.isfinite(res["klin"][[0, 2]]).all() and res["cerr"][0] == res["cerr"][2]
    res = finalize([t, t], [a, a], statuses=[2, 4], kb=0.05)
    assert np.isnan(res["klin"]).all() and np.isnan(res["cerr"]).all() and res["status"].tolist() == [2, 4]


# ---------------------------------------------------------------------------------------------------------------------
# full solves
# ---------------------------------------------------------------------------------------------------------------------
def _mixed(golden):
    from test_gpu_edges import KB_MIXED, _mixed_cases
    cases, centre_id, rows = _mixed_cases(golden)
    tracks = [dict(rt=c["rt"], nv=c["nv"], h=c["h"], name=c["name"]) for c in cases]
    return tracks, centre_id, rows, KB_MIXED


def test_both_passes_of_a_mixed_batch_against_the_replay(golden):
    tracks, centre_id, rows, kb = _mixed(golden)
    n, n_max, rt, nv, h, _ = _pack(tracks, [], pad=0.0)
    h[h == 0.0] = 1.0
    B = len(n)
    ws = _ws(B, n_max)
    npts, al = _dev(n, torch.int32), torch.zeros((B, n_max), dtype=torch.float64, device=DEV)
    st, it = torch.zeros(B, dtype=torch.int32, device=DEV), torch.zeros(B, dtype=torch.int32, device=DEV)
    ce, kl = torch.zeros(B, dtype=torch.float64, device=DEV), torch.zeros(B, dtype=torch.float64, device=DEV)
    B_._call("mc_mincurv_setup_batch_shared", B, n_max, npts, _dev(rt), _dev(nv), _dev(h), 2.0, None, B_.F_SCALE,
             _dev(centre_id, torch.int32), st, ws=ws)
    B_._call("mc_mincurv_pdip_batch", B, n_max, npts, al, st, it, ws=ws)
    before = st.cpu().numpy().copy()
    B_._call("mc_mincurv_finalize_batch", B, n_max, npts, al, kb, ce, kl, st, 0, None, ws=ws)
    passes = [(before, st.cpu().numpy().copy(), al.cpu().numpy().copy(), ce.cpu().numpy().copy(),
               kl.cpu().numpy().copy(), _read(ws))]
    B_._call("mc_mincurv_kappa_batch", B, n_max, npts, kb, al, st, it, None, ws=ws)
    before = st.cpu().numpy().copy()
    B_._call("mc_mincurv_finalize_batch", B, n_max, npts, al, kb, ce, kl, st, 0, None, ws=ws)
    passes.append((before, st.cpu().numpy().copy(), al.cpu().numpy().copy(), ce.cpu().numpy().copy(),
                   kl.cpu().numpy().copy(), _read(ws)))
    assert [b for b in range(B) if passes[0][1][b] == 4] == rows
    for p, (s0, s1, a, c, k, w) in enumerate(passes):
        worst = Worst(f"mixed batch, pass {p + 1}")
        for b, t in enumerate(tracks):
            want, zeroed = F.status_after(int(s0[b]), k[b], kb)
            assert s1[b] == want, (p, t["name"], s0[b], s1[b])
            if zeroed:
                assert c[b] == 0.0 and k[b] == 0.0
                continue
            res = dict(slab=[_slab(w, b, n[b], n_max)], klin=k[b:b + 1], cerr=c[b:b + 1])
            e, _ = _errors(res, 0, a[b, :n[b]])
            worst.add(f"{t['name']} (status {s1[b]})", e, TOL)
        worst.report(TOL)


def test_sensitivity_exports_bit_for_bit_against_the_final_slab(golden):
    tracks, _, rows, kb = _mixed(golden)
    n, n_max, rt, nv, h, _ = _pack(tracks, [], pad=0.0)
    h[h == 0.0] = 1.0
    B = len(n)
    ws = _ws(B, n_max)
    f64, i32 = dict(dtype=torch.float64, device=DEV), dict(dtype=torch.int32, device=DEV)
    out = B_._mincurv_results(B, n_max, DEV)
    sens, sens_rows = torch.full((B, 2, n_max), 7.0, **f64), torch.full((B, n_max), 7.0, **f64)
    gs, nr = torch.full((B,), 9, **i32), torch.full((B,), -9, **i32)
    B_._call("mc_mincurv_solve_batch_sens", B, n_max, _dev(n, torch.int32), _dev(rt), _dev(nv), _dev(h), kb, 2.0, None,
             B_.F_SCALE, None, *out.values(), sens, gs, sens_rows, nr, ws=ws)
    torch.cuda.synchronize()
    w, status = _read(ws), out["status"].cpu().numpy()
    sens, sens_rows, gs, nr = sens.cpu().numpy(), sens_rows.cpu().numpy(), gs.cpu().numpy(), nr.cpu().numpy()
    assert np.array_equal(gs, status)
    counts = []
    for b, t in enumerate(tracks):
        v = _slab(w, b, n[b], n_max)
        if status[b] != 0:
            assert not sens[b].any() and not sens_rows[b].any() and nr[b] == 0, t["name"]
            continue
        du, dl = F.sens_ratios(v["LU"], v["SU"], v["LL"], v["SL"])
        assert np.array_equal(sens[b, 0, :n[b]], du) and np.array_equal(sens[b, 1, :n[b]], dl), t["name"]
        assert not sens[b, :, n[b]:].any() and not sens_rows[b, n[b]:].any()
        if b in rows:
            wr, cnt = F.row_weights(v["L3"], v["S3"], v["L4"], v["S4"])
            assert np.array_equal(sens_rows[b, :n[b]], wr) and nr[b] == cnt, t["name"]
            counts.append((t["name"], cnt, float(np.abs(wr - 1.0).min())))
        else:
            assert not sens_rows[b].any() and nr[b] == 0, t["name"]
    print(f"row instances (name, strong rows, min |w - 1|): {counts}")


def test_projection_hessian_and_linear_term(golden):
    """mincurv_prox_kernel on instances that the curvature-row phase leaves alone (a limit no row reaches): the band's
    diagonal is the plain assembly's + mu bit for bit and its off-diagonals are unchanged; V_F is mu q - (H x + mu x)
    with H x through the full operator E^T E (so V_F is not the truncated band times x: the gap is printed)."""
    tracks = [track(golden(nm)["reftrack"], nm) for nm in ("handling", "synth333_kappa")]
    tracks.append(track(R.uneven_track(260, 5.0, 1), "spacing 1:5"))
    n, n_max, rt, nv, h, _ = _pack(tracks, [], pad=0.0)
    h[h == 0.0] = 1.0
    B = len(n)
    rng = np.random.default_rng(3)
    x, q = rng.standard_normal((B, n_max)) * 0.5, rng.standard_normal((B, n_max)) * 0.01
    for mu in (1e-3, 10.0):
        ws0 = _ws(B, n_max)
        st0 = torch.zeros(B, dtype=torch.int32, device=DEV)
        B_._call("mc_mincurv_setup_batch_ex", B, n_max, _dev(n, torch.int32), _dev(rt), _dev(nv), _dev(h), 2.0, None,
                 B_.F_SCALE, st0, None, ws=ws0)
        ws = _ws(B, n_max)
        out = B_._mincurv_results(B, n_max, DEV)
        B_._call("mc_mincurv_solve_batch_ex", B, n_max, _dev(n, torch.int32), _dev(rt), _dev(nv), _dev(h), 1e3, 2.0,
                 None, B_.F_SCALE, *out.values(), mu, _dev(x), _dev(q), None, None, None, None, None, None, None, 0,
                 ws=ws)
        torch.cuda.synchronize()
        w0, w = _read(ws0), _read(ws)
        for b, t in enumerate(tracks):
            assert int(out["status"][b]) == 0
            v0, v = _slab(w0, b, n[b], n_max), _slab(w, b, n[b], n_max)
            assert np.array_equal(v["HB"][:, 0], v0["HB"][:, 0] + mu), t["name"]
            assert np.array_equal(v["HB"][:, 1:], v0["HB"][:, 1:]), t["name"]
            ref = np.asarray(F.prox_linear_term(v, mu, x[b, :n[b]], q[b, :n[b]]), np.float64)
            e = float(np.abs(v["F"] - ref).max() / np.abs(ref).max())
            i = np.arange(n[b])
            band = sum(v0["HB"][:, k] * x[b, (i + k) % n[b]] + (v0["HB"][(i - k) % n[b], k] * x[b, (i - k) % n[b]]
                                                               if k else 0.0) for k in range(33))
            gap = float(np.abs(mu * q[b, :n[b]] - (band + mu * x[b, :n[b]]) - v["F"]).max() / np.abs(ref).max())
            print(f"{t['name']} mu {mu:g}: V_F {e:.2e} (bound {PROX_TOL:.0e}); truncated band instead of E^T E: {gap:.1e}")
            assert e <= PROX_TOL, (t["name"], mu, e)
