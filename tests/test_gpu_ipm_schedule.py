"""GPU tests (-m gpu) of the sliced schedule of the box-phase interior-point solver (mc_mincurv_pdip_batch, DESIGN.md
section 3.3): every instance first runs for at most K iterations and is parked if it has not stopped, and CTAs that find no
unstarted instance resume the parked ones longest first.  Only the order of the work changes, so alpha, status and iters
must be bitwise those of the unsliced schedule (MC_DEBUG_PDIP_SLICE=0) -- on every fixture in a ragged batch, with incoming non-zero statuses,
instances that stop before K, instances stopped by the iteration cap, and more instances than resident CTAs."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from global_racetrajectory_optimization_b200 import _lib, batch as B_, synth  # noqa: E402

GOLDEN = ["berlin", "berlin500_jitter_a", "berlin500_jitter_b", "handling", "modena", "synth1000", "synth128",
          "synth160_kappa", "synth200", "synth2000", "synth333", "synth333_kappa", "synth500", "synth500_narrow"]


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _ragged(tracks, w_veh):
    dev = torch.device("cuda")
    n = [t.shape[0] for t in tracks]
    rt = np.zeros((len(tracks), max(n), 4))
    for b, t in enumerate(tracks):
        rt[b, :n[b]] = t
    rt = torch.tensor(rt, device=dev)
    npts = torch.tensor(n, dtype=torch.int32, device=dev)
    _, _, nv, h = B_.calc_splines_batch(rt, n_pts=npts, want_coeffs=False)
    return rt, nv, h, npts, torch.tensor(w_veh, dtype=torch.float64, device=dev)


def _pdip(batch, slice_k, monkeypatch, status_in=None):
    """setup, then (optionally) overwrite some statuses, then the box phase with MC_DEBUG_PDIP_SLICE=slice_k"""
    rt, nv, h, npts, wv = batch
    B, n_max = rt.shape[:2]
    lib = _lib.load()
    p, s = B_._ptr, B_._stream()
    ws = B_._workspace("mincurv", lib.mc_mincurv_workspace_bytes(B, n_max), rt.device)
    st = torch.empty((B,), dtype=torch.int32, device=rt.device)
    it = torch.full((B,), -7, dtype=torch.int32, device=rt.device)
    alpha = torch.full((B, n_max), np.nan, dtype=torch.float64, device=rt.device)
    _lib.check(lib.mc_mincurv_setup_batch_ex(B, n_max, p(npts), p(rt), p(nv), p(h), 0.0, p(wv), B_.F_SCALE, p(st), p(ws),
                                             ws.numel(), s), "setup")
    if status_in is not None:
        st[status_in] = 1
    monkeypatch.setenv("MC_DEBUG_PDIP_SLICE", str(slice_k))
    _lib.check(lib.mc_mincurv_pdip_batch(B, n_max, p(npts), p(alpha), p(st), p(it), p(ws), ws.numel(), s), "pdip")
    torch.cuda.synchronize()
    return dict(alpha=alpha.cpu().numpy(), status=st.cpu().numpy(), iters=it.cpu().numpy())


def _assert_same(a, b, what):
    for k in ("alpha", "status", "iters"):
        assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), (what, k)


def _fixture_batch(golden, copies, rng):
    g = [golden(name) for name in GOLDEN]
    order = rng.permutation(copies * len(g))
    tracks = [g[i % len(g)]["reftrack"] for i in order]
    w_veh = [float(g[i % len(g)]["w_veh"]) for i in order]
    return _ragged(tracks, w_veh)


@pytest.mark.parametrize("k", [4, 6, 8, 12])
def test_fixtures_ragged_with_incoming_status_sliced_equals_one_launch(golden, monkeypatch, k):
    """every fixture, ragged n from 128 to 2000, shuffled, 20 copies (280 instances on 132 SMs x 1 CTA: three waves),
    every seventh instance entering with status 1; K = 12 lets part of the batch stop before it"""
    monkeypatch.setenv("MC_DEBUG_PDIP_CTAS_PER_SM", "1")
    batch = _fixture_batch(golden, 20, np.random.default_rng(3))
    B = batch[0].shape[0]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert B > sms
    bad = torch.arange(0, B, 7, device=batch[0].device)
    ref = _pdip(batch, 0, monkeypatch, bad)
    got = _pdip(batch, k, monkeypatch, bad)
    _assert_same(got, ref, f"K={k}")
    it, st = ref["iters"], ref["status"]
    assert np.all(st[bad.cpu().numpy()] == 1) and np.all(it[bad.cpu().numpy()] == 0)
    run = np.ones(B, bool)
    run[bad.cpu().numpy()] = False
    assert np.any(it[run] > k), "nothing was parked"
    if k == 12:
        assert np.any(it[run] <= k), "nothing stopped within the slice"
    print(f"K={k}: {B} instances, iterations {np.bincount(it[run]).nonzero()[0].tolist()}")


def test_iteration_cap_sliced_equals_one_launch(golden, monkeypatch):
    """a tolerance no instance reaches: every instance runs to max_iter (status 2) through both launches"""
    monkeypatch.setenv("MC_DEBUG_PDIP_CTAS_PER_SM", "1")
    monkeypatch.setenv("MC_DEBUG_PDIP_MU_REL", "1e-300")
    batch = _fixture_batch(golden, 12, np.random.default_rng(5))
    ref = _pdip(batch, 0, monkeypatch)
    got = _pdip(batch, 6, monkeypatch)
    _assert_same(got, ref, "cap")
    capped = ref["status"] == 2
    assert capped.sum() > len(capped) // 2 and np.all(ref["iters"][capped] == 40), (np.unique(ref["status"]), np.unique(ref["iters"]))


def test_more_instances_than_resident_ctas_sliced_equals_one_launch(monkeypatch):
    """full occupancy, three instances per resident CTA, ragged n from 100 to 400; the sliced run twice (the bucket
    order inside a bucket depends on timing, the results must not)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B = 3 * sms * 8
    rng = np.random.default_rng(11)
    ns = rng.integers(100, 400, size=B)
    tracks = [synth.make_track(int(1000 + b), int(n)) for b, n in enumerate(ns)]
    batch = _ragged(tracks, list(rng.uniform(1.6, 3.0, size=B)))
    ref = _pdip(batch, 0, monkeypatch)
    assert (ref["status"] == 0).sum() > B // 2 and ref["iters"].max() > 6
    for _ in range(2):
        _assert_same(_pdip(batch, 6, monkeypatch), ref, "full occupancy")
