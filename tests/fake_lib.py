"""Recording stand-in of libmincurv_b200.so for the CPU tests of the host logic (test infrastructure, not product code).

Every entry point only checks its argument count against the ctypes signature table and returns MC_OK (4096 for the
workspace queries); nothing is computed.  The ``fake`` fixture puts it in place of the library and lets the batched
wrappers run on CPU tensors in place of device buffers, with chunks of half the batch."""
import pytest
import torch

from global_racetrajectory_optimization_b200 import _lib, batch as B_


class FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if name not in _lib._SIGS:
            raise AttributeError(name)
        res, args = _lib._SIGS[name]

        def fn(*a):
            assert len(a) == len(args), f"{name}: {len(a)} arguments passed, {len(args)} declared"
            self.calls.append((name, a))
            if name.endswith("_workspace_bytes"):
                return 4096
            return 0
        return fn


@pytest.fixture()
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_lib, "load", lambda build_if_missing=True: lib)
    monkeypatch.setattr(_lib, "check", lambda rc, what: None)
    monkeypatch.setattr(B_, "_require_cuda", lambda: None)
    monkeypatch.setattr(B_, "_f64", lambda t, name: t.contiguous())
    monkeypatch.setattr(B_, "_stream", lambda: None)
    monkeypatch.setattr(B_, "_chunk", lambda B, per_item, dev: max(1, B // 2))      # force the chunked paths
    monkeypatch.setattr(B_, "_WS", {})
    # the stand-in writes nothing: what the wrappers allocate with torch.empty would be uninitialised memory (a NaN in
    # alpha used to reach create_raceline_batch's capacity estimate from time to time)
    monkeypatch.setattr(torch, "empty", lambda *a, **k: torch.zeros(*a, **k))
    return lib
