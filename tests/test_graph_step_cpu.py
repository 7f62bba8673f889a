"""The workspace cache and the CUDA-graph step of ``ddpo_b200.ops`` on the host: CPU tensors stand for the workspaces
and fakes for torch's graph capture, so what is captured, replayed, restored and kept alive is visible without a GPU."""
import gc
import weakref

import pytest
import torch

from ddpo_b200 import ops


class _FakeGraph:
    def __init__(self):
        self.replays = 0

    def replay(self):
        self.replays += 1


class _Capture:
    """stands for ``torch.cuda.graph(g)``: counts the captures"""
    count = 0

    def __init__(self, g):
        pass

    def __enter__(self):
        _Capture.count += 1

    def __exit__(self, *exc):
        return False


@pytest.fixture()
def fake_cuda(monkeypatch):
    monkeypatch.setattr(ops, "_WORKSPACES", {kind: {} for kind in ops._WORKSPACES})
    monkeypatch.setattr(torch.cuda, "CUDAGraph", _FakeGraph)
    monkeypatch.setattr(torch.cuda, "graph", _Capture)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    _Capture.count = 0


def test_workspace_grows_only_when_too_small(fake_cuda):
    a = ops._workspace("wgrad", "cpu", 10)
    assert a.dtype == torch.float32 and a.numel() == 1 << 20
    assert ops._workspace("wgrad", "cpu", 1 << 20) is a
    b = ops._workspace("wgrad", "cpu", (1 << 20) + 5)
    assert b is not a and b.numel() == (1 << 20) + 5
    assert ops._workspace("wgrad", "cpu", 7) is b
    # kinds are separate; the stem kernels ask for exactly what they need
    c = ops._workspace("conv_in_wgrad", "cpu", 7, min_floats=0)
    assert c.numel() == 7 and ops._workspace("wgrad", "cpu", 1) is b
    assert ops._workspace("conv_in_wgrad", "cpu", 9, min_floats=0).numel() == 9


def test_graph_step_keeps_the_captured_workspace_alive(fake_cuda):
    calls = []

    def body():
        calls.append(ops._workspace("wgrad", "cpu", 10))

    captured = ops.graph_step(None, "s", body, True)
    seen = weakref.ref(calls[-1])
    calls.clear()
    grown = ops._workspace("wgrad", "cpu", (1 << 20) + 1)   # a later step at a larger shape replaces it in the cache
    gc.collect()
    assert seen() is not None and seen() is not grown       # the graph may still write to it
    captured = ops.graph_step(captured, "s", body, True)    # replays only: holds on to the same tensor
    assert captured[1].replays == 2 and _Capture.count == 1 and seen() is not None
    del captured
    gc.collect()
    assert seen() is None                                   # nothing else keeps a superseded workspace


def test_graph_step_replays_until_the_signature_changes(fake_cuda):
    runs = []
    captured = ops.graph_step(None, ("g", 1), lambda: runs.append(1), True)
    assert len(runs) == 2 and _Capture.count == 1 and captured[1].replays == 1     # warm-up + capture, then replay
    first = captured[1]
    for _ in range(3):
        captured = ops.graph_step(captured, ("g", 1), lambda: runs.append(1), True)
    assert len(runs) == 2 and _Capture.count == 1 and captured[1] is first and first.replays == 4
    captured = ops.graph_step(captured, ("g", 2), lambda: runs.append(1), True)
    assert len(runs) == 4 and _Capture.count == 2 and captured[1] is not first and captured[1].replays == 1


def test_graph_step_restores_the_protected_tensor_after_the_warm_up(fake_cuda):
    acc = torch.arange(6, dtype=torch.float32)
    seen = []

    def body():
        acc.add_(100.0)
        seen.append(acc.clone())

    ops.graph_step(None, 0, body, True, protect=acc)
    # the warm-up adds 100, which is undone: the (fake) capture, which runs the body, starts from 0..5 again
    assert len(seen) == 2 and all(torch.equal(s, torch.arange(6) + 100.0) for s in seen)


def test_graph_step_disabled_runs_the_body_once(fake_cuda):
    runs = []
    assert ops.graph_step(None, 0, lambda: runs.append(1), False) is None
    held = ("sig", _FakeGraph(), [])
    assert ops.graph_step(held, 1, lambda: runs.append(1), False) is held
    assert runs == [1, 1] and _Capture.count == 0 and held[1].replays == 0
