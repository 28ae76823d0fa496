"""_launch.capture with Python's cyclic garbage collector: a dead network whose graph cache sits in a reference cycle
must not be freed inside another network's capture (freeing its CUDA graph releases memory with cudaFree, which
invalidates a capture in progress).  capture keeps the collector off while the capture is open."""
import gc

import pytest
import torch


def test_no_cyclic_gc_restores_the_collector_state():
    from gaussiananything_b200._launch import no_cyclic_gc
    was = gc.isenabled()
    try:
        gc.enable()
        with no_cyclic_gc():
            assert not gc.isenabled()
        assert gc.isenabled()
        with pytest.raises(ZeroDivisionError):
            with no_cyclic_gc():
                1 / 0
        assert gc.isenabled()
        gc.disable()
        with no_cyclic_gc():
            assert not gc.isenabled()
        assert not gc.isenabled()
    finally:
        (gc.enable if was else gc.disable)()


class _Net:
    """A graph cache whose launches close over the owner: the cycle a network with a GraphCache forms."""

    def __init__(self):
        from gaussiananything_b200._launch import GraphCache
        self._graphs = GraphCache("GA_TEST_UNUSED_GRAPH_SWITCH")
        self._graphs.use_graph = True
        self.junk = []
        self.me = self                                                 # the cycle: freed by the collector only

    def launches(self, x, v):
        from gaussiananything_b200 import _launch, _lib
        L, p, st = _lib.lib(), _launch.ptr, _launch.stream(x.device)
        self.junk.extend([{"a": [i]} for i in range(2000)])            # Python allocations during the capture
        acc = torch.zeros_like(x)
        _lib.check(L.ga_axpy(p(acc), p(x), 1.0, x.numel(), st), "axpy x")
        _lib.check(L.ga_axpy(p(acc), p(v), 2.0, x.numel(), st), "axpy v")
        return {"acc": acc}

    def __call__(self, x, v):
        return self._graphs.run(tuple(x.shape), lambda a, b: self.launches(a, b), (x, v))["acc"]


@pytest.mark.gpu
def test_no_collection_runs_inside_a_capture():
    """With the collector's threshold at 1, a collection starts at almost every allocation: many run during the
    eager pass and around the capture, none while the stream is capturing.  The dead network's cycle is freed later,
    and both graphs give the right values."""
    import weakref
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    x, v = torch.randn(64, 8, generator=g).to(dev), torch.randn(64, 8, generator=g).to(dev)
    dead = _Net()
    assert torch.equal(dead(x, v), x + 2 * v)                          # captured and replayed once
    ref = weakref.ref(dead)
    del dead                                                           # garbage, but only the cycle collector frees it
    assert ref() is not None
    seen = {"outside": 0, "capturing": 0}

    def watch(phase, info):
        if phase == "start":
            seen["capturing" if torch.cuda.is_current_stream_capturing() else "outside"] += 1
    old = gc.get_threshold()
    gc.callbacks.append(watch)
    gc.set_threshold(1)
    try:
        live = _Net()
        out = live(x, v)
        torch.cuda.synchronize()
    finally:
        gc.set_threshold(*old)
        gc.callbacks.remove(watch)
    assert seen["capturing"] == 0 and seen["outside"] > 0, seen
    assert torch.equal(out, x + 2 * v)
    gc.collect()
    torch.cuda.synchronize()
    assert ref() is None
    assert torch.equal(live(x, v), x + 2 * v)
