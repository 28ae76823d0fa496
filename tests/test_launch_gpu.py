"""_launch.GraphCache, the per-shape CUDA-graph cache of the DINOv2 encoder and the VAE encoder and decoder, on a
launch sequence of two library kernels: one capture per key, replay from static inputs, copies that outlive later
calls, oldest-first eviction, calls from torch.inference_mode, and eager launches into a caller's own capture."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


class Launches:
    """acc = x + 2 v (ga_axpy twice into a fresh fp32 buffer), y = bf16(acc) (ga_f32_to_bf16); counts its calls."""

    def __init__(self):
        self.calls = 0

    def __call__(self, x, v):
        from gaussiananything_b200 import _launch, _lib
        L, p, st = _lib.lib(), _launch.ptr, _launch.stream(x.device)
        self.calls += 1
        acc = torch.zeros_like(x)
        y = torch.empty(x.shape, device=x.device, dtype=torch.bfloat16)
        _lib.check(L.ga_axpy(p(acc), p(x), 1.0, x.numel(), st), "axpy x")
        _lib.check(L.ga_axpy(p(acc), p(v), 2.0, x.numel(), st), "axpy v")
        _lib.check(L.ga_f32_to_bf16(p(acc), p(y), x.numel(), st), "f32_to_bf16")
        return {"acc": acc, "y": y, "acc_col0": acc[:, 0]}           # the last one is a strided view


def _inputs(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, 8, generator=g).to(DEV), torch.randn(n, 8, generator=g).to(DEV)


def _check(out, x, v):
    want = x + 2 * v
    assert torch.equal(out["acc"], want) and torch.equal(out["y"], want.bfloat16())
    assert torch.equal(out["acc_col0"], want[:, 0]) and out["acc_col0"].is_contiguous()


def test_graph_cache_captures_once_per_key_and_replays_new_inputs():
    from gaussiananything_b200._launch import GraphCache
    cache, fn = GraphCache("GA_B200_TEST_LAUNCH_GRAPH"), Launches()
    assert cache.use_graph
    x1, v1 = _inputs(256, 1)
    x2, v2 = _inputs(256, 2)
    with torch.inference_mode():                                    # capture from inference mode
        first = cache.run(256, fn, (x1, v1))
    assert fn.calls == 2 and 256 in cache                           # eager warm-up + capture
    g = cache[256][0]
    assert isinstance(g, torch.cuda.CUDAGraph)
    second = cache.run(256, fn, (x2, v2))                           # replay, new inputs
    with torch.inference_mode():
        x3, v3 = _inputs(256, 3)                                    # inference tensors as inputs
        third = cache.run(256, fn, (x3, v3))
    torch.cuda.synchronize()
    assert fn.calls == 2 and cache[256][0] is g                     # no further capture
    _check(first, x1, v1)                                           # earlier results survive later replays
    _check(second, x2, v2)
    _check(third, x3, v3)


def test_graph_cache_evicts_the_oldest_key_at_capacity():
    from gaussiananything_b200._launch import GraphCache
    cache, fn = GraphCache("GA_B200_TEST_LAUNCH_GRAPH", capacity=2), Launches()
    ins = {n: _inputs(n, n) for n in (128, 256, 384)}
    for n in (128, 256):
        cache.run(n, fn, ins[n])
    assert set(cache) == {128, 256} and fn.calls == 4
    out = cache.run(384, fn, ins[384])
    assert set(cache) == {256, 384} and fn.calls == 6
    again = cache.run(128, fn, ins[128])                            # evicted: captured anew, 256 goes
    assert set(cache) == {384, 128} and fn.calls == 8
    torch.cuda.synchronize()
    _check(out, *ins[384])
    _check(again, *ins[128])


def test_graph_cache_off_and_inside_a_callers_capture_launches_eagerly(monkeypatch):
    from gaussiananything_b200._launch import GraphCache
    monkeypatch.setenv("GA_B200_TEST_LAUNCH_GRAPH", "0")
    off = GraphCache("GA_B200_TEST_LAUNCH_GRAPH")
    monkeypatch.delenv("GA_B200_TEST_LAUNCH_GRAPH")
    fn = Launches()
    x, v = _inputs(128, 4)
    assert not off.use_graph
    _check(off.run(128, fn, (x, v)), x, v)
    assert fn.calls == 1 and not off
    # the caller captures: run() enqueues its launches into the caller's graph and captures nothing of its own
    cache, fn = GraphCache("GA_B200_TEST_LAUNCH_GRAPH"), Launches()
    sx, sv = x.clone(), v.clone()
    outer = torch.cuda.CUDAGraph()
    with torch.cuda.graph(outer, capture_error_mode="thread_local"):
        out = cache.run(128, fn, (sx, sv))
    assert fn.calls == 1 and not cache
    x2, v2 = _inputs(128, 5)
    sx.copy_(x2)
    sv.copy_(v2)
    outer.replay()
    torch.cuda.synchronize()
    _check(out, x2, v2)
