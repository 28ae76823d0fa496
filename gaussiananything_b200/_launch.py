"""Host-side launch policy shared by the networks that run on the transformer kernels (dit, dino, vae_decoder,
vae_encoder): argument formats of the GEMM entry point, its tile width, and CUDA-graph capture and replay."""
import ctypes as C
import os

import torch

from . import _lib
from ._lib import EPI_HEADS, GaGemmEpilogue


def ptr(t):
    """A tensor's device address for a ctypes call; None is NULL."""
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def round_up(x, m):
    return (x + m - 1) // m * m


def stream(device):
    """The current CUDA stream of `device` for a ctypes call."""
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


_GEMM_CFG_ENV = None
_SMS = 132                # H100 SXM: one persistent GEMM CTA per SM


def gemm_config(M, N, mode=None):
    """Tile width (ga_b200.h) from a two-term cost model checked against the H100 sweep
    (tools/sweep_gemm.py, profiles/gemm_sweep_h100.txt):

        cost(BN) = ceil(tiles(BN) / 132) * (BN + 64)

    -- waves of the persistent grid times the per-tile work (the main loop scales with BN, the +64 is the fixed
    TMA-fill / epilogue-drain share that makes wide tiles more efficient per byte).  It picks the measured winner on
    all nine DiT shapes: 192 for 4096x768 (11.3 vs 13.1 us at 256), 4096x2304, 1536x3072 and 1536x4096, 256 for
    4096x3072 and 2738x1536, 128 for the under-filled 1536x1024 GEMMs of the deployed size.
    The HEADS epilogue (whole 64-wide heads per warpgroup: 128 or 256 only) stays at 128.  GA_B200_GEMM_CFG="big,small" overrides."""
    global _GEMM_CFG_ENV
    if _GEMM_CFG_ENV is None:
        _GEMM_CFG_ENV = os.environ.get("GA_B200_GEMM_CFG", "")
    if _GEMM_CFG_ENV:
        big, small = (int(v) for v in _GEMM_CFG_ENV.split(","))
        return big if (M >= 1024 and N >= 512) else small
    rows = -(-M // 128)
    best, best_cost = 128, None
    if mode == EPI_HEADS:
        return 128                      # 256-wide HEADS tiles measured slower at M = 1536 (deployed qkv: +1.7 % per NFE)
    for bn in (128, 192, 256):
        if bn > 128 and N < bn:
            continue
        tiles = rows * -(-N // bn)
        cost = -(-tiles // _SMS) * (bn + 64)
        if best_cost is None or cost < best_cost:
            best, best_cost = bn, cost
    return best


def epilogue(mode, **fields):
    """A GaGemmEpilogue: tensors become their addresses, eps defaults to 1e-5 and every field not given is 0.  (The
    kernel reads eps only for q/k RMSNorm in GA_EPI_HEADS, rows_per_batch only with a gate or in GA_EPI_HEADS.)"""
    e = GaGemmEpilogue(mode=mode, eps=1e-5)
    for k, v in fields.items():
        setattr(e, k, v.data_ptr() if isinstance(v, torch.Tensor) else v)
    return e


def gemm(A, W, M, N, K, epi, stream, block_n=None):
    """out = epi(A [M, K] @ W [N, K]^T), both K-contiguous, at gemm_config's tile width unless block_n is given."""
    bn = gemm_config(M, N, epi.mode) if block_n is None else block_n
    _lib.check(_lib.lib().ga_gemm_bf16_tn(ptr(A), K, ptr(W), K, M, N, K, C.byref(epi), bn, stream), "ga_gemm_bf16_tn")


def capture(launches, device):
    """Runs `launches()` once eagerly (first-use kernel attributes are set there), then captures it into a new CUDA
    graph.  Returns (graph, what launches() returned inside the capture).  Tensors made here are not inference tensors,
    so the graph may be replayed from either mode."""
    with torch.inference_mode(False), torch.no_grad():
        launches()
        torch.cuda.synchronize(device)
        g = torch.cuda.CUDAGraph()
        # thread_local: another thread of the process (NCCL's watchdog under torch.distributed) may issue CUDA calls
        # while this one captures
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            out = launches()
    return g, out


class GraphCache(dict):
    """key -> (graph, static inputs, static outputs): a launch sequence captured once per input shape and replayed
    from static input buffers.  At most `capacity` graphs are kept (each owns its activations); the oldest goes first.
    `use_graph` starts from the environment variable `env_var` ("0" turns graphs off)."""

    def __init__(self, env_var, capacity=4):
        super().__init__()
        self.use_graph = os.environ.get(env_var, "1") != "0"
        self.capacity = capacity

    def run(self, key, launches, inputs):
        """launches(*inputs) -> {name: tensor}.  Eager when graphs are off or the current stream is capturing (the
        launches then go into the caller's graph); otherwise `inputs` are copied into the static buffers of `key`'s
        graph, captured on first use, and it is replayed.  The returned tensors are contiguous copies, so they stay
        valid across later calls."""
        if not self.use_graph or torch.cuda.is_current_stream_capturing():
            return {k: v.contiguous() for k, v in launches(*inputs).items()}
        slot = self.get(key)
        if slot is None:
            while len(self) >= self.capacity:
                self.pop(next(iter(self)))
            with torch.inference_mode(False):
                static = [t.clone() for t in inputs]
            g, outs = capture(lambda: launches(*static), static[0].device)
            slot = self[key] = (g, static, outs)
        g, static, outs = slot
        for s, t in zip(static, inputs):
            s.copy_(t)
        g.replay()
        return {k: v.clone(memory_format=torch.contiguous_format) for k, v in outs.items()}


def graph_switch():
    """Class attribute `use_graph` of a network that keeps its GraphCache in `_graphs`: reads and sets the cache's."""
    return property(lambda net: net._graphs.use_graph, lambda net, on: setattr(net._graphs, "use_graph", on))
