"""GPU sweep of the wgmma GEMM tile widths on the DiT shapes (prints a table)."""
import ctypes as C
import math
import sys

import torch

sys.path.insert(0, ".")
from gaussiananything_b200 import _lib  # noqa: E402
from gaussiananything_b200._launch import ptr  # noqa: E402

L = _lib.lib()
dev = torch.device("cuda:0")
st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
shapes = [(4096, 768, 768), (4096, 2304, 768), (4096, 3072, 768), (4096, 768, 3072),
          (1536, 1024, 1024), (1536, 3072, 1024), (1536, 4096, 1024), (1536, 1024, 4096), (2738, 1536, 1024)]
cfgs = [64, 128, 192, 256]
MODE = _lib.EPI_GELU_BF16 if "gelu" in sys.argv else (_lib.EPI_RESID_GATE_F32 if "resid" in sys.argv else _lib.EPI_BF16)
for (M, N, K) in shapes:
    torch.manual_seed(0)
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    bias = torch.randn(N, device=dev)
    ref = A.float() @ W.float().T + bias
    if MODE == _lib.EPI_GELU_BF16:
        ref = torch.nn.functional.gelu(ref)
    row = []
    for cfg in cfgs:
        if MODE == _lib.EPI_RESID_GATE_F32:
            out = torch.zeros(M, N, device=dev, dtype=torch.float32)
            gate = torch.ones(2, N, device=dev)
            e = _lib.GaGemmEpilogue(mode=MODE, bias=bias.data_ptr(), out=out.data_ptr(), ld_out=N, gate=gate.data_ptr(),
                                   gate_ld=N, rows_per_batch=M // 2)
        else:
            out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
            e = _lib.GaGemmEpilogue(mode=MODE, bias=bias.data_ptr(), out=out.data_ptr(), ld_out=N)
        rc = L.ga_gemm_bf16_tn(ptr(A), K, ptr(W), K, M, N, K, C.byref(e), cfg, st)
        torch.cuda.synchronize()
        if rc != 0:
            row.append("%5d: rc=%d" % (cfg, rc))
            continue
        err = float((out.float() - ref).norm() / ref.norm())
        for _ in range(3 if MODE != _lib.EPI_RESID_GATE_F32 else 0):
            L.ga_gemm_bf16_tn(ptr(A), K, ptr(W), K, M, N, K, C.byref(e), cfg, st)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            L.ga_gemm_bf16_tn(ptr(A), K, ptr(W), K, M, N, K, C.byref(e), cfg, st)
        b.record(); b.synchronize()
        us = a.elapsed_time(b) * 1e3 / 20
        row.append("%5d: %6.1fus %5.0fTF%s" % (cfg, us, 2.0 * M * N * K / us / 1e6, "" if err < 5e-3 else " ERR%.1e" % err))
    # yardstick (not the product path): cuBLAS through torch.matmul on the same operands, bf16 output, no epilogue
    if MODE == _lib.EPI_BF16:
        Wt = W.t().contiguous()
        for _ in range(3):
            torch.matmul(A, Wt)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            torch.matmul(A, Wt)
        b.record(); b.synchronize()
        us = a.elapsed_time(b) * 1e3 / 20
        row.append("cuBLAS: %6.1fus %5.0fTF" % (us, 2.0 * M * N * K / us / 1e6))
    print("M=%d N=%d K=%d | " % (M, N, K) + " | ".join(row), flush=True)
