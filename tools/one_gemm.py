"""Run one wgmma GEMM configuration a few times (for ncu): python tools/one_gemm.py M N K cfg [gelu]."""
import ctypes as C
import math
import sys

import torch

sys.path.insert(0, ".")
from gaussiananything_b200 import _lib  # noqa: E402
from gaussiananything_b200._launch import ptr  # noqa: E402

M, N, K, cfg = (int(v) for v in sys.argv[1:5])
mode = _lib.EPI_GELU_BF16 if "gelu" in sys.argv else _lib.EPI_BF16
L = _lib.lib()
dev = torch.device("cuda:0")
st = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
A = torch.randn(M, K, device=dev).bfloat16()
W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
bias = torch.randn(N, device=dev)
out = torch.zeros(M, N, device=dev, dtype=torch.bfloat16)
e = _lib.GaGemmEpilogue(mode=mode, bias=bias.data_ptr(), out=out.data_ptr(), ld_out=N)
for _ in range(4):
    rc = L.ga_gemm_bf16_tn(ptr(A), K, ptr(W), K, M, N, K, C.byref(e), cfg, st)
    assert rc == 0, rc
torch.cuda.synchronize()
