"""GPU diagnostics for the wgmma kernels (prints errors instead of asserting)."""
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


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def gemm_case(M, N, K, bn, tag=""):
    torch.manual_seed(1)
    A = torch.randn(M, K, device=dev).bfloat16()
    W = (torch.randn(N, K, device=dev) / math.sqrt(K)).bfloat16()
    out = torch.full((M, N), 7.0, device=dev, dtype=torch.float32)
    e = _lib.GaGemmEpilogue(mode=_lib.EPI_F32, out=out.data_ptr(), ld_out=N)
    rc = L.ga_gemm_bf16_tn(ptr(A), K, ptr(W), K, M, N, K, C.byref(e), bn, st)
    torch.cuda.synchronize()
    ref = A.float() @ W.float().T
    r = rel(out, ref)
    print("GEMM %s M=%d N=%d K=%d bn=%d rc=%d rel=%.3e" % (tag, M, N, K, bn, rc, r), flush=True)
    if r > 1e-3:
        d = (out - ref).abs()
        print("   max abs err %.3f at %s ; out[0,:8]=%s ref[0,:8]=%s" % (float(d.max()), divmod(int(d.argmax()), N),
              out[0, :8].tolist(), ref[0, :8].tolist()))
        rows_bad = (d.max(1).values > 1e-2).nonzero().flatten()[:16].tolist()
        cols_bad = (d.max(0).values > 1e-2).nonzero().flatten()[:16].tolist()
        print("   bad rows", rows_bad, "bad cols", cols_bad, "untouched(7.0) frac", float((out == 7.0).float().mean()))


for args in [(128, 64, 16, 64, "1 mma"), (128, 128, 64, 128, "1 k-block"), (128, 128, 256, 128, "4 k-blocks"),
             (128, 128, 1024, 128, "ring wrap"), (256, 384, 256, 128, "multi tile"), (300, 200, 136, 64, "ragged"),
             (4096, 3072, 768, 256, "big")]:
    gemm_case(*args[:4], tag=args[4])


def attn_case(B, H, Nq, Nk):
    torch.manual_seed(2)
    pq, pk = (Nq + 127) // 128 * 128, (Nk + 127) // 128 * 128
    q = torch.zeros(B * H, pq, 64, device=dev, dtype=torch.bfloat16)
    k = torch.zeros(B * H, pk, 64, device=dev, dtype=torch.bfloat16)
    vt = torch.zeros(B * H, 64, pk, device=dev, dtype=torch.bfloat16)
    q[:, :Nq] = torch.randn(B * H, Nq, 64, device=dev)
    k[:, :Nk] = torch.randn(B * H, Nk, 64, device=dev)
    vt[:, :, :Nk] = torch.randn(B * H, 64, Nk, device=dev)
    out = torch.zeros(B, Nq, H * 64, device=dev, dtype=torch.bfloat16)
    rc = L.ga_attention_bf16(ptr(q), ptr(k), ptr(vt), ptr(out), B, H, Nq, Nk, pq, pk, 0.125, 0.0, st)
    torch.cuda.synchronize()
    ref = torch.nn.functional.scaled_dot_product_attention(
        q[:, :Nq].float().view(B, H, Nq, 64), k[:, :Nk].float().view(B, H, Nk, 64),
        vt[:, :, :Nk].float().transpose(-1, -2).reshape(B, H, Nk, 64)).transpose(1, 2).reshape(B, Nq, H * 64)
    r = rel(out.float(), ref)
    print("ATTN B=%d H=%d Nq=%d Nk=%d rc=%d rel=%.3e" % (B, H, Nq, Nk, rc, r), flush=True)
    if r > 1e-2:
        print("   out[0,0,:6]=%s ref=%s ; nan frac %.3f" % (out[0, 0, :6].float().tolist(), ref[0, 0, :6].tolist(),
              float(torch.isnan(out.float()).float().mean())))
        # is it P*V or softmax?  compare with uniform-attention (mean of V)
        meanv = vt[:, :, :Nk].float().mean(-1)
        print("   rel to mean(V): %.3e" % rel(out.float().view(B, Nq, H, 64)[:, 0], meanv.view(B, H, 64)))


for a in [(1, 1, 128, 128), (1, 1, 128, 256), (1, 2, 200, 300), (2, 12, 2048, 2048)]:
    attn_case(*a)
print("debug done", flush=True)
