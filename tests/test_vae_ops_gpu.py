"""Building-block kernels of the VAE decode path (SURVEY 8f row N1, include/ga_b200.h "VAE decode path") against the
oracle's functions (oracle/vae_decoder_oracle.py) and plain torch, through the C ABI."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def _p(t):
    return C.c_void_p(t.data_ptr() if t is not None else 0)


def _env():
    from gaussiananything_b200 import _lib
    dev = torch.device("cuda:0")
    return _lib.lib(), dev, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


@pytest.mark.parametrize("R,D", [(77, 64), (300, 768), (33, 1024)])
def test_layernorm_modulate(R, D):
    L, dev, st = _env()
    torch.manual_seed(R + D)
    x = torch.randn(R, D, device=dev) * 2 + 0.3
    mod = torch.randn(R, 6 * D, device=dev) * 0.3                 # per-token adaLN table, as DiTBlock2 produces it
    shift, scale = mod[:, :D], mod[:, D:2 * D]
    out = torch.zeros(R, D, device=dev, dtype=torch.bfloat16)
    assert L.ga_layernorm_modulate(_p(x), None, None, _p(shift), _p(scale), 6 * D, 1, _p(out), R, D, 1e-6, st) == 0
    ref = F.layer_norm(x, (D,), None, None, 1e-6) * (1 + scale) + shift
    assert rel(out.float(), ref) < 3e-3
    # PreNorm flavour: affine LayerNorm, no modulation
    w, b = torch.rand(D, device=dev) + 0.5, torch.randn(D, device=dev) * 0.1
    assert L.ga_layernorm_modulate(_p(x), _p(w), _p(b), None, None, 0, 1, _p(out), R, D, 1e-5, st) == 0
    assert rel(out.float(), F.layer_norm(x, (D,), w, b, 1e-5)) < 3e-3
    # per batch item (rows_per_batch > 1) shares one modulation row
    rpb = 11
    nb = (R + rpb - 1) // rpb
    modb = torch.randn(nb, 2 * D, device=dev) * 0.3
    assert L.ga_layernorm_modulate(_p(x), None, None, _p(modb[:, :D]), _p(modb[:, D:]), 2 * D, rpb, _p(out), R, D, 1e-6, st) == 0
    idx = torch.arange(R, device=dev) // rpb
    ref = F.layer_norm(x, (D,), None, None, 1e-6) * (1 + modb[idx, D:]) + modb[idx, :D]
    assert rel(out.float(), ref) < 3e-3


def test_thin_linear():
    L, dev, st = _env()
    torch.manual_seed(3)
    R, D, Cn = 203, 768, 13
    x = torch.randn(R, D, device=dev)
    W, b = torch.randn(Cn, D, device=dev) * 0.05, torch.randn(Cn, device=dev)
    y = torch.zeros(R, Cn, device=dev)
    assert L.ga_thin_linear(_p(x), None, None, 1, _p(W), _p(b), _p(y), R, D, Cn, 0.0, st) == 0        # conv_sr
    assert rel(y, F.linear(F.silu(x), W, b)) < 1e-5
    lw, lb = torch.rand(D, device=dev) + 0.5, torch.randn(D, device=dev) * 0.1
    assert L.ga_thin_linear(_p(x), _p(lw), _p(lb), 0, _p(W), _p(b), _p(y), R, D, Cn, 1e-5, st) == 0   # PreNorm head
    assert rel(y, F.linear(F.layer_norm(x, (D,), lw, lb, 1e-5), W, b)) < 1e-5


@pytest.mark.parametrize("S,Lq,H", [(5, 4, 1), (37, 5, 2), (64, 9, 12), (3, 16, 2)])
def test_micro_attention(S, Lq, H):
    from oracle.dit_oracle import rmsnorm
    L, dev, st = _env()
    torch.manual_seed(S * Lq)
    Cw = H * 64
    qkv = (torch.randn(S * Lq, 3 * Cw, device=dev) * 1.5).bfloat16()
    qn, kn = torch.rand(64, device=dev) + 0.5, torch.rand(64, device=dev) + 0.5
    out = torch.zeros(S * Lq, Cw, device=dev, dtype=torch.bfloat16)
    assert L.ga_micro_attention_bf16(_p(qkv), _p(qn), _p(kn), _p(out), S, Lq, H, 1e-5, st) == 0
    t = qkv.float().view(S, Lq, 3, H, 64).permute(2, 0, 3, 1, 4)              # K, S, H, L, d
    q, k = rmsnorm(t[0], qn), rmsnorm(t[1], kn)
    ref = F.scaled_dot_product_attention(q, k, t[2]).transpose(1, 2).reshape(S * Lq, Cw)
    assert rel(out.float(), ref) < 4e-3


def test_micro_seq_build():
    L, dev, st = _env()
    torch.manual_seed(0)
    D, S0, f1, f2 = 64, 10, 8, 4
    tok = torch.randn(S0, D, device=dev)
    q1, q2 = torch.randn(f1, D, device=dev), torch.randn(f2, D, device=dev)
    seq1 = torch.zeros(S0, 1 + f1, D, device=dev)
    assert L.ga_micro_seq_build(_p(tok), 0, _p(q1), _p(seq1), S0, f1, D, st) == 0
    assert torch.equal(seq1, torch.cat([tok[:, None], q1[None].expand(S0, -1, -1)], 1))
    S1 = S0 * f1                                               # next stage: the children of stage 1 are the parents
    seq2 = torch.zeros(S1, 1 + f2, D, device=dev)
    assert L.ga_micro_seq_build(_p(seq1), f1, _p(q2), _p(seq2), S1, f2, D, st) == 0
    parents = seq1[:, 1:].reshape(S1, D)
    assert torch.equal(seq2, torch.cat([parents[:, None], q2[None].expand(S1, -1, -1)], 1))


def test_surfel_cascade_pack_matches_oracle_activations():
    from oracle import vae_decoder_oracle as vo
    L, dev, st = _env()
    torch.manual_seed(1)
    act = vo.Activations(0.45)
    N, f, skip = 50, 8, 0.1
    base_pre = torch.randn(N, 13, device=dev) * 2
    xyz = (torch.rand(N, 3, device=dev) - 0.5) * 0.8
    g = torch.zeros(N, 13, device=dev)
    sf = float(act.scaling_factor)
    assert L.ga_surfel_cascade_pack(_p(base_pre), 0, None, _p(xyz), 3, 1, 0.45 * 0.5 * skip, sf, _p(g), None, N, st) == 0
    ref = act.pack(act.offset(base_pre[:, :3]) * skip + xyz, base_pre)
    assert rel(g, ref) < 1e-5
    # child level: residual on the parent's pre-activation, offset from the parent's position (no skip weight)
    res = torch.randn(N * f, 13, device=dev) * 2
    gc, pre = torch.zeros(N * f, 13, device=dev), torch.zeros(N * f, 13, device=dev)
    assert L.ga_surfel_cascade_pack(_p(res), 0, _p(base_pre), _p(g), 13, f, 0.45 * 0.5, sf, _p(gc), _p(pre), N * f, st) == 0
    pre_ref = res.view(N, f, 13) + base_pre[:, None]
    pos_ref = act.offset(res.view(N, f, 13)[..., :3]) + g[:, None, :3]
    assert rel(pre, pre_ref.reshape(N * f, 13)) < 1e-6
    assert rel(gc, act.pack(pos_ref, pre_ref).reshape(N * f, 13)) < 1e-5
    assert torch.allclose(gc[:, 6:10].norm(dim=-1), torch.ones(N * f, device=dev), atol=1e-5)
    # the same with the residuals still in the [N, 1+f] sequence layout (row 0 of every sequence is the parent token)
    res_seq = torch.randn(N, 1 + f, 13, device=dev)
    res_seq[:, 1:] = res.view(N, f, 13)
    gc2 = torch.zeros_like(gc)
    assert L.ga_surfel_cascade_pack(_p(res_seq), 1, _p(base_pre), _p(g), 13, f, 0.45 * 0.5, sf, _p(gc2), None, N * f, st) == 0
    assert torch.equal(gc2, gc)


def test_silu_to_bf16():
    L, dev, st = _env()
    x = torch.randn(1000, device=dev) * 3
    y = torch.zeros(1000, device=dev, dtype=torch.bfloat16)
    assert L.ga_silu_to_bf16(_p(x), _p(y), 1000, st) == 0
    assert rel(y.float(), F.silu(x)) < 3e-3
