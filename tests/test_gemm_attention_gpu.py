"""The tensor-core GEMM (ga_gemm_bf16_tn) and flash attention (ga_attention_bf16, ga_attention_causal_bf16) against
the fp64 references of tests/tc_ref.py, element by element, at the shapes, epilogues, tile widths and edges the
networks use.  Every call:
  - reads operands whose padding is hostile: A's and W's columns between K and lda / ldw and their rows past M / N
    are NaN; K rows past Nk are +-30, Vt columns past Nk 1e4, Q rows past Nq 30;
  - writes into sentinel-filled buffers with slack before, after and between rows (ld_out > N, once with
    ld_out % 4 == 0 and once odd, which takes the scalar stores), and for HEADS the tokens past rows_per_batch and
    the buffers of the parts the columns do not reach; everything outside the written region is compared bitwise;
  - is repeated and must give the same bits.
TC_REF_REPORT=<file> records the largest |err| / bound of every check (see tests/tc_ref.py)."""
import ctypes as C

import pytest
import torch

from tests import tc_ref as tr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

BLOCK_N = (64, 128, 192, 256)


def _lib():
    from gaussiananything_b200 import _lib
    return _lib, _lib.lib()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _round_up(x, m):
    return (x + m - 1) // m * m


def _ld(n, kind):
    """ld_out > n: 'vec' keeps ld_out % 4 == 0, 'odd' forces the scalar stores."""
    return _round_up(n + 1, 4) if kind == "vec" else (n + 1) | 1


def _bits(t):
    return t.view(torch.int32 if t.dtype == torch.float32 else torch.int16)


def _gemm_call(Abuf, lda, Wbuf, ldw, M, N, K, epi, bn):
    _, L = _lib()
    rc = L.ga_gemm_bf16_tn(C.c_void_p(Abuf.data_ptr()), lda, C.c_void_p(Wbuf.data_ptr()), ldw, M, N, K, C.byref(epi),
                           bn, _st())
    assert rc == 0, rc
    torch.cuda.synchronize()


def run_gemm(mode, M, N, K, bn, ld_kind="vec", gate_kind=None, group="gemm", seed=0, D_gate=None):
    """One elementwise-epilogue GEMM checked against fp64; returns max |err| / bound.  gate_kind (RESID_GATE):
    'batch' (rows_per_batch 23, straddling the 16-row warp slices), 'token' (rows_per_batch 1, the gate a column
    slice of a wider table, as the VAE decoder's per-token adaLN), 'layerscale' (one [N] gate for all rows,
    rows_per_batch = M, as DINOv2), or 'none0' / 'none1' / 'noneM' (NULL gate with rows_per_batch 0, 1 or M)."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(seed * 7919 + M * 31 + N * 17 + K + mode)
    Abuf, A, lda = tr.hostile_operand(M, K, dev, gen)
    Wbuf, W, ldw = tr.hostile_operand(N, K, dev, gen, scale=K ** -0.5)
    bias = (torch.randn(N, generator=gen) * 0.5).to(dev)
    n_out = N // 2 if mode == tr.GEGLU else N
    ld = _ld(n_out, ld_kind)
    f32 = mode in (tr.F32_OUT, tr.RESID_GATE)
    out = tr.GuardBuf((M + 3, ld), torch.float32 if f32 else torch.bfloat16, dev)
    written = tr.region(out.shape, slice(0, M), slice(0, n_out), device=dev)
    fields = dict(bias=bias.data_ptr(), out=out.t.data_ptr(), ld_out=ld)
    x0 = gate = table = None
    if mode == tr.RESID_GATE:
        x0 = torch.randn(M, N, generator=gen).to(dev)
        out.t[:M, :N] = x0
        if gate_kind == "batch":
            rpb = 23
            nb = -(-M // rpb)
            table = torch.randn(nb, N + 5, generator=gen).to(dev)
            gate = table[:, :N].repeat_interleave(rpb, 0)[:M]
            fields.update(gate=table.data_ptr(), gate_ld=N + 5, rows_per_batch=rpb)
        elif gate_kind == "token":
            mw = D_gate if D_gate else 3 * N + 8
            off = mw - N - 3                                   # a column slice, not 16-byte aligned
            table = torch.randn(M, mw, generator=gen).to(dev)
            gate = table[:, off:off + N]
            fields.update(gate=table.data_ptr() + 4 * off, gate_ld=mw, rows_per_batch=1)
        elif gate_kind == "layerscale":
            table = (torch.rand(N, generator=gen) * 2.0 - 1.0).to(dev)
            gate = table[None, :].expand(M, N)
            fields.update(gate=table.data_ptr(), gate_ld=N, rows_per_batch=M)
        else:
            fields.update(rows_per_batch={"none0": 0, "none1": 1, "noneM": M}[gate_kind])
    epi = lib.GaGemmEpilogue(mode=mode, eps=1e-5, **fields)
    _gemm_call(Abuf, lda, Wbuf, ldw, M, N, K, epi, bn)
    got = out.t[:M, :n_out].clone()
    Y, S = tr.gemm_ref(A, W, bias)
    ref, tol = tr.epilogue_ref(mode, Y, S, x0=x0, gate=gate)
    what = "mode %d M=%d N=%d K=%d block_n=%d ld_out=%d gate=%s" % (mode, M, N, K, bn, ld, gate_kind)
    worst, msg = tr.check(got, ref, tol, group, what)
    assert msg == "", msg
    ok, gmsg = out.intact(written)
    assert ok, what + ": " + gmsg
    del Y, S, ref, tol
    if mode == tr.RESID_GATE:
        out.t[:M, :N] = x0
    _gemm_call(Abuf, lda, Wbuf, ldw, M, N, K, epi, bn)
    assert torch.equal(_bits(out.t[:M, :n_out]), _bits(got)), what + ": a repeat gave different bits"
    return worst


def run_heads(bn, variant, norm, use_bias, heads, rpb, B=2, K=200, group="heads", seed=0):
    """One HEADS GEMM: variant 'qkv' (first_part 0, q k v), 'q' (first_part 0, q only), 'kv' (first_part 1, k v).
    All three buffers are always passed: the ones the columns do not reach must stay untouched."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    first_part, parts = {"qkv": (0, 3), "q": (0, 1), "kv": (1, 2)}[variant]
    N, M, tp = parts * 64 * heads, B * rpb, _round_up(rpb, 128)
    gen = torch.Generator().manual_seed(seed * 7919 + heads * 1000 + rpb + parts)
    Abuf, A, lda = tr.hostile_operand(M, K, dev, gen)
    Wbuf, W, ldw = tr.hostile_operand(N, K, dev, gen, scale=K ** -0.5)
    bias = (torch.randn(N, generator=gen) * 0.3).to(dev) if use_bias else None
    qn = (torch.rand(64, generator=gen) + 0.5).to(dev) if norm else None
    kn = (torch.rand(64, generator=gen) + 0.5).to(dev) if norm else None
    bufs = {"q": tr.GuardBuf((B * heads, tp, 64), torch.bfloat16, dev),
            "k": tr.GuardBuf((B * heads, tp, 64), torch.bfloat16, dev),
            "v": tr.GuardBuf((B * heads, 64, tp), torch.bfloat16, dev)}
    epi = lib.GaGemmEpilogue(mode=tr.HEADS, bias=bias.data_ptr() if use_bias else 0, q=bufs["q"].t.data_ptr(),
                             k=bufs["k"].t.data_ptr(), vt=bufs["v"].t.data_ptr(), qn_w=qn.data_ptr() if norm else 0,
                             kn_w=kn.data_ptr() if norm else 0, heads=heads, first_part=first_part, tok_pitch=tp,
                             rows_per_batch=rpb, eps=1e-5)
    _gemm_call(Abuf, lda, Wbuf, ldw, M, N, K, epi, bn)
    Y, S = tr.gemm_ref(A, W, bias)
    refs = tr.heads_ref(Y, S, B, rpb, heads, first_part, qn_w=qn, kn_w=kn)
    what = "HEADS %s block_n=%d norm=%d bias=%d heads=%d rows_per_batch=%d tok_pitch=%d" % (
        variant, bn, norm, use_bias, heads, rpb, tp)
    worst = 0.0
    got, written = {}, {}
    for name, g in bufs.items():
        if name not in refs:
            written[name] = None
            continue
        if name == "v":
            view = g.t.view(B, heads, 64, tp)[..., :rpb]
            written[name] = tr.region(g.shape, slice(None), slice(None), slice(0, rpb), device=dev)
        else:
            view = g.t.view(B, heads, tp, 64)[:, :, :rpb]
            written[name] = tr.region(g.shape, slice(None), slice(0, rpb), device=dev)
        got[name] = view.clone()
        w, msg = tr.check(view, *refs[name], group, what + " part " + name)
        assert msg == "", msg
        worst = max(worst, w)
    for name, g in bufs.items():
        ok, gmsg = g.intact(written[name])
        assert ok, what + " buffer " + name + ": " + gmsg
    _gemm_call(Abuf, lda, Wbuf, ldw, M, N, K, epi, bn)
    for name, v in got.items():
        view = bufs[name].t.view(B, heads, 64, tp)[..., :rpb] if name == "v" else bufs[name].t.view(B, heads, tp, 64)[:, :, :rpb]
        assert torch.equal(_bits(view), _bits(v)), what + ": a repeat gave different bits in " + name
    return worst


# ---- GEMM edge matrix ----------------------------------------------------------------------------------------------

EDGE_SHAPES = [(1, 64, 8), (15, 96, 72), (17, 102, 136), (129, 190, 64), (200, 500, 1000), (1000, 768, 3072)]
EDGE_MODES = [(tr.BF16_OUT, None), (tr.GELU_OUT, None), (tr.F32_OUT, None), (tr.GEGLU, None),
              (tr.RESID_GATE, "batch"), (tr.RESID_GATE, "token"), (tr.RESID_GATE, "none0")]


@pytest.mark.parametrize("ld_kind", ["vec", "odd"])
@pytest.mark.parametrize("bn", BLOCK_N)
@pytest.mark.parametrize("mode,gate_kind", EDGE_MODES, ids=lambda v: str(v))
@pytest.mark.parametrize("M,N,K", EDGE_SHAPES, ids=lambda v: str(v))
def test_gemm_edges(M, N, K, mode, gate_kind, bn, ld_kind):
    run_gemm(mode, M, N, K, bn, ld_kind, gate_kind, group="gemm_edge")


@pytest.mark.parametrize("mode,gate_kind", [(tr.BF16_OUT, None), (tr.GELU_OUT, None), (tr.F32_OUT, None),
                                            (tr.GEGLU, None), (tr.RESID_GATE, "batch")], ids=lambda v: str(v))
def test_gemm_persistent_wrap(mode, gate_kind):
    """4096 x 3072 x 768 at 128 x 64 tiles: 1536 tiles, so every CTA loops ~12 times and the smem ring wraps many
    times over."""
    run_gemm(mode, 4096, 3072, 768, 64, "vec", gate_kind, group="gemm_wrap")


@pytest.mark.parametrize("M,N,K", [(129, 190, 64), (200, 500, 1000), (1000, 768, 3072)], ids=lambda v: str(v))
def test_gemm_f32_bits_do_not_depend_on_tile_width(M, N, K):
    """Every tile width runs the same k16 wgmma sequence for an output element, so the fp32 results are bitwise
    equal across block_n."""
    lib, _ = _lib()
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(M + N + K)
    Abuf, _, lda = tr.hostile_operand(M, K, dev, gen)
    Wbuf, _, ldw = tr.hostile_operand(N, K, dev, gen, scale=K ** -0.5)
    bias = (torch.randn(N, generator=gen) * 0.5).to(dev)
    outs = []
    for bn in BLOCK_N:
        out = torch.empty(M, N, device=dev)
        _gemm_call(Abuf, lda, Wbuf, ldw, M, N, K,
                   lib.GaGemmEpilogue(mode=tr.F32_OUT, bias=bias.data_ptr(), out=out.data_ptr(), ld_out=N), bn)
        outs.append(out)
    for bn, o in zip(BLOCK_N[1:], outs[1:]):
        assert torch.equal(_bits(o), _bits(outs[0])), "block_n %d differs from block_n 64" % bn


# ---- HEADS ---------------------------------------------------------------------------------------------------------

def _heads_cases():
    """Every (variant, heads, rows_per_batch) triple; tile width, qk-norm and bias follow from their indices so that
    every pair of values of any two options occurs (and each option at both widths)."""
    out = []
    for iv, variant in enumerate(("qkv", "q", "kv")):
        for ih, heads in enumerate((1, 2, 16)):
            for ir, rpb in enumerate((77, 200, 1369)):
                bn = (128, 256)[(iv + ih + ir) % 2]
                out.append((bn, variant, (iv + ih) % 2, (iv + ir) % 2, heads, rpb))
    return out


def test_heads_cases_cover_every_pair():
    cases = _heads_cases()
    levels = [(128, 256), ("qkv", "q", "kv"), (0, 1), (0, 1), (1, 2, 16), (77, 200, 1369)]
    for i in range(6):
        for j in range(i + 1, 6):
            seen = {(c[i], c[j]) for c in cases}
            assert len(seen) == len(levels[i]) * len(levels[j]), (i, j)


@pytest.mark.parametrize("bn,variant,norm,use_bias,heads,rpb", _heads_cases())
def test_gemm_heads(bn, variant, norm, use_bias, heads, rpb):
    run_heads(bn, variant, norm, use_bias, heads, rpb)


# ---- production census ---------------------------------------------------------------------------------------------
# Every call site of the networks at its deployed size, with the tile width the engines pick.  Sizes: DiT-L (D 1024,
# 16 heads) at N = 768 points, B = 2, image context M = 1369 (Dc 1024) and text context M = 77 (Dc 768); CLIP ViT-L/14
# text (D 768, 12 heads, 77 tokens, B = 2); DINOv2 ViT-L/14 (D 1024, 1374 tokens, patch GEMM K = 640); the VAE decoder
# (D 768, depth 12, B = 2 x 768 tokens, adaLN table N = 12 * 6 * 768); the VAE encoder (8 views of 64 x 64 tokens =
# 32768, D 256, inner 512, 768 queries).
CENSUS_ELEMENTWISE = {
    "dit_fc2_f32": (tr.F32_OUT, 1536, 1024, 1024, None),
    "dit_xyz_resid_none": (tr.RESID_GATE, 1536, 1024, 64, "none1"),
    "dit_ca_out_resid_none": (tr.RESID_GATE, 1536, 1024, 1024, "none1"),
    "dit_proj_resid_batch_gate": (tr.RESID_GATE, 1536, 1024, 1024, "batch"),
    "dit_fc1_gelu": (tr.GELU_OUT, 1536, 4096, 1024, None),
    "dit_fc2_resid_batch_gate": (tr.RESID_GATE, 1536, 1024, 4096, "batch"),
    "clip_out_resid_none": (tr.RESID_GATE, 154, 768, 768, "noneM"),
    "clip_fc_bf16": (tr.BF16_OUT, 154, 3072, 768, None),
    "clip_proj_resid_none": (tr.RESID_GATE, 154, 768, 3072, "noneM"),
    "dino_patch_f32_k640": (tr.F32_OUT, 1369, 1024, 640, None),
    "dino_proj_layerscale": (tr.RESID_GATE, 1374, 1024, 1024, "layerscale"),
    "dino_fc1_gelu": (tr.GELU_OUT, 1374, 4096, 1024, None),
    "dino_fc2_layerscale": (tr.RESID_GATE, 1374, 1024, 4096, "layerscale"),
    "dec_adaln_table_f32": (tr.F32_OUT, 1536, 12 * 6 * 768, 768, None),
    "dec_proj_token_gate": (tr.RESID_GATE, 1536, 768, 768, "token"),
    "dec_fc2_token_gate": (tr.RESID_GATE, 1536, 768, 3072, "token"),
    "dec_upsampler_resid_none": (tr.RESID_GATE, 7680, 768, 768, "none1"),
    "enc_geglu": (tr.GEGLU, 32768, 4096, 512, None),
    "enc_ff2_resid_none": (tr.RESID_GATE, 32768, 512, 2048, "none0"),
    "enc_srt_fc1_gelu": (tr.GELU_OUT, 768, 1024, 256, None),
}
CENSUS_HEADS = {   # variant, norm, bias, heads, rows_per_batch, B, K
    "dit_ctx_kv_1369": ("kv", 1, 0, 16, 1369, 2, 1024),
    "t23d_ctx_kv_77": ("kv", 1, 0, 16, 77, 2, 768),
    "dit_ca_q": ("q", 1, 0, 16, 768, 2, 1024),
    "dit_qkv": ("qkv", 1, 1, 16, 768, 2, 1024),
    "clip_qkv": ("qkv", 0, 1, 12, 77, 2, 768),
    "dino_qkv": ("qkv", 0, 1, 16, 1374, 1, 1024),
    "dec_qkv": ("qkv", 1, 1, 12, 768, 2, 768),
    "enc_self_qkv_all_views": ("qkv", 0, 0, 8, 32768, 1, 512),
    "enc_agg_kv_32768": ("kv", 1, 0, 8, 32768, 1, 256),
    "enc_agg_q_768": ("q", 1, 0, 8, 768, 1, 256),
}


@pytest.mark.parametrize("site", sorted(CENSUS_ELEMENTWISE) + sorted(CENSUS_HEADS))
def test_gemm_production_census(site):
    from gaussiananything_b200._launch import gemm_config
    if site in CENSUS_HEADS:
        variant, norm, use_bias, heads, rpb, B, K = CENSUS_HEADS[site]
        parts = {"qkv": 3, "q": 1, "kv": 2}[variant]
        bn = gemm_config(B * rpb, parts * 64 * heads, tr.HEADS)
        run_heads(bn, variant, norm, use_bias, heads, rpb, B=B, K=K, group="census")
    else:
        mode, M, N, K, gate_kind = CENSUS_ELEMENTWISE[site]
        D_gate = 12 * 6 * 768 if gate_kind == "token" else None       # the decoder's gate rows are the adaLN table
        run_gemm(mode, M, N, K, gemm_config(M, N, mode), "vec", gate_kind, group="census", D_gate=D_gate)


# ---- attention -----------------------------------------------------------------------------------------------------

def run_attention(B, H, Nq, Nk, pitch_q_kind, bound_kind, scale, causal=False, rows=None, group="attention"):
    _, L = _lib()
    dev = torch.device("cuda:0")
    pk = _round_up(Nk, 128)
    pq = Nq if pitch_q_kind == "tight" else _round_up(Nq, 128)
    gen = torch.Generator().manual_seed(B * 1000003 + H * 10007 + Nq * 101 + Nk + int(causal))
    q, k, vt = tr.attention_inputs(B, H, Nq, Nk, pq, pk, dev, gen, qk_scale=1.0)
    bound = 0.0
    if bound_kind == "static":
        bound = tr.static_bound(q, k, Nq, Nk, scale)
        assert 0.0 < bound <= 40.0, bound               # inside the range where the kernel takes the static path
    out = tr.GuardBuf((B, Nq, H * 64), torch.bfloat16, dev)
    fn = L.ga_attention_causal_bf16 if causal else L.ga_attention_bf16
    args = [C.c_void_p(t.data_ptr()) for t in (q, k, vt, out.t)] + [B, H, Nq, Nk, pq, pk, scale, bound, _st()]
    assert fn(*args) == 0
    torch.cuda.synchronize()
    got = out.t.clone()
    ref, tol = tr.attention_ref(q, k, vt, B, H, Nq, Nk, scale, causal=causal, rows=rows)
    what = "%sattention B=%d H=%d Nq=%d Nk=%d pitch_q=%d pitch_k=%d scale=%.4f bound=%.3f" % (
        "causal " if causal else "", B, H, Nq, Nk, pq, pk, scale, bound)
    worst, msg = tr.check(got if rows is None else got[:, rows.to(dev)], ref, tol, group, what)
    assert msg == "", msg
    ok, gmsg = out.intact(tr.region(out.shape, slice(None), device=dev))
    assert ok, what + ": " + gmsg
    assert fn(*args) == 0
    torch.cuda.synchronize()
    assert torch.equal(_bits(out.t), _bits(got)), what + ": a repeat gave different bits"
    return worst


ATTN_SHAPES = [(1, 1, 1, 1), (2, 3, 1, 1369), (3, 5, 17, 5), (2, 12, 77, 77), (1, 2, 128, 129), (1, 2, 129, 128),
               (2, 16, 768, 1369), (2, 16, 768, 77), (2, 16, 1374, 1374)]


def _attn_cases():
    out = []
    for s in ATTN_SHAPES:
        for pk in (("tight", "round") if s[2] % 128 else ("round",)):
            for bound in ("online", "static"):
                for scale in (0.125, 32 ** -0.5):
                    out.append(s + (pk, bound, scale))
    return out


@pytest.mark.parametrize("B,H,Nq,Nk,pitch_q_kind,bound_kind,scale", _attn_cases())
def test_attention_matrix(B, H, Nq, Nk, pitch_q_kind, bound_kind, scale):
    run_attention(B, H, Nq, Nk, pitch_q_kind, bound_kind, scale)


@pytest.mark.parametrize("bound_kind", ["online", "static"])
@pytest.mark.parametrize("N", [1, 2, 77, 127, 128, 129, 255, 256, 257, 1000])
def test_attention_causal(N, bound_kind):
    run_attention(2, 3, N, N, "round", bound_kind, 0.125, causal=True, group="causal")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("scale", [0.125, 32 ** -0.5])
def test_attention_32k_keys_static_bound(scale):
    """The VAE encoder's aggregation cross-attention: 768 queries over all 8 x 64 x 64 view tokens."""
    run_attention(1, 8, 768, 32768, "round", "static", scale, group="attention_32k")


@pytest.mark.timeout(600)
@pytest.mark.parametrize("bound_kind", ["online", "static"])
def test_attention_32k_self_sampled_rows(bound_kind):
    """The VAE encoder's all-views self-attention, 32768 x 32768, checked on every row of the first and last
    128-query blocks and 256 random rows."""
    g = torch.Generator().manual_seed(11)
    N = 32768
    rows = torch.cat([torch.arange(128), torch.arange(N - 128, N), 128 + torch.randperm(N - 256, generator=g)[:256]])
    run_attention(1, 8, N, N, "round", bound_kind, 0.125, rows=rows, group="attention_32k")
