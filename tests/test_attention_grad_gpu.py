"""memory_efficient_attention forward and backward on the GPU against the fp64 reference of
tests/attention_grad_ref.py: O and lse element by element, dq, dk, dv within 1.5 times the bf16 emulation's distance
from fp64, at the training shapes of the reference's transformers and at the tile edges."""
import pytest
import torch

from tests import attention_grad_ref as R
from tests import tc_ref

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _mea():
    from gaussiananything_b200 import attention
    return attention


def _bmhk(t, B, H):
    """[B*H, N, d] -> [B, N, H, d] (a permuted view, not contiguous)."""
    return t.view(B, H, t.shape[1], t.shape[2]).permute(0, 2, 1, 3)


def _bh(t):
    """[B, N, H, d] or [B, N, d] -> [B*H, N, d] (contiguous copy)."""
    if t.dim() == 3:
        return t.contiguous()
    B, N, H, d = t.shape
    return t.permute(0, 2, 1, 3).reshape(B * H, N, d)


def _check_case(q, k, v, do, scale, B, H, layout="bmhk", need=(True, True, True)):
    """q, k, v, do bf16 [B*H, N, d] on the GPU.  Runs the module in `layout`, checks everything against fp64."""
    A = _mea()
    if layout == "bmk":
        qi, ki, vi, doi = (t.clone() for t in (q, k, v, do))
    else:
        qi, ki, vi, doi = (_bmhk(t.clone(), B, H) for t in (q, k, v, do))
    for t, n in zip((qi, ki, vi), need):
        t.requires_grad_(n)
    out = A.memory_efficient_attention(qi, ki, vi, scale=scale)
    out.backward(doi)
    torch.cuda.synchronize()
    # lse from the same entry point the autograd function uses
    _, lse = A._forward(*(A._prepare(t.detach().unsqueeze(2) if t.dim() == 3 else t.detach()) for t in (qi, ki, vi)),
                        scale)
    O64, L64, To, Tl = R.attention_fwd(q, k, v, scale)
    Oe, Le, _, _ = R.attention_fwd(q, k, v, scale, emulate=True)
    got_o = _bh(out.detach())
    assert torch.isfinite(got_o).all()
    w, msg = tc_ref.check(got_o, O64, To, "attn_grad", "O")
    assert not msg, msg
    w, msg = tc_ref.check(lse.view_as(L64), L64, Tl, "attn_grad", "lse")
    assert not msg, msg
    g64 = R.attention_bwd(q, k, v, O64, L64, do, scale)
    ge = R.attention_bwd(q, k, v, Oe, Le, do, scale, emulate=True)
    floors = R.grad_floors(q, k, v, do, scale)
    for name, t, n, ref, emu, fl in zip("qkv", (qi, ki, vi), need, g64, ge, floors):
        if not n:
            assert t.grad is None
            continue
        g = _bh(t.grad)
        assert t.grad.shape == t.shape and t.grad.stride() == t.stride() and t.grad.dtype == t.dtype
        assert torch.isfinite(g).all(), name
        _check_grad("d" + name, g, ref, emu, fl)
    return out


def _check_grad(name, got, ref, emu, floor):
    e_gpu, e_emu = float((got.double() - ref).norm()), float((emu - ref).norm())
    assert e_gpu <= 1.5 * e_emu + floor, (name, "L2 from fp64", e_gpu, "emulation", e_emu, "floor", floor,
                                          "relative", R.rel_l2(got, ref), R.rel_l2(emu, ref))


def _inputs(BH, Nq, Nk, d, seed, dv=None):
    g = torch.Generator().manual_seed(seed)
    return R.inputs(BH, Nq, Nk, d, g, dv=dv, device=DEV)


# the reference's training shapes: (B, H, Nq, Nk, d, layout)
TRAINING = [
    (2, 16, 768, 768, 64, "bmhk"),      # DiT-L self-attention
    (2, 12, 768, 768, 64, "bmhk"),      # DiT2-B (VAE decoder) self-attention
    (24, 1, 768, 1369, 64, "bmk"),      # DiT cross-attention to DINOv2 tokens, [B*H, N, d]
    (24, 1, 768, 77, 64, "bmk"),        # cross-attention to CLIP text tokens
    (4, 1, 768, 32768, 64, "bmk"),      # SRT encoder agg_ca
    (1, 8, 32768, 32768, 64, "bmk"),    # VAE encoder mid attention over 8 views x 64^2 tokens, batch 1
    (8, 8, 4096, 4096, 64, "bmk"),      # VAE encoder attention per view
    (2, 8, 768, 768, 32, "bmhk"),       # SRT blocks, head dimension 32
    (768, 12, 9, 9, 64, "bmhk"),        # decoder up-samplers per object: 768, 6144, 24576 sequences of 9, 5, 4
    (6144, 12, 5, 5, 64, "bmhk"),
    (24576, 12, 4, 4, 64, "bmhk"),
]


@pytest.mark.parametrize("B,H,Nq,Nk,d,layout", TRAINING)
def test_training_shapes(B, H, Nq, Nk, d, layout):
    if layout == "bmk":
        B, H = B * H, 1
    q, k, v, do = _inputs(B * H, Nq, Nk, d, 1000 + Nq + Nk)
    _check_case(q, k, v, do, d ** -0.5, B, H, layout)


EDGES = [1, 15, 16, 17, 127, 129]


@pytest.mark.parametrize("Nq,Nk", [(a, b) for a in EDGES for b in EDGES if a != b] + [(n, n) for n in EDGES])
def test_edges(Nq, Nk):
    q, k, v, do = _inputs(6, Nq, Nk, 64, 7 * Nq + Nk)
    _check_case(q, k, v, do, 0.125, 2, 3)


@pytest.mark.parametrize("scale", [1.0, -0.3, 0.01])
@pytest.mark.parametrize("N", [9, 200])
def test_any_scale(scale, N):
    q, k, v, do = _inputs(4, N, N + 3, 64, 11)
    _check_case(q, k, v, do, scale, 2, 2)


@pytest.mark.parametrize("dqk,dv", [(32, 32), (64, 32), (32, 64)])
@pytest.mark.parametrize("N", [9, 130])
def test_head_dim_32(dqk, dv, N):
    q, k, v, do = _inputs(4, N, N, dqk, 5, dv=dv)
    _check_case(q, k, v, do, 0.17, 2, 2)


@pytest.mark.parametrize("need", [(True, False, False), (False, True, False), (False, False, True), (False, True, True)])
@pytest.mark.parametrize("N", [9, 100])
def test_some_inputs_need_grad(need, N):
    q, k, v, do = _inputs(4, N, N, 64, 3)
    _check_case(q, k, v, do, 0.125, 2, 2, need=need)


@pytest.mark.parametrize("B,H,N,d", [(2, 4, 9, 64), (2, 4, 300, 64), (2, 4, 300, 32), (24576, 12, 4, 64)])
def test_unbind_views_and_nan_padding(B, H, N, d):
    """q, k, v are unbind views of a packed qkv [B, N, 3, H, d] cut out of a NaN-filled buffer: NaN past N and past d
    (d = 32 in a 64-wide row), never read.  The last case is the decoder up-samplers' 4-token layout per object."""
    A = _mea()
    g = torch.Generator().manual_seed(21)
    buf = torch.full((B, N + 7, 3, H, 64), float("nan"), dtype=torch.bfloat16, device=DEV)
    vals = (torch.randn(B, N, 3, H, d, generator=g) * 1.2).to(torch.bfloat16).to(DEV)
    buf[:, :N, :, :, :d] = vals
    leaf = buf[:, :N, :, :, :d].clone()                           # the reference's operands
    src = buf.detach().requires_grad_(True)
    q, k, v = src[:, :N, :, :, :d].unbind(2)
    assert not q.is_contiguous()
    do = torch.randn(B, N, H, d, generator=g).to(torch.bfloat16).to(DEV)
    out = A.memory_efficient_attention(q, k, v)
    out.backward(do)
    assert torch.isfinite(out).all()
    grad = src.grad[:, :N, :, :, :d]
    assert torch.isfinite(grad).all(), "a padded NaN reached a gradient"
    assert (src.grad[:, N:] == 0).all() and (src.grad[..., d:] == 0).all()
    ql, kl, vl = (_bh(t) for t in leaf.unbind(2))
    O64, L64, To, _ = R.attention_fwd(ql, kl, vl, d ** -0.5)
    w, msg = tc_ref.check(_bh(out.detach()), O64, To, "attn_grad", "O")
    assert not msg, msg
    Oe, Le, _, _ = R.attention_fwd(ql, kl, vl, d ** -0.5, emulate=True)
    g64 = R.attention_bwd(ql, kl, vl, O64, L64, _bh(do), d ** -0.5)
    ge = R.attention_bwd(ql, kl, vl, Oe, Le, _bh(do), d ** -0.5, emulate=True)
    floors = R.grad_floors(ql, kl, vl, _bh(do), d ** -0.5)
    for i, name in enumerate("qkv"):
        _check_grad("d" + name, _bh(grad[:, :, i]), g64[i], ge[i], floors[i])


@pytest.mark.parametrize("N", [9, 200])
def test_expanded_query_and_key(N):
    """q and k broadcast over the batch with expand (batch stride 0), as a learned token set is: each gradient is the
    sum over the batch of the per-batch gradients, not one batch's gradient repeated."""
    A = _mea()
    B, H, d, Nk = 4, 2, 64, N + 3
    g = torch.Generator().manual_seed(41)
    qb = (torch.randn(1, N, H, d, generator=g) * 1.2).to(torch.bfloat16).to(DEV).requires_grad_(True)
    kb = (torch.randn(1, Nk, H, d, generator=g) * 1.2).to(torch.bfloat16).to(DEV).requires_grad_(True)
    v = torch.randn(B, Nk, H, d, generator=g).to(torch.bfloat16).to(DEV).requires_grad_(True)
    do = torch.randn(B, N, H, d, generator=g).to(torch.bfloat16).to(DEV)
    out = A.memory_efficient_attention(qb.expand(B, -1, -1, -1), kb.expand(B, -1, -1, -1), v)
    out.backward(do)
    q, k = (_bh(t.detach().expand(B, -1, -1, -1)) for t in (qb, kb))
    vv, dd = _bh(v.detach()), _bh(do)
    scale = d ** -0.5
    O64, L64, To, _ = R.attention_fwd(q, k, vv, scale)
    w, msg = tc_ref.check(_bh(out.detach()), O64, To, "attn_grad", "O")
    assert not msg, msg
    Oe, Le, _, _ = R.attention_fwd(q, k, vv, scale, emulate=True)
    g64 = R.attention_bwd(q, k, vv, O64, L64, dd, scale)
    ge = R.attention_bwd(q, k, vv, Oe, Le, dd, scale, emulate=True)
    fq, fk, fv = R.grad_floors(q, k, vv, dd, scale)
    bsum = lambda t: t.view(B, H, t.shape[1], d).sum(0)                       # [H, N, d]
    for name, got, ref, emu, fl in (("dq", qb.grad, g64[0], ge[0], fq), ("dk", kb.grad, g64[1], ge[1], fk)):
        assert torch.isfinite(got).all()
        _check_grad(name, got[0].permute(1, 0, 2), bsum(ref), R.bf16(bsum(emu)), B * fl)
    _check_grad("dv", _bh(v.grad), g64[2], ge[2], fv)


@pytest.mark.parametrize("B,H,N", [(5462, 12, 9), (5462, 12, 17)])
def test_many_heads(B, H, N):
    """batch * heads = 65544 > 65535 on the short path (9 tokens) and on the tiled path (17 tokens)."""
    q, k, v, do = _inputs(B * H, N, N, 64, 31)
    _check_case(q, k, v, do, 0.125, B, H)


@pytest.mark.parametrize("N", [9, 129])
def test_zero_grad_out_gives_zero_gradients(N):
    A = _mea()
    q, k, v, _ = _inputs(4, N, N, 64, 8)
    q, k, v = (_bmhk(t, 2, 2).requires_grad_(True) for t in (q, k, v))
    out = A.memory_efficient_attention(q, k, v)
    out.backward(torch.zeros_like(out))
    for t in (q, k, v):
        assert (t.grad == 0).all() and not torch.signbit(t.grad).any()


@pytest.mark.parametrize("N", [9, 300])
def test_repeatable_bits(N):
    A = _mea()
    q, k, v, do = _inputs(8, N, N + 5, 64, 9)
    runs = []
    for _ in range(3):
        qi, ki, vi = (_bmhk(t, 2, 4).detach().requires_grad_(True) for t in (q, k, v))
        out = A.memory_efficient_attention(qi, ki, vi)
        out.backward(_bmhk(do, 2, 4))
        runs.append([out.detach().clone()] + [t.grad.clone() for t in (qi, ki, vi)])
    for r in runs[1:]:
        for a, b in zip(runs[0], r):
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_reference_chunking_matches_one_call():
    """The reference's up-samplers call the function on batch chunks of 32768 and concatenate: same bits."""
    A = _mea()
    B, H, N = 40000, 2, 5
    g = torch.Generator().manual_seed(4)
    q, k, v, do = (torch.randn(B, N, H, 64, generator=g).to(torch.bfloat16).to(DEV) for _ in range(4))
    res = []
    for chunked in (False, True):
        qi, ki, vi = (t.clone().requires_grad_(True) for t in (q, k, v))
        if chunked:
            out = torch.cat([A.memory_efficient_attention(qi[i:i + 32768], ki[i:i + 32768], vi[i:i + 32768])
                             for i in range(0, B, 32768)])
        else:
            out = A.memory_efficient_attention(qi, ki, vi)
        out.backward(do)
        res.append([out.detach()] + [t.grad for t in (qi, ki, vi)])
    for a, b in zip(*res):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def test_inplace_change_before_backward_raises():
    A = _mea()
    qkv = torch.randn(2, 64, 3, 4, 64, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    x = qkv * 1.0
    q, k, v = x.unbind(2)
    out = A.memory_efficient_attention(q, k, v)
    x.mul_(2.0)
    with pytest.raises(RuntimeError):
        out.sum().backward()


def test_double_backward_raises():
    A = _mea()
    q, k, v = (torch.randn(2, 40, 2, 64, device=DEV, dtype=torch.bfloat16, requires_grad=True) for _ in range(3))
    out = A.memory_efficient_attention(q, k, v)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(out.float().sum(), (q,), create_graph=True)


def test_no_grad_runs_forward_only_and_fp32_inputs():
    A = _mea()
    q, k, v = (torch.randn(2, 50, 2, 64, device=DEV) for _ in range(3))
    with torch.no_grad():
        out = A.memory_efficient_attention(q, k, v)
    assert out.dtype == torch.float32 and out.shape == (2, 50, 2, 64) and not out.requires_grad
    qb, kb, vb = (t.to(torch.bfloat16) for t in (q, k, v))
    ref = A.memory_efficient_attention(qb, kb, vb)
    assert torch.equal(out, ref.float())
    qf = q.clone().requires_grad_(True)
    A.memory_efficient_attention(qf, k, v).sum().backward()
    assert qf.grad.dtype == torch.float32 and qf.grad.shape == q.shape


class _MemEffAttentionBlock(torch.nn.Module):
    """The reference's MemEffAttention with qk RMSNorm: qkv Linear -> unbind -> per-head RMSNorm -> attention -> proj."""

    def __init__(self, dim, heads, attn):
        super().__init__()
        self.heads, self.attn = heads, attn
        self.qkv = torch.nn.Linear(dim, 3 * dim)
        self.proj = torch.nn.Linear(dim, dim)
        self.q_norm = torch.nn.RMSNorm(dim // heads, eps=1e-5)
        self.k_norm = torch.nn.RMSNorm(dim // heads, eps=1e-5)

    def forward(self, x):
        B, N, C = x.shape
        q, k, v = self.qkv(x).reshape(B, N, 3, self.heads, C // self.heads).unbind(2)
        q, k = self.q_norm(q).to(v.dtype), self.k_norm(k).to(v.dtype)
        return self.proj(self.attn(q, k, v).reshape(B, N, C))


def _sdpa(q, k, v):
    return torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2),
                                                            v.transpose(1, 2)).transpose(1, 2)


def test_memeff_block_trains_under_autocast():
    """Five AdamW steps of a MemEffAttention-shaped block under bf16 autocast: the parameters stay as close to an
    fp32 SDPA run as a bf16-autocast SDPA run does."""
    A = _mea()
    torch.manual_seed(0)
    dim, heads, B, N = 256, 4, 4, 200
    base = _MemEffAttentionBlock(dim, heads, None).to(DEV)
    xs = [torch.randn(B, N, dim, device=DEV) for _ in range(5)]
    ys = [torch.randn(B, N, dim, device=DEV) for _ in range(5)]

    def train(attn, autocast):
        m = _MemEffAttentionBlock(dim, heads, attn).to(DEV)
        m.load_state_dict(base.state_dict())
        opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
        for x, y in zip(xs, ys):
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                loss = (m(x).float() - y).pow(2).mean()
            opt.zero_grad()
            loss.backward()
            opt.step()
        return torch.cat([p.detach().flatten() for p in m.parameters()]), float(loss)

    ref, _ = train(_sdpa, False)
    sdpa_bf16, _ = train(_sdpa, True)
    ours, loss = train(A.memory_efficient_attention, True)
    start = torch.cat([p.detach().flatten() for p in base.parameters()])
    d_ours = float((ours - ref).norm() / (ref - start).norm())
    d_sdpa = float((sdpa_bf16 - ref).norm() / (ref - start).norm())
    assert torch.isfinite(ours).all() and loss == loss
    assert d_ours <= 1.5 * d_sdpa + 1e-3, (d_ours, d_sdpa)
