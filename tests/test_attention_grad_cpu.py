"""CPU checks of memory_efficient_attention: the fp64 reference against torch autograd, argument validation (Python
and the host-only C validator), the layout handling of the Python layer through a stub library, and install_shims()
on a stub xformers.ops module."""
import ctypes as C
import sys
import types

import pytest
import torch

from tests import attention_grad_ref as R


def _attention():
    from gaussiananything_b200 import attention
    return attention


@pytest.mark.parametrize("BH,Nq,Nk,d,dv", [(2, 17, 5, 64, 64), (3, 1, 129, 32, 64), (2, 70, 70, 64, 32)])
@pytest.mark.parametrize("scale", [0.125, -0.7])
def test_fp64_reference_matches_autograd(BH, Nq, Nk, d, dv, scale):
    g = torch.Generator().manual_seed(BH * 100 + Nq + Nk)
    q, k, v, do = R.inputs(BH, Nq, Nk, d, g, dv=dv)
    O, L, _, _ = R.attention_fwd(q, k, v, scale, chunk=16)
    dq, dk, dv_ = R.attention_bwd(q, k, v, O, L, do, scale, chunk=16)
    qq, kk, vv = (t.double().requires_grad_(True) for t in (q, k, v))
    s = qq @ kk.transpose(1, 2) * scale
    o = torch.softmax(s, -1) @ vv
    o.backward(do.double())
    assert torch.allclose(O, o.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(L, torch.logsumexp(s.detach(), -1), rtol=1e-12, atol=1e-12)
    for a, b in zip((dq, dk, dv_), (qq.grad, kk.grad, vv.grad)):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-12)


def test_emulation_rounds_to_bf16_and_stays_close():
    g = torch.Generator().manual_seed(3)
    q, k, v, do = R.inputs(2, 40, 33, 64, g)
    O, L, To, _ = R.attention_fwd(q, k, v, 0.125)
    Oe, Le, _, _ = R.attention_fwd(q, k, v, 0.125, emulate=True)
    assert torch.equal(Oe, R.bf16(Oe))
    assert ((Oe - O).abs() <= To).all()
    for a, b in zip(R.attention_bwd(q, k, v, Oe, Le, do, 0.125, emulate=True), R.attention_bwd(q, k, v, O, L, do, 0.125)):
        assert torch.equal(a, R.bf16(a))
        assert 1e-4 < R.rel_l2(a, b) < 1e-2


# ---- argument refusals of the Python layer (raised before any device or library access) ----

def _t(*shape, dtype=torch.bfloat16):
    return torch.zeros(*shape, dtype=dtype)


def test_refusals():
    A = _attention()
    q = _t(2, 8, 4, 64)
    with pytest.raises(NotImplementedError, match="attn_bias"):
        A.memory_efficient_attention(q, q, q, attn_bias=torch.zeros(1))
    with pytest.raises(NotImplementedError, match="dropout"):
        A.memory_efficient_attention(q, q, q, p=0.1)
    with pytest.raises(NotImplementedError, match="head dimension 128"):
        A.memory_efficient_attention(_t(2, 8, 4, 128), _t(2, 8, 4, 128), _t(2, 8, 4, 128))
    with pytest.raises(NotImplementedError, match="head dimension 48 of value"):
        A.memory_efficient_attention(q, q, _t(2, 8, 4, 48))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        A.memory_efficient_attention(q, q, q)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        A.memory_efficient_attention(_t(2, 8, 64, dtype=torch.float32), _t(2, 8, 64), _t(2, 8, 64))


@pytest.mark.parametrize("q,k,v,match", [
    ((2, 8, 4, 64), (2, 9, 4, 64), (2, 8, 4, 64), "disagree outside"),
    ((2, 8, 4, 64), (3, 9, 4, 64), (3, 9, 4, 64), "batch or heads"),
    ((2, 8, 4, 64), (2, 9, 2, 64), (2, 9, 2, 64), "batch or heads"),
    ((2, 8, 4, 64), (2, 9, 4, 32), (2, 9, 4, 32), "head dimensions differ"),
    ((2, 8, 64), (2, 9, 4, 64), (2, 9, 4, 64), "must all be BMHK or all BMK"),
    ((8, 64), (8, 64), (8, 64), "BMHK"),
    ((2, 0, 4, 64), (2, 9, 4, 64), (2, 9, 4, 64), "empty"),
])
def test_shape_mismatches(q, k, v, match):
    A = _attention()
    with pytest.raises(ValueError, match=match):
        A.memory_efficient_attention(_t(*q), _t(*k), _t(*v))


def test_dtype_refused():
    A = _attention()
    q = _t(2, 8, 4, 64, dtype=torch.float64)
    with pytest.raises(TypeError, match="bf16, fp16 or fp32"):
        A.memory_efficient_attention(q, q, q)


# ---- the host-only C validator ----

def _validate(**kw):
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    a = dict(q=0x1000, k=0x2000, v=0x3000, o=0x4000, lse=0x5000, dout=0x6000, delta=0x7000, dq=0x8000, dk=0x9000,
             dv=0xa000, batch=2, heads=4, Nq=100, Nk=77, d_qk=64, d_v=64, strides=[8 * i for i in range(24)],
             backward=1)
    a.update(kw)
    st = (C.c_int64 * 24)(*a["strides"]) if a["strides"] is not None else None
    p = lambda x: C.c_void_p(x)
    return L.ga_attention_grad_validate(p(a["q"]), p(a["k"]), p(a["v"]), p(a["o"]), p(a["lse"]), p(a["dout"]),
                                        p(a["delta"]), p(a["dq"]), p(a["dk"]), p(a["dv"]), a["batch"], a["heads"],
                                        a["Nq"], a["Nk"], a["d_qk"], a["d_v"], st, a["backward"])


def test_c_validator():
    BAD, SIZE = -1, -3
    assert _validate() == 0
    assert _validate(d_qk=32, d_v=32) == 0 and _validate(d_v=32) == 0
    assert _validate(dq=None, dk=None, dv=None) == 0                  # gradients not formed
    assert _validate(backward=0, dout=None, delta=None) == 0
    assert _validate(backward=1, dout=None) == BAD
    assert _validate(backward=1, delta=None) == BAD
    for name in ("q", "k", "v", "o", "lse"):
        assert _validate(**{name: None}) == BAD, name
    assert _validate(strides=None) == BAD
    for name in ("batch", "heads", "Nq", "Nk"):
        assert _validate(**{name: 0}) == BAD, name
    assert _validate(d_qk=48) == BAD and _validate(d_v=128) == BAD
    assert _validate(q=0x1008) == BAD and _validate(dk=0x9004) == BAD
    assert _validate(lse=0x5002) == BAD
    s = [8 * i for i in range(24)]
    s[4] = 12
    assert _validate(strides=s) == BAD                               # k's token stride not a multiple of 8
    s[4] = -8
    assert _validate(strides=s) == BAD
    s = [8 * i for i in range(24)]
    s[22] = 4
    assert _validate(strides=s) == BAD                               # dv's token stride
    assert _validate(strides=s, dv=None) == 0                         # ... not in use
    assert _validate(strides=s, backward=0) == 0
    # a zero stride on an output dimension of size > 1 (CTAs would write the same elements); inputs may broadcast
    for i in (9, 10, 11, 15, 16, 17, 18, 19, 20, 21, 22, 23):
        s = [8 * (i + 1) for i in range(24)]
        s[i] = 0
        assert _validate(strides=s) == BAD, i
    s = [8 * (i + 1) for i in range(24)]
    s[0] = s[3] = s[6] = 0                                           # q, k, v broadcast over the batch
    assert _validate(strides=s) == 0
    s = [8 * (i + 1) for i in range(24)]
    s[9] = s[15] = 0
    assert _validate(strides=s, batch=1) == 0                         # a size-1 dimension's stride is irrelevant
    # batch * heads past 65535 is accepted (one-dimensional grid); past 2^31 - 1 CTAs it is not
    assert _validate(batch=300000, heads=12, Nq=9, Nk=9) == 0
    assert _validate(batch=70000, heads=12, Nq=300, Nk=300) == 0
    assert _validate(batch=2 ** 30, heads=2, Nq=100, Nk=100) == SIZE


# ---- layout handling of the Python layer, through a stub library on the host ----

class _StubLib:
    """Records the calls the autograd function makes."""

    def __init__(self):
        self.calls = []

    def ga_attention_fwd_lse_bf16(self, q, k, v, o, lse, B, H, Nq, Nk, D, Dv, strides, scale, stream):
        self.calls.append(("fwd", [q.value, k.value, v.value, o.value], (B, H, Nq, Nk, D, Dv), list(strides)[:12],
                           scale))
        return 0

    def ga_attention_bwd_bf16(self, q, k, v, o, lse, dout, delta, dq, dk, dv, B, H, Nq, Nk, D, Dv, strides, scale,
                              stream):
        self.calls.append(("bwd", [q.value, k.value, v.value, dq.value, dk.value, dv.value], (B, H, Nq, Nk, D, Dv),
                           list(strides), scale))
        return 0


@pytest.fixture
def stub(monkeypatch):
    """The Python layer run on the host: a stub library, and the CUDA checks of torch bypassed."""
    A = _attention()
    lib = _StubLib()
    monkeypatch.setattr(A._lib, "lib", lambda: lib)

    class _Dev:
        def __init__(self, *a):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False
    monkeypatch.setattr(torch.cuda, "device", _Dev)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a: types.SimpleNamespace(cuda_stream=0))
    monkeypatch.setattr(A, "_check_args", lambda *a: None)
    return A, lib


def test_bmhk_unbind_views_are_read_in_place(stub):
    A, lib = stub
    B, N, H, D = 2, 10, 4, 64
    qkv = torch.randn(B, N, 3, H, D).to(torch.bfloat16).requires_grad_(True)
    q, k, v = qkv.unbind(2)
    out = A.memory_efficient_attention(q, k, v)
    assert out.shape == (B, N, H, D) and out.dtype == torch.bfloat16
    kind, ptrs, dims, strides, scale = lib.calls[0]
    assert kind == "fwd" and dims == (B, H, N, N, D, D) and scale == pytest.approx(D ** -0.5)
    assert ptrs[:3] == [q.data_ptr(), k.data_ptr(), v.data_ptr()]          # no copy
    assert strides[:3] == [N * 3 * H * D, 3 * H * D, D]
    assert strides[9:12] == [N * H * D, H * D, D]                            # o: contiguous BMHK
    out.backward(torch.ones_like(out))
    kind, ptrs, dims, strides, _ = lib.calls[1]
    assert kind == "bwd"
    assert strides[15:24] == [N * 3 * H * D, 3 * H * D, D] * 3             # gradients in the inputs' strides
    assert qkv.grad.shape == qkv.shape


def test_bmk_and_dtype_conversion(stub):
    A, lib = stub
    q = torch.randn(6, 20, 32, requires_grad=True)
    k = torch.randn(6, 9, 32, requires_grad=True)
    v = torch.randn(6, 9, 64, dtype=torch.float16)
    out = A.memory_efficient_attention(q, k, v, scale=0.3, op=object())
    assert out.shape == (6, 20, 64) and out.dtype == torch.float32
    kind, ptrs, dims, strides, scale = lib.calls[0]
    assert dims == (6, 1, 20, 9, 32, 64) and scale == pytest.approx(0.3)
    assert strides[:3] == [20 * 32, 32, 0] and strides[6:9] == [9 * 64, 64, 0]
    out.sum().backward()
    assert lib.calls[1][0] == "bwd"
    assert q.grad.dtype == torch.float32 and q.grad.shape == q.shape and k.grad.shape == k.shape
    _, ptrs, _, _, _ = lib.calls[1]
    assert ptrs[5] is None                                                   # v needs no gradient: dv not formed


def test_expanded_inputs_get_fresh_gradients(stub):
    """An input broadcast with expand (stride 0 over the batch) must not lend its strides to its gradient: every
    (batch, head) CTA would write the same elements."""
    A, lib = stub
    kb = torch.randn(1, 10, 2, 64).to(torch.bfloat16).requires_grad_(True)
    q = torch.randn(4, 7, 2, 64).to(torch.bfloat16).requires_grad_(True)
    v = torch.randn(4, 10, 2, 64).to(torch.bfloat16)
    A.memory_efficient_attention(q, kb.expand(4, 10, 2, 64), v).sum().backward()
    kind, ptrs, dims, strides, _ = lib.calls[1]
    assert kind == "bwd" and strides[3:6] == [0, 128, 64]                    # k is read where it lies
    assert strides[18:21] == [10 * 2 * 64, 128, 64]                          # dk: a contiguous buffer of its own
    assert kb.grad.shape == kb.shape
    assert not A._non_overlapping((4, 10, 2, 64), (0, 128, 64, 1))
    assert A._non_overlapping((4, 10, 2, 64), (3 * 1280, 3 * 128, 64, 1))    # unbind views of a packed qkv
    assert A._grad_like(torch.zeros(4, 10, 2, 64, dtype=torch.bfloat16),
                        ((4, 10, 2, 64), (0, 128, 64, 1), torch.float32)).stride() == (1280, 128, 64, 1)


def test_unaddressable_strides_are_copied(stub):
    A, lib = stub
    base = torch.randn(2, 12, 3, 65).to(torch.bfloat16)
    q = base[..., :64]                                                       # token stride 195: not a multiple of 8
    A.memory_efficient_attention(q, q, q)
    _, ptrs, _, strides, _ = lib.calls[0]
    assert ptrs[0] != q.data_ptr() and strides[:3] == [12 * 3 * 64, 3 * 64, 64]


def test_no_grad_and_partial_gradients(stub):
    A, lib = stub
    q, k, v = (torch.randn(2, 30, 2, 64).to(torch.bfloat16) for _ in range(3))
    with torch.no_grad():
        A.memory_efficient_attention(q, k, v)
    assert [c[0] for c in lib.calls] == ["fwd"]
    k.requires_grad_(True)
    A.memory_efficient_attention(q, k, v).sum().backward()
    _, ptrs, _, _, _ = lib.calls[-1]
    assert ptrs[3] is None and ptrs[4] is not None and ptrs[5] is None
    assert q.grad is None and v.grad is None and k.grad.shape == k.shape


def test_double_backward_raises(stub):
    A, lib = stub
    q = torch.randn(2, 30, 2, 64).to(torch.bfloat16).requires_grad_(True)
    out = A.memory_efficient_attention(q, q, q)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(out.float().sum(), q, create_graph=True)


def test_inplace_change_before_backward_raises(stub):
    A, lib = stub
    x = torch.randn(2, 30, 3, 2, 64).to(torch.bfloat16).requires_grad_(True) * 1.0
    q, k, v = x.unbind(2)
    out = A.memory_efficient_attention(q, k, v)
    x.add_(1.0)
    with pytest.raises(RuntimeError, match="inplace"):
        out.sum().backward()


# ---- install_shims ----

def test_install_shims_patches_a_stub_xformers(monkeypatch):
    A = _attention()
    orig = object()
    xops = types.ModuleType("xformers.ops")
    xops.memory_efficient_attention = orig
    xf = types.ModuleType("xformers")
    xf.ops = xops
    vt = types.ModuleType("vit.vision_transformer")
    vt.memory_efficient_attention = orig
    monkeypatch.setitem(sys.modules, "xformers", xf)
    monkeypatch.setitem(sys.modules, "xformers.ops", xops)
    monkeypatch.setitem(sys.modules, "vit.vision_transformer", vt)
    assert A.install_shims() is True
    assert xops.memory_efficient_attention is A.memory_efficient_attention
    assert vt.memory_efficient_attention is A.memory_efficient_attention


def test_install_shims_without_xformers(monkeypatch):
    A = _attention()
    monkeypatch.setitem(sys.modules, "xformers", None)                 # import xformers raises ImportError
    monkeypatch.setitem(sys.modules, "xformers.ops", None)
    vt = types.ModuleType("vit.vision_transformer")
    orig = object()
    vt.memory_efficient_attention = orig
    monkeypatch.setitem(sys.modules, "vit.vision_transformer", vt)
    assert A.install_shims() is False
    assert vt.memory_efficient_attention is orig


def test_package_install_shims_leaves_xformers_alone(monkeypatch):
    """The package-level switch does not swap attention in (INTEGRATION.md section 3k)."""
    import gaussiananything_b200 as ga
    orig = object()
    xops = types.ModuleType("xformers.ops")
    xops.memory_efficient_attention = orig
    monkeypatch.setitem(sys.modules, "xformers.ops", xops)
    ga.install_shims(replace_classes=True)
    assert xops.memory_efficient_attention is orig
