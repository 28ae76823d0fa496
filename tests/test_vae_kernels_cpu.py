"""Argument checks of the 3D VAE's kernels (include/ga_b200.h Part 5 and the VAE decode path of Part 2): the alignment
of every pointer a kernel reads or writes as a vector (float2, float4, uint2, __nv_bfloat162), and the argument rules
next to each declaration.  Each refused call must be refused by host code before any launch.

The pointers are made-up device addresses that nothing dereferences.  A call that passed its checks would launch a
kernel on them, so the whole file is skipped where a CUDA device is present.  Without a device, a call that gets past
its checks returns a CUDA error instead of a GA_ERR_* code, so a missing check fails its test cleanly; each case first
shows that the unchanged call does get that far.  That a refused call writes nothing is checked with real buffers in
tests/test_vae_kernels_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="calls the entry points with made-up device pointers; run without a GPU")

BADARG, WORKSPACE = -1, -2
A = 1 << 24


def ptr(k):
    """The k-th made-up device address (16-byte aligned)."""
    return A * k


def _entries(L):
    """{name: (call, arguments that pass every check)}; call(L, args) returns the entry point's code."""
    e = {}
    e["conv"] = (lambda L, a: L.ga_conv3x3_bf16(a["x"], 2, 16, 16, a["Cin"], a["w"], a["kp"], a["bias"], a["Cout"],
                                                a["stride"], a["res"], a["f32"], a["bf16"], None),
                 dict(x=ptr(1), Cin=64, w=ptr(2), kp=576, bias=ptr(3), Cout=128, stride=1, res=ptr(4), f32=ptr(5),
                      bf16=ptr(6)))
    e["conv relu"] = (lambda L, a: L.ga_conv3x3_relu_bf16(a["x"], 2, 16, 16, a["Cin"], a["w"], a["kp"], a["bias"],
                                                          a["Cout"], a["bf16"], None),
                      dict(x=ptr(1), Cin=512, w=ptr(2), kp=4608, bias=None, Cout=64, bf16=ptr(6)))
    e["gn"] = (lambda L, a: L.ga_group_norm_nhwc(a["x"], ptr(2), ptr(3), 2, 4096, a["C"], 1e-6, 1, a["out"],
                                                 a["out_bf16"], ptr(5), a["sb"], None),
               dict(x=ptr(1), C=64, out=ptr(4), out_bf16=0, sb=L.ga_group_norm_scratch_bytes(2, 4096)))
    e["gn bf16"] = (e["gn"][0], dict(e["gn"][1], out_bf16=1))
    e["micro"] = (lambda L, a: L.ga_micro_attention_bf16(a["qkv"], a["qn"], a["kn"], a["out"], 64, a["L"], 12, 1e-5,
                                                         None),
                  dict(qkv=ptr(1), qn=ptr(2), kn=ptr(3), out=ptr(4), L=9))
    e["micro generic"] = (e["micro"][0], dict(e["micro"][1], L=7))
    return e


def _shift(name, by):
    """name's pointer moved by `by` bytes."""
    f = lambda a: {name: a[name] + by}
    f.label = "%s%+d" % (name, by)
    return f


def _label(change):
    if hasattr(change, "label"):
        return change.label
    return ",".join("%s=%s" % kv for kv in change({"sb": 0}).items())


# (entry, change to the good arguments, the code it must return)
CASES = [
    # float2 residual reads and fp32 stores: 8 bytes; __nv_bfloat162 stores: 4 bytes; the gathered x: 16 bytes
    ("conv", _shift("res", 4), BADARG), ("conv", _shift("f32", 4), BADARG), ("conv", _shift("bf16", 2), BADARG),
    ("conv", _shift("x", 8), BADARG), ("conv", _shift("w", 8), BADARG), ("conv relu", _shift("bf16", 2), BADARG),
    # float4 loads, float4 / uint2 stores
    ("gn", _shift("x", 4), BADARG), ("gn", _shift("x", 8), BADARG), ("gn", _shift("out", 8), BADARG),
    ("gn", _shift("out", 4), BADARG), ("gn bf16", _shift("out", 4), BADARG), ("gn bf16", _shift("x", 4), BADARG),
    # __nv_bfloat162 loads and stores, float2 norm weights
    ("micro", _shift("qkv", 2), BADARG), ("micro", _shift("out", 2), BADARG), ("micro", _shift("qn", 4), BADARG),
    ("micro", _shift("kn", 4), BADARG), ("micro generic", _shift("qkv", 2), BADARG),
    ("micro generic", _shift("kn", 4), BADARG),
    # argument rules
    ("conv", lambda a: dict(Cin=60), BADARG), ("conv", lambda a: dict(Cin=0), BADARG),
    ("conv", lambda a: dict(Cout=96), BADARG), ("conv", lambda a: dict(kp=512), BADARG),
    ("conv", lambda a: dict(f32=None, bf16=None), BADARG), ("conv", lambda a: dict(stride=3), BADARG),
    ("conv relu", lambda a: dict(kp=4544), BADARG), ("conv relu", lambda a: dict(Cout=32), BADARG),
    ("gn", lambda a: dict(C=48), BADARG), ("gn", lambda a: dict(C=1056), BADARG), ("gn", lambda a: dict(C=0), BADARG),
    ("gn", lambda a: dict(C=-32), BADARG),
    ("gn", lambda a: dict(sb=a["sb"] - 1), WORKSPACE), ("gn bf16", lambda a: dict(sb=0), WORKSPACE),
    ("micro", lambda a: dict(L=17), BADARG), ("micro", lambda a: dict(L=0), BADARG),
    ("micro", lambda a: dict(qn=None), BADARG),
]

# arguments the checks must let through: the alignment each vector access needs and no more, NULL optional pointers
PASS = [
    ("conv", _shift("res", 8)), ("conv", _shift("f32", 8)), ("conv", _shift("bf16", 4)),
    ("conv", lambda a: dict(bias=None, res=None, f32=None)), ("conv", lambda a: dict(bf16=None, stride=2)),
    ("conv", lambda a: dict(Cin=8, kp=128, Cout=192)), ("conv relu", _shift("bf16", 4)),
    ("gn bf16", _shift("out", 8)), ("gn", lambda a: dict(C=1024)), ("gn", lambda a: dict(C=96)),
    ("micro", _shift("qkv", 4)), ("micro", _shift("out", 4)), ("micro", _shift("qn", 8)),
    ("micro generic", _shift("kn", 8)), ("micro", lambda a: dict(L=16)),
]


@pytest.fixture(scope="module")
def L():
    from gaussiananything_b200 import _lib
    return _lib.lib()


@pytest.mark.parametrize("name,change,want", CASES, ids=["%s %s" % (c[0], _label(c[1])) for c in CASES])
def test_refused_before_launch(L, name, change, want):
    call, good = _entries(L)[name]
    rc = call(L, good)
    assert rc > 0, "%s: the unchanged call should pass its checks and fail only at the launch, got %d" % (name, rc)
    bad = dict(good, **change(good))
    assert call(L, bad) == want, (name, change(good))


@pytest.mark.parametrize("name,change", PASS, ids=["%s %s" % (c[0], _label(c[1])) for c in PASS])
def test_accepted(L, name, change):
    """Calls the rules allow reach the launch (a CUDA error here, not a GA_ERR_* code)."""
    call, good = _entries(L)[name]
    rc = call(L, dict(good, **change(good)))
    assert rc > 0, (name, change(good), rc)
