"""Argument checks of the PatchGAN discriminator's entry points (include/ga_b200.h Part 11): alignment of the pointers
the kernels access as float2 or __nv_bfloat162, channel multiples, sizes and workspaces.  Each refused call must be
refused by host code before any launch.

The pointers are made-up device addresses that nothing dereferences.  A call that passed its checks would launch a
kernel on them, so the whole file is skipped where a CUDA device is present.  Without a device, a call that gets past
its checks returns a CUDA error instead of GA_ERR_BADARG, so a missing check fails its test cleanly; each case first
shows that the unchanged call does get that far."""
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
    e["lrelu"] = (lambda L, a: L.ga_conv4x4_lrelu_bf16(a["x"], a["n"], a["H"], a["W"], a["Cin"], a["w"], a["kp"],
                                                       a["bias"], a["Cout"], a["stride"], a["out"], None),
                  dict(x=ptr(1), n=2, H=24, W=24, Cin=8, w=ptr(2), kp=128, bias=ptr(3), Cout=64, stride=2,
                       out=ptr(4)))
    e["stats"] = (lambda L, a: L.ga_conv4x4_stats(a["x"], a["n"], a["H"], a["W"], a["Cin"], a["w"], a["kp"],
                                                  a["Cout"], a["stride"], a["z"], a["partial"], None),
                  dict(x=ptr(1), n=4, H=12, W=12, Cin=64, w=ptr(2), kp=1024, Cout=128, stride=2, z=ptr(3),
                       partial=ptr(4)))
    e["bn_forward"] = (lambda L, a: L.ga_disc_bn_forward(a["z"], a["partial"], a["M"], a["C"], a["gamma"], a["beta"],
                                                         a["training"], 0.1, 1e-5, a["rm"], a["rv"], a["mean"],
                                                         a["rstd"], a["a"], None),
                       dict(z=ptr(1), partial=ptr(2), M=144, C=128, gamma=ptr(3), beta=ptr(4), training=1,
                            rm=ptr(5), rv=ptr(6), mean=ptr(7), rstd=ptr(8), a=ptr(9)))
    e["conv5"] = (lambda L, a: L.ga_disc_conv5(a["x"], a["n"], a["H"], a["W"], a["w5"], a["bias"], a["out"], None),
                  dict(x=ptr(1), n=4, H=5, W=7, w5=ptr(2), bias=ptr(3), out=ptr(4)))
    e["conv5_backward"] = (lambda L, a: L.ga_disc_conv5_backward(a["g5"], a["n"], a["H"], a["W"], a["w5"], a["a4"],
                                                                 a["z4"], a["mean4"], a["rstd4"], a["gy4"],
                                                                 a["bn_partial"], a["dw_partial"], a["dw5"], None),
                           dict(g5=ptr(1), n=4, H=5, W=7, w5=ptr(2), a4=ptr(3), z4=ptr(4), mean4=ptr(5),
                                rstd4=ptr(6), gy4=ptr(7), bn_partial=ptr(8), dw_partial=ptr(9), dw5=ptr(10)))
    dgrad = lambda L, a: L.ga_disc_dgrad(a["g"], a["n"], a["H"], a["W"], a["Cg"], a["w"], a["kp"], a["Cout"],
                                         a["stride"], a["act"], a["z"], a["mean"], a["rstd"], a["gy"], a["partial"],
                                         a["out"], None)
    e["dgrad_bn"] = (dgrad, dict(g=ptr(1), n=4, H=6, W=6, Cg=256, w=ptr(2), kp=1024, Cout=128, stride=2, act=ptr(3),
                                 z=ptr(4), mean=ptr(5), rstd=ptr(6), gy=ptr(7), partial=ptr(8), out=None))
    e["dgrad_lrelu"] = (dgrad, dict(g=ptr(1), n=2, H=12, W=12, Cg=128, w=ptr(2), kp=512, Cout=64, stride=2,
                                    act=ptr(3), z=None, mean=None, rstd=None, gy=None, partial=None, out=ptr(4)))
    e["bn_backward"] = (lambda L, a: L.ga_disc_bn_backward(a["gy"], a["z"], a["M"], a["C"], a["mean"], a["rstd"],
                                                           a["gamma"], a["partial"], a["n_partial"], 1, a["dgamma"],
                                                           a["dbeta"], a["k"], a["dz"], None),
                        dict(gy=ptr(1), z=ptr(2), M=144, C=128, mean=ptr(3), rstd=ptr(4), gamma=ptr(5),
                             partial=ptr(6), n_partial=2, dgamma=ptr(7), dbeta=ptr(8), k=ptr(9), dz=ptr(10)))
    e["wgrad"] = (lambda L, a: L.ga_disc_wgrad(a["dy"], a["x"], a["n"], a["H"], a["W"], a["Cin"], a["Co"],
                                               a["stride"], a["cin_out"], a["ws"], a["ws_bytes"], a["dw"], None),
                  dict(dy=ptr(1), x=ptr(2), n=2, H=24, W=24, Cin=8, Co=64, stride=2, cin_out=3, ws=ptr(3),
                       ws_bytes=L.ga_disc_wgrad_workspace_bytes(2, 12, 12, 64, 8), dw=ptr(4)))
    e["colsum"] = (lambda L, a: L.ga_disc_colsum(a["x"], 1, a["rows"], a["C"], a["scratch"], a["bytes"], a["out"],
                                                 None),
                   dict(x=ptr(1), rows=1025, C=64, scratch=ptr(2), bytes=L.ga_disc_colsum_scratch_bytes(1025, 64),
                        out=ptr(3)))
    e["input_backward"] = (lambda L, a: L.ga_disc_input_backward(a["g1"], a["n"], a["H"], a["W"], a["w1"], a["dx"],
                                                                 None),
                           dict(g1=ptr(1), n=2, H=24, W=24, w1=ptr(2), dx=ptr(3)))
    return e


def _shift(name, by):
    """name's pointer or byte count moved by `by`."""
    f = lambda a: {name: a[name] + by}
    f.label = "%s%+d" % (name, by)
    return f


def _label(change):
    if hasattr(change, "label"):
        return change.label
    return ",".join("%s=%s" % kv for kv in change(dict.fromkeys(("ws_bytes", "bytes"), 0)).items())


# (entry, change to the good arguments, the code it must return)
CASES = [
    # float2 pointers: 8 bytes
    ("stats", _shift("z", 4), BADARG), ("stats", _shift("partial", 4), BADARG),
    ("bn_forward", _shift("z", 4), BADARG), ("bn_forward", _shift("partial", 4), BADARG),
    ("conv5_backward", _shift("z4", 4), BADARG), ("conv5_backward", _shift("gy4", 4), BADARG),
    ("conv5_backward", _shift("bn_partial", 4), BADARG), ("conv5_backward", _shift("dw_partial", 4), BADARG),
    ("dgrad_bn", _shift("z", 4), BADARG), ("dgrad_bn", _shift("gy", 4), BADARG),
    ("dgrad_bn", _shift("partial", 4), BADARG),
    ("bn_backward", _shift("gy", 4), BADARG), ("bn_backward", _shift("z", 4), BADARG),
    ("bn_backward", _shift("partial", 4), BADARG), ("bn_backward", _shift("k", 4), BADARG),
    ("wgrad", _shift("ws", 4), BADARG),
    # __nv_bfloat162 pointers: 4 bytes
    ("lrelu", _shift("out", 2), BADARG), ("bn_forward", _shift("a", 2), BADARG),
    ("dgrad_lrelu", _shift("out", 2), BADARG), ("dgrad_bn", _shift("act", 2), BADARG),
    ("bn_backward", _shift("dz", 2), BADARG), ("conv5_backward", _shift("a4", 2), BADARG),
    # 16-byte operands of the convolutions
    ("lrelu", _shift("x", 8), BADARG), ("stats", _shift("w", 8), BADARG), ("conv5", _shift("x", 8), BADARG),
    ("wgrad", _shift("dy", 8), BADARG), ("input_backward", _shift("g1", 8), BADARG),
    # channel multiples
    ("lrelu", lambda a: dict(Cin=4, kp=64), BADARG), ("stats", lambda a: dict(Cin=60), BADARG),
    ("wgrad", lambda a: dict(Cin=12), BADARG), ("dgrad_bn", lambda a: dict(Cg=252), BADARG),
    ("lrelu", lambda a: dict(Cout=96), BADARG), ("stats", lambda a: dict(Cout=32), BADARG),
    ("wgrad", lambda a: dict(Co=96), BADARG), ("dgrad_bn", lambda a: dict(Cout=96), BADARG),
    ("stats", lambda a: dict(kp=960), BADARG),
    # BatchNorm: C odd, training needs partials and M >= 2
    ("bn_forward", lambda a: dict(C=127), BADARG), ("bn_backward", lambda a: dict(C=127), BADARG),
    ("bn_forward", lambda a: dict(partial=None), BADARG), ("bn_forward", lambda a: dict(M=1), BADARG),
    ("bn_backward", lambda a: dict(n_partial=0), BADARG),
    # colsum: 256 % C
    ("colsum", lambda a: dict(C=3, bytes=10 ** 6), BADARG), ("colsum", lambda a: dict(C=512, bytes=10 ** 6), BADARG),
    # workspaces too small
    ("wgrad", _shift("ws_bytes", -4), WORKSPACE), ("colsum", _shift("bytes", -4), WORKSPACE),
    # wgrad: cin_out in [1, Cin]
    ("wgrad", lambda a: dict(cin_out=9), BADARG), ("wgrad", lambda a: dict(cin_out=0), BADARG),
    # sizes below 2
    ("conv5", lambda a: dict(H=1), BADARG), ("conv5_backward", lambda a: dict(W=1), BADARG),
    ("input_backward", lambda a: dict(H=1), BADARG), ("lrelu", lambda a: dict(W=1), BADARG),
    ("stats", lambda a: dict(H=1), BADARG), ("dgrad_bn", lambda a: dict(H=1), BADARG),
    ("wgrad", lambda a: dict(W=1), BADARG),
    # dgrad: the BatchNorm epilogue's pointers and conv 1's bf16 output are exclusive
    ("dgrad_bn", lambda a: dict(out=ptr(11)), BADARG), ("dgrad_lrelu", lambda a: dict(gy=ptr(11)), BADARG),
    # conv 5's weight gradient needs both its partials and dw5
    ("conv5_backward", lambda a: dict(dw5=None), BADARG),
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
