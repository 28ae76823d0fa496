"""Argument checks of the networks' row-wise and element-wise entry points (include/ga_b200.h Parts 2, 3 and 5): the
alignment of every pointer a kernel reads as float4 or writes as uint2 / __nv_bfloat162, and the argument rules
next to each declaration.  Each refused call must be refused by host code before any launch.

The pointers are made-up device addresses that nothing dereferences.  A call that passed its checks would launch a
kernel on them, so the whole file is skipped where a CUDA device is present.  Without a device, a call that gets past
its checks returns a CUDA error instead of GA_ERR_BADARG, so a missing check fails its test cleanly; each case first
shows that the unchanged call does get that far.  That ga_vae_enc_input refuses bad token_xyz arguments before it
writes x_bf16 is checked with real buffers in tests/test_row_kernels_gpu.py."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.skipif(torch.cuda.is_available(),
                                reason="calls the entry points with made-up device pointers; run without a GPU")

BADARG, SIZE = -1, -3
A = 1 << 24


def ptr(k):
    """The k-th made-up device address (16-byte aligned)."""
    return A * k


def _head(L, a):
    from gaussiananything_b200._lib import GaVaeEncHead
    h = GaVaeEncHead(*[ptr(20 + i) for i in range(10)], 1e-6)
    return L.ga_vae_enc_head(C.byref(h), a["x"], a["noise"], a["R"], a["D"], a["hid"], a["zc"], a["h"], a["mean"],
                             a["logvar"], a["std"], a["latent"], None)


def _entries():
    """{name: (call, arguments that pass every check)}; call(L, args) returns the entry point's code."""
    e = {}
    e["rmsnorm"] = (lambda L, a: L.ga_rmsnorm_modulate(a["x"], a["w"], a["shift"], a["scale"], a["mod_ld"], a["rpb"],
                                                       a["out"], a["R"], a["D"], 1e-6, None),
                    dict(x=ptr(1), w=ptr(2), shift=ptr(3), scale=ptr(3) + 4 * 768, mod_ld=6 * 768, rpb=64,
                         out=ptr(4), R=128, D=768))
    ln_mod = lambda L, a: L.ga_layernorm_modulate(a["x"], a["w"], a["b"], a["shift"], a["scale"], a["mod_ld"],
                                                  a["rpb"], a["out"], a["R"], a["D"], 1e-6, None)
    e["ln_mod affine"] = (ln_mod, dict(x=ptr(1), w=ptr(2), b=ptr(3), shift=None, scale=None, mod_ld=0, rpb=1,
                                       out=ptr(4), R=257, D=1024))
    e["ln_mod shift"] = (ln_mod, dict(x=ptr(1), w=None, b=None, shift=ptr(3), scale=ptr(3) + 4 * 1024,
                                      mod_ld=6 * 24 * 1024, rpb=1, out=ptr(4), R=257, D=1024))
    e["ln_rows"] = (lambda L, a: L.ga_layernorm_rows(a["x"], a["w"], a["b"], a["y"], a["R"], a["D"], 1e-5, None),
                    dict(x=ptr(1), w=ptr(2), b=ptr(3), y=ptr(4), R=3, D=768))
    e["ln_rows scalar"] = (e["ln_rows"][0], dict(x=ptr(1) + 4, w=ptr(2) + 4, b=ptr(3) + 4, y=ptr(4) + 4, R=3, D=770))
    e["linear"] = (lambda L, a: L.ga_linear_small(a["x"], a["W"], a["bias"], a["y"], a["rows"], a["N"], a["K"],
                                                  a["act_in"], a["act_out"], a["acc"], None),
                   dict(x=ptr(1), W=ptr(2), bias=ptr(3), y=ptr(4), rows=2, N=1024, K=256, act_in=1, act_out=1, acc=1))
    e["linear scalar"] = (e["linear"][0], dict(e["linear"][1], x=ptr(1) + 4, W=ptr(2) + 4, K=300))
    e["final"] = (lambda L, a: L.ga_final_layer(a["x"], a["mod"], a["W"], a["bias"], a["y"], a["R"], a["D"],
                                                a["Cout"], a["rpb"], 1e-6, None),
                  dict(x=ptr(1), mod=ptr(2), W=ptr(3), bias=ptr(4), y=ptr(5), R=100, D=1024, Cout=14, rpb=50))
    e["final scalar"] = (e["final"][0], dict(e["final"][1], x=ptr(1) + 4, mod=ptr(2) + 4, W=ptr(3) + 4, D=1025))
    e["embed"] = (lambda L, a: L.ga_embed_fc1(a["xin"], a["Cx"], a["xin2"], a["C2"], a["W1"], a["b1"], a["h"], a["R"],
                                              a["D"], None),
                  dict(xin=ptr(1), Cx=14, xin2=ptr(2), C2=3, W1=ptr(3), b1=ptr(4), h=ptr(5), R=100, D=1024))
    e["thin"] = (lambda L, a: L.ga_thin_linear(a["x"], a["ln_w"], a["ln_b"], 1, a["W"], a["bias"], a["y"], a["R"],
                                               a["D"], 13, 1e-6, None),
                 dict(x=ptr(1), ln_w=ptr(2), ln_b=ptr(3), W=ptr(4), bias=ptr(5) + 4, y=ptr(6) + 4, R=17, D=768))
    e["seq"] = (lambda L, a: L.ga_micro_seq_build(a["parents"], a["prev_f"], a["queries"], a["seq"], a["S"], a["f"],
                                                  a["D"], None),
                dict(parents=ptr(1), prev_f=8, queries=ptr(2), seq=ptr(3), S=64, f=4, D=768))
    e["dino"] = (lambda L, a: L.ga_dino_tokens(a["patch"], a["cls"], a["reg"], 4, a["pos"], a["x"], 2, 1369, 1024,
                                               None),
                 dict(patch=ptr(1), cls=ptr(2), reg=ptr(3), pos=ptr(4), x=ptr(5)))
    e["enc_input"] = (lambda L, a: L.ga_vae_enc_input(a["img"], 2, 15, a["H"], a["W"], 16, a["x"], 12, a["step"],
                                                      a["off"], a["txyz"], None),
                      dict(img=ptr(1), H=64, W=48, x=ptr(2), step=8, off=4, txyz=ptr(3)))
    e["head"] = (_head, dict(x=ptr(1), noise=ptr(2), R=4, D=1024, hid=1024, zc=10, h=ptr(3), mean=ptr(4),
                             logvar=ptr(5), std=ptr(6), latent=ptr(7)))
    return e


def _shift(name, by):
    """name's pointer moved by `by` bytes."""
    f = lambda a: {name: a[name] + by}
    f.label = "%s%+d" % (name, by)
    return f


def _label(change):
    if hasattr(change, "label"):
        return change.label
    return ",".join("%s=%s" % kv for kv in change({}).items())


# (entry, change to the good arguments, the code it must return)
CASES = [
    # float4 reads and writes: 16 bytes
    ("rmsnorm", _shift("x", 4), BADARG), ("rmsnorm", _shift("w", 8), BADARG),
    ("rmsnorm", lambda a: dict(shift=ptr(3) + 4, scale=ptr(3) + 4 * 769), BADARG),
    ("rmsnorm", lambda a: dict(scale=ptr(3) + 4 * 770), BADARG),
    ("ln_mod affine", _shift("x", 4), BADARG), ("ln_mod affine", _shift("w", 4), BADARG),
    ("ln_mod affine", _shift("b", 8), BADARG),
    ("ln_mod shift", _shift("shift", 4), BADARG), ("ln_mod shift", _shift("scale", 12), BADARG),
    ("ln_rows", _shift("x", 4), BADARG), ("ln_rows", _shift("w", 4), BADARG), ("ln_rows", _shift("b", 4), BADARG),
    ("ln_rows", _shift("y", 8), BADARG),
    ("linear", _shift("x", 4), BADARG), ("linear", _shift("W", 8), BADARG),
    ("final", _shift("x", 4), BADARG), ("final", _shift("mod", 4), BADARG), ("final", _shift("W", 8), BADARG),
    ("thin", _shift("x", 4), BADARG), ("thin", _shift("ln_w", 4), BADARG), ("thin", _shift("ln_b", 8), BADARG),
    ("thin", _shift("W", 4), BADARG),
    ("seq", _shift("parents", 4), BADARG), ("seq", _shift("queries", 8), BADARG), ("seq", _shift("seq", 4), BADARG),
    ("dino", _shift("patch", 4), BADARG), ("dino", _shift("cls", 4), BADARG), ("dino", _shift("reg", 8), BADARG),
    ("dino", _shift("pos", 4), BADARG), ("dino", _shift("x", 12), BADARG),
    # uint2 bf16 stores: 8 bytes; __nv_bfloat162 stores: 4 bytes
    ("rmsnorm", _shift("out", 4), BADARG), ("ln_mod affine", _shift("out", 4), BADARG),
    ("ln_mod shift", _shift("out", 2), BADARG), ("enc_input", _shift("x", 2), BADARG),
    # argument rules
    ("rmsnorm", lambda a: dict(mod_ld=6 * 768 + 2), BADARG), ("rmsnorm", lambda a: dict(scale=None), BADARG),
    ("final", lambda a: dict(rpb=0), BADARG), ("final", lambda a: dict(rpb=-50), BADARG),
    ("final scalar", lambda a: dict(rpb=0), BADARG),
    ("linear", lambda a: dict(act_in=2), BADARG), ("linear", lambda a: dict(act_out=-1), BADARG),
    ("linear scalar", lambda a: dict(act_out=2), BADARG), ("linear scalar", lambda a: dict(act_in=3), BADARG),
    ("ln_rows", lambda a: dict(w=None), BADARG), ("ln_rows scalar", lambda a: dict(w=None), BADARG),
    ("embed", lambda a: dict(C2=-1), BADARG), ("embed", lambda a: dict(C2=-3, xin2=None), BADARG),
    ("ln_mod affine", lambda a: dict(w=None), BADARG), ("thin", lambda a: dict(ln_w=None), BADARG),
    ("ln_mod shift", lambda a: dict(mod_ld=6 * 24 * 1024 + 1), BADARG),
    # token_xyz arguments
    ("enc_input", lambda a: dict(off=48), BADARG), ("enc_input", lambda a: dict(off=-1), BADARG),
    ("enc_input", lambda a: dict(step=0), BADARG), ("enc_input", lambda a: dict(H=3, W=3, off=3), BADARG),
    # readout head: static + dynamic shared memory past 48 KiB
    ("head", lambda a: dict(D=12280 - 1024 - 60 + 1), SIZE), ("head", lambda a: dict(hid=12288 - 1024 - 60), SIZE),
]

# arguments the checks must let through: the scalar paths take any alignment, the head's largest size fits
PASS = [
    ("ln_rows scalar", lambda a: {}), ("linear scalar", lambda a: {}), ("final scalar", lambda a: {}),
    ("linear", lambda a: dict(K=1152, x=ptr(1) + 4, W=ptr(2) + 4)),
    ("ln_rows", lambda a: dict(D=1028, x=ptr(1) + 4, w=None, b=None, y=ptr(4) + 4)),
    ("rmsnorm", lambda a: dict(shift=None, scale=None, mod_ld=3)),
    ("embed", lambda a: dict(C2=0, xin2=None)), ("enc_input", lambda a: dict(txyz=None, off=99, step=0)),
    ("enc_input", lambda a: dict(step=1, off=47)),
    ("thin", lambda a: dict(ln_w=None, ln_b=None, bias=None)),
    ("seq", lambda a: dict(prev_f=0)), ("dino", lambda a: {}),
    ("head", lambda a: dict(D=12280 - 1024 - 60)),
]


@pytest.fixture(scope="module")
def L():
    from gaussiananything_b200 import _lib
    return _lib.lib()


@pytest.mark.parametrize("name,change,want", CASES, ids=["%s %s" % (c[0], _label(c[1])) for c in CASES])
def test_refused_before_launch(L, name, change, want):
    call, good = _entries()[name]
    rc = call(L, good)
    assert rc > 0, "%s: the unchanged call should pass its checks and fail only at the launch, got %d" % (name, rc)
    bad = dict(good, **change(good))
    assert call(L, bad) == want, (name, change(good))


@pytest.mark.parametrize("name,change", PASS, ids=["%s %s" % (c[0], _label(c[1])) for c in PASS])
def test_accepted(L, name, change):
    """Calls the rules allow reach the launch (a CUDA error here, not a GA_ERR_* code)."""
    call, good = _entries()[name]
    rc = call(L, dict(good, **change(good)))
    assert rc > 0, (name, change(good), rc)
