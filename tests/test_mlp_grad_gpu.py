"""The linear-gradient kernels and the differentiable FusedMLP on the GPU (include/ga_b200.h Part 13) against the fp64
reference of tests/mlp_grad_ref.py: every kernel's output element by element, and every result within 1.5 times the
bf16 emulation's L2 distance from fp64, at the reference's training shapes and at the tile edges."""
import pytest
import torch

from tests import mlp_grad_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"

# (rows M, D, hidden): the training shapes of the reference's FusedMLPs
SHAPES = {
    "DiT-L": (3072, 1024, 4096),
    "DiT-B": (3072, 768, 3072),
    "decoder-block": (768, 768, 3072),
    "upsampler-1": (6912, 768, 3072),
    "upsampler-2": (30720, 768, 3072),
    "upsampler-3": (98304, 768, 3072),
    "SRT": (768, 256, 1024),
}
EDGES = [(1, 8, 8), (63, 72, 136), (127, 8, 72), (129, 136, 72), (200, 72, 8), (257, 200, 328)]


def _M():
    from gaussiananything_b200 import mlp
    return mlp


def _params(D, Hd, gen, bias_scale=0.1):
    w1 = (torch.rand(Hd, D, generator=gen) * 2 - 1) / D ** 0.5
    b1 = bias_scale * torch.randn(Hd, generator=gen)
    w2 = (torch.rand(D, Hd, generator=gen) * 2 - 1) / Hd ** 0.5
    b2 = bias_scale * torch.randn(D, generator=gen)
    return [t.to(DEV) for t in (w1, b1, w2, b2)]


def _bf(t):
    return t.to(torch.bfloat16)


def _l2(name, got, ref, emu, floor):
    e_gpu, e_emu = float((got.double() - ref).norm()), float((emu - ref).norm())
    assert e_gpu <= 1.5 * e_emu + floor, (name, "L2 from fp64", e_gpu, "emulation", e_emu, "floor", floor,
                                          "relative", R.rel_l2(got, ref), R.rel_l2(emu, ref))


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _run_kernels(M, D, Hd, seed):
    """Every kernel of the MLP's training step on random operands, each checked element by element against fp64
    on the operands it was given; then the chain's results against the fp64 MLP within 1.5 times the emulation's
    distance."""
    mlp = _M()
    gen = torch.Generator().manual_seed(seed)
    x = _bf(torch.randn(M, D, generator=gen).to(DEV))
    w1, b1, w2, b2 = _params(D, Hd, gen)
    dy = _bf(torch.randn(M, D, generator=gen).to(DEV))
    w1b, w2b = mlp._pack(w1), mlp._pack(w2)
    out = {}
    # fc1: H and Z
    h, z = mlp._fc1(x, w1b, b1, keep_pre=True)
    v, ztol, href, htol = R.fc1_bounds(x, w1b, b1)
    for name, got, ref, tol in (("Z", z, v, ztol), ("H", h, href, htol)):
        msg = R.check(got, ref, tol, name)
        assert not msg, msg
    del v, ztol, href, htol
    # dgrad with gelu': dZ = (dY W2) o gelu'(Z)
    dz = mlp._dgrad(dy, w2b, z=z)
    ref, tol = R.dgrad_bounds(dy, w2b, z)
    msg = R.check(dz, ref, tol, "dZ")
    assert not msg, msg
    del ref, tol
    # plain dgrad, bf16 and fp32 output: dx = dZ W1
    for f32 in (False, True):
        dx = mlp._dgrad(dz, w1b, f32=f32)
        assert dx.dtype == (torch.float32 if f32 else torch.bfloat16)
        ref, tol = R.dgrad_bounds(dz, w1b, out_bf16=not f32)
        msg = R.check(dx, ref, tol, "dx f32=%s" % f32)
        assert not msg, msg
        out["dx"] = dx
    del ref, tol
    # wgrad: dW2 = dY^T H, dW1 = dZ^T x
    for name, g, a in (("dW2", dy, h), ("dW1", dz, x)):
        dw = mlp._wgrad(g, a)
        ref, tol = R.wgrad_bounds(g, a)
        msg = R.check(dw, ref, tol, name)
        assert not msg, msg
        out[name] = dw
        del ref, tol
    # bias gradients
    for name, g in (("db2", dy), ("db1", dz)):
        db = mlp._bgrad(g)
        ref, tol = R.colsum_bounds(g)
        msg = R.check(db, ref, tol, name)
        assert not msg, msg
        out[name] = db
    # the chain against the fp64 MLP, within 1.5 times the emulation's distance
    out.update(H=h, Z=z, dZ=dz)
    ref = R.mlp(x, w1, b1, w2, b2, dy)
    emu = R.mlp(x, w1, b1, w2, b2, dy, emulate=True)
    floors = dict(H=R.floor(x, w1), Z=R.floor(x, w1), dZ=R.floor(dy, w2), dx=R.floor(dy, w2, w1),
                  dW1=R.floor(dy, w2, x), dW2=R.floor(dy, x, w1), db1=R.floor(dy, w2), db2=R.floor(dy))
    for k, fl in floors.items():
        _l2(k, out[k], ref[k], emu[k], fl + 1e-30)
    return out


@pytest.mark.parametrize("name", list(SHAPES))
def test_kernels_at_training_shapes(name):
    M, D, Hd = SHAPES[name]
    _run_kernels(M, D, Hd, seed=M + D)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("M,D,Hd", EDGES)
def test_kernels_at_tile_edges(M, D, Hd):
    _run_kernels(M, D, Hd, seed=M * 7 + D)


def test_outputs_stay_inside_their_tensors():
    """A kernel writes its output's elements and nothing next to them (sentinel-filled slack)."""
    from gaussiananything_b200 import _lib
    mlp = _M()
    L = _lib.lib()
    gen = torch.Generator().manual_seed(5)
    M, N, K = 129, 72, 200
    g = _bf(torch.randn(M, N, generator=gen)).to(DEV)
    w = _bf(torch.randn(N, K, generator=gen)).to(DEV)
    x = _bf(torch.randn(M, K, generator=gen)).to(DEV)
    stream = mlp.stream(g.device)
    for dtype, n, call in (
            (torch.bfloat16, M * K, lambda o: L.ga_linear_dgrad_bf16(mlp.ptr(g), mlp.ptr(w), None, o, 0, M, N, K, stream)),
            (torch.float32, M * K, lambda o: L.ga_linear_dgrad_bf16(mlp.ptr(g), mlp.ptr(w), None, o, 1, M, N, K, stream)),
            (torch.float32, N * K, lambda o: L.ga_linear_wgrad_bf16(mlp.ptr(g), mlp.ptr(x), o, M, N, K, None, 0,
                                                                    stream)),
            (torch.float32, N, lambda o: L.ga_linear_bias_grad_bf16(mlp.ptr(g), o, M, N, None, 0, stream))):
        buf = torch.full((n + 128,), float("nan"), dtype=dtype, device=DEV)
        assert call(buf.data_ptr() + 64 * buf.element_size()) == 0
        torch.cuda.synchronize()
        assert torch.isnan(buf[:64]).all() and torch.isnan(buf[64 + n:]).all()
        assert torch.isfinite(buf[64:64 + n]).all()


def test_repeated_calls_give_the_same_bits():
    mlp = _M()
    from gaussiananything_b200 import _lib
    L = _lib.lib()
    gen = torch.Generator().manual_seed(11)
    D, Hd = 256, 1024                                    # the SRT's weights: wgrad splits over M
    w1, b1, w2, b2 = _params(D, Hd, gen)
    splits = set()
    for M in (768, 3072):
        x = _bf(torch.randn(M, D, generator=gen)).to(DEV)
        dy = _bf(torch.randn(M, D, generator=gen)).to(DEV)
        splits.add(L.ga_linear_wgrad_splits(M, Hd, D))
        runs = []
        for _ in range(3):
            h, z = mlp._fc1(x, mlp._pack(w1), b1, keep_pre=True)
            dz = mlp._dgrad(dy, mlp._pack(w2), z=z)
            runs.append([h, z, dz, mlp._dgrad(dz, mlp._pack(w1)), mlp._dgrad(dz, mlp._pack(w1), f32=True),
                         mlp._wgrad(dz, x), mlp._wgrad(dy, h), mlp._bgrad(dz), mlp._bgrad(dy)])
        for r in runs[1:]:
            for a, b in zip(runs[0], r):
                assert torch.equal(_bits(a), _bits(b))
        # and the split run is within its bounds
        ref, tol = R.wgrad_bounds(dz, x)
        msg = R.check(runs[0][5], ref, tol, "dW1 M=%d" % M)
        assert not msg, msg
    assert len(splits) == 2 and max(splits) > 1, splits


# ---- the module ---------------------------------------------------------------------------------------------------

def _module(D, Hd, seed):
    torch.manual_seed(seed)
    m = _M().FusedMLP(dim_model=D, dropout=0.0, activation="gelu", hidden_layer_multiplier=Hd // D).to(DEV)
    with torch.no_grad():
        m.mlp[1].bias.normal_(0, 0.1)
        m.mlp[3].bias.normal_(0, 0.1)
    return m


def _check_module_grads(m, x, dy, need=(True, True, True, True, True), out=None):
    """Runs m on x (requires_grad as need[0]), backward with dy, and checks y, x.grad and the parameter gradients."""
    params = [m.mlp[0].weight, m.mlp[1].bias, m.mlp[2].weight, m.mlp[3].bias]
    for p, n in zip(params, need[1:]):
        p.requires_grad_(n)
        p.grad = None
    xi = x.detach().clone().requires_grad_(need[0])
    y = m(xi) if out is None else out(m, xi)
    assert y.shape == x.shape
    y.backward(dy)
    torch.cuda.synchronize()
    D = x.shape[-1]
    x2, dy2 = x.detach().reshape(-1, D), dy.detach().reshape(-1, D)
    ps = [p.detach() for p in params]
    ref = R.mlp(x2, *ps, dy2)
    emu = R.mlp(x2, *ps, dy2, emulate=True)
    w1, _, w2, _ = ps
    _l2("y", y.detach().reshape(-1, D), ref["y"], emu["y"], R.floor(x2, w1, w2) + 2.0 ** -8 * float(ref["y"].norm()) *
        (y.dtype != torch.float32))
    grads = [xi.grad] + [p.grad for p in params]
    names = ["dx", "dW1", "db1", "dW2", "db2"]
    floors = [R.floor(dy2, w2, w1), R.floor(dy2, w2, x2), R.floor(dy2, w2), R.floor(dy2, x2, w1), R.floor(dy2)]
    for name, g, n, fl, t in zip(names, grads, need, floors, [xi] + params):
        if not n:
            assert g is None, name
            continue
        assert g is not None and g.dtype == t.dtype and g.shape == t.shape, name
        assert torch.isfinite(g).all(), name
        _l2(name, g.reshape(ref[name].shape), ref[name], emu[name], fl)
    return y, grads


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_module_gradients_per_input_dtype(dtype):
    m = _module(256, 1024, seed=1)
    gen = torch.Generator().manual_seed(2)
    x = torch.randn(768, 256, generator=gen).to(DEV, dtype)
    dy = torch.randn(768, 256, generator=gen).to(DEV, dtype)
    y, grads = _check_module_grads(m, x, dy)
    assert y.dtype == dtype and grads[0].dtype == dtype
    assert all(g.dtype == torch.float32 for g in grads[1:])


def test_module_gradients_under_bf16_autocast():
    m = _module(256, 1024, seed=3)
    gen = torch.Generator().manual_seed(4)
    x = torch.randn(4, 192, 256, generator=gen).to(DEV)
    dy = torch.randn(4, 192, 256, generator=gen).to(DEV)

    def run(mod, xi):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return mod(xi)
    _check_module_grads(m, x, dy, out=run)


def test_module_gradients_3d_and_non_contiguous():
    m = _module(768, 3072, seed=5)
    gen = torch.Generator().manual_seed(6)
    x = _bf(torch.randn(2, 768, 384, generator=gen)).to(DEV).transpose(1, 2)      # [2, 384, 768], not contiguous
    assert not x.is_contiguous()
    dy = _bf(torch.randn(2, 384, 768, generator=gen)).to(DEV)
    _check_module_grads(m, x, dy)


@pytest.mark.parametrize("need", [(False, True, True, True, True), (True, False, False, True, True),
                                  (False, False, False, True, False), (True, True, True, False, False),
                                  (False, True, False, False, False)])
def test_partial_gradients_skip_their_gemms(need, monkeypatch):
    mlp = _M()
    calls = []
    for fn in ("_dgrad", "_wgrad", "_bgrad"):
        orig = getattr(mlp, fn)
        monkeypatch.setattr(mlp, fn, lambda *a, _f=orig, _n=fn, **k: (calls.append(_n), _f(*a, **k))[1])
    m = _module(256, 1024, seed=7)
    gen = torch.Generator().manual_seed(8)
    x = _bf(torch.randn(300, 256, generator=gen)).to(DEV)
    dy = _bf(torch.randn(300, 256, generator=gen)).to(DEV)
    _check_module_grads(m, x, dy, need=need)
    nx, nw1, nb1, nw2, nb2 = need
    want_dgrad = (nx or nw1 or nb1) + nx
    assert calls.count("_dgrad") == want_dgrad, calls
    assert calls.count("_wgrad") == nw1 + nw2, calls
    assert calls.count("_bgrad") == nb1 + nb2, calls


def test_zero_output_gradient_gives_exact_zeros():
    m = _module(256, 1024, seed=9)
    x = torch.randn(130, 256, device=DEV, dtype=torch.bfloat16)
    xi = x.clone().requires_grad_(True)
    m(xi).backward(torch.zeros_like(x))
    for g in [xi.grad] + [p.grad for p in m.parameters()]:
        assert g is not None and not g.any()


def test_no_grad_forward_saves_nothing_and_matches():
    m = _module(256, 1024, seed=10)
    x = torch.randn(3, 100, 256, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        y0 = m(x)
    assert y0.grad_fn is None
    y1 = m(x)                       # parameters require grad: the training forward
    assert y1.grad_fn is not None
    assert torch.equal(y0, y1.detach())
    for p in m.parameters():
        p.requires_grad_(False)
    assert m(x).grad_fn is None


def test_in_place_parameter_change_before_backward_raises():
    m = _module(256, 1024, seed=12)
    x = torch.randn(64, 256, device=DEV, requires_grad=True)
    y = m(x)
    with torch.no_grad():
        m.mlp[2].weight.mul_(0.5)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        y.sum().backward()


def test_double_backward_raises():
    m = _module(256, 1024, seed=13)
    x = torch.randn(64, 256, device=DEV, requires_grad=True)
    y = m(x)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(y.sum(), x, create_graph=True)


@pytest.mark.parametrize("M,N,K", [(4, 6144, 1024), (3072, 1024, 1024), (129, 72, 200)])
def test_linear_gradients(M, N, K):
    """DiT-L's adaLN (4 conditioning rows -> 6 x 1024) and attention projection shapes, and a tile edge."""
    mlp = _M()
    gen = torch.Generator().manual_seed(M + N)
    lin = torch.nn.Linear(K, N).to(DEV)
    x = torch.randn(M, K, generator=gen).to(DEV).requires_grad_(True)
    dy = torch.randn(M, N, generator=gen).to(DEV)
    y = mlp.linear(x, lin.weight, lin.bias)
    y.backward(dy)
    xd, wd, bd, gd = x.detach().double(), lin.weight.detach().double(), lin.bias.detach().double(), dy.double()
    r = R.bf16
    ref = dict(y=xd @ wd.T + bd, dx=gd @ wd, dW=gd.T @ xd, db=gd.sum(0))
    emu = dict(y=r(xd) @ r(wd).T + bd, dx=r(gd) @ r(wd), dW=r(gd).T @ r(xd), db=r(gd).sum(0))
    got = dict(y=y.detach(), dx=x.grad, dW=lin.weight.grad, db=lin.bias.grad)
    floors = dict(y=R.floor(xd, wd), dx=R.floor(gd, wd), dW=R.floor(gd, xd), db=R.floor(gd))
    for k in ref:
        assert got[k].dtype == torch.float32
        _l2(k, got[k], ref[k], emu[k], floors[k])
    # bias None and a frozen weight: only dx
    x.grad = None
    lin.weight.requires_grad_(False)
    mlp.linear(x, lin.weight).backward(dy)
    _l2("dx (no bias)", x.grad, ref["dx"], emu["dx"], floors["dx"])


def test_adamw_training_lowers_the_loss():
    m = _module(256, 1024, seed=14)
    gen = torch.Generator().manual_seed(15)
    x = torch.randn(768, 256, generator=gen).to(DEV)
    target = torch.randn(768, 256, generator=gen).to(DEV)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(20):
        opt.zero_grad(set_to_none=True)
        loss = torch.nn.functional.mse_loss(m(x), target)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(torch.isfinite(torch.tensor(losses)))
    assert losses[-1] < 0.9 * losses[0], losses
