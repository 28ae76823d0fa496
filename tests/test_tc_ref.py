"""The checker of tests/tc_ref.py has teeth (CPU only): on synthetic outputs -- the fp64 reference rounded the way the
kernels round -- it passes the unmodified output and flags each of the faults a subtly wrong kernel makes: one large
element off by 2 %, two adjacent columns swapped, the bias dropped from one column, one guard element overwritten,
one attention row computed with a padded key left unmasked."""
import pytest
import torch

from tests import tc_ref as tr

GEMM_MODES = [tr.BF16_OUT, tr.GELU_OUT, tr.F32_OUT, tr.RESID_GATE, tr.GEGLU]


def _round_like_kernel(mode, ref):
    """fp64 -> the kernel's output type: fp32 for F32_OUT / RESID_GATE, fp32 then bf16 for the bf16 modes."""
    out = ref.float()
    return out if mode in (tr.F32_OUT, tr.RESID_GATE) else out.bfloat16()


def _gemm_case(mode, M=40, N=96, K=200, seed=0):
    gen = torch.Generator().manual_seed(seed + 10 * mode)
    _, A, _ = tr.hostile_operand(M, K, "cpu", gen)
    _, W, _ = tr.hostile_operand(N, K, "cpu", gen, scale=K ** -0.5)
    bias = torch.randn(N, generator=gen) * 0.5
    x0 = torch.randn(M, N, generator=gen) if mode == tr.RESID_GATE else None
    gate = (torch.rand(M, N, generator=gen) + 0.5) if mode == tr.RESID_GATE else None
    Y, S = tr.gemm_ref(A, W, bias)
    ref, tol = tr.epilogue_ref(mode, Y, S, x0=x0, gate=gate)
    return Y, S, bias, x0, gate, ref, tol


def test_hostile_operand_is_nan_outside_the_operand():
    buf, view, ld = tr.hostile_operand(5, 24, "cpu", torch.Generator().manual_seed(0))
    assert ld == 32 and buf.shape == (13, 32)
    assert torch.isfinite(view.float()).all()
    assert torch.isnan(buf[:5, 24:].float()).all() and torch.isnan(buf[5:].float()).all()


@pytest.mark.parametrize("mode", GEMM_MODES)
def test_gemm_checker_passes_rounded_reference(mode):
    _, _, _, _, _, ref, tol = _gemm_case(mode)
    worst, msg = tr.check(_round_like_kernel(mode, ref), ref, tol)
    assert msg == "", msg
    assert worst < 1.0


@pytest.mark.parametrize("mode", GEMM_MODES)
def test_gemm_checker_flags_largest_element_off_by_two_percent(mode):
    _, _, _, _, _, ref, tol = _gemm_case(mode)
    got = _round_like_kernel(mode, ref)
    i = int(ref.abs().argmax())
    got.view(-1)[i] = got.view(-1)[i] * 1.02
    assert tr.check(got, ref, tol)[1] != ""


@pytest.mark.parametrize("mode", GEMM_MODES)
def test_gemm_checker_flags_two_adjacent_columns_swapped(mode):
    _, _, _, _, _, ref, tol = _gemm_case(mode)
    got = _round_like_kernel(mode, ref)
    r = ref.shape[0] // 2
    got[r, 6], got[r, 7] = got[r, 7].clone(), got[r, 6].clone()
    if torch.equal(got[r, 6], got[r, 7]):
        pytest.skip("equal neighbours")
    assert tr.check(got, ref, tol)[1] != ""


@pytest.mark.parametrize("mode", GEMM_MODES)
def test_gemm_checker_flags_bias_dropped_from_one_column(mode):
    Y, S, bias, x0, gate, ref, tol = _gemm_case(mode)
    j = 10                                           # for GEGLU: the x half of output column 5
    Yb = Y.clone()
    Yb[:, j] -= bias[j].double()
    ref_b, _ = tr.epilogue_ref(mode, Yb, S, x0=x0, gate=gate)
    jo = j // 2 if mode == tr.GEGLU else j
    got = _round_like_kernel(mode, ref)
    got[:, jo] = _round_like_kernel(mode, ref_b)[:, jo]
    assert tr.check(got, ref, tol)[1] != ""


def test_heads_checker_passes_rounded_reference_and_flags_a_swap():
    gen = torch.Generator().manual_seed(3)
    B, rpb, H, K = 2, 21, 2, 72
    _, A, _ = tr.hostile_operand(B * rpb, K, "cpu", gen)
    _, W, _ = tr.hostile_operand(3 * H * 64, K, "cpu", gen, scale=K ** -0.5)
    bias = torch.randn(3 * H * 64, generator=gen) * 0.2
    qn, kn = torch.rand(64, generator=gen) + 0.5, torch.rand(64, generator=gen) + 0.5
    Y, S = tr.gemm_ref(A, W, bias)
    parts = tr.heads_ref(Y, S, B, rpb, H, 0, qn_w=qn, kn_w=kn)
    assert sorted(parts) == ["k", "q", "v"] and parts["v"][0].shape == (B, H, 64, rpb)
    for name, (ref, tol) in parts.items():
        got = ref.float().bfloat16()
        assert tr.check(got, ref, tol)[1] == "", name
        got[1, 1, 3, 10], got[1, 1, 3, 11] = got[1, 1, 3, 11].clone(), got[1, 1, 3, 10].clone()
        assert tr.check(got, ref, tol)[1] != "", name


def test_guard_flags_one_overwritten_element():
    M, N, ld = 5, 6, 9
    for dt in (torch.float32, torch.bfloat16):
        g = tr.GuardBuf((M + 2, ld), dt, "cpu")
        written = tr.region(g.shape, slice(0, M), slice(0, N))
        g.t[:M, :N] = 1.5
        assert g.intact(written) == (True, "")
        g.t[2, N] = 0.0                                  # the ld_out slack of one row
        ok, msg = g.intact(written)
        assert not ok and "element (2, 6)" in msg
        g.fill_outside(written)
        assert g.intact(written)[0] and float(g.t[0, 0]) == 1.5
        g.buf[-1] = 0.0                                  # past the tensor
        assert not g.intact(written)[0]
        g.fill_outside(written)
        g.t[M, 0] = float("nan")                         # a canonical NaN is not the sentinel
        assert not g.intact(written)[0]


def _attention_like_kernel(q, k, vt, Nq, Nk, scale, causal=False, extra_key=None, row=None):
    """The kernel's rounding: fp32 scores and probabilities, P rounded to bf16 in P V, l summed from the fp32
    probabilities, O rounded to bf16.  extra_key / row: row `row` also sees key index `extra_key` (unmasked)."""
    BH = q.shape[0]
    out = torch.empty(BH, Nq, 64, dtype=torch.bfloat16)
    for bh in range(BH):
        s = (q[bh, :Nq].float() @ k[bh].float().T) * scale
        mask = torch.arange(k.shape[1])[None, :] >= Nk
        mask = mask.expand(Nq, -1).clone()
        if causal:
            mask |= torch.arange(k.shape[1])[None, :] > torch.arange(Nq)[:, None]
        if extra_key is not None:
            mask[row, extra_key] = False
        s = s.masked_fill(mask, float("-inf"))
        p = torch.exp(s - s.max(-1, keepdim=True).values)
        o = (p.bfloat16().float() @ vt[bh].float().T) / p.sum(-1, keepdim=True)
        out[bh] = o.bfloat16()
    return out


@pytest.mark.parametrize("causal", [False, True])
def test_attention_checker_passes_rounded_reference_and_flags_an_unmasked_padded_key(causal):
    B, H, N, pitch = 1, 2, 77, 128
    gen = torch.Generator().manual_seed(7)
    q, k, vt = tr.attention_inputs(B, H, N, N, pitch, pitch, "cpu", gen)
    ref, tol = tr.attention_ref(q, k, vt, B, H, N, N, 0.125, causal=causal)
    fold = lambda o: o.view(B, H, N, 64).permute(0, 2, 1, 3).reshape(B, N, H * 64)
    got = fold(_attention_like_kernel(q, k, vt, N, N, 0.125, causal))
    worst, msg = tr.check(got, ref, tol)
    assert msg == "" and worst < 1.0, msg
    # padded key N unmasked in one row: flagged in every row where it scores above the real keys' maximum
    s = (q[:, :N].double() @ k[:, N].double()[:, :, None])[..., 0]               # [B*H, N] scores of key N
    row = int(s[0].argmax())
    bad = fold(_attention_like_kernel(q, k, vt, N, N, 0.125, causal, extra_key=N, row=row))
    assert tr.check(bad, ref, tol)[1] != ""
    assert torch.equal(bad[:, :row], got[:, :row]) and torch.equal(bad[:, row + 1:], got[:, row + 1:])
    # the same key unmasked in every row (a mask shifted by one key) is flagged as a whole
    assert tr.check(fold(_attention_like_kernel(q, k, vt, N, N, 0.125, causal, extra_key=N, row=slice(None))),
                    ref, tol)[1] != ""


def test_attention_reference_on_sampled_rows_matches_the_full_one():
    B, H, Nq, Nk = 1, 2, 150, 140
    gen = torch.Generator().manual_seed(8)
    q, k, vt = tr.attention_inputs(B, H, Nq, Nk, 256, 256, "cpu", gen)
    full, tfull = tr.attention_ref(q, k, vt, B, H, Nq, Nk, 0.2)
    rows = torch.tensor([0, 5, 127, 128, 149])
    part, tpart = tr.attention_ref(q, k, vt, B, H, Nq, Nk, 0.2, rows=rows, chunk=2)
    assert torch.allclose(part, full[:, rows], rtol=1e-12, atol=1e-14)
    assert torch.allclose(tpart, tfull[:, rows], rtol=1e-12, atol=1e-14)
    assert tr.static_bound(q, k, Nq, Nk, 0.125) >= float(
        (q[:, :Nq].double() @ k[:, :Nk].double().transpose(1, 2)).abs().max()) * 0.125
