"""The decode references of tests/kernel_ref.py on the CPU, on small seeded inputs: the step GEMM's normalise-on-load
operand and bracket, the decode qkv fix-up chain, the two decode attention references and the bracket checker's
pooled tally (test_step_gemm_gpu.py, test_decode_attn_gpu.py and test_frame_tail_gpu.py run them against the
kernels)."""
from __future__ import annotations

import pytest
import torch

from oracle import lm_oracle as O
from tests import kernel_ref as R
from tests.kernel_ref import rbf


def _operand(rows, K, seed):
    """bf16 rows of different scales, a norm weight and the fp32 per-tile sums of squares the finalize leaves."""
    g = torch.Generator().manual_seed(seed)
    scale = torch.tensor([2.0 ** (j % 7 - 3) for j in range(rows)])[:, None]
    x = (torch.randn(rows, K, generator=g) * scale).bfloat16()
    nw = (1 + 0.1 * torch.randn(K, generator=g)).bfloat16()
    return x, nw, R.tile_ssq(x).float()


@pytest.mark.parametrize("K", [256, 1000])
def test_norm_operand_brackets_the_float64_rsqrt(K):
    eps = 1e-6
    x, nw, ssq = _operand(16, K, K)
    mid, lo, hi = R.norm_operand(x, ssq, nw, eps, K)
    assert (lo <= mid).all() and (mid <= hi).all()
    assert float((lo != hi).double().mean()) < 0.01
    # X' with r at its float64 value, and with torch's fp32 rsqrt (another rsqrtf) over another summation order
    r64 = torch.rsqrt((x.double() ** 2).sum(-1) / K + eps).float()
    r32 = torch.rsqrt((x.float() ** 2).sum(-1) / K + torch.tensor(eps, dtype=torch.float32))
    for r, what in ((r64, "float64 rsqrt"), (r32, "fp32 rsqrt")):
        R.check_bracket(rbf(rbf(x.float() * r[:, None]) * nw.float()[None, :]), lo, hi, what)


def test_step_gemm_bracket_holds_fp32_accumulations():
    eps, K, n = 1e-6, 1000, 96
    x, nw, ssq = _operand(16, K, 3)
    W = (torch.randn(n, K, generator=torch.Generator().manual_seed(4)) * 0.05).bfloat16()
    mid, lo, hi = R.norm_operand(x, ssq, nw, eps, K)
    # the worst-case accumulation bound (ACC) around an fp32 GEMM
    ref, absprod = R.fp64_gemm(mid, W)
    err = (mid @ W.float().T).double() - ref
    assert (err.abs() <= R.acc_bound(absprod, K, 1)).all()
    # the C_AMB bracket of rbf(W X') holds the fp32 GEMM on either end of X''s bracket and its float64 value
    v, E = R.normed_gemm(x, ssq, nw, eps, W)
    assert torch.equal(v, ref)
    b_lo, b_hi = R.bracket_bf16(v, E)
    assert (b_lo <= rbf(v)).all() and (rbf(v) <= b_hi).all()
    for xp, what in ((lo, "lo"), (hi, "hi"), (mid, "mid")):
        R.check_bracket(rbf(xp @ W.float().T), b_lo, b_hi, f"fp32 GEMM of X' {what}")
        R.check_bracket(rbf(R.fp64_gemm(xp, W)[0]), b_lo, b_hi, f"float64 GEMM of X' {what}")


@pytest.mark.parametrize("Dh", [64, 128])
def test_fixup_chain_holds_the_prefill_emulation(Dh):
    """The decode fix-up (step GEMM normalised on load, bias, qk-norm, RoPE) over an fp32 GEMM of its operand agrees
    with qkv_prep_row_kernel's emulation: the same arithmetic after the GEMM."""
    eps, D, H, Hkv, n = 1e-6, 256, 4, 2, 24
    g = torch.Generator().manual_seed(Dh)
    x, nw, ssq = _operand(n, D, Dh + 1)
    W = (torch.randn((H + 2 * Hkv) * Dh, D, generator=g) * 0.05).bfloat16()
    b = (torch.randn((H + 2 * Hkv) * Dh, generator=g) * 0.02).bfloat16()
    qn, kn = (1 + 0.1 * torch.randn(Dh, generator=g)).bfloat16(), (1 + 0.1 * torch.randn(Dh, generator=g)).bfloat16()
    cs = O.precompute_freqs_cis(512, Dh, 1e6)[torch.randint(0, 512, (n,), generator=g)].float()
    q_pre, k_pre, v = R.fixup_ref64(x, ssq, nw, W, b, H, Hkv, Dh, qn, kn, eps)
    ref = (R.rope_bracket(*q_pre, cs), R.rope_bracket(*k_pre, cs), v)
    mid = R.norm_operand(x, ssq, nw, eps, D)[0]
    emul = R.qkv_emul(mid @ W.float().T, b, H, Hkv, Dh, qn, kn, eps, cs)
    for (elo, ehi, emid), (rlo, rhi, rmid), what in zip(emul, ref, "qkv"):
        assert (rlo <= rmid).all() and (rmid <= rhi).all(), what
        R.check_bracket(emid, rlo, rhi, f"{what}: emulation in the fix-up bracket", rmid, share=0.05)


def _attn_case(Dh, L, seed):
    g = torch.Generator().manual_seed(seed)
    Hkv, G = 2, 4
    K = torch.randn(Hkv, L, Dh, generator=g).bfloat16().double()
    V = torch.randn(Hkv, L, Dh, generator=g).bfloat16().double()
    q = torch.randn(Hkv, G, Dh, generator=g).bfloat16().double()
    scale32 = float(torch.tensor(1.0) / torch.sqrt(torch.tensor(float(Dh))))
    o64 = torch.nn.functional.scaled_dot_product_attention(q, K, V, scale=scale32)  # [Hkv, G, Dh]
    return q, K, V, scale32, o64


@pytest.mark.parametrize("Dh", [64, 128])
@pytest.mark.parametrize("L", [1, 37, 300])
def test_attn_decode_fp32_brackets_the_float64_softmax(Dh, L):
    q, K, V, scale, o64 = _attn_case(Dh, L, Dh + L)
    o, E = R.attn_decode_fp32(q, torch.zeros_like(q), K, V, scale)
    assert torch.allclose(o, o64, rtol=1e-12, atol=1e-12)
    assert (E > 0).all()
    R.check_bracket(rbf(o64), rbf(o - E), rbf(o + E), "float64 softmax")
    # an fp32 evaluation, and a q anywhere inside a bracket of width qd around it
    o32 = torch.softmax((q.float() @ K.float().transpose(1, 2)) * scale, -1) @ V.float()
    R.check_bracket(rbf(o32), rbf(o - E), rbf(o + E), "fp32 softmax")
    qd = 2.0 ** -8 * q.abs()
    o, E = R.attn_decode_fp32(q, qd, K, V, scale)
    for q2 in (q - qd, q + qd):
        o2 = torch.nn.functional.scaled_dot_product_attention(q2, K, V, scale=scale)
        R.check_bracket(rbf(o2), rbf(o - E), rbf(o + E), "float64 softmax of a q inside the bracket")


@pytest.mark.parametrize("Dh", [64, 128])
@pytest.mark.parametrize("L", [1, 5, 10])
def test_attn_decode_bf16_brackets_the_bf16_chain(Dh, L):
    """The all-bf16 attention (oracle.lm_oracle._eq_sdpa) rounds the scores, the scaled scores, the probabilities and
    the output to bf16: mid is torch's float64 softmax through those roundings, and the bracket holds the chain
    evaluated in fp32."""
    q, K, V, scale, _ = _attn_case(Dh, L, Dh + L + 1)
    lo, hi, mid = R.attn_decode_bf16(q, q, q, K, V, scale)
    assert (lo <= mid).all() and (mid <= hi).all()
    Kt = K.transpose(1, 2)
    s64 = rbf(rbf(q @ Kt) * scale).double()
    assert torch.equal(mid, rbf(rbf(torch.softmax(s64, -1)).double() @ V))
    s32 = rbf(rbf(q.float() @ Kt.float()) * scale)
    R.check_bracket(rbf(rbf(torch.softmax(s32, -1)) @ V.float()), lo, hi, "fp32 evaluation of the bf16 chain")


def test_check_bracket_pools_its_share_in_a_tally():
    got = torch.zeros(1000)
    lo, hi = got - 1, got + 1
    for n_diff, ok in ((9, True), (11, False)):
        mid = got.clone()
        mid[:n_diff] = 0.5
        tally = [0, 0]
        R.check_bracket(got[:500], lo[:500], hi[:500], "first half", mid[:500], tally=tally)  # no share per call
        R.check_bracket(got[500:], lo[500:], hi[500:], "second half", mid[500:], tally=tally)
        assert tally == [n_diff, 1000]
        if ok:
            R.check_tally(tally, "pooled")
            R.check_bracket(got, lo, hi, "one call", mid)
        else:
            with pytest.raises(AssertionError, match="11 of 1000"):
                R.check_tally(tally, "pooled")
            with pytest.raises(AssertionError, match="differ"):
                R.check_bracket(got, lo, hi, "one call", mid)
    with pytest.raises(AssertionError, match="off"):
        R.check_bracket(got, lo + 1.5, hi, "outside")
