"""The prefill float64 references and fp32 emulations of tests/kernel_ref.py on the CPU: shapes, orderings and the
bounds' logic, without a GPU (tests/test_prefill_gpu.py runs them against the kernels)."""
from __future__ import annotations

import math

import torch

from oracle import lm_oracle as O
from tests import kernel_ref as R
from tests.kernel_ref import rbf


def test_gate_row_matches_interleave_w13():
    from fish_speech_b200.engine import interleave_w13

    I, D = 528, 8
    w1 = torch.arange(I * D, dtype=torch.float32).view(I, D)
    w3 = -w1 - 1
    m = interleave_w13(w1, w3)
    gi = R.gate_row(torch.arange(I))
    assert torch.equal(m[gi], w1) and torch.equal(m[gi + 16], w3)
    Ip = math.ceil(I / 64) * 64
    pad = R.gate_row(torch.arange(I, Ip))
    assert (m[pad] == 0).all() and (m[pad + 16] == 0).all() and m.shape[0] == 2 * Ip


def test_embed_ref_is_the_oracle_and_brackets_its_rounding():
    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=3)
    C, cs = cfg.num_codebooks, cfg.codebook_size
    g = torch.Generator().manual_seed(1)
    tok = torch.randint(0, cfg.vocab_size, (64, C + 1), generator=g)
    tok[:, 1:] = torch.randint(0, cs, (64, C), generator=g)
    tok[:6, 0] = torch.tensor([cfg.semantic_begin_id - 1, cfg.semantic_begin_id, cfg.semantic_end_id,
                               cfg.semantic_end_id + 1, cfg.im_end_id, 0])
    tok[10:40, 0] = torch.randint(cfg.semantic_begin_id, cfg.semantic_end_id + 1, (30,), generator=g)
    for scale in (True, False):
        lo, hi, mid, x64 = R.embed_ref(tok, w["embeddings.weight"], w["codebook_embeddings.weight"], C, cs,
                                       cfg.semantic_begin_id, cfg.semantic_end_id, scale)
        c2 = O.tiny_config(scale_codebook_embeddings=scale)
        st = O.LMState(c2, {k: v.double() for k, v in w.items()})
        assert torch.allclose(x64, O.embed(st, tok.t()[None])[0], rtol=1e-12, atol=1e-15)
        assert (lo <= mid).all() and (mid <= hi).all() and (lo <= rbf(x64) + 1e-2).all()
        # the oracle in bf16 (one rounding of the codebook sum, of the add, of the scale) lies in the bracket
        stb = O.LMState(c2, w)
        xb = O.embed(stb, tok.t()[None])[0].float()
        R.check_bracket(xb, lo, hi, f"bf16 oracle, scale={scale}")
        # non-semantic rows are the embedding row itself
        plain = ~((tok[:, 0] >= cfg.semantic_begin_id) & (tok[:, 0] <= cfg.semantic_end_id))
        assert torch.equal(mid[plain], w["embeddings.weight"][tok[plain, 0]].float())
        # the wrong embeds the GPU test relies on falling outside: scale on non-semantic rows, sem_end exclusive
        sem_end_row = 2
        wrong = rbf(mid[sem_end_row] * 0 + w["embeddings.weight"][tok[sem_end_row, 0]].float())
        assert not ((wrong >= lo[sem_end_row]) & (wrong <= hi[sem_end_row])).all()


def test_row_norm_brackets_an_fp32_block_sum():
    g = torch.Generator().manual_seed(2)
    x = rbf(torch.randn(16, 2560, generator=g))
    w = (1 + 0.1 * torch.randn(2560, generator=g)).bfloat16()
    lo, hi, mid = R.row_norm(x, w, 1e-6)
    # the kernel's arithmetic with another summation order
    ss = (x.view(16, 10, 256) ** 2).sum(-1).sum(-1, keepdim=True)
    r = torch.rsqrt(ss / 2560 + torch.tensor(1e-6, dtype=torch.float32))
    got = rbf(rbf(x * r) * w.float())
    R.check_bracket(got, lo, hi, "norm", mid)
    assert float((lo != hi).double().mean()) < 0.01


def test_qkv_emulation_and_float64_chain_agree():
    g = torch.Generator().manual_seed(4)
    H, Hkv, Dh, D, n = 4, 2, 64, 256, 40
    W = (torch.randn((H + 2 * Hkv) * Dh, D, generator=g) * 0.05).bfloat16()
    b = (torch.randn((H + 2 * Hkv) * Dh, generator=g) * 0.02).bfloat16()
    qn, kn = (1 + 0.1 * torch.randn(Dh, generator=g)).bfloat16(), (1 + 0.1 * torch.randn(Dh, generator=g)).bfloat16()
    xn = torch.randn(n, D, generator=g).bfloat16()
    cs = O.precompute_freqs_cis(512, Dh, 1e6)[torch.randint(0, 512, (n,), generator=g)].float()
    ws = (xn.float() @ W.float().T)  # an fp32 GEMM result
    e = R.qkv_emul(ws, b, H, Hkv, Dh, qn, kn, 1e-6, cs)
    r = R.qkv_ref64(xn, W, b, H, Hkv, Dh, qn, kn, 1e-6, cs)
    for (elo, ehi, emid), (rlo, rhi, rmid), what in zip(e, r, "qkv"):
        assert elo.shape == rlo.shape
        # the emulation's value lies in the float64 bracket and is mostly its rounding
        R.check_bracket(emid, rlo, rhi, f"{what}: emulation in the float64 bracket", rmid, share=0.05)
        assert float((elo != ehi).double().mean()) < 0.01, f"{what}: emulation brackets too wide"
    # and both match the oracle's layer in bf16 (nn.RMSNorm, apply_rotary) to within bf16 rounding
    q = (xn.float() @ W.float().T + b.float())[:, : H * Dh].bfloat16().view(1, n, H, Dh)
    q = torch.nn.functional.rms_norm(q, (Dh,), qn, 1e-6)
    q = O.apply_rotary(q, cs.bfloat16().view(n, Dh // 2, 2))[0].float()
    assert float((q - r[0][2]).abs().max()) <= 0.05 * float(q.abs().max())


def test_swiglu_and_residual():
    g = torch.Generator().manual_seed(5)
    I, D, n = 528, 256, 20
    w1 = (torch.randn(I, D, generator=g) * 0.05).bfloat16()
    w3 = (torch.randn(I, D, generator=g) * 0.05).bfloat16()
    xn = torch.randn(n, D, generator=g).bfloat16()
    from fish_speech_b200.engine import interleave_w13

    ws = xn.float() @ interleave_w13(w1, w3).float().T
    lo, hi, mid = R.swiglu_emul(ws, I)
    rlo, rhi, rmid = R.swiglu_ref64(xn, w1, w3)
    R.check_bracket(mid, rlo, rhi, "swiglu emulation in the float64 bracket", rmid, share=0.05)
    assert lo.shape == (n, I)
    x = torch.randn(n, D, generator=g).bfloat16()
    wo = (torch.randn(D, I, generator=g) * 0.05).bfloat16()
    a = mid.bfloat16()
    got = R.resid_emul(x, a.float() @ wo.float().T, None)
    rlo, rhi, rmid = R.resid_ref64(x, a, wo, None)
    R.check_bracket(got, rlo, rhi, "residual emulation in the float64 bracket", rmid, share=0.05)


def test_attention_reference_and_its_teeth():
    g = torch.Generator().manual_seed(6)
    Hkv, G, Dh, L = 2, 2, 64, 300
    K = torch.randn(Hkv, L, Dh, generator=g).bfloat16().double()
    V = torch.randn(Hkv, L, Dh, generator=g).bfloat16().double()
    pos = torch.tensor([0, 1, 63, 64, 65, 150, 298])
    q = torch.randn(len(pos), Hkv, G, Dh, generator=g).bfloat16().double()
    scale = 1 / math.sqrt(Dh)
    o, E = R.attn_ref64(q, K, V, pos, scale)
    for i, p in enumerate(pos.tolist()):  # a plain softmax, row by row
        s = torch.einsum("hgd,hld->hgl", q[i], K[:, : p + 1]) * scale
        want = torch.einsum("hgl,hld->hgd", torch.softmax(s, -1), V[:, : p + 1])
        assert torch.allclose(o[i], want, rtol=1e-12, atol=1e-12)
    assert (E > 0).all() and (E < 2.0 ** -10 * V.abs().max()).all()
    # an fp32 evaluation of the same softmax stays inside the bracket
    o32 = torch.stack([torch.einsum("hgl,hld->hgd", torch.softmax(
        (torch.einsum("hgd,hld->hgl", q[i].float(), K[:, : p + 1].float()) * scale), -1), V[:, : p + 1].float())
        for i, p in enumerate(pos.tolist())])
    R.check_bracket(rbf(o32), rbf(o - E), rbf(o + E), "fp32 softmax")
    # p rounded to one bf16 is far outside for most rows, a causal leak for every row with a next position
    hi_only = R.attn_ref64(q, K, V, pos, scale, p_hi_only=True)[0]
    out = ((rbf(o) < rbf(hi_only - E)) | (rbf(o) > rbf(hi_only + E))).flatten(1).any(1)
    assert int(out.sum()) >= len(pos) - 2
    leak = R.attn_ref64(q, K, V, pos + 1, scale)[0]
    assert ((rbf(o) < rbf(leak - E)) | (rbf(o) > rbf(leak + E))).flatten(1).any(1).all()
    # rotate_by one position: the table's row 1
    cs1 = O.precompute_freqs_cis(4, Dh, 1e6)[1].float()
    assert R.rotate_by(q, cs1).shape == q.shape


def test_paged_history():
    pages, Hkv, Dh = 6, 2, 8
    cache = torch.arange(pages * Hkv * 64 * Dh, dtype=torch.float32).view(pages, Hkv, 64, Dh)
    row = torch.tensor([4, -1, 2, 0], dtype=torch.int32)
    h = R.paged_history(cache, row, 150)
    assert h.shape == (Hkv, 150, Dh)
    assert torch.equal(h[:, :64], cache[4].double()) and (h[:, 64:128] == 0).all()
    assert torch.equal(h[:, 128:150], cache[2, :, :22].double())
