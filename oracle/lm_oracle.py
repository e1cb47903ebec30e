"""ORACLE — TEST INFRASTRUCTURE ONLY (never imported by the product path).

CPU restatement (PyTorch CPU tensors, bf16 storage, the same operator sequence and therefore the same
rounding points) of the reference's Dual-AR text2semantic inference algorithm:

  fish_speech/models/text2semantic/llama.py      (model math)
  fish_speech/models/text2semantic/inference.py  (sampling, per-frame decode, generate loop)

Every function cites the reference lines it follows.  The oracle is *pinned*: oracle/make_golden.py
imports the real reference modules from a checkout of the reference (with the stubs in oracle/ref_stubs.py), runs
both on the same seeded weights and inputs, asserts bit-equality and writes tests/golden/*.npz; the
CPU test-suite re-checks the oracle against those fixtures without needing the reference.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

RAS_WIN_SIZE = 10  # inference.py:49-51
RAS_HIGH_TEMP = 1.0
RAS_HIGH_TOP_P = 0.9


@dataclass
class LMConfig:
    """DualARModelArgs after __post_init__ (llama.py:28-73, 156-193) + tokenizer ids."""

    dim: int = 2560
    n_layer: int = 36
    n_head: int = 32
    n_local_heads: int = 8
    head_dim: int = 128
    intermediate_size: int = 9728
    rope_base: float = 1e6
    norm_eps: float = 1e-6
    max_seq_len: int = 4096
    vocab_size: int = 155776
    tie_word_embeddings: bool = True
    attention_qk_norm: bool = True
    attention_qkv_bias: bool = False
    attention_o_bias: bool = False
    codebook_size: int = 4096
    num_codebooks: int = 10
    semantic_begin_id: int = 151678
    semantic_end_id: int = 155773
    im_end_id: int = 151645
    scale_codebook_embeddings: bool = True
    norm_fastlayer_input: bool = True
    n_fast_layer: int = 4
    fast_dim: int = 2560
    fast_n_head: int = 32
    fast_n_local_heads: int = 8
    fast_head_dim: int = 128
    fast_intermediate_size: int = 9728
    fast_attention_qk_norm: bool = False
    fast_attention_qkv_bias: bool = False
    fast_attention_o_bias: bool = False
    initializer_range: float = 0.02

    @property
    def has_fast_project_in(self) -> bool:  # llama.py:665-668
        return self.fast_dim != self.dim


def s2pro_config(**over) -> LMConfig:
    """Assumed S2-Pro geometry (SURVEY.md §8): Qwen3-4B slow stack + 4-layer fast stack."""
    return LMConfig(**over)


def tiny_config(**over) -> LMConfig:
    """Small geometry with the same structure (GQA 4:1, qk-norm, tied head) for fast CPU parity."""
    base = dict(
        dim=256, n_layer=2, n_head=4, n_local_heads=1, head_dim=64, intermediate_size=512,
        max_seq_len=128, vocab_size=1200, codebook_size=96, num_codebooks=4,
        semantic_begin_id=1000, semantic_end_id=1095, im_end_id=999,
        n_fast_layer=2, fast_dim=256, fast_n_head=4, fast_n_local_heads=1, fast_head_dim=64,
        fast_intermediate_size=512,
    )
    base.update(over)
    return LMConfig(**base)


# ------------------------------------------------------------------------------------------------
# weights: reference state_dict key names (llama.py:249-306, 660-706, 831-866, 979-996)
# ------------------------------------------------------------------------------------------------
def make_weights(cfg: LMConfig, seed: int = 1234, dtype=torch.bfloat16, head_gain: float = 1.0,
                 norm_jitter: float = 0.1) -> dict[str, torch.Tensor]:
    """Seeded synthetic weights. Linear / Embedding ~ N(0, initializer_range) as the reference's
    _init_weights (llama.py:468-477); norm weights 1 + jitter so the norm multiply is exercised;
    `head_gain` widens the logit gaps of the two output heads so greedy decisions are far from bf16
    ties (SURVEY.md §8c)."""
    g = torch.Generator().manual_seed(seed)
    std = cfg.initializer_range

    def lin(o, i, gain=1.0):
        return (torch.randn(o, i, generator=g) * std * gain).to(dtype)

    def nrm(n):
        return (1.0 + norm_jitter * torch.randn(n, generator=g)).to(dtype)

    w: dict[str, torch.Tensor] = {}
    w["embeddings.weight"] = lin(cfg.vocab_size, cfg.dim, head_gain)
    w["codebook_embeddings.weight"] = lin(cfg.codebook_size * cfg.num_codebooks, cfg.dim)

    def block(prefix, dim, nh, nkv, hd, inter, qk_norm, qkv_bias, o_bias):
        w[f"{prefix}.attention.wqkv.weight"] = lin((nh + 2 * nkv) * hd, dim)
        if qkv_bias:
            w[f"{prefix}.attention.wqkv.bias"] = (torch.randn((nh + 2 * nkv) * hd, generator=g) * std).to(dtype)
        w[f"{prefix}.attention.wo.weight"] = lin(dim, nh * hd)
        if o_bias:
            w[f"{prefix}.attention.wo.bias"] = (torch.randn(dim, generator=g) * std).to(dtype)
        if qk_norm:
            w[f"{prefix}.attention.q_norm.weight"] = nrm(hd)
            w[f"{prefix}.attention.k_norm.weight"] = nrm(hd)
        w[f"{prefix}.feed_forward.w1.weight"] = lin(inter, dim)
        w[f"{prefix}.feed_forward.w3.weight"] = lin(inter, dim)
        w[f"{prefix}.feed_forward.w2.weight"] = lin(dim, inter)
        w[f"{prefix}.ffn_norm.weight"] = nrm(dim)
        w[f"{prefix}.attention_norm.weight"] = nrm(dim)

    for l in range(cfg.n_layer):
        block(f"layers.{l}", cfg.dim, cfg.n_head, cfg.n_local_heads, cfg.head_dim, cfg.intermediate_size,
              cfg.attention_qk_norm, cfg.attention_qkv_bias, cfg.attention_o_bias)
    w["norm.weight"] = nrm(cfg.dim)
    if not cfg.tie_word_embeddings:
        w["output.weight"] = lin(cfg.vocab_size, cfg.dim, head_gain)
    if cfg.has_fast_project_in:
        w["fast_project_in.weight"] = lin(cfg.fast_dim, cfg.dim)
        w["fast_project_in.bias"] = (torch.randn(cfg.fast_dim, generator=g) * std).to(dtype)
    w["fast_embeddings.weight"] = lin(cfg.codebook_size, cfg.fast_dim)
    for l in range(cfg.n_fast_layer):
        block(f"fast_layers.{l}", cfg.fast_dim, cfg.fast_n_head, cfg.fast_n_local_heads, cfg.fast_head_dim,
              cfg.fast_intermediate_size, cfg.fast_attention_qk_norm, cfg.fast_attention_qkv_bias,
              cfg.fast_attention_o_bias)
    w["fast_norm.weight"] = nrm(cfg.fast_dim)
    w["fast_output.weight"] = lin(cfg.codebook_size, cfg.fast_dim, head_gain)
    return w


# ------------------------------------------------------------------------------------------------
# primitives
# ------------------------------------------------------------------------------------------------
def precompute_freqs_cis(seq_len: int, n_elem: int, base: float) -> torch.Tensor:
    """llama.py:1004-1023 — cos/sin table stored in bf16, shape [seq_len, n_elem/2, 2]."""
    inv = 1.0 / (base ** (torch.arange(0, n_elem, 2)[: n_elem // 2].float() / n_elem))
    ang = torch.outer(torch.arange(seq_len), inv)
    cis = torch.polar(torch.ones_like(ang), ang)
    return torch.stack([cis.real, cis.imag], dim=-1).to(torch.bfloat16)


def apply_rotary(x: torch.Tensor, freqs: torch.Tensor) -> torch.Tensor:
    """llama.py:1026-1038 — interleaved pairs, fp32 math, cast back. x [B,S,H,D], freqs [S,D/2,2]."""
    xs = x.float().reshape(*x.shape[:-1], -1, 2)
    fr = freqs.view(1, xs.size(1), 1, xs.size(3), 2)
    out = torch.stack(
        [xs[..., 0] * fr[..., 0] - xs[..., 1] * fr[..., 1],
         xs[..., 1] * fr[..., 0] + xs[..., 0] * fr[..., 1]], -1)
    return out.flatten(3).type_as(x)


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float) -> torch.Tensor:
    """llama.py:990-1001 — normalise in fp32, round to x.dtype, THEN multiply by the weight."""
    xf = x.float()
    y = (xf * torch.rsqrt(torch.mean(xf * xf, dim=-1, keepdim=True) + eps)).type_as(x)
    return y * weight


def _eq_sdpa(q, k, v, mask):
    """llama.py:948-976 — the fast stack's hand-rolled attention (all-bf16 matmul / softmax)."""
    scale = 1 / math.sqrt(q.size(-1))
    bias = torch.zeros(1, 1, q.size(-2), k.size(-2), dtype=q.dtype)
    bias = torch.where(mask.logical_not(), float("-inf"), bias)
    aw = q @ k.transpose(-2, -1) * scale
    aw += bias
    aw = torch.softmax(aw, dim=-1)
    return aw @ v


@dataclass
class KV:
    k: torch.Tensor  # [B, Hkv, S, D]
    v: torch.Tensor


@dataclass
class LMState:
    """Static caches (llama.py:196-214, 307-325, 708-721) and tables of one model instance."""

    cfg: LMConfig
    w: dict
    max_batch: int = 1
    kv: list = field(default_factory=list)
    fast_kv: list = field(default_factory=list)
    freqs: Optional[torch.Tensor] = None
    fast_freqs: Optional[torch.Tensor] = None
    causal: Optional[torch.Tensor] = None


def setup(cfg: LMConfig, w: dict, max_batch: int = 1) -> LMState:
    dt = w["embeddings.weight"].dtype
    assert cfg.max_seq_len % 8 == 0, "max_seq_len must be a multiple of 8 (find_multiple, llama.py:313)"
    S = cfg.max_seq_len
    st = LMState(cfg, w, max_batch)
    st.kv = [KV(torch.zeros(max_batch, cfg.n_local_heads, S, cfg.head_dim, dtype=dt),
                torch.zeros(max_batch, cfg.n_local_heads, S, cfg.head_dim, dtype=dt)) for _ in range(cfg.n_layer)]
    st.fast_kv = [KV(torch.zeros(max_batch, cfg.fast_n_local_heads, cfg.num_codebooks, cfg.fast_head_dim, dtype=dt),
                     torch.zeros(max_batch, cfg.fast_n_local_heads, cfg.num_codebooks, cfg.fast_head_dim, dtype=dt))
                  for _ in range(cfg.n_fast_layer)]
    st.freqs = precompute_freqs_cis(cfg.max_seq_len, cfg.head_dim, cfg.rope_base)
    st.fast_freqs = precompute_freqs_cis(cfg.num_codebooks, cfg.fast_head_dim, cfg.rope_base)
    st.causal = torch.tril(torch.ones(cfg.max_seq_len, cfg.max_seq_len, dtype=torch.bool))
    st.S = S
    return st


def _block(st: LMState, prefix: str, x, freqs, mask, input_pos, kv: KV, nh, nkv, hd, qk_norm, use_sdpa, eps):
    """TransformerBlock.forward + Attention.forward + FeedForward.forward (llama.py:838-845, 884-946, 986-987)."""
    w = st.w
    B, S, _ = x.shape
    h_in = rms_norm(x, w[f"{prefix}.attention_norm.weight"], eps)
    qkv = F.linear(h_in, w[f"{prefix}.attention.wqkv.weight"], w.get(f"{prefix}.attention.wqkv.bias"))
    q, k, v = qkv.split([nh * hd, nkv * hd, nkv * hd], dim=-1)
    q = q.view(B, S, nh, hd)
    k = k.view(B, S, nkv, hd)
    v = v.view(B, S, nkv, hd)
    if qk_norm:  # nn.RMSNorm(head_dim): single rounding
        q = F.rms_norm(q, (hd,), w[f"{prefix}.attention.q_norm.weight"], eps)
        k = F.rms_norm(k, (hd,), w[f"{prefix}.attention.k_norm.weight"], eps)
    q = apply_rotary(q, freqs)
    k = apply_rotary(k, freqs)
    q, k, v = (t.transpose(1, 2) for t in (q, k, v))
    kv.k[:B, :, input_pos] = k
    kv.v[:B, :, input_pos] = v
    kk = kv.k[:B].repeat_interleave(nh // nkv, dim=1)
    vv = kv.v[:B].repeat_interleave(nh // nkv, dim=1)
    if use_sdpa:
        y = F.scaled_dot_product_attention(q, kk, vv, attn_mask=mask)
    else:
        y = _eq_sdpa(q, kk, vv, mask)
    y = y.transpose(1, 2).contiguous().view(B, S, nh * hd)
    h = x + F.linear(y, w[f"{prefix}.attention.wo.weight"], w.get(f"{prefix}.attention.wo.bias"))
    n2 = rms_norm(h, w[f"{prefix}.ffn_norm.weight"], eps)
    ff = F.linear(F.silu(F.linear(n2, w[f"{prefix}.feed_forward.w1.weight"])) *
                  F.linear(n2, w[f"{prefix}.feed_forward.w3.weight"]), w[f"{prefix}.feed_forward.w2.weight"])
    return h + ff


def embed(st: LMState, inp: torch.Tensor) -> torch.Tensor:
    """llama.py:399-420. inp [B, C+1, S] integer."""
    cfg, w = st.cfg, st.w
    embs = [F.embedding(inp[:, i + 1] + i * cfg.codebook_size, w["codebook_embeddings.weight"])
            for i in range(cfg.num_codebooks)]
    vq = torch.stack(embs, dim=1).sum(dim=1)
    sem = (inp[:, 0] >= cfg.semantic_begin_id) & (inp[:, 0] <= cfg.semantic_end_id)
    vq[~sem] = 0
    x = F.embedding(inp[:, 0], w["embeddings.weight"]) + vq
    if cfg.scale_codebook_embeddings:
        x = torch.where(sem.unsqueeze(-1).expand_as(x), x / math.sqrt(cfg.num_codebooks + 1), x)
    return x


def forward_generate(st: LMState, inp: torch.Tensor, input_pos: torch.Tensor, per_layer=None):
    """BaseTransformer.forward_generate + DualARTransformer.forward_generate (llama.py:390-466, 819-828).
    Returns (token_logits [B,1,V], hidden [B,1,fast_dim])."""
    cfg, w = st.cfg, st.w
    x = embed(st, inp)
    mask = st.causal[None, None, input_pos, : st.S]
    freqs = st.freqs[input_pos]
    if per_layer is not None:
        per_layer.append(x.clone())
    for l in range(cfg.n_layer):
        x = _block(st, f"layers.{l}", x, freqs, mask, input_pos, st.kv[l], cfg.n_head, cfg.n_local_heads,
                   cfg.head_dim, cfg.attention_qk_norm, True, cfg.norm_eps)
        if per_layer is not None:
            per_layer.append(x.clone())
    if x.size(1) > 1:
        x = x[:, -1:]
    slow_out = rms_norm(x, w["norm.weight"], cfg.norm_eps)
    head = w["embeddings.weight"] if cfg.tie_word_embeddings else w["output.weight"]
    logits = F.linear(slow_out, head)
    hidden = slow_out if cfg.norm_fastlayer_input else x
    if cfg.has_fast_project_in:
        hidden = F.linear(hidden, w["fast_project_in.weight"], w["fast_project_in.bias"])
    return logits, hidden


def forward_generate_fast(st: LMState, x: torch.Tensor, input_pos: torch.Tensor) -> torch.Tensor:
    """llama.py:799-817. x [B, fast_dim]-like; returns codebook logits [B,1,codebook_size]."""
    cfg, w = st.cfg, st.w
    x = x.view(x.shape[0], 1, -1)
    mask = st.causal[None, None, input_pos, : cfg.num_codebooks]
    freqs = st.fast_freqs[input_pos]
    for l in range(cfg.n_fast_layer):
        x = _block(st, f"fast_layers.{l}", x, freqs, mask, input_pos, st.fast_kv[l], cfg.fast_n_head,
                   cfg.fast_n_local_heads, cfg.fast_head_dim, cfg.fast_attention_qk_norm, False, cfg.norm_eps)
    return F.linear(rms_norm(x, w["fast_norm.weight"], cfg.norm_eps), w["fast_output.weight"])


# ------------------------------------------------------------------------------------------------
# sampling (inference.py:43-93)
# ------------------------------------------------------------------------------------------------
def logits_to_probs(logits, temperature, top_p, top_k: int, rec_cum: Optional[list] = None):
    sorted_logits, sorted_idx = torch.sort(logits, descending=True)
    cum = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
    if rec_cum is not None:
        rec_cum.append(cum[: max(2, top_k)].float().clone())
        rec_cum.append(sorted_logits[: top_k + 1].float().clone())
    ranks = torch.arange(sorted_logits.shape[-1])
    remove = (cum > top_p) | (ranks >= top_k)
    remove[0] = False
    remove = remove.scatter(dim=-1, index=sorted_idx, src=remove)
    logits = torch.where(remove, float("-Inf"), logits)
    logits = logits / torch.clip(temperature, min=1e-5)
    return F.softmax(logits, dim=-1)


NOISE = True
"""multinomial_sample_one_no_sync (inference.py:43-46) divides the probabilities by -log(U) with U drawn
in the probs dtype.  In bf16 U takes only 256 values and is EXACTLY 0 with probability 1/256; then
-log(U) = inf, every score becomes 0 and argmax returns index 0 — even with top_k=1, where the result
should not depend on the noise at all.  This is a quirk of the reference (verified against it: the
pinned runs reproduce it bit for bit).  NOISE=False drops the division so that the top_k=1 path is the
deterministic argmax the reference intends; CUDA parity is defined against that."""


def sample(logits, temperature, top_p, top_k: int, generator=None, rec: Optional[list] = None):
    """`rec` (tests): receives the score vector probs / q the reference takes the argmax of."""
    cums = [] if rec is not None else None
    probs = logits_to_probs(logits[0, -1], temperature, top_p, top_k, cums)
    if not NOISE:
        return torch.argmax(probs, dim=-1, keepdim=True).to(torch.int), probs
    q = -torch.log(torch.rand(probs.shape, dtype=probs.dtype, generator=generator))
    if rec is not None:
        # (scores the argmax is taken of, sorted cumulative probabilities the top-p cut compares with top_p, top_p,
        #  the top_k + 1 largest logits: the top-k cut falls between the last two)
        rec.append(((probs / q).float().clone(), cums[0], float(top_p), cums[1]))
    return torch.argmax(probs / q, dim=-1, keepdim=True).to(torch.int), probs


def semantic_logit_bias(cfg: LMConfig, dtype) -> torch.Tensor:
    """inference.py:306-320."""
    b = torch.full((1, 1, cfg.vocab_size), float("-inf"), dtype=dtype)
    b[0, 0, cfg.semantic_begin_id: cfg.semantic_end_id + 1] = 0.0
    b[0, 0, cfg.im_end_id] = 0.0
    return b


def decode_one_token_ar(st: LMState, x, input_pos, temperature, top_p, top_k: int, bias,
                        previous_tokens=None, generator=None, trace: Optional[dict] = None):
    """inference.py:96-181 — one frame for ONE sequence (batch row 0), returns [C+1, 1] int."""
    cfg = st.cfg
    logits, hidden = forward_generate(st, x, input_pos)
    biased = logits + bias
    rec = trace.setdefault("scores", []) if trace is not None else None  # [main, RAS re-draw, codebook 1, 2, ...]
    main = sample(biased, temperature, top_p, top_k, generator, rec)[0]
    ht = torch.tensor(RAS_HIGH_TEMP, dtype=temperature.dtype)
    hp = torch.tensor(RAS_HIGH_TOP_P, dtype=top_p.dtype)
    main_high = sample(biased, ht, hp, top_k, generator, rec)[0]
    if previous_tokens is not None:
        in_window = (previous_tokens[0] == main).any()
        is_sem = (main >= cfg.semantic_begin_id) & (main <= cfg.semantic_end_id)
        if trace is not None:
            trace["ras_hit"] = bool(in_window & is_sem)
            trace["ras_changed"] = bool(in_window & is_sem) and int(main_high) != int(main)
        main = torch.where(in_window & is_sem, main_high, main)
    if trace is not None:
        trace["slow_logits"] = biased[0, -1].float().clone()
        trace["hidden"] = hidden[0, -1].float().clone()
        trace["fast_logits"] = []
    codebooks = [main]
    forward_generate_fast(st, hidden, torch.tensor([0], dtype=torch.long))
    a = torch.clamp(main - cfg.semantic_begin_id, min=0, max=cfg.codebook_size - 1)
    hs = F.embedding(a, st.w["fast_embeddings.weight"])
    codebooks.append(a)
    for cb in range(1, cfg.num_codebooks):
        fl = forward_generate_fast(st, hs, torch.tensor([cb], dtype=torch.long))
        if trace is not None:
            trace["fast_logits"].append(fl[0, -1].float().clone())
        a = sample(fl, temperature, top_p, top_k, generator, rec)[0]
        hs = F.embedding(a, st.w["fast_embeddings.weight"])
        codebooks.append(a)
    return torch.stack(codebooks, dim=1).T


def generate(st: LMState, prompt: torch.Tensor, max_new_tokens: int, temperature=1.0, top_p=0.9, top_k=30,
             generator=None, traces: Optional[list] = None, stop_on_im_end: bool = True,
             noise: bool = True) -> torch.Tensor:
    """inference.py:243-359 + decode_n_tokens :184-238. prompt [C+1, T] -> [C+1, T+n].
    noise=False: deterministic top_k=1 (see NOISE)."""
    global NOISE
    saved, NOISE = NOISE, noise
    try:
        return _generate(st, prompt, max_new_tokens, temperature, top_p, top_k, generator, traces, stop_on_im_end)
    finally:
        NOISE = saved


def _generate(st, prompt, max_new_tokens, temperature, top_p, top_k, generator, traces, stop_on_im_end):
    cfg = st.cfg
    dt = st.w["embeddings.weight"].dtype
    T = prompt.size(1)
    if T >= cfg.max_seq_len:
        raise ValueError(f"Input sequence length {T} exceeds max_seq_len {cfg.max_seq_len}")
    if max_new_tokens:
        if T + max_new_tokens > cfg.max_seq_len:
            max_new_tokens = cfg.max_seq_len - T
    else:
        max_new_tokens = cfg.max_seq_len - T
    temperature = torch.tensor(temperature, dtype=dt)
    top_p = torch.tensor(top_p, dtype=dt)
    bias = semantic_logit_bias(cfg, dt)
    C1 = cfg.num_codebooks + 1
    tr = {} if traces is not None else None
    first = decode_one_token_ar(st, prompt.view(1, C1, -1), torch.arange(0, T), temperature, top_p, top_k, bias,
                                None, generator, tr)
    if traces is not None:
        traces.append(tr)
    out = [first]
    cur = first.view(1, C1, -1)
    input_pos = torch.tensor([T], dtype=torch.long)
    prev = torch.zeros((C1, RAS_WIN_SIZE), dtype=torch.int)
    for _ in range(max_new_tokens - 1):
        tr = {} if traces is not None else None
        with sdpa_kernel(SDPBackend.MATH):
            nxt = decode_one_token_ar(st, cur, input_pos, temperature, top_p, top_k, bias, prev, generator, tr).clone()
        if traces is not None:
            traces.append(tr)
        input_pos = input_pos + 1
        cur = nxt.view(1, C1, -1)
        prev = prev.roll(-1, dims=1)
        prev[:, -1] = nxt.view(C1, -1)[:, 0]
        out.append(nxt)
        if stop_on_im_end and cur[0, 0, -1] == cfg.im_end_id:
            break
    return torch.cat([prompt.to(torch.int)] + out, dim=1)
