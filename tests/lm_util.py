"""Shared helpers for the LM tests: oracle config -> product model, the kernel tests' configurations and sweep tables,
and the plumbing of their GPU modules."""
from __future__ import annotations

import ast

import numpy as np
import pytest
import torch

from oracle import lm_oracle as O


def _lib():
    from fish_speech_b200 import _lib

    return _lib


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, seed, scale=1.0) -> torch.Tensor:
    return (torch.randn(shape, generator=_gen(seed), device="cuda") * scale).bfloat16()


def _sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------------------------
# the decode step GEMM's sweep (test_step_gemm_gpu, test_decode64_gpu)
# ---------------------------------------------------------------------------------------------------------------------
STAGES = (2, 3, 4, 8)  # 8 does not fit two CTAs per SM: step_plan_init shrinks it

SHAPES = [
    pytest.param(6144, 2560, id="s2pro-qkv"),
    pytest.param(2560, 4096, id="s2pro-wo"),
    pytest.param(19456, 2560, id="s2pro-w13"),
    pytest.param(2560, 9728, id="s2pro-w2"),
    pytest.param(4097, 2560, id="s2pro-head"),
    pytest.param(4096, 2560, id="s2pro-fast-out"),
    pytest.param(384, 256, id="tiny-qkv"),
    pytest.param(96, 256, id="tiny-fast-out"),
    pytest.param(97, 256, id="tiny-head"),
    pytest.param(1, 1000, id="one-row-K1000"),  # partial last k-block (40 of 64) and a one-feature tile
    pytest.param(200, 528, id="K528"),  # w2 with an intermediate size that is not a multiple of 64
]


def _ctas():
    return (1, 2, 3, 7, 132, 2 * _sms(), 10 ** 6)  # 10^6: clamped to what one wave holds


def layer_configs():
    """name -> config of the decode layer GEMM tests."""
    return {
        # wo bias in both stacks; intermediate sizes that are not multiples of 64 (w1|w3 padded, w2 with K % 64 != 0)
        "tiny": O.tiny_config(attention_o_bias=True, fast_attention_o_bias=True, intermediate_size=528,
                              fast_intermediate_size=400),
        # S2-Pro layer shapes with two layers per stack and a reduced vocabulary (test_lm_gpu.py builds it so too)
        "s2pro": O.LMConfig(n_layer=2, n_fast_layer=2, vocab_size=8192, max_seq_len=256, semantic_begin_id=4000,
                            semantic_end_id=8095, im_end_id=3999),
    }


def attn_configs():
    """name -> (config, slots): every (head_dim, group) instance of the attention kernels in one stack or the other.
    (Dh, G) per stack in the comments; both row tiles; qk-norm and qkv bias on and off."""
    s2 = dict(vocab_size=8192, semantic_begin_id=4000, semantic_end_id=8095, im_end_id=3999, max_seq_len=32768)
    return {
        # slow (64, 8) norm; fast (128, 2) norm + bias
        "tiny-a": (O.tiny_config(max_seq_len=1024, n_head=8, n_local_heads=1, head_dim=64, fast_n_head=2,
                                 fast_n_local_heads=1, fast_head_dim=128, fast_attention_qk_norm=True,
                                 fast_attention_qkv_bias=True), 32),
        # slow (128, 1) bias; fast (64, 2) plain, behind fast_project_in (fast_dim != dim)
        "tiny-b": (O.tiny_config(max_seq_len=1024, n_head=2, n_local_heads=2, head_dim=128, attention_qk_norm=False,
                                 attention_qkv_bias=True, fast_dim=128, fast_n_head=4, fast_n_local_heads=2,
                                 fast_head_dim=64), 64),
        # slow (64, 1) norm + bias; fast (128, 8) norm
        "tiny-c": (O.tiny_config(max_seq_len=1024, n_head=2, n_local_heads=2, head_dim=64, attention_qkv_bias=True,
                                 fast_n_head=8, fast_n_local_heads=1, fast_head_dim=128, fast_attention_qk_norm=True),
                   32),
        # slow (128, 2) plain; fast (64, 4) bias
        "tiny-d": (O.tiny_config(max_seq_len=1024, n_head=4, n_local_heads=2, head_dim=128, attention_qk_norm=False,
                                 fast_attention_qkv_bias=True), 64),
        # S2-Pro layers: slow (128, 4) norm, fast (128, 4) plain; 32 768 positions per slot
        "s2pro": (O.LMConfig(n_layer=2, n_fast_layer=2, **s2), 64),
        # slow (128, 8) norm: the smallest score buffer per position
        "s2pro-g8": (O.LMConfig(n_layer=2, n_fast_layer=1, n_local_heads=4, **s2), 32),
    }


def model_args(cfg: O.LMConfig):
    from fish_speech_b200.models.text2semantic.llama import DualARModelArgs

    return DualARModelArgs(
        model_type="dual_ar", vocab_size=cfg.vocab_size, n_layer=cfg.n_layer, n_head=cfg.n_head, dim=cfg.dim,
        intermediate_size=cfg.intermediate_size, n_local_heads=cfg.n_local_heads, head_dim=cfg.head_dim,
        rope_base=cfg.rope_base, norm_eps=cfg.norm_eps, max_seq_len=cfg.max_seq_len,
        tie_word_embeddings=cfg.tie_word_embeddings, attention_qkv_bias=cfg.attention_qkv_bias,
        attention_o_bias=cfg.attention_o_bias, attention_qk_norm=cfg.attention_qk_norm,
        codebook_size=cfg.codebook_size, num_codebooks=cfg.num_codebooks,
        semantic_begin_id=cfg.semantic_begin_id, semantic_end_id=cfg.semantic_end_id,
        scale_codebook_embeddings=cfg.scale_codebook_embeddings, n_fast_layer=cfg.n_fast_layer,
        fast_dim=cfg.fast_dim, fast_n_head=cfg.fast_n_head, fast_n_local_heads=cfg.fast_n_local_heads,
        fast_head_dim=cfg.fast_head_dim, fast_intermediate_size=cfg.fast_intermediate_size,
        fast_attention_qkv_bias=cfg.fast_attention_qkv_bias, fast_attention_qk_norm=cfg.fast_attention_qk_norm,
        fast_attention_o_bias=cfg.fast_attention_o_bias, norm_fastlayer_input=cfg.norm_fastlayer_input,
    )


def split_w13(weights: dict) -> dict:
    """The product loads checkpoints in the reference's key naming (w1/w3 separate) — already the case."""
    return weights


def build_model(cfg: O.LMConfig, weights: dict, max_batch=1, debug=True, max_rows=2048):
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    m = DualARTransformer(model_args(cfg), weights, device="cuda", im_end_id=cfg.im_end_id)
    m.debug = debug
    m.max_rows = max_rows
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len)
    m._cache_setup_done = True
    return m


def make_prompt(cfg: O.LMConfig, seed: int, T: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    prompt = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.long)
    prompt[0] = torch.randint(0, cfg.im_end_id, (T,), generator=g)
    a, b = T // 3, min(T - 1, T // 3 + 3)
    prompt[0, a:b] = cfg.semantic_begin_id + torch.randint(0, cfg.codebook_size, (b - a,), generator=g)
    prompt[1:, a:b] = torch.randint(0, cfg.codebook_size, (cfg.num_codebooks, b - a), generator=g)
    return prompt


def load_golden(path):
    z = np.load(path, allow_pickle=False)
    over = ast.literal_eval(str(z["config"]))
    cfg = O.tiny_config(**over)
    w = O.make_weights(cfg, seed=int(z["weight_seed"]), head_gain=float(z["head_gain"]))
    return cfg, w, z


def restricted(cfg: O.LMConfig, full_logits: torch.Tensor) -> torch.Tensor:
    """Selectable rows of a full-vocabulary logit vector: semantic ids, then <|im_end|>."""
    return torch.cat([full_logits[..., cfg.semantic_begin_id: cfg.semantic_end_id + 1],
                      full_logits[..., cfg.im_end_id: cfg.im_end_id + 1]], dim=-1)


def assert_tokens_match(got: torch.Tensor, ref: torch.Tensor, traces: list, cfg: O.LMConfig, T: int, what: str = "",
                        tie_ulps: float = 2.0):
    """Free-running greedy parity. Token ids / codes must be identical; the only tolerated divergence
    is a decision the oracle itself took on a bf16 near-tie (top-2 logit gap within 2 bf16 ulps), after
    which the two runs legitimately follow different histories. Returns the number of frames compared."""
    got, ref = got.to(torch.int32).cpu(), ref.to(torch.int32).cpu()
    n = min(got.shape[1], ref.shape[1])
    for f in range(T, n):
        if torch.equal(got[:, f], ref[:, f]):
            continue
        r = int((got[:, f] != ref[:, f]).nonzero()[0])
        tr = traces[f - T]
        logits = restricted(cfg, tr["slow_logits"]) if r <= 1 else tr["fast_logits"][r - 2]
        top2 = torch.topk(logits.float(), 2).values
        gap = float(top2[0] - top2[1])
        ulp = float(top2[0].abs()) * 2 ** -7
        assert gap <= tie_ulps * ulp, (f"{what}: frame {f - T} row {r}: got {got[:, f].tolist()} want {ref[:, f].tolist()} "
                                       f"(oracle top-2 gap {gap:.4g}, {tie_ulps} ulp = {tie_ulps * ulp:.4g})")
        return f - T
    assert got.shape == ref.shape, f"{what}: length {got.shape} vs {ref.shape}"
    return n - T


def teacher_forced_check(model, cfg: O.LMConfig, w: dict, prompt: torch.Tensor, n: int, what: str = ""):
    """Frame-by-frame parity with the ORACLE's history fed back (so one near-tie cannot hide the rest of
    the run). For every frame the CUDA engine decodes one frame from the oracle's previous frame; its
    token id / codes are compared row by row. A mismatch is tolerated only where the oracle's own
    decision was a bf16 near-tie (top-2 gap <= 2 ulp); the rest of that frame (which then sees a
    different code history) is skipped. Returns (frames_fully_equal, near_ties, decisions_verified)."""
    from fish_speech_b200.models.text2semantic.inference import decode_one_token_ar

    T = prompt.shape[1]
    traces = []
    ref = O.generate(O.setup(cfg, w), prompt, n, temperature=0.7, top_p=0.7, top_k=1, traces=traces,
                     stop_on_im_end=False, noise=False)
    temp, top_p = torch.tensor(0.7), torch.tensor(0.7)
    C1 = cfg.num_codebooks + 1
    prev = torch.zeros((C1, 10), dtype=torch.int32)
    equal, ties, decisions = 0, 0, 0
    for f in range(n):
        if f == 0:
            x, pos, pt = prompt.view(1, C1, -1).cuda(), torch.arange(T).cuda(), None
        else:
            x = ref[:, T + f - 1].view(1, C1, 1).cuda()
            pos, pt = torch.tensor([T + f - 1]).cuda(), prev.cuda()
        tok = decode_one_token_ar(model, x, pos, temp, top_p, 1, None, None, None, previous_tokens=pt).cpu().view(-1)
        want = ref[:, T + f].to(torch.int32)
        if torch.equal(tok.to(torch.int32), want):
            equal += 1
            decisions += cfg.num_codebooks  # slow token + C-1 sampled codes (row 1 is derived from row 0)
        else:
            r = int((tok.to(torch.int32) != want).nonzero()[0])
            decisions += max(0, r - 1) if r >= 2 else 0
            tr = traces[f]
            logits = restricted(cfg, tr["slow_logits"]) if r <= 1 else tr["fast_logits"][r - 2]
            top2 = torch.topk(logits.float(), 2).values
            gap, ulp = float(top2[0] - top2[1]), float(top2[0].abs()) * 2 ** -7
            assert gap <= 2 * ulp, (f"{what}: frame {f} row {r}: got {tok.tolist()} want {want.tolist()} "
                                   f"(oracle top-2 gap {gap:.4g} > 2 ulp = {2 * ulp:.4g})")
            ties += 1
        if f > 0:
            prev = prev.roll(-1, dims=1)
            prev[:, -1] = want
    return equal, ties, decisions
