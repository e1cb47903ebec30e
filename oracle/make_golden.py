"""Pin the oracle against the REAL reference and write the golden fixtures (test infrastructure).

Run where a checkout of the reference exists (its directory in $FISH_SPEECH_REFERENCE):

    python -m oracle.make_golden

For every case it (1) runs the unmodified reference (imported through oracle/ref_stubs.py), (2) runs the
oracle restatement on the same seeded weights / inputs, (3) asserts bit-equality, (4) stores inputs,
seeds and the reference's outputs under tests/golden/.  The committed fixtures let the CPU test-suite
and the GPU suite (no reference needed) re-check both the oracle and the CUDA path
against outputs of the reference itself.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import lm_oracle as O  # noqa: E402
from oracle import ref_stubs as R  # noqa: E402

GOLD = ROOT / "tests" / "golden"

# (name, config overrides, weight seed, head_gain, prompt len, new frames, top_k, temperature, top_p)
LM_CASES = [
    ("lm_tiny_greedy", {}, 11, 8.0, 12, 12, 1, 0.7, 0.7),
    ("lm_tiny_topk", {}, 12, 1.0, 9, 10, 30, 0.7, 0.8),
    ("lm_tiny_proj", dict(fast_dim=128, fast_n_head=2, fast_n_local_heads=1, fast_head_dim=64, fast_intermediate_size=256, attention_qk_norm=False,
                          fast_attention_qk_norm=True, norm_fastlayer_input=False,
                          scale_codebook_embeddings=False), 13, 8.0, 10, 8, 1, 0.7, 0.7),
    # stochastic decode that exercises the RAS substitution (inference.py:114-144): a peaky 96-token semantic head
    # repeats tokens inside the 10-frame window, so the high-temperature re-draw replaces the main token
    ("lm_tiny_ras", {}, 16, 2.0, 9, 24, 30, 0.7, 0.8),
    ("lm_tiny_bias", dict(attention_qkv_bias=True, attention_o_bias=True, fast_attention_qkv_bias=True,
                          fast_attention_o_bias=True, n_local_heads=2, fast_n_local_heads=4), 14, 8.0, 16, 8, 1, 0.7, 0.7),
]


def make_prompt(cfg: O.LMConfig, seed: int, T: int) -> torch.Tensor:
    """Text ids with a short span of semantic tokens + codes in the middle (a voice-clone-like prompt)."""
    g = torch.Generator().manual_seed(seed)
    prompt = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.long)
    prompt[0] = torch.randint(0, cfg.im_end_id, (T,), generator=g)
    a, b = T // 3, min(T - 1, T // 3 + 3)
    prompt[0, a:b] = cfg.semantic_begin_id + torch.randint(0, cfg.codebook_size, (b - a,), generator=g)
    prompt[1:, a:b] = torch.randint(0, cfg.codebook_size, (cfg.num_codebooks, b - a), generator=g)
    return prompt


def min_decision_gap(traces, cfg) -> float:
    """Smallest top-2 logit gap (in bf16 ulps of the winner) over every greedy decision of a run."""
    worst = float("inf")
    for tr in traces:
        sel = torch.cat([tr["slow_logits"][cfg.semantic_begin_id: cfg.semantic_end_id + 1],
                         tr["slow_logits"][cfg.im_end_id: cfg.im_end_id + 1]])
        for lg in [sel] + list(tr["fast_logits"]):
            top = torch.topk(lg.float(), 2).values
            worst = min(worst, float((top[0] - top[1]) / (top[0].abs() * 2 ** -7 + 1e-12)))
    return worst


def run_lm_case(name, over, seed, head_gain, T, n, top_k, temp, top_p):
    R.install()
    from fish_speech.models.text2semantic import inference as ref_inf

    cfg = O.tiny_config(**over)
    wseed, rng_seed = seed, seed
    while True:
        w = O.make_weights(cfg, seed=wseed, head_gain=head_gain)
        model = R.reference_lm(cfg, w)
        prompt = make_prompt(cfg, wseed, T)
        torch.manual_seed(rng_seed)
        ref = ref_inf.generate(model=model, prompt=prompt, max_new_tokens=n, audio_masks=None, audio_parts=None,
                               temperature=temp, top_p=top_p, top_k=top_k).to(torch.int32)
        st = O.setup(cfg, w)
        traces = []
        torch.manual_seed(rng_seed)
        got = O.generate(st, prompt, n, temperature=temp, top_p=top_p, top_k=top_k, traces=traces)
        assert torch.equal(ref, got), f"{name}: oracle differs from the reference"
        if top_k != 1:
            break
        # Greedy fixtures must be the deterministic argmax sequence with no bf16 near-ties, so that a
        # different (but correct) summation order cannot legitimately change a decision:
        #  * the reference's bf16 noise must never have hit U == 0 (see lm_oracle.NOISE) -> next RNG seed
        #  * every decision's top-2 gap must exceed 4 bf16 ulps                       -> next weight seed
        ctr = []
        clean = O.generate(O.setup(cfg, w), prompt, n, temperature=temp, top_p=top_p, top_k=top_k, noise=False,
                           traces=ctr)
        gap = min_decision_gap(ctr, cfg)
        if gap <= 4.0:
            print(f"{name}: weight seed {wseed} has a near-tie (min gap {gap:.2f} ulp), trying the next one")
            wseed += 100
            continue
        if not torch.equal(clean, ref):
            print(f"{name}: rng seed {rng_seed} hits the U==0 quirk, trying the next one")
            rng_seed += 1000
            continue
        break
    extra = {}
    if name == "lm_tiny_ras":
        extra = dict(ras_hits=sum(bool(t.get("ras_hit")) for t in traces),
                     ras_changed=sum(bool(t.get("ras_changed")) for t in traces))
        assert extra["ras_changed"] >= 5, "the RAS fixture must exercise the substitution"
    np.savez_compressed(
        GOLD / f"{name}.npz",
        config=np.array(repr(over)), weight_seed=wseed, head_gain=head_gain, prompt=prompt.numpy(),
        new_frames=n, top_k=top_k, temperature=temp, top_p=top_p, rng_seed=rng_seed,
        ref_tokens=ref.numpy(),
        ref_slow_logits=torch.stack([t["slow_logits"] for t in traces]).numpy().astype(np.float32),
        **extra,
    )
    print(f"{name}: reference == oracle, {ref.shape[1] - T} frames -> {GOLD / (name + '.npz')}")


def main():
    GOLD.mkdir(parents=True, exist_ok=True)
    for case in LM_CASES:
        run_lm_case(*case)
    try:
        from oracle import make_golden_codec

        make_golden_codec.main()
    except ImportError:
        print("codec goldens: oracle.make_golden_codec not present yet")


if __name__ == "__main__":
    main()
