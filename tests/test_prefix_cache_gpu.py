"""Prefix cache of the KV page pool on the GPU (LmEngine(prefix_cache=True), setup_caches(prefix_cache=)).

A cached prefix is K/V a prefill wrote; prefill is row-independent and batch-invariant, so a request that maps it (and
copies its partly matched last page) must produce bitwise the tokens of a cold run on a fresh engine. These tests check
that for voices whose slots other voices took over, under evictions, with every serving option beside the cache, at
S2-Pro geometry, and on the one-request-at-a-time `generate` path."""
from __future__ import annotations

import pytest
import torch

from oracle import lm_oracle as O
from tests.lm_util import make_prompt

pytestmark = pytest.mark.gpu

GREEDY = dict(temperature=0.7, top_p=0.7, top_k=1)
SAMPLED = dict(temperature=0.8, top_p=0.9, top_k=30)


def _model(cfg, w, slots, prefix_cache, kv_pages=None, args=None, im_end=None, max_rows=2048):
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from tests.lm_util import model_args

    m = DualARTransformer(args or model_args(cfg), w, device="cuda", im_end_id=cfg.im_end_id if im_end is None else im_end)
    m.max_rows = max_rows
    m.setup_caches(max_batch_size=slots, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages, prefix_cache=prefix_cache)
    m._cache_setup_done = True
    return m


def _voices(cfg, lengths, seed=0):
    return [make_prompt(cfg, 7000 + seed + v, n) for v, n in enumerate(lengths)]


def _specs(voices, picks, cfg, tail=(20, 60), n=(12, 30), seed=0):
    """(prompt, budget, sampling seed) per request: voice `picks[i]` + a tail of its own."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for i, v in enumerate(picks):
        t = int(torch.randint(tail[0], tail[1] + 1, (1,), generator=g))
        budget = int(torch.randint(n[0], n[1] + 1, (1,), generator=g))
        out.append((torch.cat([voices[v], make_prompt(cfg, 90_000 + 31 * seed + i, t)], 1), budget, 1000 + i))
    return out


def _serve(model, phases, sp, paced=False, **kw):
    """Run each phase's requests through one ContinuousBatcher, a phase after the previous one has finished. Returns
    the results in order and the batcher."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    slots = model.engine.max_batch
    b = ContinuousBatcher(model, max_slots=slots, frames_per_poll=4, max_live=2 * slots if paced else None, **kw)
    out = []
    for phase in phases:
        reqs = [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=n, seed=s, reuse_prefix=True,
                                     pace=400.0 if paced else None, **sp)) for p, n, s in phase]
        b.run()
        for r in reqs:
            assert r.error is None, r.error
            out.append(r.result.cpu())
    if b.kv_growth:
        assert not b.eng.buffer("kv_miss").any()
    return out, b


def _cold(cfg, w, specs, sp, slots):
    """Every request alone on a fresh engine without the cache."""
    m = _model(cfg, w, slots, prefix_cache=False)
    out = [_serve(m, [[s]], sp)[0][0] for s in specs]
    m.engine.close()
    return out


@pytest.mark.parametrize("sp", [GREEDY, SAMPLED], ids=["greedy", "sampled"])
def test_a_voice_whose_slot_moved_on_is_served_from_the_cache(sp):
    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=21, head_gain=3.0)
    voices = _voices(cfg, [150, 233, 97])  # not multiples of 64: the partly matched page is copied on write
    a1, b1, c1, a2 = _specs(voices, [0, 1, 2, 0], cfg)
    cold = _cold(cfg, w, [a1, b1, c1, a2], sp, slots=2)
    m = _model(cfg, w, 2, prefix_cache=True)
    eng = m.engine
    got, b = _serve(m, [[a1], [b1, c1]], sp)
    assert eng.kv_pool.hits == 0 and len(eng.kv_pool.cached) >= 2  # both slots have served other voices since a1
    before = eng.rows_prefilled
    more, _ = _serve_more(b, [a2], sp)
    assert eng.kv_pool.hits == 1 and eng.rows_prefilled - before == a2[0].shape[1] - 150
    for i, (x, y) in enumerate(zip(got + more, cold)):
        assert torch.equal(x, y), f"request {i}: tokens differ from a cold run at {(x != y).nonzero()[:4].tolist()}"
    assert eng.pages_cached > 0 and eng.prefix_hits == 1
    b.close()
    eng.close()


def _serve_more(b, phase, sp):
    from fish_speech_b200.scheduler import SlotRequest

    reqs = [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=n, seed=s, reuse_prefix=True, **sp))
            for p, n, s in phase]
    b.run()
    assert all(r.error is None for r in reqs)
    return [r.result.cpu() for r in reqs], b


def test_a_small_pool_evicts_and_keeps_the_tokens():
    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=22, head_gain=3.0)
    voices = _voices(cfg, [150, 233, 97, 180, 301, 77], seed=1)
    picks = [0, 1, 2, 3, 0, 4, 5, 1, 0, 2, 3, 4, 0, 5, 1, 0]
    specs = _specs(voices, picks, cfg, seed=1)
    phases = [specs[i:i + 2] for i in range(0, len(specs), 2)]
    ref, _ = _serve(_model(cfg, w, 3, prefix_cache=False, kv_pages=24), phases, SAMPLED, kv_growth=True)
    m = _model(cfg, w, 3, prefix_cache=True, kv_pages=24)
    got, b = _serve(m, phases, SAMPLED, kv_growth=True)
    assert b.kv_growth and m.engine.prefix_evictions > 0 and m.engine.prefix_hits > 0
    for i, (x, y) in enumerate(zip(got, ref)):
        assert torch.equal(x, y), f"request {i}: tokens differ with the cache"
    assert m.engine.rows_prefilled < sum(p.shape[1] for p, _, _ in specs)


@pytest.mark.parametrize("opt", ["fused_admission", "kv_growth", "compact_rows", "paced"])
def test_each_serving_option_gives_the_same_tokens_with_the_cache(opt):
    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=23, head_gain=3.0)
    voices = _voices(cfg, [150, 233, 97, 180], seed=2)
    picks = [0, 1, 2, 3, 0, 1, 0, 2, 3, 1, 0, 0]
    specs = _specs(voices, picks, cfg, seed=2)
    phases = [specs[:5], specs[5:9], specs[9:]]
    kw = {} if opt == "paced" else {opt: True}
    slots = 36 if opt == "compact_rows" else 4
    pages = 40 if opt == "kv_growth" else None
    runs = []
    for cache in (False, True):
        m = _model(cfg, w, slots, prefix_cache=cache, kv_pages=pages)
        runs.append(_serve(m, phases, SAMPLED, paced=opt == "paced", **kw)[0])
        if cache:
            assert m.engine.prefix_hits > 0
        m.engine.close()
    for i, (x, y) in enumerate(zip(*runs)):
        assert torch.equal(x, y), f"{opt}: request {i} differs with the cache"


@pytest.mark.parametrize("slots", [32, 64])
def test_s2pro_geometry_with_a_700_row_cached_prefix(slots):
    """Full S2-Pro layer geometry (36 slow + 4 fast layers, synthetic weights, <|im_end|> zeroed so budgets set the
    lengths), greedy: a 700-row voice prefix cached, its slot taken over, then reused."""
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    dev = torch.device("cuda", 0)
    cfg = s2pro_args(max_seq_len=1024)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    g = torch.Generator().manual_seed(5)

    def rows(n):
        p = torch.zeros(cfg.num_codebooks + 1, n, dtype=torch.int32)
        p[0] = torch.randint(0, 151643, (n,), generator=g, dtype=torch.int32)
        return p

    voice, other = rows(700), rows(650)
    specs = [(torch.cat([voice, rows(40)], 1), 12, 1), (torch.cat([other, rows(50)], 1), 12, 2),
             (torch.cat([voice, rows(33)], 1), 12, 3)]
    runs, engines = [], []
    for cache in (False, True):
        m = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        m.max_rows = 1024
        m.setup_caches(max_batch_size=slots, max_seq_len=cfg.max_seq_len, kv_pages=2 * 17, prefix_cache=cache)
        # two slots' worth of pages: the second voice takes over the first one's pages unless they are cached
        out, b = _serve(m, [[specs[0]], [specs[1]], [specs[2]]], GREEDY)
        runs.append(out)
        engines.append((m.engine.rows_prefilled, m.engine.prefix_hits))
        b.close()
        m.engine.close()
    for i, (x, y) in enumerate(zip(*runs)):
        assert torch.equal(x, y), f"{slots} slots: request {i} differs with the cache"
    assert engines[1][1] == 1 and engines[0][0] - engines[1][0] == 700


def test_one_at_a_time_generate_alternating_voices():
    from fish_speech_b200.models.text2semantic.inference import generate

    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=24, head_gain=3.0)
    voices = _voices(cfg, [170, 140], seed=3)
    specs = _specs(voices, [0, 1, 0], cfg, seed=3)
    outs = []
    for cache in (False, True):
        m = _model(cfg, w, 1, prefix_cache=cache)
        eng = m.engine
        res, prefilled = [], []
        for p, n, s in specs:
            before = eng.rows_prefilled
            res.append(generate(model=m, prompt=p.cuda(), max_new_tokens=n, reuse_prefix=True, seed=s,
                                **SAMPLED).cpu())
            prefilled.append(eng.rows_prefilled - before)
        outs.append((res, prefilled))
        eng.close()
    (off, pre_off), (on, pre_on) = outs
    for i, (x, y) in enumerate(zip(off, on)):
        assert torch.equal(x, y), f"call {i} differs with the cache"
    T = [p.shape[1] for p, _, _ in specs]
    assert pre_off == T  # without the cache voice A is gone once B has used the slot
    assert pre_on == [T[0], T[1], T[2] - 170]  # the third call prefills only its tail
