"""Paged slow KV cache (include/fishb200.h fsb_lm_config.kv_pages, engine.KvPagePool): a sequence's K/V lives in
64-position pages of a shared pool, found through a page table the kernels read at run time.

The page walk visits the same positions in the same order as the contiguous layout did, so every result here must be
bit-identical to an engine whose pool holds every slot at full capacity -- however the pages are scattered, shared,
copied on write or reclaimed."""
from __future__ import annotations

import random

import pytest
import torch

from oracle import lm_oracle as O
from tests.lm_util import build_model, make_prompt

pytestmark = pytest.mark.gpu


def _paged_model(cfg, w, kv_pages, max_batch=1, max_rows=2048, scramble=None):
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from tests.lm_util import model_args

    m = DualARTransformer(model_args(cfg), w, device="cuda", im_end_id=cfg.im_end_id)
    m.max_rows = max_rows
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages)
    m._cache_setup_done = True
    if scramble is not None:  # pages handed out in a fixed random order: a sequence's pages are neither ordered nor adjacent
        random.Random(scramble).shuffle(m.engine.kv_pool.free)
    return m


def _gen(model, prompt, n, **kw):
    from fish_speech_b200.models.text2semantic.inference import generate

    return generate(model=model, prompt=prompt.cuda(), max_new_tokens=n, **kw).cpu()


def _table_is_scrambled(eng, slot, n):
    pages = eng.kv_pool.table[slot, :n].tolist()
    return all(p >= 0 for p in pages) and pages != sorted(pages)


SAMPLED = dict(temperature=0.8, top_p=0.9, top_k=30, seed=4242)
GREEDY = dict(temperature=0.7, top_p=0.7, top_k=1)


@pytest.mark.parametrize("kw", [GREEDY, SAMPLED], ids=["greedy", "sampled"])
def test_scrambled_pages_equal_the_default_pool_tiny(kw):
    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=11, head_gain=4.0)
    ref = build_model(cfg, w, debug=False, max_rows=100)
    paged = _paged_model(cfg, w, kv_pages=24, max_rows=100, scramble=5)  # 100-row prefill pieces: splits mid-page
    scrambled = []
    for seed, T, n in ((1, 150, 40), (2, 333, 30), (3, 70, 90)):
        prompt = make_prompt(cfg, seed, T)
        a = _gen(ref, prompt, n, **kw)
        b = _gen(paged, prompt, n, **kw)
        assert torch.equal(a, b), f"T={T}: paged != contiguous-capacity pool at {(a != b).nonzero()[:4].tolist()}"
        scrambled.append(_table_is_scrambled(paged.engine, 0, -(-T // 64)))
    assert any(scrambled)


def test_scrambled_pages_with_chunked_attention():
    """attend() walks a long context in score chunks; with a 32-position chunk every chunk boundary and page
    boundary is crossed in both the prefill (per-row path) and the decode attention."""
    from fish_speech_b200 import _lib

    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=12, head_gain=4.0)
    prompt = make_prompt(cfg, 9, 260)
    L = _lib.lib()
    try:
        L.fsb_op_attn_score_chunk(32)
        L.fsb_op_attn_per_row(1)
        ref = _gen(build_model(cfg, w, debug=False, max_rows=100), prompt, 24, **SAMPLED)
        got = _gen(_paged_model(cfg, w, kv_pages=16, max_rows=100, scramble=6), prompt, 24, **SAMPLED)
    finally:
        L.fsb_op_attn_score_chunk(0)
        L.fsb_op_attn_per_row(0)
    assert torch.equal(ref, got)


def _s2pro_small(max_seq_len, n_layer=2, n_fast_layer=2):
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args

    cfg = s2pro_args(max_seq_len=max_seq_len, n_layer=n_layer, n_fast_layer=n_fast_layer)
    w = synthetic.lm_state_dict(cfg, torch.device("cuda", 0))
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    return cfg, w


def _s2pro_model(cfg, w, max_batch, kv_pages=None, max_rows=2048):
    from fish_speech_b200.configs import S2PRO_IM_END_ID
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    m = DualARTransformer(cfg, w, device="cuda", im_end_id=S2PRO_IM_END_ID)
    m.max_rows = max_rows
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages)
    m._cache_setup_done = True
    return m


def _s2pro_prompt(cfg, seed, T):
    g = torch.Generator().manual_seed(seed)
    p = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.int32)
    p[0] = torch.randint(0, 151643, (T,), generator=g, dtype=torch.int32)
    return p


def test_scrambled_pages_equal_the_default_pool_s2pro_layers():
    cfg, w = _s2pro_small(2048)
    ref = _s2pro_model(cfg, w, 1, max_rows=200)
    paged = _s2pro_model(cfg, w, 1, kv_pages=12, max_rows=200)
    random.Random(7).shuffle(paged.engine.kv_pool.free)
    prompt = _s2pro_prompt(cfg, 3, 450)
    for kw in (GREEDY, SAMPLED):
        a, b = _gen(ref, prompt, 12, **kw), _gen(paged, prompt, 12, **kw)
        assert torch.equal(a, b), kw
    assert _table_is_scrambled(paged.engine, 0, 8)


def test_pool_smaller_than_the_work():
    """Three times more requests than the pool holds at once: admissions wait for pages (FIFO), every result equals
    the request alone, and the pages in use never exceed the pool."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=21, head_gain=2.5)
    pages = 12
    model = _paged_model(cfg, w, kv_pages=pages, max_batch=8, max_rows=512, scramble=8)
    specs = [dict(prompt=make_prompt(cfg, 900 + i, 60 + (37 * i) % 130), max_new_tokens=20 + (11 * i) % 40,
                  temperature=0.8, top_p=0.9, top_k=30, seed=100 + i) for i in range(16)]
    need = sum(-(-(s["prompt"].shape[1] + s["max_new_tokens"]) // 64) for s in specs)
    assert need >= 3 * pages
    b = ContinuousBatcher(model, max_slots=8, frames_per_poll=4)
    reqs = [b.submit(SlotRequest(**{**s, "prompt": s["prompt"].cuda()})) for s in specs]
    in_use = []
    while not b.idle():
        b.step()
        in_use.append(model.engine.kv_pool.in_use())
    b.close()
    pool = model.engine.kv_pool
    assert max(in_use) <= pages and pool.peak <= pages
    with pytest.raises(ValueError, match="kv_pages"):
        b.submit(SlotRequest(prompt=make_prompt(cfg, 1, 700).cuda(), max_new_tokens=100))
    solo = build_model(cfg, w, debug=False)
    for i, (s, r) in enumerate(zip(specs, reqs)):
        one = _gen(solo, s["prompt"], s["max_new_tokens"], temperature=0.8, top_p=0.9, top_k=30, seed=s["seed"])
        assert torch.equal(r.result.cpu(), one), f"request {i} != its solo run"


def test_shared_prefix_pages_and_copy_on_write():
    """16 requests share a 200-row prefix: its 3 whole pages are mapped once (refcount 16), the partial 4th is copied.
    The donor's slot is then re-prefilled from position 0 with an unrelated prompt while the 15 sharers still decode:
    copy-on-write keeps their pages, and every request equals a fresh prefill of its own prompt."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=31, head_gain=2.5)
    prefix = make_prompt(cfg, 5, 200)
    tail = lambda i: make_prompt(cfg, 600 + i, 24)
    prompts = [torch.cat([prefix, tail(i)], dim=1) for i in range(16)]
    model = _paged_model(cfg, w, kv_pages=None, max_batch=16, max_rows=4096, scramble=9)
    eng = model.engine
    b = ContinuousBatcher(model, max_slots=16, frames_per_poll=4)
    kw = dict(temperature=0.8, top_p=0.9, top_k=30)
    r0 = b.submit(SlotRequest(prompt=prompts[0].cuda(), max_new_tokens=9, reuse_prefix=True, seed=0, **kw))
    b.step()
    sharers = [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=48, reuse_prefix=True, seed=i, **kw))
               for i, p in enumerate(prompts[1:], 1)]
    b._admit()
    pool = eng.kv_pool
    assert not r0.done.is_set() and sorted(r.slot for r in sharers) == list(range(1, 16))
    shared = pool.table[r0.slot, :3]
    assert pool.ref[shared].tolist() == [16, 16, 16]
    assert all(pool.table[r.slot, :3].tolist() == shared.tolist() for r in sharers)
    assert all(pool.table[r.slot, 3] != pool.table[r0.slot, 3] for r in sharers)  # the partial page was copied
    rebel_prompt = make_prompt(cfg, 77, 150)
    rebel = b.submit(SlotRequest(prompt=rebel_prompt.cuda(), max_new_tokens=20, seed=99, **kw))
    b.run()
    b.close()
    assert rebel.slot == r0.slot
    solo = build_model(cfg, w, debug=False)
    for i, r in enumerate([r0] + sharers):
        one = _gen(solo, prompts[i], r.max_new_tokens, seed=i, **kw)
        assert torch.equal(r.result.cpu(), one), f"request {i} (slot {r.slot}) != a fresh prefill"
    assert torch.equal(rebel.result.cpu(), _gen(solo, rebel_prompt, 20, seed=99, **kw))


def test_retired_prefix_is_reclaimed_under_pressure():
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=41, head_gain=2.5)
    model = _paged_model(cfg, w, kv_pages=8, max_batch=4)
    eng = model.engine
    kw = dict(temperature=0.8, top_p=0.9, top_k=30)
    first = make_prompt(cfg, 1, 180)
    b = ContinuousBatcher(model, max_slots=4, frames_per_poll=4)
    b.submit(SlotRequest(prompt=make_prompt(cfg, 4, 100).cuda(), max_new_tokens=6, seed=4, **kw))
    a = b.submit(SlotRequest(prompt=first.cuda(), max_new_tokens=6, reuse_prefix=True, seed=1, **kw))
    b.run()
    assert a.slot == 1 and a.slot in eng._slot_tokens  # retired, its 3 pages kept as a prefix
    big = b.submit(SlotRequest(prompt=make_prompt(cfg, 2, 400).cuda(), max_new_tokens=40, reuse_prefix=True, seed=2,
                               **kw))
    b.run()
    assert big.slot != a.slot and a.slot not in eng._slot_tokens  # 7 pages: the retired prefix had to go
    assert eng.kv_pool.table[a.slot].max() < 0
    again = torch.cat([first, make_prompt(cfg, 3, 30)], dim=1)
    reused = eng.rows_reused
    c = b.submit(SlotRequest(prompt=again.cuda(), max_new_tokens=10, reuse_prefix=True, seed=3, **kw))
    b.run()
    b.close()
    assert eng.rows_reused == reused  # nothing left to reuse: prefilled in full
    solo = build_model(cfg, w, debug=False)
    for r, p, n, seed in ((a, first, 6, 1), (c, again, 10, 3)):
        assert torch.equal(r.result.cpu(), _gen(solo, p, n, seed=seed, **kw))


def test_64_slots_long_prompt_beside_short_ones_s2pro_layers():
    """Capacity 32 768 positions per slot with a pool far below 64 x 32 768: one 4000-row prompt among 63 short
    requests; each result equals its solo run."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg, w = _s2pro_small(32768)
    pages = 160  # 64 x 512 pages would be the contiguous-capacity pool
    model = _s2pro_model(cfg, w, 64, kv_pages=pages, max_rows=4096)
    kw = dict(temperature=0.8, top_p=0.9, top_k=30)
    specs = [dict(prompt=_s2pro_prompt(cfg, 0, 4000), max_new_tokens=8, seed=0)]
    specs += [dict(prompt=_s2pro_prompt(cfg, i, 10 + i % 17), max_new_tokens=4 + i % 6, seed=i) for i in range(1, 64)]
    b = ContinuousBatcher(model, max_slots=64, frames_per_poll=4)
    reqs = [b.submit(SlotRequest(**{**s, "prompt": s["prompt"].cuda()}, **kw)) for s in specs]
    b.run()
    b.close()
    assert model.engine.kv_pool.peak <= pages
    model.engine.close()
    solo = _s2pro_model(cfg, w, 1)
    for i in (0, 1, 2, 31, 63):
        s = specs[i]
        one = _gen(solo, s["prompt"], s["max_new_tokens"], seed=s["seed"], **kw)
        assert torch.equal(reqs[i].result.cpu(), one), f"request {i} != its solo run"
