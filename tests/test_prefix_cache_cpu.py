"""Prefix cache of the KV page pool without a GPU (KvPagePool prefix_cache, LmEngine(prefix_cache=True)): a finished
request's prompt pages stay in the pool as a cached row, later requests with the same prefix map them instead of
prefilling those rows, and a reservation short of pages drops cached rows least recently used first. The page
bookkeeping is LmEngine's own; only the device work is faked."""
import random
import time

import numpy as np
import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200.engine import KV_PAGE, KvPagePool, kv_pages_for
from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
from tests.test_engine_cpu import _SchedModel
from tests.test_kv_grow_cpu import _GrowFakeEngine
from tests.test_paged_kv_cpu import _S2ProSizedModel


class _CacheFakeEngine(_GrowFakeEngine):
    """_GrowFakeEngine on a pool with the prefix cache on or off; records the rows each prefill computes and every page
    copy."""

    def __init__(self, slots, pages, stop=None, prefix_cache=True, **kw):
        super().__init__(slots, pages, stop, **kw)
        self.copies, self.pieces = [], []
        self.kv_pool = KvPagePool(slots, kv_pages_for(self.kv_len), pages, on_reclaim=self._forget_slot,
                                  copy_page=lambda s, d, n: self.copies.append((s, d, n)), prefix_cache=prefix_cache)

    def prefill(self, prompts, slots, sp, start_pos=None, do_sample=True, kv_end=None):
        self.pieces += [(int(s), int(s0), int(p.shape[1]), p, len(self.prefills)) for p, s, s0 in
                        zip(prompts, slots, start_pos or [0] * len(prompts))]
        super().prefill(prompts, slots, sp, start_pos, do_sample, kv_end)


def _batcher(slots, pages, stop=None, kv_len=2048, fpp=8, growth=False, prefix_cache=True, **kw):
    eng = _CacheFakeEngine(slots, pages, stop, prefix_cache=prefix_cache, kv_len=kv_len, max_frames=kv_len,
                           max_rows=1 << 16)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=kv_len), max_slots=slots, frames_per_poll=fpp,
                          kv_growth=growth, **kw)
    return b, eng


def _check_pages(eng):
    """Every reference is a row's -- slots, parked rows, cached rows -- and every page is free or referenced."""
    pool = eng.kv_pool
    rows = [pool.table[s] for s in range(pool.slots)] + list(pool.detached) + [e.row for e in pool.cached]
    refs = np.zeros(pool.n_pages, dtype=np.int64)
    for row in rows:
        np.add.at(refs, row[row >= 0], 1)
    assert (refs == pool.ref).all()
    assert len(pool.free) == len(set(pool.free)) and not (refs[pool.free] > 0).any()
    assert len(pool.free) + int((refs > 0).sum()) == pool.n_pages


def _voice(seed, n):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 4000, (3, n), generator=g, dtype=torch.int32)


def _req(prefix, tail_seed, tail, n, seed, **kw):
    return SlotRequest(prompt=torch.cat([prefix, _voice(10_000 + tail_seed, tail)], 1), max_new_tokens=n, seed=seed,
                       reuse_prefix=True, **kw)


# ---- the pool ----------------------------------------------------------------------------------------------------------
def test_insert_keeps_only_the_prompt_pages_and_frees_decode_pages():
    pool = KvPagePool(2, 16, 20, prefix_cache=True)
    pool.reserve(0, 150 + 200)  # prompt of 150 rows + 200 frames: 6 pages
    pages = pool.table[0, :6].tolist()
    pool.insert(0, _voice(1, 150))
    (entry,) = pool.cached
    assert entry.n == 150 and entry.row[:3].tolist() == pages[:3] and (entry.row[3:] < 0).all()
    assert (pool.table[0] < 0).all() and pool.ref[pages[:3]].tolist() == [1, 1, 1]
    assert set(pages[3:]) <= set(pool.free) and pool.in_use() == 3 and pool.cached_pages() == 3
    assert pool.available() == 20  # pages only the cache maps are available
    # a covering entry is only touched; an entry that is a prefix of a new one is dropped
    pool.reserve(1, 100)
    pool.insert(1, _voice(1, 150)[:, :100])
    assert list(pool.cached) == [entry] and pool.in_use() == 3
    longer = torch.cat([_voice(1, 150), _voice(2, 80)], 1)
    pool.reserve(1, 230)
    pool.insert(1, longer)
    (entry2,) = pool.cached
    assert entry2.n == 230 and pool.in_use() == 4 and pool.lookup(np.ascontiguousarray(longer.numpy().T))[0] == 230


def test_retire_caches_the_prompt_and_decode_pages_go_back():
    b, eng = _batcher(2, 40)
    r = b.submit(_req(_voice(1, 150), 0, 40, 300, seed=1))
    b.step()
    assert eng.kv_pool.in_use() == kv_pages_for(190 + 300)
    b.run()
    assert r.error is None and r.done.is_set()
    (entry,) = eng.kv_pool.cached
    assert entry.n == 190 and eng.kv_pool.in_use() == kv_pages_for(190) and (eng.kv_pool.table < 0).all()
    _check_pages(eng)


def test_cache_off_keeps_the_retired_slot_as_before():
    b, eng = _batcher(2, 40, prefix_cache=False)
    b.submit(_req(_voice(1, 150), 0, 40, 300, seed=1))
    b.run()
    assert not eng.kv_pool.cached and eng.kv_pool.in_use() == kv_pages_for(190 + 300)


def test_lookup_takes_the_longest_prefix_over_slots_and_cache_and_copies_the_partial_page():
    """A live slot shares 130 rows with the new prompt, a cached row 200: the cached row wins, its 3 whole pages are
    mapped by reference and the 4th is copied, exactly 200 % 64 = 8 positions of it."""
    eng = _CacheFakeEngine(4, 40, kv_len=1024, max_frames=1024, max_rows=4096)
    voice = _voice(7, 200)
    eng.prefill_reusing([torch.cat([voice, _voice(8, 30)], 1)], [0], None, kv_end=[300])
    eng.retire_slot(0)
    (entry,) = eng.kv_pool.cached
    eng.prefill_reusing([torch.cat([voice[:, :130], _voice(9, 90)], 1)], [1], None, kv_end=[260])  # live, shares 130
    eng.copies.clear()
    new = torch.cat([voice, _voice(10, 50)], 1)
    assert eng._donor(new, 2, {2}) == (200, entry)
    reused = eng.prefill_reusing([new], [2], None, kv_end=[300])
    assert reused == [200] and eng.pieces[-1][:3] == (2, 200, 50)
    pool = eng.kv_pool
    assert pool.table[2, :3].tolist() == entry.row[:3].tolist() and pool.table[2, 3] != entry.row[3]
    assert eng.copies == [(int(entry.row[3]), int(pool.table[2, 3]), 200 % KV_PAGE)]
    assert pool.hits == 2 and eng.rows_reused == 130 + 200  # slot 1 took its 130 rows from the cache too
    # shorter than MIN_REUSE: nothing is reused
    assert eng._donor(torch.cat([voice[:, :10], _voice(11, 40)], 1), 3, {3}) == (0, 3)
    _check_pages(eng)


# ---- eviction ------------------------------------------------------------------------------------------------------------
def _cache_voices(eng, voices, slot=0):
    for v in voices:
        eng.prefill_reusing([v], [slot], None, kv_end=[v.shape[1] + 10])
        eng.retire_slot(slot)


def _which(pool, voices):
    """Index of the voice each cached row starts with, least recently used first."""
    return [next(i for i, v in enumerate(voices) if np.array_equal(e.rows[:v.shape[1]], v.numpy().T))
            for e in pool.cached]


def test_eviction_only_under_pressure_and_least_recently_used_first():
    eng = _CacheFakeEngine(2, 10, kv_len=1024, max_frames=1024, max_rows=4096)
    voices = [_voice(20 + i, 130) for i in range(4)]  # 3 pages each
    _cache_voices(eng, voices[:3])
    pool = eng.kv_pool
    assert _which(pool, voices) == [0, 1, 2] and pool.evictions == 0 and len(pool.free) == 1
    # reuse voice 0: its partial page is copied into the free page, no pressure; it becomes the most recently used
    eng.prefill_reusing([torch.cat([voices[0], _voice(99, 20)], 1)], [1], None, kv_end=[160])
    assert pool.hits == 1 and pool.evictions == 0
    eng.retire_slot(1)  # voice 0 + its tail replaces the cached voice 0, which is a prefix of it
    assert _which(pool, voices) == [1, 2, 0] and len(pool.free) == 1
    _cache_voices(eng, voices[3:], slot=0)  # needs 3 pages: the least recently used, voice 1, goes
    assert pool.evictions == 1 and _which(pool, voices) == [2, 0, 3]
    _check_pages(eng)


def test_eviction_never_frees_a_page_a_live_or_parked_row_maps():
    eng = _CacheFakeEngine(3, 10, kv_len=1024, max_frames=1024, max_rows=4096)
    voice = _voice(30, 200)  # 3 whole pages and 8 rows of a 4th
    _cache_voices(eng, [voice])
    (entry,) = eng.kv_pool.cached
    shared = entry.row[:3].tolist()
    eng.prefill_reusing([torch.cat([voice, _voice(31, 20)], 1)], [0], None, kv_end=[228])  # live sharer
    eng.prefill_reusing([torch.cat([voice, _voice(32, 20)], 1)], [1], None, kv_end=[228])
    parked = eng.park_slot(1, 228)
    pool = eng.kv_pool
    assert len(pool.free) == 4
    pool.reserve(2, 5 * KV_PAGE)  # one page short: the cached row goes, and only its own 4th page is freed
    assert not pool.cached and pool.evictions == 1
    assert pool.table[0, :3].tolist() == shared and parked.row[:3].tolist() == shared
    assert pool.ref[shared].tolist() == [2, 2, 2] and not set(shared) & set(pool.free)
    _check_pages(eng)
    with pytest.raises(RuntimeError, match="exhausted"):
        pool.reserve(2, 8 * KV_PAGE)  # only live and parked rows left


@pytest.mark.parametrize("seed", range(24))
def test_randomized_schedules_with_growth_and_the_cache_finish_and_leak_nothing(seed):
    """Seeded schedules over a few voices: bounded pools, KV growth on or off, cancels in every state. The cache-on run
    finishes every request the cache-off run finishes, with the same tokens, never runs out of pages, and after
    release_kv every page is free."""
    rnd = random.Random(seed)
    slots, fpp = rnd.choice([2, 3, 4, 8]), rnd.choice([4, 8])
    growth = rnd.random() < 0.6
    voices = [_voice(100 * seed + v, rnd.randint(20, 300)) for v in range(rnd.randint(1, 4))]
    specs = []
    for i in range(rnd.randint(6, 20)):
        v = rnd.randrange(len(voices) + 1)
        T, n = rnd.randint(1, 90), rnd.randint(8, 300)
        specs.append((v, T, n, rnd.randint(1, n)))
    worst = max(kv_pages_for((voices[v].shape[1] if v < len(voices) else 0) + T + n) for v, T, n, _ in specs)
    pages = rnd.randint(worst, 3 * worst)
    cancel_at = {rnd.randrange(len(specs)): rnd.randint(0, 30) for _ in range(2)}

    cancelled = set()

    def run(cache):
        b, eng = _batcher(slots, pages, {i: s[3] for i, s in enumerate(specs)}, fpp=fpp, growth=growth,
                          prefix_cache=cache)
        reqs = []
        for i, (v, T, n, _) in enumerate(specs):
            prefix = voices[v] if v < len(voices) else torch.zeros(3, 0, dtype=torch.int32)
            reqs.append(_req(prefix, 1000 * seed + i, T, n, seed=i))
        pending = list(reqs)
        for step in range(5000):
            while pending and (rnd_run.random() < 0.5 or b.idle()):
                b.submit(pending.pop(0))
            for i, at in cancel_at.items():
                if step == at and not reqs[i].done.is_set() and (reqs[i] in b.waiting or reqs[i].slot >= 0
                                                                 or reqs[i]._parked is not None):
                    b.cancel(reqs[i])
                    cancelled.add(i)
            if b.idle() and not pending:
                break
            b.step()
            _check_pages(eng)
        assert b.idle() and not pending
        eng.release_kv()
        assert eng.kv_pool.in_use() == 0 and not eng.kv_pool.ref.any() and not eng.kv_pool.cached
        return reqs, eng

    rnd_run = random.Random(seed)
    off, _ = run(False)
    rnd_run = random.Random(seed)
    on, eng = run(True)
    for i, (a, c) in enumerate(zip(off, on)):
        assert a.done.is_set() and c.done.is_set()
        if i not in cancelled:
            assert a.error is None and c.error is None, (a.error, c.error)
            assert torch.equal(a.result, c.result)
    if growth:
        assert not eng.bufs["kv_miss"].any()


# ---- a voice-clone queue ---------------------------------------------------------------------------------------------------
def _zipf_queue(cache, V=6, n_req=40, seed=3, engine=_CacheFakeEngine, pages=400):
    rnd = random.Random(seed)
    w = [1.0 / (k + 1) ** 1.1 for k in range(V)]
    voices = [_voice(500 + v, rnd.randint(100, 300)) for v in range(V)]
    kw = dict(prefix_cache=cache) if engine is _CacheFakeEngine else {}
    eng = engine(4, pages, {i: 20 + i % 17 for i in range(n_req)}, kv_len=2048, max_frames=2048, max_rows=1 << 16, **kw)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=2048), max_slots=4, frames_per_poll=8)
    reqs = []
    for i in range(n_req):
        v = rnd.choices(range(V), w)[0]
        reqs.append(b.submit(_req(voices[v], i, rnd.randint(30, 100), 64, seed=i, tag=v)))
    b.run()
    assert all(r.error is None for r in reqs)
    return reqs, eng, voices


def test_zipf_voice_queue_cache_off_makes_todays_calls():
    reqs, eng, _ = _zipf_queue(False)
    base, base_eng, _ = _zipf_queue(None, engine=_GrowFakeEngine)
    assert eng.calls == base_eng.calls and eng.prefills == base_eng.prefills
    assert all(torch.equal(a.result, c.result) for a, c in zip(reqs, base))
    assert not eng.kv_pool.cached and eng.kv_pool.hits == 0


def test_zipf_voice_queue_cache_on_prefills_only_what_is_not_cached():
    off, eng_off, voices = _zipf_queue(False)
    on, eng, _ = _zipf_queue(True)
    assert all(torch.equal(a.result, c.result) for a, c in zip(off, on))
    assert eng.kv_pool.evictions == 0  # the pool is large enough to keep every voice
    first = {}  # voice -> first prefill call that computed it
    for r in on:
        T = r.prompt.shape[1]
        (start, rows, call), = [(s0, n, k) for _, s0, n, p, k in eng.pieces
                                if s0 + n == T and torch.equal(p, r.prompt[:, s0:])]
        assert rows == T - start
        if first.setdefault(r.tag, call) < call:  # not prefilled beside its voice's first request
            assert start >= voices[r.tag].shape[1], "a voice served before must come from the cache or a live slot"
    assert eng.rows_prefilled + eng.rows_reused == sum(r.prompt.shape[1] for r in on)
    assert eng.rows_prefilled < eng_off.rows_prefilled and eng.kv_pool.hits > 0


def test_lookup_stays_cheap_with_hundreds_of_cached_voices():
    pool = KvPagePool(1, 32, 4000, prefix_cache=True)
    for v in range(300):
        pool.reserve(0, 700)
        pool.insert(0, _voice(2000 + v, 700))
    probe = np.ascontiguousarray(torch.cat([_voice(2150, 700), _voice(1, 60)], 1).numpy().T)
    t0 = time.perf_counter()
    for _ in range(20):
        n, e = pool.lookup(probe)
    dt = (time.perf_counter() - t0) / 20
    assert n == 700 and e.n == 700
    assert dt < 5e-3, f"lookup over 300 cached rows took {dt * 1e3:.2f} ms"


# ---- the serving worker ----------------------------------------------------------------------------------------------------
def test_serve_prefix_cache_variable(monkeypatch):
    assert inf.serve_prefix_cache(None) is False and inf.serve_prefix_cache("") is False
    assert inf.serve_prefix_cache("0") is False and inf.serve_prefix_cache("1") is True
    for bad in ("yes", "2", "on"):
        with pytest.raises(ValueError, match="FSB_SERVE_PREFIX_CACHE"):
            inf.serve_prefix_cache(bad)
    loaded = []
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: loaded.append(1))
    monkeypatch.setenv("FSB_SERVE_PREFIX_CACHE", "true")
    with pytest.raises(ValueError, match="FSB_SERVE_PREFIX_CACHE"):
        inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
    assert not loaded  # refused before the model loads


@pytest.mark.parametrize("slots", ["1", "64"])
@pytest.mark.parametrize("env,want", [(None, False), ("0", False), ("1", True)])
def test_serving_worker_hands_the_variable_to_setup_caches(monkeypatch, slots, env, want):
    seen = []
    model = _S2ProSizedModel()
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (model, inf.decode_one_token_ar))
    monkeypatch.setattr(inf, "serve_requests", lambda m, q, s: seen.append(m.caches))
    monkeypatch.setenv("FSB_SERVE_SLOTS", slots)
    monkeypatch.setenv("FSB_SERVE_KV_LEN", "1024")
    monkeypatch.delenv("FSB_SERVE_KV_GB", raising=False)
    if env is None:
        monkeypatch.delenv("FSB_SERVE_PREFIX_CACHE", raising=False)
    else:
        monkeypatch.setenv("FSB_SERVE_PREFIX_CACHE", env)
    q = inf.launch_thread_safe_queue("ckpt", "cpu", torch.bfloat16)
    if slots == "1":
        q.put(None)
        assert model.caches["prefix_cache"] is want and model.caches["max_batch_size"] == 1
        return
    for _ in range(200):
        if seen:
            break
        time.sleep(0.01)
    assert seen[0]["prefix_cache"] is want and seen[0]["max_batch_size"] == 64


# ---- voice-clone prompts of the reference's prompt builder ------------------------------------------------------------------
VOICE_TEXTS = ("Hello there, this is the first request.", "A different text entirely for the second one.")


def voice_clone_prompts(frontend=None):
    """The first prompt of two requests with one reference (text and codes) and different texts, built by the REAL body
    of the generate_long plan with the byte-level tokenizer of test_engine_cpu.py. `frontend` replaces the reference's
    prompt builder when given. Returns (prompts, conversations the builder saw or None, end of the system message: one
    past its <|im_end|>, from the live builder's token ids, or None)."""
    from tests.test_engine_cpu import _ByteTokenizer

    class Model:
        class config:
            max_seq_len, num_codebooks = 8192, 10

        tokenizer = _ByteTokenizer()

    ref_codes = torch.arange(10 * 40).view(10, 40) % 1024
    saved = inf._reference_frontend
    if frontend is not None:
        inf._reference_frontend = frontend
    try:
        prompts = []
        for text in VOICE_TEXTS:
            plan = inf._generate_long_plan(model=Model, device="cpu", text=text, chunk_length=200, max_new_tokens=64,
                                           temperature=0.8, top_p=0.8, top_k=30,
                                           prompt_text=["reference words spoken in the clip"], prompt_tokens=[ref_codes])
            kind, payload = plan.send(None)
            assert kind == "generate" and payload["reuse_prefix"] is True
            prompts.append(payload["prompt"].clone())
            plan.close()
    finally:
        inf._reference_frontend = saved
    im_end = Model.tokenizer.special.get("<|im_end|>")
    end = None if im_end is None else int((prompts[0][0] == im_end).nonzero()[0]) + 1
    return prompts, getattr(frontend, "calls", None), end


def test_two_requests_with_one_reference_share_the_whole_system_message():
    from tests.test_engine_cpu import GOLD, _ReplayFrontend

    z = np.load(GOLD / "voice_clone_prompts.npz")
    golden = [z["prompt_0"], z["prompt_1"]]
    system_end = int(z["system_end"])
    try:
        import fish_speech.conversation  # noqa: F401
    except ImportError:
        pass
    else:
        live, _, end = voice_clone_prompts()
        assert all(np.array_equal(a.numpy(), b) for a, b in zip(live, golden)) and end == system_end
    fe = _ReplayFrontend(golden)
    prompts, calls, _ = voice_clone_prompts(fe)
    (sys_a, *_), (sys_b, *_) = calls
    assert sys_a[:4] == sys_b[:4] and sys_a[0] == "system" and all(torch.equal(x, y) for x, y in zip(sys_a[4], sys_b[4]))
    a, b = (np.ascontiguousarray(p.numpy().T, dtype=np.int32) for p in prompts)
    shared = int(np.flatnonzero((a[:len(b)] != b[:len(a)]).any(axis=1))[0])
    assert shared >= system_end > 40  # the reference codes and text sit inside the system message
    pool = KvPagePool(2, 16, 20, prefix_cache=True)
    pool.reserve(0, a.shape[0] + 64)
    pool.insert(0, prompts[0].to(torch.int32))
    assert pool.lookup(b)[0] == shared
