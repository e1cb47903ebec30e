"""Host rules of the paged slow KV cache (no GPU): the page allocator (engine.KvPagePool), page-aware FIFO admission
of the slot scheduler, and the FSB_SERVE_KV_GB pool sizing of the serving worker."""
import time

import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200.engine import KV_PAGE, KvPagePool, kv_pages_for
from tests.test_engine_cpu import _FakeEngine, _FakeModel, _SchedModel


def _pool(slots=4, per_slot=8, pages=16):
    copies, reclaimed = [], []
    pool = KvPagePool(slots, per_slot, pages, copy_page=lambda s, d, n: copies.append((s, d, n)),
                      on_reclaim=reclaimed.append)
    return pool, copies, reclaimed


def test_reserve_maps_private_pages_and_trims():
    pool, copies, _ = _pool()
    assert kv_pages_for(1) == 1 and kv_pages_for(64) == 1 and kv_pages_for(65) == 2
    pool.reserve(0, 130)
    assert (pool.table[0, :3] >= 0).all() and (pool.table[0, 3:] < 0).all()
    assert pool.in_use() == 3 and pool.ref[pool.table[0, :3]].tolist() == [1, 1, 1]
    before = pool.table[0, :3].tolist()
    pool.reserve(0, 200, start=130)  # grows in place
    assert pool.table[0, :3].tolist() == before and pool.in_use() == 4
    pool.reserve(0, 64)  # pages past the end go back
    assert pool.in_use() == 1 and pool.table[0, 0] == before[0]
    assert not copies and pool.peak == 4
    with pytest.raises(ValueError, match="capacity"):
        pool.reserve(0, 8 * KV_PAGE + 1)


def test_shared_prefix_refcounts_and_copy_on_write():
    pool, copies, _ = _pool()
    pool.reserve(0, 300)  # donor: 5 pages
    donor = pool.table[0].tolist()
    p = 200  # 3 whole pages + 8 rows of the 4th
    pool.share(1, 0, kv_pages_for(p))
    pool.reserve(1, 260, start=p)
    assert pool.table[1, :3].tolist() == donor[:3] and pool.ref[donor[:3]].tolist() == [2, 2, 2]
    assert pool.table[1, 3] != donor[3] and pool.ref[donor[3]] == 1
    assert copies == [(donor[3], int(pool.table[1, 3]), p - 3 * KV_PAGE)]  # the partial page keeps rows [192, 200)
    # the donor re-prefilled from 0: shared pages are replaced, not overwritten; nothing to keep
    pool.reserve(0, 100, start=0)
    assert pool.table[1, :3].tolist() == donor[:3] and pool.ref[donor[:3]].tolist() == [1, 1, 1]
    assert not set(pool.table[0, :2].tolist()) & set(donor[:3])
    assert len(copies) == 1
    # a write starting mid-page into a shared page keeps the rows before it
    pool.share(2, 1, 2)
    pool.reserve(2, 150, start=100)
    assert copies[-1] == (donor[1], int(pool.table[2, 1]), 100 - KV_PAGE)
    assert pool.table[2, 0] == donor[0] and pool.ref[donor[0]] == 2
    # releasing a sharer only drops its reference
    pool.release(2)
    assert pool.ref[donor[0]] == 1 and donor[0] not in pool.free


def test_retired_slots_are_reclaimed_least_recently_retired_first():
    pool, _, reclaimed = _pool(slots=4, per_slot=8, pages=8)
    for s in range(3):
        pool.reserve(s, 2 * KV_PAGE)
    pool.retire(1)
    pool.retire(0)
    assert pool.available() == 8 - 2  # slot 2 is live
    pool.reserve(3, 3 * KV_PAGE)  # 2 free pages: one retired slot must go, slot 1 first
    assert reclaimed == [1] and (pool.table[1] < 0).all() and (pool.table[0, :2] >= 0).all()
    pool.reserve(3, 5 * KV_PAGE)  # 1 free page for 2 more: slot 0 goes too
    assert reclaimed == [1, 0]
    with pytest.raises(RuntimeError, match="kv_pages"):
        pool.reserve(3, 8 * KV_PAGE)  # only live slots left
    assert pool.in_use() <= pool.n_pages


def test_reclaiming_a_donor_keeps_the_pages_its_sharers_map():
    pool, _, reclaimed = _pool(slots=3, per_slot=8, pages=6)
    pool.reserve(0, 3 * KV_PAGE)
    pool.share(1, 0, 2)
    pool.reserve(1, 3 * KV_PAGE, start=2 * KV_PAGE)
    pool.retire(0)
    assert pool.available() == 6 - 3
    pool.reserve(2, 3 * KV_PAGE)  # needs the donor's private page
    assert reclaimed == [0] and pool.ref[pool.table[1, :2]].tolist() == [1, 1]


def test_pages_shared_among_re_prefilled_slots_are_released_before_allocating():
    """Two retired slots share a prefix; both are re-prefilled from position 0 in a pool with no other free page.
    What they shared must not be counted twice: the first reservation drops its reference before allocating."""
    pool, copies, _ = _pool(slots=3, per_slot=8, pages=4)
    pool.reserve(0, 2 * KV_PAGE)
    pool.share(1, 0, 2)
    pool.reserve(1, 2 * KV_PAGE, start=2 * KV_PAGE)
    pool.retire(0)
    pool.retire(1)
    assert pool.available() == 4
    pool.hold(0, 2 * KV_PAGE, 0)
    pool.hold(1, 2 * KV_PAGE, 0)
    pool.reserve(0, 2 * KV_PAGE)
    pool.reserve(1, 2 * KV_PAGE)
    assert pool.in_use() == 4 and not copies
    assert not set(pool.table[0, :2].tolist()) & set(pool.table[1, :2].tolist())


class _PagedFakeEngine(_FakeEngine):
    """_FakeEngine with a page pool: reservations at prefill, pages kept on retirement."""

    def __init__(self, slots, pages, **kw):
        super().__init__(slots, **kw)
        self.kv_pool = KvPagePool(slots, kv_pages_for(self.kv_len), pages)
        self.peaks = []

    def kv_pages_available(self):
        return self.kv_pool.available()

    def kv_pages_needed(self, prompt, n_positions, slot, busy=(), reuse=False):
        return kv_pages_for(min(n_positions, self.kv_len))

    def retire_slot(self, slot):
        self.kv_pool.retire(slot)

    def release_kv(self):
        for s in range(self.max_batch):
            self.kv_pool.release(s)

    def prefill(self, prompts, slots, sp, start_pos=None, do_sample=True, kv_end=None):
        for p, s, e in zip(prompts, slots, kv_end):
            self.kv_pool.reserve(s, e)
        self.peaks.append(self.kv_pool.in_use())
        super().prefill(prompts, slots, sp, start_pos, do_sample)


def test_admission_waits_for_pages_in_fifo_order():
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    eng = _PagedFakeEngine(slots=4, pages=3, kv_len=256, max_frames=200, max_rows=1024)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=256), max_slots=4, frames_per_poll=4)
    mk = lambda T, n, tag: SlotRequest(prompt=torch.full((3, T), tag), max_new_tokens=n, tag=tag)
    with pytest.raises(ValueError, match="kv_pages"):
        b.submit(mk(200, 100, 9))  # 4 pages: more than the whole pool
    reqs = [b.submit(mk(100, 20, 0)), b.submit(mk(150, 40, 1)), b.submit(mk(10, 2, 2))]
    b.step()
    # 2 + 3 pages do not fit in 3: request 1 waits, and the small request 2 does not overtake it
    assert [r.slot for r in reqs] == [0, -1, -1] and len(b.waiting) == 2
    b.run()
    assert all(r.done.is_set() for r in reqs) and max(eng.peaks) <= 3
    order = [p for p in eng.prefills]
    assert order[0] == [0] and order[1][0] == reqs[1].slot and reqs[2].slot >= 0
    b.close()


class _ReusingFakeEngine(_FakeEngine):
    """_FakeEngine whose page bookkeeping is LmEngine's own: donor choice, page-limited admission accounting and
    prefill_reusing's sharing run unchanged; only the device work (page-table upload, kernels) is left out."""

    from fish_speech_b200.engine import LmEngine as _E

    MIN_REUSE = _E.MIN_REUSE
    _common_prefix = staticmethod(_E._common_prefix)
    _donor = _E._donor
    _forget_slot = _E._forget_slot
    kv_pages_needed = _E.kv_pages_needed
    kv_pages_available = _E.kv_pages_available
    retire_slot = _E.retire_slot
    release_kv = _E.release_kv
    prefill_reusing = _E.prefill_reusing

    def __init__(self, slots, pages, **kw):
        super().__init__(slots, **kw)
        self.kv_pool = KvPagePool(slots, kv_pages_for(self.kv_len), pages, on_reclaim=self._forget_slot)
        self._slot_tokens, self._covered, self.in_use = {}, {}, []
        self.rows_reused = self.rows_prefilled = 0

    def _reserve(self, items):
        for s, end, start in items:
            self.kv_pool.hold(int(s), end, start)
        for s, end, start in items:
            self.kv_pool.reserve(int(s), end, start)

    def prefill(self, prompts, slots, sp, start_pos=None, do_sample=True, kv_end=None):
        start_pos = start_pos or [0] * len(prompts)
        self._reserve([(s, max(s0 + p.shape[1], e), s0) for p, s, s0, e in zip(prompts, slots, start_pos, kv_end)])
        self.in_use.append(self.kv_pool.in_use())
        super().prefill(prompts, slots, sp)


def test_page_limited_admission_counts_pages_shared_with_a_live_donor():
    """A pool too small for 8 private copies of a 200-row prefix: requests that reuse the prefix of a live slot need
    only their own pages, so all 8 are admitted together beside the donor, and no reservation runs out of pages."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    eng = _ReusingFakeEngine(slots=9, pages=13, kv_len=1024, max_frames=100, max_rows=4096)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=1024), max_slots=9, frames_per_poll=4)
    prefix = torch.arange(200).repeat(3, 1)
    mk = lambda i, n: SlotRequest(prompt=torch.cat([prefix, torch.full((3, 20), 1000 + i)], dim=1), max_new_tokens=n,
                                  reuse_prefix=True, tag=i)
    donor = b.submit(mk(0, 60))  # 280 positions: 5 pages
    b.step()
    assert donor.slot == 0 and not donor.done.is_set()
    sharers = [b.submit(mk(i, 30)) for i in range(1, 9)]  # 250 positions: 4 pages, 3 of them the donor's
    assert eng.kv_pages_needed(sharers[0].prompt, 250, 1, reuse=True) == 1
    b._admit()
    assert sorted(r.slot for r in sharers) == list(range(1, 9)) and not b.waiting
    pool = eng.kv_pool
    assert pool.ref[pool.table[0, :3]].tolist() == [9, 9, 9] and pool.in_use() == 13
    assert eng.rows_reused == 8 * 200
    b.run()
    b.close()
    assert all(r.done.is_set() for r in [donor] + sharers) and max(eng.in_use) <= 13


class _S2ProSizedModel(_FakeModel):
    class config:
        max_seq_len = 32768
        n_layer, n_local_heads, head_dim = 36, 8, 128


def test_serve_kv_pool_sizing():
    cfg = _S2ProSizedModel.config
    assert inf.kv_page_bytes(cfg) == 64 * 147456
    assert inf.serve_kv_pool_pages(24, cfg, 80 * 10 ** 9) == int(24e9 // (64 * 147456))
    with pytest.raises(ValueError, match="FSB_SERVE_KV_GB"):
        inf.serve_kv_pool_pages(24, cfg, 20 * 10 ** 9)
    with pytest.raises(ValueError, match="FSB_SERVE_KV_GB"):
        inf.serve_kv_pool_pages(0.001, cfg, 80 * 10 ** 9)


def test_serve_kv_gb_builds_a_paged_engine(monkeypatch):
    seen = []
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (_S2ProSizedModel(), inf.decode_one_token_ar))
    monkeypatch.setattr(inf, "serve_requests", lambda model, q, slots: seen.append((slots, model.caches)))
    monkeypatch.setenv("FSB_SERVE_SLOTS", "64")
    monkeypatch.setenv("FSB_SERVE_KV_GB", "24")
    monkeypatch.delenv("FSB_SERVE_KV_LEN", raising=False)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (60 * 10 ** 9, 80 * 10 ** 9))
    inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
    for _ in range(200):
        if seen:
            break
        time.sleep(0.01)
    caches = seen[0][1]
    assert caches["max_batch_size"] == 64 and caches["max_seq_len"] == 32768
    assert caches["kv_pages"] == int(24e9 // (64 * 147456))
    monkeypatch.setenv("FSB_SERVE_KV_LEN", "16384")
    monkeypatch.setenv("FSB_SERVE_KV_GB", "70")
    with pytest.raises(ValueError, match="FSB_SERVE_KV_GB"):
        inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
    assert len(seen) == 1
