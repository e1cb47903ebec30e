"""KV growth of the slot scheduler without a GPU (ContinuousBatcher(kv_growth=True)): requests map pages as they
decode under the banker's rule (scheduler.kv_safe), wait parked for pages when a grant would be unsafe, and every
request finishes with the tokens it would produce alone. The page bookkeeping is LmEngine's own; only the device
work is faked."""
import random

import numpy as np
import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200.engine import KV_PAGE, LmEngine, ParkedSlot, kv_pages_for
from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest, kv_safe
from tests.test_engine_cpu import _SchedModel
from tests.test_paged_kv_cpu import _ReusingFakeEngine


class _GrowFakeEngine(_ReusingFakeEngine):
    """_ReusingFakeEngine with park / resume, LmEngine.grow_kv, and a decode that, like the kernels, records in
    "kv_miss" a live row whose write position has no page. Tokens name the request (1000 * seed + frame), and a
    request stops after `stop[seed]` frames (its <|im_end|>) when that comes before its budget."""

    grow_kv = LmEngine.grow_kv
    SAVED = ("slot_state", "slot_limit", "slot_seed", "n_out", "pos", "out_tokens")

    def __init__(self, slots, pages, stop=None, **kw):
        super().__init__(slots, pages, **kw)
        self.stop = stop or {}
        self.bufs["pos"] = torch.zeros(max(32, slots), dtype=torch.int32)
        self.bufs["kv_miss"] = torch.zeros(slots, dtype=torch.int32)
        self.calls = []

    def _reserve(self, items):
        items = list(items)
        self.calls.append(("reserve", [(int(s), int(e), int(b)) for s, e, b in items]))
        super()._reserve(items)
        for s, end, _ in items:
            self._covered[int(s)] = kv_pages_for(end)

    def _emit(self, s):
        b = self.bufs
        f = int(b["n_out"][s])
        b["out_tokens"][s, :, f] = 1000 * int(b["slot_seed"][s]) + f
        b["n_out"][s] = f + 1
        if f + 1 >= int(b["slot_limit"][s]) or f + 1 >= self.stop.get(int(b["slot_seed"][s]), 1 << 30):
            b["slot_state"][s] = 2

    def prefill(self, prompts, slots, sp, start_pos=None, do_sample=True, kv_end=None):
        start_pos = start_pos or [0] * len(prompts)
        self.calls.append(("prefill", list(slots), list(kv_end)))
        for s, s0 in zip(slots, start_pos):
            if s0 == 0:
                self._slot_tokens.pop(int(s), None)  # as LmEngine.prefill: overwritten from position 0
        self._reserve([(s, max(s0 + p.shape[1], e), s0) for p, s, s0, e in zip(prompts, slots, start_pos, kv_end)])
        self.prefills.append(list(slots))
        for p, s, s0 in zip(prompts, slots, start_pos):
            self.bufs["pos"][s] = s0 + p.shape[1]
            self._emit(s)

    def decode(self, batch, nframes, sp, use_graph=True):
        self.calls.append(("decode", nframes))
        b = self.bufs
        for _ in range(nframes):
            for s in range(batch):
                p = int(b["pos"][s])
                if p >= 0 and self.kv_pool.table[s, p // KV_PAGE] < 0 and int(b["kv_miss"][s]) == 0:
                    b["kv_miss"][s] = p + 1  # idle rows too, as the kernels do for any row at a position >= 0
                if int(b["slot_state"][s]) != 1:
                    continue
                self._emit(s)
                b["pos"][s] = p + 1

    def park_slot(self, slot, ctx_len=0):
        self.calls.append(("park", slot))
        blob = {k: self.bufs[k][slot].clone() for k in self.SAVED}
        self.bufs["slot_state"][slot] = 0
        self.bufs["pos"][slot] = -1
        return ParkedSlot(blob, self.kv_pool.detach(slot), self._slot_tokens.pop(slot, None),
                          self._covered.pop(slot, None), ctx_len)

    def resume_slot(self, slot, parked):
        self.calls.append(("resume", slot))
        self.kv_pool.attach(slot, parked.row)
        if parked.tokens is not None:
            self._slot_tokens[slot] = parked.tokens
        if parked.covered is not None:
            self._covered[slot] = parked.covered
        for k, v in parked.blob.items():
            self.bufs[k][slot] = v

    def drop_parked(self, parked):
        self.calls.append(("drop",))
        self.kv_pool.drop(parked.row)


def _batcher(slots, pages, stop=None, kv_len=1024, fpp=8, growth=True, **kw):
    eng = _GrowFakeEngine(slots, pages, stop, kv_len=kv_len, max_frames=kv_len, max_rows=1 << 16)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=kv_len), max_slots=slots, frames_per_poll=fpp,
                          kv_growth=growth, **kw)
    return b, eng


def _check_pool(b, eng):
    """Pages are conserved and every reference is a row's; the admitted requests form a safe state."""
    pool = eng.kv_pool
    rows = [pool.table[s] for s in range(pool.slots)] + list(pool.detached)
    refs = np.zeros(pool.n_pages, dtype=np.int64)
    for row in rows:
        np.add.at(refs, row[row >= 0], 1)
    assert (refs == pool.ref).all()
    assert len(pool.free) == len(set(pool.free)) and not (refs[pool.free] > 0).any()
    assert len(pool.free) + int((refs > 0).sum()) == pool.n_pages
    avail, claims = b._kv_state()
    assert kv_safe(avail, claims.values())
    assert all(need >= 0 for need, _ in claims.values())


def _frames(reqs):
    return sum(int(r.result.shape[1]) if r.result is not None else 0 for r in reqs)


def test_kv_safe_banker_rule():
    assert kv_safe(3, [(5, 0), (3, 2)])  # the one needing 3 ends and gives back its 2 pages: then 5 fit
    assert not kv_safe(3, [(3, 0), (5, 2)])
    assert not kv_safe(3, [(4, 9)])
    assert not kv_safe(2, [(2, 0), (3, 0)])
    assert kv_safe(0, [])
    assert kv_safe(1, [(1, 1), (2, 0)]) and not kv_safe(1, [(1, 0), (2, 0)])


@pytest.mark.parametrize("seed", range(40))
def test_randomized_schedules_are_safe_and_finish(seed):
    """Seeded schedules: pools from one worst case to several, ragged prompts with and without a shared prefix,
    lengths below budgets, cancels in every state. After every step: pages conserved, the state safe, progress."""
    rnd = random.Random(seed)
    slots = rnd.choice([2, 3, 4, 6, 8])
    fpp = rnd.choice([4, 8, 16])
    budget_max = rnd.choice([128, 256, 400])
    prefix = torch.arange(rnd.choice([70, 130, 200])).repeat(3, 1) + 7
    n_req = rnd.randint(6, 24)
    reqs, stop = [], {}
    for i in range(n_req):
        T = rnd.randint(1, 150)
        shared = rnd.random() < 0.4
        p = torch.cat([prefix, torch.full((3, T), 5000 + i)], 1) if shared else torch.full((3, T), 9000 + i)
        n = rnd.randint(8, budget_max)
        stop[i] = rnd.randint(1, n)
        reqs.append(SlotRequest(prompt=p, max_new_tokens=n, seed=i, reuse_prefix=shared))
    worst = max(kv_pages_for(r.prompt.shape[1] + r.max_new_tokens) for r in reqs)
    pages = rnd.randint(worst, 3 * worst)
    b, eng = _batcher(slots, pages, stop, fpp=fpp)
    assert b.kv_growth
    pending = list(reqs)
    cancelled = set()
    for step in range(5000):
        while pending and rnd.random() < 0.5:
            b.submit(pending.pop(0))
        if b.idle() and not pending:
            break
        if rnd.random() < 0.04:  # cancel one request wherever it is: waiting, running, parked for pages
            live = [r for r in reqs if not r.done.is_set() and (r in b.waiting or r.slot >= 0 or r._parked is not None)]
            if live:
                r = rnd.choice(live)
                assert b.cancel(r)
                cancelled.add(r.seed)
        before = (_frames(reqs), sum(r.done.is_set() for r in reqs),
                  sum(int(eng.bufs["n_out"][s]) for s in b.active))
        work = not b.idle()
        b.step()
        _check_pool(b, eng)
        after = (_frames(reqs), sum(r.done.is_set() for r in reqs),
                 sum(int(eng.bufs["n_out"][s]) for s in b.active))
        if work:
            assert after != before or b.active, f"step {step}: no request made progress"
    assert b.idle() and not pending
    for r in reqs:
        assert r.done.is_set()
        if r.seed in cancelled:
            continue
        assert r.error is None, r.error
        n = min(stop[r.seed], r._limit)
        assert r.result[1:, r.prompt.shape[1]:].tolist() == [[1000 * r.seed + f for f in range(n)]] * 2
    assert not eng.bufs["kv_miss"].any()
    eng.release_kv()
    assert eng.kv_pool.in_use() == 0 and not eng.kv_pool.ref.any()


def test_every_step_progresses_with_a_pool_of_one_worst_case():
    """The tightest pool: one request's worst case. Requests take turns, each finishes, none is starved."""
    stop = {i: 40 + 10 * i for i in range(6)}
    b, eng = _batcher(4, kv_pages_for(64 + 200), stop, fpp=8)
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 64), i), max_new_tokens=200, seed=i)) for i in range(6)]
    steps = 0
    while not b.idle():
        n = _frames(reqs) + sum(int(eng.bufs["n_out"][s]) for s in b.active)
        b.step()
        _check_pool(b, eng)
        steps += 1
        assert steps < 1000
    assert all(r.error is None and r.result.shape[1] == 64 + stop[r.seed] for r in reqs)


def test_fifo_admission_and_fifo_resume_of_requests_parked_for_pages():
    """The head of the queue is never overtaken, and requests parked for pages resume in the order they were
    parked. Equal requests on a pool of two worst cases: all four run at first, two are parked for pages."""
    T, n = 60, 190
    stop = {i: n for i in range(6)}
    b, eng = _batcher(4, 2 * kv_pages_for(T + n), stop, fpp=8)
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, T), i), max_new_tokens=n, seed=i)) for i in range(6)]
    admitted, short_order, resumed = [], [], []
    was_short = set()
    while not b.idle():
        waiting = list(b.waiting)
        b.step()
        newly = [r for r in waiting if r not in b.waiting]
        assert newly == waiting[:len(newly)]  # FIFO: a prefix of the queue is admitted
        admitted += newly
        for r in b.short:
            if r.seed not in was_short:
                was_short.add(r.seed)
                short_order.append(r.seed)
        for r in reqs:
            if r.seed in was_short and r.seed not in resumed and r.slot >= 0:
                resumed.append(r.seed)
    assert [r.seed for r in admitted] == list(range(6))
    assert len(short_order) >= 2 and resumed == short_order
    assert sum(r.page_parks for r in reqs) >= 2
    assert all(r.error is None and r.result.shape[1] == T + n for r in reqs)


def _run_counting(growth, pages):
    stop = {i: 64 for i in range(16)}
    b, eng = _batcher(16, pages, stop, fpp=8, growth=growth)
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 64), i), max_new_tokens=256, seed=i)) for i in range(16)]
    peak = 0
    while not b.idle():
        b.step()
        peak = max(peak, len(b.active))
    assert all(r.error is None and r.result.shape[1] == 64 + 64 for r in reqs)
    return peak, [r.result for r in reqs]


def test_growth_admits_more_requests_than_reserving_the_budget():
    """Budgets four times the actual length (256 frames, stop at 64) on a 20-page pool: reserving prompt + budget
    (5 pages of 64 positions) runs 4 requests at a time. Growth maps 2 pages at admission (64 + 8 positions) and
    keeps 3 in reserve for the worst case: the k-th admission is safe while 3 <= 20 - 2k, so 8 run at a time.
    Same tokens."""
    fixed, res_fixed = _run_counting(False, 20)
    grown, res_grown = _run_counting(True, 20)
    assert fixed == 4 and grown == 8
    assert all(torch.equal(a, b) for a, b in zip(res_fixed, res_grown))


@pytest.mark.parametrize("pages", [None, 40])
def test_growth_is_opt_in(pages):
    """kv_growth=False, and kv_growth=True on a pool that holds every slot at full capacity (None: 4 slots x 16
    pages), make the same engine calls."""
    def run(growth):
        stop = {i: 30 + 7 * i for i in range(7)}
        b, eng = _batcher(4, pages or 4 * kv_pages_for(1024), stop, fpp=8, growth=growth)
        for i in range(7):
            b.submit(SlotRequest(prompt=torch.full((3, 40 + 9 * i), i), max_new_tokens=120, seed=i))
        b.run()
        return b, eng.calls

    b_off, off = run(False)
    b_on, on = run(True)
    assert not b_off.kv_growth
    if pages is None:
        assert not b_on.kv_growth and on == off
    else:
        assert b_on.kv_growth and on != off  # a bounded pool: growth maps pages as requests decode


def test_kv_miss_fails_the_request_alone():
    """A row that meets an unmapped page (recorded by the decode kernels in "kv_miss") fails with the slot and
    position; its neighbour finishes."""
    stop = {0: 100, 1: 100}
    b, eng = _batcher(2, 8, stop, fpp=8)
    r0 = b.submit(SlotRequest(prompt=torch.full((3, 60), 0), max_new_tokens=100, seed=0))
    r1 = b.submit(SlotRequest(prompt=torch.full((3, 60), 1), max_new_tokens=100, seed=1))
    b.step()
    orig = b.eng.grow_kv
    b.eng.grow_kv = lambda ends: orig({s: e for s, e in ends.items() if s != r0.slot})  # r0's next page is withheld
    b.run()
    assert isinstance(r0.error, RuntimeError) and "slot 0" in str(r0.error) and "position 128" in str(r0.error)  # admission mapped [0, 128)
    assert r1.error is None and r1.result.shape[1] == 160
    assert not eng.bufs["kv_miss"].any()


def test_serve_kv_grow_needs_a_bounded_pool(monkeypatch):
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (None, None))
    monkeypatch.setenv("FSB_SERVE_KV_GROW", "1")
    monkeypatch.delenv("FSB_SERVE_KV_GB", raising=False)
    with pytest.raises(ValueError, match="FSB_SERVE_KV_GROW.*FSB_SERVE_KV_GB"):
        inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
    monkeypatch.setenv("FSB_SERVE_KV_GROW", "yes")
    monkeypatch.setenv("FSB_SERVE_KV_GB", "24")
    with pytest.raises(ValueError, match="FSB_SERVE_KV_GROW"):
        inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
