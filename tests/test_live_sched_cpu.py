"""Host rules of serving more live streams than slots (no GPU): the pacing policy (scheduler.schedule_live), the
page pool's detached rows (engine.KvPagePool.detach / attach / drop), ContinuousBatcher.cancel, parking through a
fake engine with a fake clock, and the worker loop's `cancel` event."""
import queue as Q
import threading

import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200.engine import KV_PAGE, KvPagePool, ParkedSlot
from fish_speech_b200.scheduler import (PARK_POLLS, RESUME_POLLS, Cancelled, ContinuousBatcher, SlotRequest,
                                        StreamClock, schedule_live)
from tests.test_engine_cpu import _FakeBatcher, _FakeEngine, _FakeModel, _SchedModel, _fake_plan
from tests.test_paged_kv_cpu import _PagedFakeEngine

NOW, FPP = 100.0, 4
RESUME_AT, PARK_AT = RESUME_POLLS * FPP, PARK_POLLS * FPP


def _req(lead=None, tag=None, pace=10.0):
    """A request whose lead at NOW is `lead` frames; None: unpaced."""
    r = SlotRequest(prompt=torch.zeros(3, 1, dtype=torch.long), max_new_tokens=8, tag=tag)
    if lead is not None:
        r.pace, r.stream = pace, StreamClock(t_first=0.0, frames=lead + pace * NOW)
        assert r.lead(NOW) == pytest.approx(lead)
    return r


def _plan(running, parked, waiting, slots, max_live):
    return schedule_live(running, parked, waiting, NOW, slots, max_live, FPP)


def _tags(rs):
    return [r.tag for r in rs]


# ---- the policy function ---------------------------------------------------------------------------------------------
def test_unpaced_requests_are_scheduled_first_in_first_out():
    running = [_req(tag="r0"), _req(tag="r1")]
    waiting = [_req(tag=i) for i in range(5)]
    p = _plan(running, [], waiting, slots=4, max_live=4)
    assert not p.park and not p.resume and not p.fill and _tags(p.admit) == [0, 1]
    p = _plan(running + [_req(), _req()], [], waiting, slots=4, max_live=4)
    assert not p.park and not p.admit  # no free slot: nobody moves


def test_parks_the_largest_leads_first_and_only_as_many_as_are_needed():
    running = [_req(PARK_AT + 5, "a"), _req(PARK_AT + 30, "b"), _req(PARK_AT + 10, "c"), _req(PARK_AT - 1, "d")]
    parked = [_req(RESUME_AT - 1, "p")]
    waiting = [_req(-3.0, "w")]
    p = _plan(running, parked, waiting, slots=4, max_live=8)
    assert _tags(p.park) == ["b", "c"]  # two candidates below the resume threshold -> the two largest leads
    assert _tags(p.resume) == ["p"] and _tags(p.admit) == ["w"]  # the parked one resumes before the admission
    # with a free slot nobody is parked: the slot goes to the parked request, the new one waits
    p = _plan(running[:3], parked, waiting, slots=4, max_live=8)
    assert not p.park and _tags(p.resume) == ["p"] and not p.admit


def test_never_parks_an_unpaced_request_or_one_below_the_park_threshold():
    running = [_req(None, "u0"), _req(None, "u1"), _req(PARK_AT - 0.5, "x"), _req(PARK_AT, "y")]
    p = _plan(running, [_req(0.0, "p0"), _req(1.0, "p1")], [], slots=4, max_live=8)
    assert _tags(p.park) == ["y"] and _tags(p.resume) == ["p0"]  # the smallest lead gets the one slot
    p = _plan(running[:3] + [_req(None, "u2")], [_req(0.0, "p0")], [_req(-9.0, "w")], slots=4, max_live=8)
    assert not p.park and not p.resume and not p.admit


def test_nothing_is_parked_for_requests_that_are_not_short_of_frames():
    running = [_req(PARK_AT + 9, "a"), _req(PARK_AT + 9, "b")]
    p = _plan(running, [_req(RESUME_AT, "p")], [_req(None, "u")], slots=2, max_live=8)
    assert not p.park and not p.resume and not p.admit  # a parked request at the threshold and an unpaced arrival
    # a continuation chunk that is still far ahead does not take a slot from anybody either
    p = _plan(running, [], [_req(RESUME_AT + 3, "chunk2")], slots=2, max_live=8)
    assert not p.park and not p.admit


def test_an_overdue_continuation_chunk_goes_ahead_of_later_arrivals():
    chunk2 = _req(-6.0, "chunk2")  # its utterance is playing and has run dry
    waiting = [_req(None, "u"), _req(-0.5, "new0"), _req(-0.2, "new1"), chunk2, _req(2.0, "early")]
    p = _plan([], [], waiting, slots=8, max_live=8)
    # overdue paced ones by smallest lead; the rest (unpaced, and paced ones that still have audio) as they arrived
    assert _tags(p.admit) == ["chunk2", "new0", "new1", "u", "early"]
    p = _plan([_req(PARK_AT + 1, "a"), _req(None, "b")], [], waiting, slots=2, max_live=3)
    assert _tags(p.park) == ["a"] and _tags(p.admit) == ["chunk2"]  # max_live leaves room for one more


def test_no_flapping_between_the_thresholds():
    assert PARK_POLLS - RESUME_POLLS >= 3  # several polls of hysteresis
    mid = (RESUME_AT + PARK_AT) / 2
    running = [_req(mid, f"r{i}") for i in range(4)]
    parked = [_req(mid - 1, f"p{i}") for i in range(4)]
    p = _plan(running, parked, [], slots=4, max_live=8)
    assert not p.park and not p.resume and not p.admit
    # what was just resumed (lead below the resume threshold) cannot be parked in the next poll, even if every slot
    # is wanted: it is below the park threshold until it has run for several polls
    p = _plan([_req(RESUME_AT - 1 + FPP, f"r{i}") for i in range(4)], [_req(0.0, "p")], [], slots=4, max_live=8)
    assert not p.park and not p.resume


def test_free_slots_never_idle_while_requests_are_parked():
    p = _plan([_req(mid := 12.0, "r")], [_req(mid + 5, "p1"), _req(mid, "p0")], [_req(None, "u")], slots=4, max_live=8)
    assert not p.resume and _tags(p.admit) == ["u"] and _tags(p.fill) == ["p0", "p1"]


# ---- the page pool's detached rows -----------------------------------------------------------------------------------
def _pool(slots=4, per_slot=8, pages=8):
    reclaimed = []
    return KvPagePool(slots, per_slot, pages, on_reclaim=reclaimed.append), reclaimed


def test_detached_pages_keep_their_references_and_count_as_live():
    pool, reclaimed = _pool()
    pool.reserve(0, 3 * KV_PAGE)
    pages = pool.table[0, :3].tolist()
    row = pool.detach(0)
    assert row[:3].tolist() == pages and (pool.table[0] < 0).all() and 0 in pool.retired
    assert pool.ref[pages].tolist() == [1, 1, 1] and pool.in_use() == 3 and pool.available() == 8 - 3
    with pytest.raises(ValueError, match="retired"):
        pool.detach(0)
    # other requests fill the pool, retire, and are all reclaimed: the detached pages are not touched
    pool.reserve(1, 3 * KV_PAGE)
    pool.reserve(2, 2 * KV_PAGE)
    pool.retire(1)
    pool.retire(2)
    pool.reserve(3, 5 * KV_PAGE)
    assert set(reclaimed) >= {1, 2} and pool.ref[pages].tolist() == [1, 1, 1]
    assert not set(pool.table[3, :5].tolist()) & set(pages)
    with pytest.raises(RuntimeError, match="kv_pages"):
        pool.reserve(0, 1 * KV_PAGE)  # 5 live + 3 detached pages: the pool is full, and the parked pages stay
    assert pool.ref[pages].tolist() == [1, 1, 1] and all(p not in pool.free for p in pages)
    pool.retire(0)
    pool.retire(3)
    pool.attach(1, row)  # another slot than it left
    assert pool.table[1, :3].tolist() == pages and 1 not in pool.retired and not pool.detached
    assert pool.ref[pages].tolist() == [1, 1, 1] and pool.available() == 8 - 3
    with pytest.raises(ValueError, match="detached row"):
        pool.attach(0, row)  # only once
    assert int(pool.ref.sum()) == int((pool.table >= 0).sum())  # every reference is a table entry again


def test_a_shared_prefix_stays_shared_through_detach_and_attach():
    pool, _ = _pool(pages=12)
    pool.reserve(0, 3 * KV_PAGE)
    pool.share(1, 0, 2)
    pool.reserve(1, 4 * KV_PAGE, start=2 * KV_PAGE)
    shared = pool.table[0, :2].tolist()
    assert pool.ref[shared].tolist() == [2, 2]
    row = pool.detach(1)
    assert pool.ref[shared].tolist() == [2, 2] and pool.available() == 12 - 5  # 3 of slot 0 + 2 private ones
    pool.reserve(2, 2 * KV_PAGE)  # slot 2 held nothing; the target of the attach below holds pages of its own
    pool.retire(2)
    held = pool.table[2, :2].tolist()
    pool.attach(2, row)
    assert pool.table[2, :2].tolist() == shared and pool.ref[shared].tolist() == [2, 2]
    assert all(p in pool.free for p in held)  # the slot's retired pages were released first
    pool.retire(0)
    pool.release(0)  # the donor goes: the resumed request still holds the prefix
    assert pool.ref[shared].tolist() == [1, 1] and all(p not in pool.free for p in shared)


def test_dropping_a_detached_row_frees_what_nobody_else_maps():
    pool, _ = _pool()
    pool.reserve(0, 2 * KV_PAGE)
    pool.share(1, 0, 1)
    pool.reserve(1, 3 * KV_PAGE, start=KV_PAGE)
    row = pool.detach(1)
    pool.drop(row)
    assert pool.in_use() == 2 and pool.ref[pool.table[0, :2]].tolist() == [1, 1] and pool.available() == 8 - 2
    with pytest.raises(ValueError):
        pool.drop(row)


# ---- the batcher with a fake engine and a fake clock -----------------------------------------------------------------
class _ParkingFakeEngine(_PagedFakeEngine):
    """_PagedFakeEngine whose tokens name the request (1000 * seed + frame), so that a request's result does not
    depend on the slots it ran in, with LmEngine's park / resume on the CPU buffers."""

    SAVED = ("slot_state", "slot_limit", "slot_temperature", "slot_top_p", "slot_top_k", "slot_seed", "n_out", "pos",
             "ras_window", "out_tokens")

    def __init__(self, slots, pages, **kw):
        super().__init__(slots, pages, **kw)
        self.log = []

    def _frame(self, s):
        b = self.bufs
        if int(b["slot_state"][s]) == 1:
            b["out_tokens"][s, :, int(b["n_out"][s])] = 1000 * int(b["slot_seed"][s]) + int(b["n_out"][s])
            tok = b["out_tokens"][s, :, int(b["n_out"][s])].clone()
            super()._frame(s)
            b["out_tokens"][s, :, int(b["n_out"][s]) - 1] = tok

    def park_slot(self, slot, ctx_len=0):
        self.log.append(("park", slot))
        blob = {k: self.bufs[k][slot].clone() for k in self.SAVED}
        self.bufs["slot_state"][slot] = 0
        self.bufs["pos"][slot] = -1
        return ParkedSlot(blob, self.kv_pool.detach(slot), None, None, ctx_len)

    def resume_slot(self, slot, parked):
        self.log.append(("resume", slot))
        assert int(self.bufs["slot_state"][slot]) == 0
        self.kv_pool.attach(slot, parked.row)
        for k, v in parked.blob.items():
            self.bufs[k][slot] = v

    def drop_parked(self, parked):
        self.log.append(("drop", None))
        self.kv_pool.drop(parked.row)


def _live_batcher(slots=2, max_live=4, pages=64, fpp=2, **kw):
    eng = _ParkingFakeEngine(slots, pages, kv_len=256, max_frames=64, max_rows=1024)
    clk = [0.0]
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=256), max_slots=slots, frames_per_poll=fpp, max_live=max_live,
                          clock=lambda: clk[0], **kw)
    return b, eng, clk


def _want(r, n):
    return [1000 * r.seed + f for f in range(n)]


def test_default_batcher_admits_and_retires_as_before():
    """pace=None everywhere and the default max_live: the scenario of test_engine_cpu's host-logic test."""
    eng = _FakeEngine(slots=2)
    b = ContinuousBatcher(_SchedModel(eng), max_slots=2, frames_per_poll=4)
    assert b.max_live == 2
    order = []
    mk = lambda T, n, tag: SlotRequest(prompt=torch.full((3, T), tag), max_new_tokens=n, tag=tag,
                                       on_done=lambda r: order.append(r.tag))
    reqs = [b.submit(mk(5, 3, 0)), b.submit(mk(7, 9, 1)), b.submit(mk(4, 1, 2)), b.submit(mk(6, 0, 3))]
    b.run()
    # admissions, retirements, frames and context bounds of the scheduler before it knew about pacing
    assert order == [0, 1, 2, 3] and eng.prefills == [[0, 1], [0], [0]] and [r.slot for r in reqs] == [0, 1, 0, 0]
    assert (b.frames_run, b.slot_frames) == (40, 48)
    assert eng.bounds == [9, 13, 13, 17, 8, 12, 16, 20, 24, 28, 32, 36, 40]
    assert all(r.parks == 0 and r.stream is None for r in reqs) and not b.parked
    eng2 = _FakeEngine(slots=2)
    b2 = ContinuousBatcher(_SchedModel(eng2), max_slots=2, frames_per_poll=2, min_free_to_admit=2)
    for tag, n in enumerate([2, 8, 4, 4]):
        b2.submit(mk(3, n, tag))
    b2.run()
    assert eng2.prefills == [[0, 1], [0, 1]]
    with pytest.raises(ValueError, match="max_live"):
        ContinuousBatcher(_SchedModel(_FakeEngine(slots=2)), max_slots=2, max_live=1)


def test_paced_requests_are_parked_and_resumed_with_their_frames_in_order():
    b, eng, clk = _live_batcher(slots=2, max_live=4)
    pieces = {i: [] for i in range(4)}
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 5 + i), i), max_new_tokens=40, seed=i + 1, tag=i, pace=1.0,
                                 on_frames=lambda r, c: pieces[r.tag].append(c.clone()))) for i in range(4)]
    unpaced = b.submit(SlotRequest(prompt=torch.full((3, 4), 9), max_new_tokens=30, seed=9))
    with pytest.raises(ValueError, match="pace"):
        b.submit(SlotRequest(prompt=torch.full((3, 4), 9), max_new_tokens=3, pace=0.0))
    live_peak = 0
    while not b.idle():
        b.step()
        clk[0] += 0.25  # a poll makes 2 frames and the listeners play a quarter of one
        live_peak = max(live_peak, len(b.active) + len(b.parked))
        assert len(b.active) <= 2 and eng.kv_pool.available() >= 0
    assert live_peak == 4 and not b.parked and not eng.kv_pool.detached
    assert sum(r.parks for r in reqs) >= 2 and all(r.parks == r.resumes for r in reqs) and unpaced.parks == 0
    assert ("park", 0) in eng.log and any(k == "resume" for k, _ in eng.log)
    for r in reqs + [unpaced]:
        T = r.prompt.size(1)
        assert r.error is None and r.result[0, T:].tolist() == _want(r, r._limit)
    for r in reqs:
        T = r.prompt.size(1)
        assert torch.equal(torch.cat(pieces[r.tag], dim=1), r.result[1:, T:-1])
        assert r.stream.frames == r._limit - 1
    b.close()


def test_chunks_of_one_stream_share_a_playback_clock():
    b, eng, clk = _live_batcher(slots=1, max_live=1)
    st = StreamClock()
    r1 = b.submit(SlotRequest(prompt=torch.zeros(3, 4, dtype=torch.long), max_new_tokens=7, seed=1, pace=2.0, stream=st))
    b.run()
    assert st.frames == 6 and st.t_first == 0.0
    clk[0] = 10.0
    r2 = b.submit(SlotRequest(prompt=torch.zeros(3, 9, dtype=torch.long), max_new_tokens=5, seed=2, pace=2.0, stream=st))
    assert r2.lead(10.0) == 6 - 2.0 * 10.0  # the utterance has been playing for 10 s: not a new arrival's lead of 0
    fresh = b.submit(SlotRequest(prompt=torch.zeros(3, 4, dtype=torch.long), max_new_tokens=5, seed=3, pace=2.0))
    assert fresh.lead(10.0) == 0.0 and fresh.lead(11.0) == -2.0
    b.run()
    assert st.frames == 6 + 4 and r1.done.is_set() and r2.done.is_set()


def test_cancel_in_each_state_fires_on_done_once():
    b, eng, clk = _live_batcher(slots=2, max_live=3)
    done = []
    mk = lambda i, **kw: SlotRequest(prompt=torch.full((3, 70), i), max_new_tokens=40, seed=i + 1, tag=i,
                                     on_done=lambda r: done.append(r.tag), **kw)
    r0, r1, r2, r3 = [b.submit(mk(i, pace=1.0)) for i in range(3)] + [b.submit(mk(3))]
    for _ in range(30):  # r0 and r1 run ahead, then one of them makes room for r2
        if b.parked:
            break
        b.step()
        clk[0] += 0.25
    (parked,) = b.parked
    survivor = r0 if parked is r1 else r1
    assert parked in (r0, r1) and parked._parked is not None and r2.slot >= 0 and r3.slot == -1
    free_before = eng.kv_pool.available()
    assert b.cancel(r3) and r3 not in b.waiting  # waiting
    slot = r2.slot
    assert b.cancel(r2) and slot not in b.active  # running: the slot idles, its pages become reclaimable
    assert int(eng.bufs["slot_state"][slot]) == 0 and int(eng.bufs["pos"][slot]) == -1
    assert slot in eng.kv_pool.retired and eng.kv_pool.available() == free_before + 2
    assert b.cancel(parked) and not b.parked and not eng.kv_pool.detached  # parked: its pages go back
    assert eng.kv_pool.available() == free_before + 4 and eng.log[-1] == ("drop", None)
    for r in (parked, r2, r3):
        assert isinstance(r.error, Cancelled) and r.done.is_set() and r.result is None
        assert not b.cancel(r)  # once
    assert sorted(done) == sorted([parked.tag, 2, 3])
    late = b.submit(mk(7))
    b.run()  # the freed slot and pages serve the next request; the survivor finishes untouched
    assert sorted(done) == sorted([parked.tag, 2, 3, survivor.tag, 7]) and late.slot == slot
    for r in (survivor, late):
        assert r.error is None and r.result[0, 70:].tolist() == _want(r, r._limit)


# ---- the worker loop -------------------------------------------------------------------------------------------------
class _CancellableBatcher(_FakeBatcher):
    max_slots = max_live = 3

    def __init__(self, slots, event_after):
        super().__init__(slots)
        self.steps, self.event_after, self.cancelled = 0, event_after, []

    def step(self):
        self.steps += 1
        super().step()
        for n, ev in self.event_after:
            if self.steps == n:
                ev.set()

    def cancel(self, r):
        self.cancelled.append(r)
        self.waiting = [x for x in self.waiting if x is not r]
        self.active = [e for e in self.active if e[0] is not r]
        r.error = Cancelled()
        r.on_done(r)


def _serve(texts, cancel_at):
    ev = {t: threading.Event() for t in cancel_at}
    fb = _CancellableBatcher(3, [(n, ev[t]) for t, n in cancel_at.items()])
    q, outs = Q.Queue(), {}
    for t in texts:
        outs[t] = Q.Queue()
        request = dict(text=t, chunks=2)
        if t in ev:
            request["cancel"] = ev[t]
        q.put(inf.GenerateRequest(request=request, response_queue=outs[t]))
    q.put(None)
    inf.serve_requests(_FakeModel(), q, 3, batcher=fb)
    got = {}
    for t, rq in outs.items():
        got[t] = []
        while not rq.empty():
            it = rq.get_nowait()
            got[t].append((it.status, it.response.action, getattr(it.response, "text", None)))
    return fb, got


def test_cancel_event_ends_a_plan_and_leaves_the_others_alone(monkeypatch):
    monkeypatch.setattr(inf, "_generate_long_plan", _fake_plan)
    texts = ["a", "bbbbbb", "ddd"]
    _, plain = _serve(texts, {})
    fb, got = _serve(texts, {"bbbbbb": 1})  # its listener leaves during chunk 0
    assert fb.closed and len(fb.cancelled) == 1 and fb.idle()
    assert got["bbbbbb"] == []  # no sample, no "next", no error
    assert got["a"] == plain["a"] and got["ddd"] == plain["ddd"]
    assert [a for _, a, _ in got["a"]] == ["sample", "sample", "next"]
    fb, got = _serve(texts, {"bbbbbb": 4})  # ... or between its chunks' ends: what was sent stays, nothing follows
    assert got["bbbbbb"] == plain["bbbbbb"][:len(got["bbbbbb"])] and ("success", "next", None) not in got["bbbbbb"]
    assert got["a"] == plain["a"] and got["ddd"] == plain["ddd"]
    # an event set after the request is over changes nothing
    _, got = _serve(texts, {"a": 50})
    assert got == plain


def test_one_at_a_time_worker_ignores_cancel_and_pacing_keys(monkeypatch):
    seen = {}
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (_FakeModel(), None))
    monkeypatch.setattr(inf, "generate_long", lambda **kw: seen.update(kw) or iter(()))
    monkeypatch.delenv("FSB_SERVE_SLOTS", raising=False)
    q = inf.launch_thread_safe_queue("x", "cpu", torch.bfloat16)
    rq = Q.Queue()
    q.put(inf.GenerateRequest(request=dict(text="t", cancel=threading.Event()), response_queue=rq))
    q.put(None)
    for _ in range(200):
        if "text" in seen:
            break
        threading.Event().wait(0.01)
    assert seen["text"] == "t" and "cancel" not in seen


def test_live_mode_paces_streaming_requests_only(monkeypatch):
    """FSB_SERVE_LIVE > slots: streaming requests carry the playback pace and one clock per plan; others do not."""
    monkeypatch.setattr(inf, "_generate_long_plan", _fake_plan)
    subs = []

    class _Rec(_FakeBatcher):
        max_slots, max_live = 3, 6

        def submit(self, r):
            subs.append(r)
            super().submit(r)

    q = Q.Queue()
    q.put(inf.GenerateRequest(request=dict(text="s", chunks=2, stream_frames=8), response_queue=Q.Queue()))
    q.put(inf.GenerateRequest(request=dict(text="p", chunks=1), response_queue=Q.Queue()))
    q.put(None)
    inf.serve_requests(_FakeModel(), q, 3, batcher=_Rec(3))
    s = [r for r in subs if r.on_frames is not None]
    assert len(s) == 2 and all(r.pace == pytest.approx(44100 / 2048) for r in s) and s[0].stream is s[1].stream
    assert [r.pace for r in subs if r.on_frames is None] == [None]
    subs.clear()
    _Rec.max_live = 3  # not live: as before
    q.put(inf.GenerateRequest(request=dict(text="s", chunks=1, stream_frames=8), response_queue=Q.Queue()))
    q.put(None)
    inf.serve_requests(_FakeModel(), q, 3, batcher=_Rec(3))
    assert [r.pace for r in subs] == [None]
