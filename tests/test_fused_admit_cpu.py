"""Fused admission without a GPU (ContinuousBatcher(fused_admission=True)): the engine calls with the mode on, a
scheduler with the mode off that decides exactly as before, no request moved or parked before its first frame, and
FSB_SERVE_FUSED_ADMIT. The page bookkeeping and park / resume are LmEngine's own or their CPU twins; only device work is
faked, with the rules of fsb_lm_prefill_deferred: a deferred slot idles at position -1 and the next decode's first frame
makes its frame 0."""
import random

import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200 import scheduler as sched
from fish_speech_b200.scheduler import Cancelled, ContinuousBatcher, SlotRequest, StreamClock
from tests.test_decode_rows_cpu import _RowsFakeEngine, _got, _ramp, _run_waves, _want
from tests.test_engine_cpu import _SchedModel
from tests.test_kv_grow_cpu import _check_pool


class _FusedFakeEngine(_RowsFakeEngine):
    """_RowsFakeEngine whose prefill can defer the first frames: the slots are marked pending at position -1, and the
    first frame of the next decode makes their frame 0 (position = prompt end) beside the running rows. Parking or
    moving a pending slot, or a decode whose rows miss one, fails as fsb_lm_slot_save / fsb_lm_decode do."""

    def __init__(self, slots, pages, stop=None, **kw):
        super().__init__(slots, pages, stop, **kw)
        self.pending = {}  # slot -> position of its last prompt row

    def prefill(self, prompts, slots, sp, start_pos=None, do_sample=True, kv_end=None, defer_first_frame=False):
        if not defer_first_frame:
            return super().prefill(prompts, slots, sp, start_pos, do_sample, kv_end)
        start_pos = start_pos or [0] * len(prompts)
        self.calls.append(("prefill_deferred", list(slots), list(kv_end)))
        for s, s0 in zip(slots, start_pos):
            if s0 == 0:
                self._slot_tokens.pop(int(s), None)
        self._reserve([(s, max(s0 + p.shape[1], e), s0) for p, s, s0, e in zip(prompts, slots, start_pos, kv_end)])
        self.prefills.append(list(slots))
        for p, s, s0 in zip(prompts, slots, start_pos):
            self.pending[int(s)] = s0 + p.shape[1] - 1
            self.bufs["pos"][s] = -1

    def decode(self, batch, nframes, sp, use_graph=True):
        if self.pending and nframes >= 1:
            assert max(self.pending) < batch, (sorted(self.pending), batch)
            b = self.bufs
            for s, last in self.pending.items():
                if int(b["slot_state"][s]) == 1:  # a vacated slot is dropped, as the splice kernel does
                    b["pos"][s] = last
            live = {s for s in self.pending if int(b["slot_state"][s]) == 1}
            self.pending = {}
            self.calls.append(("fused_frame", sorted(live)))
            # the first frame: every live row, the new ones from their prompt end (as _GrowFakeEngine.decode)
            super().decode(batch, 1, sp, use_graph)
            nframes -= 1
        if nframes:
            super().decode(batch, nframes, sp, use_graph)

    def park_slot(self, slot, ctx_len=0):
        assert slot not in self.pending, f"slot {slot} parked before its first frame"
        return super().park_slot(slot, ctx_len)


def _batcher(slots=64, pages=4096, stop=None, kv_len=1024, fpp=4, **kw):
    eng = _FusedFakeEngine(slots, pages, stop, kv_len=kv_len, max_frames=kv_len, max_rows=1 << 16)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=kv_len), max_slots=slots, frames_per_poll=fpp, **kw)
    eng.batcher = b
    return b, eng


def test_call_sequence_with_the_mode_on():
    """Admissions prefill deferred, the poll's first decode frame serves them, and a request makes frames_per_poll
    frames in its first poll (not one more)."""
    b, eng = _batcher(slots=4, fpp=3, fused_admission=True)
    r0 = b.submit(SlotRequest(prompt=torch.full((3, 5), 0), max_new_tokens=7, seed=1))
    r1 = b.submit(SlotRequest(prompt=torch.full((3, 9), 1), max_new_tokens=1, seed=2))
    b.step()
    calls = [c for c in eng.calls if c[0] != "reserve"]
    assert [c[0] for c in calls] == ["prefill_deferred", "fused_frame", "decode", "decode"], calls
    assert calls[2:] == [("decode", 1), ("decode", 2)]  # the fused frame, then the poll's other frames
    assert ("prefill_deferred", [0, 1], [5 + 7, 9 + 1]) in eng.calls
    assert eng.calls[[c[0] for c in eng.calls].index("fused_frame")] == ("fused_frame", [0, 1])
    assert int(eng.bufs["n_out"][0]) == 3 and r1.done.is_set() and _got(r1) == _want(r1) == [2000]
    r2 = b.submit(SlotRequest(prompt=torch.full((3, 4), 2), max_new_tokens=5, seed=3))
    b.run()
    b.close()
    assert all(r.error is None and _got(r) == _want(r) for r in (r0, r1, r2))
    assert not any(c[0] == "prefill" for c in eng.calls)
    assert b._pending == set() and eng.pending == {}


@pytest.mark.parametrize("seed", range(6))
def test_switch_off_decides_exactly_as_before(seed):
    """fused_admission=False is the default and changes nothing: the same engine calls as a batcher built without the
    argument, and no prefill is deferred. On: the same tokens, in fewer frames."""
    def run(**kw):
        rnd = random.Random(seed)
        b, eng = _batcher(slots=48, pages=rnd.choice([80, 4096]), kv_len=512, fpp=4, kv_growth=seed % 2 == 0,
                          compact_rows=seed % 3 == 0, **kw)
        reqs = _ramp(b, rnd, 70)
        _run_waves(b, reqs, [6, 30, 20, 0, 14])
        b.close()
        return eng, reqs, b

    eng0, reqs0, b0 = run()
    eng1, reqs1, b1 = run(fused_admission=False)
    assert not b0.fused_admission and eng0.calls == eng1.calls and eng0.rows == eng1.rows
    assert not any(c[0] in ("prefill_deferred", "fused_frame") for c in eng0.calls)
    assert [r.slot for r in reqs0] == [r.slot for r in reqs1]
    eng2, reqs2, b2 = run(fused_admission=True)
    assert [_got(r) for r in reqs2] == [_got(r) for r in reqs0]
    assert any(c[0] == "fused_frame" for c in eng2.calls) and not any(c[0] == "prefill" for c in eng2.calls)
    assert b2.frames_run <= b0.frames_run


@pytest.mark.parametrize("seed", range(16))
def test_no_pending_row_is_moved_or_parked(seed):
    """Seeded queues with compaction, page growth from a small pool (requests parked for pages), paced streams and
    cancels, the mode on. The fake engine fails a park or move of a pending slot; every request returns its own
    tokens and pages are conserved."""
    rnd = random.Random(seed)
    slots = rnd.choice([34, 48, 64])
    growth = seed % 2 == 0
    paced = seed % 4 < 2
    clk = [0.0]
    kw = dict(kv_growth=growth, max_live=slots + 16 if paced else None, clock=lambda: clk[0])
    b, eng = _batcher(slots=slots, pages=rnd.choice([60, 120]) if growth else 4096, kv_len=512,
                      fpp=rnd.choice([2, 4, 8]), compact_rows=True, fused_admission=True, **kw)
    reqs, cancelled = [], set()
    for i in range(rnd.randint(50, 90)):
        r = SlotRequest(prompt=torch.full((3, rnd.randint(1, 100)), i), max_new_tokens=rnd.randint(1, 120), seed=i + 1)
        if paced and rnd.random() < 0.5:
            r.pace, r.stream = 40.0, StreamClock()
        reqs.append(r)
    todo = list(reqs)
    while todo or not b.idle():
        for _ in range(rnd.randint(0, 12)):
            if todo:
                b.submit(todo.pop(0))
        if rnd.random() < 0.1:
            live = [r for r in reqs if not r.done.is_set() and (r.slot >= 0 or r._parked is not None)]
            if live:
                v = rnd.choice(live)
                assert b.cancel(v)
                cancelled.add(id(v))
        b.step()
        clk[0] += 0.05
        if growth:
            _check_pool(b, eng)
    b.close()
    for r in reqs:
        if id(r) in cancelled:
            assert isinstance(r.error, Cancelled)
            continue
        assert r.error is None and _got(r) == _want(r), f"request {r.seed}"


def test_a_pending_row_above_32_is_not_moved_when_growth_parks_requests_below_it():
    """The reachable case: kv_growth parks running requests for pages after an admission, which frees slots below 32;
    compaction would then move the new request above 32 down before its first frame. It stays and runs its first frame
    there; the compaction of that poll moves nobody else's request into a pending slot either."""
    b, eng = _batcher(slots=48, pages=10 ** 6, kv_len=512, fpp=4, kv_growth=True, compact_rows=True,
                      fused_admission=True, max_live=96)
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 8), i), max_new_tokens=200, seed=i + 1)) for i in range(40)]
    b.step()
    assert len(b.active) == 40
    new = b.submit(SlotRequest(prompt=torch.full((3, 8), 99), max_new_tokens=30, seed=100))
    parked_for_pages = [b.active[s] for s in range(30)]
    real_grow = b._grow

    def grow():  # pages run short for 30 requests below slot 32 right after the admission
        for r in parked_for_pages:
            b._park(r)
            b._to_short(r)
        return real_grow()

    b._grow = grow
    b.step()
    b._grow = real_grow
    assert new.slot == 40 and new.moves == 0, (new.slot, new.moves)  # 40 is the lowest free slot at admission
    assert len(b.active) <= 32 and int(eng.bufs["n_out"][40]) == 4
    b.run()
    b.close()
    assert all(r.error is None and _got(r) == _want(r) for r in reqs + [new])


# ---- FSB_SERVE_FUSED_ADMIT -------------------------------------------------------------------------------------------
def test_serve_fused_admit_parsing():
    assert inf.serve_fused_admit(None) is False
    for v in ("", " ", "0", " 0 "):
        assert inf.serve_fused_admit(v) is False
    assert inf.serve_fused_admit("1") is True and inf.serve_fused_admit(" 1 ") is True
    for v in ("2", "yes", "true", "-1", "1.0", "on"):
        with pytest.raises(ValueError, match="FSB_SERVE_FUSED_ADMIT"):
            inf.serve_fused_admit(v)


def test_launch_refuses_a_bad_fused_admit_value_before_loading_anything(monkeypatch):
    monkeypatch.setenv("FSB_SERVE_FUSED_ADMIT", "yes")
    monkeypatch.delenv("FSB_SERVE_KV_GROW", raising=False)
    monkeypatch.delenv("FSB_SERVE_COMPACT", raising=False)
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: pytest.fail("the model was loaded"))
    with pytest.raises(ValueError, match="FSB_SERVE_FUSED_ADMIT='yes'"):
        inf.launch_thread_safe_queue("nowhere", "cpu", torch.bfloat16)


@pytest.mark.parametrize("value,want", [(None, False), ("0", False), ("1", True)])
def test_serve_requests_passes_the_switch_to_the_batcher(monkeypatch, value, want):
    seen = {}

    class _Stop(Exception):
        pass

    class _Batcher:
        def __init__(self, model, **kw):
            seen.update(kw)
            raise _Stop

    monkeypatch.setattr(sched, "ContinuousBatcher", _Batcher)
    if value is None:
        monkeypatch.delenv("FSB_SERVE_FUSED_ADMIT", raising=False)
    else:
        monkeypatch.setenv("FSB_SERVE_FUSED_ADMIT", value)
    monkeypatch.delenv("FSB_SERVE_KV_GROW", raising=False)
    monkeypatch.delenv("FSB_SERVE_COMPACT", raising=False)
    with pytest.raises(_Stop):
        inf.serve_requests(object(), None, 48)
    assert seen["fused_admission"] is want and seen["max_slots"] == 48
