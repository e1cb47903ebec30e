"""Compact rows without a GPU (ContinuousBatcher(compact_rows=True)): the move policy (scheduler.compact_moves), the
row count each poll hands to the engine, FSB_SERVE_COMPACT, and a scheduler with the switch off that decides exactly
as before. The page bookkeeping and park / resume are LmEngine's own or their CPU twins; only device work is faked."""
import random

import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200 import scheduler as sched
from fish_speech_b200.scheduler import Cancelled, ContinuousBatcher, SlotRequest, StreamClock, compact_moves
from tests.test_engine_cpu import _SchedModel
from tests.test_kv_grow_cpu import _GrowFakeEngine, _check_pool


class _RowsFakeEngine(_GrowFakeEngine):
    """_GrowFakeEngine that records the row count of every decode call and checks it covers every live request."""

    def __init__(self, slots, pages, stop=None, **kw):
        super().__init__(slots, pages, stop, **kw)
        self.rows = []
        self.batcher = None

    def decode(self, batch, nframes, sp, use_graph=True):
        assert 1 <= batch <= self.max_batch
        if self.batcher is not None and self.batcher.compact_rows:
            assert batch == 1 + max(self.batcher.active), (batch, sorted(self.batcher.active))
        self.rows.append(batch)
        super().decode(batch, nframes, sp, use_graph)


def _batcher(slots=64, pages=4096, stop=None, kv_len=1024, fpp=4, **kw):
    eng = _RowsFakeEngine(slots, pages, stop, kv_len=kv_len, max_frames=kv_len, max_rows=1 << 16)
    b = ContinuousBatcher(_SchedModel(eng, max_seq_len=kv_len), max_slots=slots, frames_per_poll=fpp, **kw)
    eng.batcher = b
    return b, eng


def _want(r):
    return [1000 * r.seed + f for f in range(r.result.shape[1] - r.prompt.shape[1])]


def _got(r):
    return r.result[0, r.prompt.shape[1]:].tolist()


# ---- the policy function ---------------------------------------------------------------------------------------------
def test_compact_moves_only_when_everything_fits_below_the_tile():
    assert compact_moves([], list(range(64))) == []
    assert compact_moves([0, 1, 5], [2, 3, 4] + list(range(6, 64))) == []  # nothing above slot 31
    # the high ones, lowest first, into the lowest free slots below 32
    running = [0, 2, 40, 33, 63]
    free = [s for s in range(64) if s not in running]
    assert compact_moves(running, free) == [(33, 1), (40, 3), (63, 4)]
    # exactly 32 running: every slot below 32 ends up used
    running = list(range(1, 32)) + [50]
    free = [s for s in range(64) if s not in running]
    assert compact_moves(running, free) == [(50, 0)]
    # 33 running: they cannot all fit, nobody moves
    running = list(range(1, 32)) + [50, 60]
    assert compact_moves(running, [s for s in range(64) if s not in running]) == []
    # every move goes downward and to a slot that was free; the order of the inputs does not matter
    rnd = random.Random(5)
    for _ in range(200):
        k = rnd.randint(0, 40)
        running = rnd.sample(range(64), k)
        free = [s for s in range(64) if s not in running]
        rnd.shuffle(free)
        moves = compact_moves(running, free)
        assert all(to < 32 <= frm and to in free and frm in running for frm, to in moves)
        assert len({to for _, to in moves}) == len(moves)
        after = sorted([s for s in running if s not in {f for f, _ in moves}] + [t for _, t in moves])
        assert len(after) == k and (k > 32 or not after or after[-1] < 32)
    assert compact_moves([3, 20], [0, 1], rows=4) == [(20, 0)]


# ---- the row count of each poll --------------------------------------------------------------------------------------
def _ramp(b, rnd, n, seed0=1):
    """Requests of ragged prompts and budgets, submitted in waves so that load rises above 32 and falls back."""
    reqs = []
    for i in range(n):
        r = SlotRequest(prompt=torch.full((3, rnd.randint(1, 40)), i), max_new_tokens=rnd.randint(3, 60),
                        seed=seed0 + i)
        reqs.append(r)
    return reqs


def _run_waves(b, reqs, waves):
    k = 0
    for w in waves:
        for r in reqs[k:k + w]:
            b.submit(r)
        k += w
        for _ in range(3):
            b.step()
    while not b.idle():
        b.step()


@pytest.mark.parametrize("fpp", [1, 4, 8])
def test_step_decodes_rows_up_to_the_highest_live_slot_and_compacts(fpp):
    rnd = random.Random(fpp)
    b, eng = _batcher(fpp=fpp, compact_rows=True)
    reqs = _ramp(b, rnd, 90)
    _run_waves(b, reqs, [8, 30, 30, 0, 0, 22])
    b.close()
    assert all(r.error is None and _got(r) == _want(r) for r in reqs)
    assert max(eng.rows) > 32 and min(eng.rows) < 32  # load went above 32 rows and came back down
    assert b.moves == sum(r.moves for r in reqs) > 0
    assert all(r.parks == 0 and r.resumes == 0 for r in reqs)  # a move is not a park
    # a poll with at most 32 live requests never decodes more than 32 rows
    moves = [c for c in eng.calls if c[0] in ("park", "resume")]
    assert all(a[0] == "park" and a[1] >= 32 and c[0] == "resume" and c[1] < 32 for a, c in zip(moves[::2], moves[1::2]))


def test_the_row_count_follows_the_highest_slot_below_the_tile_too():
    """A 32-slot engine has one tile; the rows still shrink to the live ones, and nothing moves."""
    b, eng = _batcher(slots=8, fpp=2, compact_rows=True)
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 4), i), max_new_tokens=2 + 4 * i, seed=10 + i))
            for i in range(3)]
    b.run()
    b.close()
    assert set(eng.rows) == {3}  # slot 2 runs longest: the rows never shrink below it
    assert b.moves == 0 and all(_got(r) == _want(r) for r in reqs)
    b, eng = _batcher(slots=8, fpp=2, compact_rows=True)
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 4), i), max_new_tokens=14 - 4 * i, seed=10 + i))
            for i in range(3)]
    b.run()
    b.close()
    assert eng.rows == sorted(eng.rows, reverse=True) and eng.rows[0] == 3 and eng.rows[-1] == 1


# ---- composition -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(12))
def test_compaction_with_growth_parking_streaming_and_cancel(seed):
    """Seeded queues with every feature the scheduler composes with: pages granted as requests decode (a small pool, so
    some wait parked for pages), paced streams parked and resumed (max_live), shared prefixes, streamed frames and
    cancels. Every request that is not cancelled returns its own tokens, streamed frames arrive in order, and pages
    are conserved after every poll."""
    rnd = random.Random(seed)
    slots = rnd.choice([34, 48, 64])
    growth = seed % 2 == 0
    paced = seed % 3 == 0
    clk = [0.0]
    kw = dict(kv_growth=growth, max_live=slots + 16 if paced else None, clock=lambda: clk[0])
    pages = rnd.choice([60, 120, 400]) if growth else 4096
    b, eng = _batcher(slots=slots, pages=pages, kv_len=512, fpp=rnd.choice([2, 4, 8]), compact_rows=True, **kw)
    prefix = torch.arange(130).repeat(3, 1) + 7
    reqs, streamed = [], {}
    for i in range(rnd.randint(50, 90)):
        T = rnd.randint(1, 100)
        p = torch.cat([prefix[:, :T], torch.full((3, rnd.randint(1, 20)), i)], 1) if rnd.random() < 0.3 else \
            torch.full((3, T), i)
        r = SlotRequest(prompt=p, max_new_tokens=rnd.randint(2, 120), seed=i + 1, reuse_prefix=rnd.random() < 0.3,
                        on_frames=lambda r, c: streamed.setdefault(id(r), []).extend(c[0].tolist()))
        if paced and rnd.random() < 0.5:
            r.pace, r.stream = 40.0, StreamClock()
        reqs.append(r)
    pending = list(reqs)
    cancelled = set()
    while pending or not b.idle():
        for _ in range(rnd.randint(0, 12)):
            if pending:
                b.submit(pending.pop(0))
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
        assert streamed.get(id(r), []) == _want(r)[:-1]
    assert b.moves > 0


# ---- the switch off --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_switch_off_decides_exactly_as_before(seed):
    """compact_rows=False is the default and changes nothing: the same engine calls (prefills, slots, decodes of all
    max_slots rows, parks) as a batcher built without the argument, and no request is moved."""
    def run(**kw):
        rnd = random.Random(seed)
        b, eng = _batcher(slots=48, pages=rnd.choice([80, 4096]), kv_len=512, fpp=4,
                          kv_growth=seed % 2 == 0, **kw)
        reqs = _ramp(b, rnd, 70)
        _run_waves(b, reqs, [6, 30, 20, 0, 14])
        b.close()
        return eng, reqs, b

    eng0, reqs0, b0 = run()
    eng1, reqs1, b1 = run(compact_rows=False)
    assert not b0.compact_rows and eng0.calls == eng1.calls and eng0.rows == eng1.rows
    assert all(n == 48 for n in eng0.rows) and b0.moves == b1.moves == 0
    assert [r.slot for r in reqs0] == [r.slot for r in reqs1] and all(r.moves == 0 for r in reqs0 + reqs1)
    eng2, reqs2, b2 = run(compact_rows=True)  # on: other slots and rows, the same tokens
    assert [_got(r) for r in reqs2] == [_got(r) for r in reqs0] and b2.moves > 0 and min(eng2.rows) < 48


# ---- FSB_SERVE_COMPACT -----------------------------------------------------------------------------------------------
def test_serve_compact_parsing():
    assert inf.serve_compact(None) is False
    for v in ("", " ", "0", " 0 "):
        assert inf.serve_compact(v) is False
    assert inf.serve_compact("1") is True and inf.serve_compact(" 1") is True
    for v in ("2", "yes", "true", "-1", "1.0", "on"):
        with pytest.raises(ValueError, match="FSB_SERVE_COMPACT"):
            inf.serve_compact(v)


def test_launch_refuses_a_bad_compact_value_before_loading_anything(monkeypatch):
    monkeypatch.setenv("FSB_SERVE_COMPACT", "yes")
    monkeypatch.delenv("FSB_SERVE_KV_GROW", raising=False)
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: pytest.fail("the model was loaded"))
    with pytest.raises(ValueError, match="FSB_SERVE_COMPACT='yes'"):
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
        monkeypatch.delenv("FSB_SERVE_COMPACT", raising=False)
    else:
        monkeypatch.setenv("FSB_SERVE_COMPACT", value)
    monkeypatch.delenv("FSB_SERVE_KV_GROW", raising=False)
    with pytest.raises(_Stop):
        inf.serve_requests(object(), None, 48)
    assert seen["compact_rows"] is want and seen["max_slots"] == 48
