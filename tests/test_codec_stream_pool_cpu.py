"""Host side of the shared streaming-decode pool (no GPU): CodecStreamWorker coalescing, ordering, error delivery and
the fall-back to a private stream, and TTSInferenceEngine with FSB_STREAM_POOL, with the device work replaced by a
stand-in pool whose sample values are the absolute frame index of each stream."""
import queue
import threading

import numpy as np
import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from fish_speech_b200.inference_engine import CodecStreamWorker, TTSInferenceEngine, _ChunkAudio
from fish_speech_b200.inference_engine.schema import ServeTTSRequest
from fish_speech_b200.models.dac.modded_dac import DAC

FL = 2048


class _FakePool:
    def __init__(self, slots=4, k_max=32, gate=None, fail_on=None):
        self.slots, self.k_max = slots, k_max
        self.live = [False] * slots
        self.pos = [0] * slots
        self.calls = []  # {slot: frames} of every push
        self.gate = gate  # threading.Event the first push waits for
        self.fail_on = fail_on  # a push that contains this slot raises

    def open(self):
        for s in range(self.slots):
            if not self.live[s]:
                self.live[s], self.pos[s] = True, 0
                return s
        raise ValueError("full")

    def close(self, slot):
        if not self.live[slot]:
            raise ValueError("closed")
        self.live[slot] = False

    def push(self, pieces):
        if self.gate is not None and not self.calls:
            self.calls.append({s: c.shape[-1] for s, c in pieces.items()})
            assert self.gate.wait(10)
        else:
            self.calls.append({s: c.shape[-1] for s, c in pieces.items()})
        if self.fail_on is not None and self.fail_on in pieces:
            raise RuntimeError("codec failed")
        out = {}
        for s, c in pieces.items():
            k = c.shape[-1]
            if not self.live[s] or k > self.k_max:
                raise ValueError("bad push")
            out[s] = torch.arange(self.pos[s], self.pos[s] + k, dtype=torch.float32).repeat_interleave(FL)
            self.pos[s] += k
        return out


def _codes(k):
    return torch.zeros(10, k, dtype=torch.long)


def _frames(wav):
    return list(wav[::FL].astype(int))


def test_pieces_from_several_threads_share_one_push_and_come_back_to_their_caller():
    gate = threading.Event()
    pool = _FakePool(slots=4, gate=gate)
    w = CodecStreamWorker(pool)
    slots = [w.open() for _ in range(4)]
    first = w.submit(slots[0], _codes(2))  # the worker blocks inside this push
    while not pool.calls:
        pass
    results = {}

    def caller(s, k):
        results[s] = w.decode(s, _codes(k))

    ts = [threading.Thread(target=caller, args=(s, k)) for s, k in zip(slots[1:], (3, 5, 7))]
    for t in ts:
        t.start()
    while w._q.qsize() < 3:
        pass
    gate.set()
    for t in ts:
        t.join(10)
    assert _frames(first.result(10)) == [0, 1]
    assert pool.calls[1] == {slots[1]: 3, slots[2]: 5, slots[3]: 7}  # one push for all three callers
    for s, k in zip(slots[1:], (3, 5, 7)):
        assert _frames(results[s]) == list(range(k))
    assert w.pushes == 2


def test_queued_pieces_of_one_stream_keep_their_order_and_respect_k_max():
    gate = threading.Event()
    pool = _FakePool(slots=2, k_max=8, gate=gate)
    w = CodecStreamWorker(pool)
    a, b = w.open(), w.open()
    blocker = w.submit(b, _codes(1))
    while not pool.calls:
        pass
    futs = [w.submit(a, _codes(k)) for k in (3, 4, 2, 8)]
    gate.set()
    got = [f.result(10) for f in futs]
    blocker.result(10)
    assert [_frames(x) for x in got] == [[0, 1, 2], [3, 4, 5, 6], [7, 8], list(range(9, 17))]
    # 3 + 4 fit one push of at most 8 frames; 2 and 8 need one push each
    assert [c.get(a) for c in pool.calls[1:]] == [7, 2, 8]
    with pytest.raises(ValueError):
        w.submit(a, _codes(9))
    assert _frames(w.decode(a, _codes(19))) == list(range(17, 36))  # split into pieces of k_max


def test_a_failing_push_errors_every_waiter_and_the_worker_survives():
    gate = threading.Event()
    pool = _FakePool(slots=3, gate=gate, fail_on=2)
    w = CodecStreamWorker(pool)
    s = [w.open() for _ in range(3)]
    blocker = w.submit(s[0], _codes(1))
    while not pool.calls:
        pass
    f1, f2 = w.submit(s[1], _codes(2)), w.submit(s[2], _codes(3))
    gate.set()
    blocker.result(10)
    for f in (f1, f2):
        with pytest.raises(RuntimeError, match="codec failed"):
            f.result(10)
    pool.fail_on = None
    assert _frames(w.decode(s[1], _codes(2))) == [0, 1]


def _fake_dac(pool_slots=None):
    d = object.__new__(DAC)
    d.sample_rate = 44100
    d._device = torch.device("cpu")
    d.from_indices = lambda codes: torch.full((codes.shape[0], 1, codes.shape[-1] * FL), 0.25)
    d.streams_opened = 0

    class _Stream:
        def __init__(self):
            self.pos = 0

        def push(self, codes):
            k = codes.shape[-1]
            out = torch.arange(self.pos, self.pos + k, dtype=torch.float32).repeat_interleave(FL).view(1, 1, -1)
            self.pos += k
            return out

    def open_decode_stream(batch=1, max_frames=4096):
        d.streams_opened += 1
        return _Stream()

    d.open_decode_stream = open_decode_stream
    d.pools = []

    def open_stream_pool(slots, k_max=32, **kw):
        d.pools.append(_FakePool(slots=slots, k_max=k_max))
        return d.pools[-1]

    d.open_stream_pool = open_stream_pool
    return d


def test_a_full_pool_falls_back_to_a_private_stream(monkeypatch):
    monkeypatch.setenv("FSB_STREAM_POOL", "1")
    dac = _fake_dac()
    eng = TTSInferenceEngine(queue.Queue(), dac, torch.bfloat16, compile=False)
    a, b = _ChunkAudio(eng), _ChunkAudio(eng)
    assert _frames(a.push_partial(_codes(3))) == [0, 1, 2] and a.slot == 0
    assert _frames(b.push_partial(_codes(2))) == [0, 1] and b.slot is None and dac.streams_opened == 1
    assert _frames(a.push_partial(_codes(2))) == [3, 4]
    a.finish(_codes(5))
    assert dac.pools[0].live == [False]  # the chunk's slot is closed when the chunk ends
    c = _ChunkAudio(eng)
    c.push_partial(_codes(1))
    assert c.slot == 0  # and reused


def _run_streaming_request(monkeypatch, pool):
    if pool:
        monkeypatch.setenv("FSB_STREAM_POOL", "4")
    else:
        monkeypatch.delenv("FSB_STREAM_POOL", raising=False)

    def serve(q):
        item = q.get()
        put = lambda a, n=0: item.response_queue.put(inf.WrappedGenerateResponse(
            status="success", response=inf.GenerateResponse(action=a, codes=_codes(n) if n else None)))
        put("partial", 8)
        put("partial", 5)
        put("sample", 15)
        put("partial", 40)  # more than one push of k_max frames
        put("sample", 41)
        put("sample", 4)
        put("next")

    q = queue.Queue()
    threading.Thread(target=serve, args=(q,), daemon=True).start()
    dac = _fake_dac()
    eng = TTSInferenceEngine(q, dac, torch.bfloat16, compile=False)
    res = list(eng.inference(ServeTTSRequest(text="hi", streaming=True)))
    return res, dac


def test_engine_with_a_stream_pool_yields_the_same_segments(monkeypatch):
    plain, d0 = _run_streaming_request(monkeypatch, pool=False)
    pooled, d1 = _run_streaming_request(monkeypatch, pool=True)
    assert d0.pools == [] and d0.streams_opened == 2
    assert len(d1.pools) == 1 and d1.streams_opened == 0 and len(d1.pools[0].calls) >= 5
    assert [r.code for r in pooled] == [r.code for r in plain] == ["header"] + ["segment"] * 6 + ["final"]
    for a, b in zip(plain[1:], pooled[1:]):
        assert np.array_equal(a.audio[1], b.audio[1])
    assert d1.pools[0].live == [False] * 4


def test_a_failure_while_grouping_errors_the_round_and_close_stops_the_worker():
    gate = threading.Event()
    pool = _FakePool(slots=2, gate=gate)
    w = CodecStreamWorker(pool)
    a, b = w.open(), w.open()
    blocker = w.submit(b, _codes(1))
    while not pool.calls:
        pass
    f1 = w.submit(a, _codes(2))
    f2 = w.submit(a, torch.zeros(9, 1, dtype=torch.long))  # cannot be joined with the piece before it
    gate.set()
    blocker.result(10)
    for f in (f1, f2):
        with pytest.raises(RuntimeError):
            f.result(10)
    assert _frames(w.decode(b, _codes(2))) == [1, 2]  # the worker survived
    w.release(a)
    w.close()
    assert not w._thread.is_alive()
