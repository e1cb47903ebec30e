"""Host side of the 64-slot engine (no GPU): the row-tile rule, the scheduler at 64 slots with the fake engine of
test_engine_cpu.py, the FSB_SERVE_SLOTS clamp and the slow-KV memory check of the serving worker."""
import time

import pytest
import torch

import fish_speech_b200.models.text2semantic.inference as inf
from tests.test_engine_cpu import _FakeEngine, _FakeModel, _SchedModel


def test_row_tile_follows_the_engine_size():
    from fish_speech_b200.engine import MAX_DECODE_BATCH, decode_row_tile

    assert MAX_DECODE_BATCH == 64
    assert [decode_row_tile(n) for n in (1, 2, 31, 32, 33, 47, 64)] == [32, 32, 32, 32, 64, 64, 64]


class _FakeEngine64(_FakeEngine):
    def __init__(self, slots, **kw):
        super().__init__(slots, **kw)
        self.bufs["pos"] = torch.zeros(64, dtype=torch.int32)  # the decode state has the 64-row tile


def test_continuous_batcher_host_logic_at_64_slots():
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    eng = _FakeEngine64(slots=64, max_rows=1024)  # room to prefill every slot in one pass
    b = ContinuousBatcher(_SchedModel(eng), max_slots=64, frames_per_poll=4)
    done = []
    reqs = [b.submit(SlotRequest(prompt=torch.full((3, 3 + i % 5), i), max_new_tokens=1 + i % 11, tag=i,
                                 on_done=lambda r: done.append(r.tag))) for i in range(100)]
    b.run()
    assert b.idle() and sorted(done) == list(range(100))
    assert eng.prefills[0] == list(range(64))  # every slot filled at once
    assert sum(len(p) for p in eng.prefills) == 100
    assert max(r.slot for r in reqs) == 63
    for r in reqs:
        T, n = r.prompt.size(1), 1 + r.tag % 11
        assert r.result.shape == (3, T + n) and r.result[0, T:].tolist() == [100 * r.slot + f for f in range(n)]
    b.close()
    with pytest.raises(ValueError, match="max_slots"):
        ContinuousBatcher(_SchedModel(_FakeEngine64(slots=64)), max_slots=65)


def test_generate_batch_rejects_more_than_64_prompts():
    with pytest.raises(ValueError, match="1..64"):
        inf.generate_batch(model=_FakeModel(), prompts=[torch.zeros(3, 4, dtype=torch.long)] * 65, max_new_tokens=1)


class _S2ProSizedModel(_FakeModel):
    class config:
        max_seq_len = 32768
        n_layer, n_local_heads, head_dim = 36, 8, 128


def test_slow_kv_memory_check():
    cfg = _S2ProSizedModel.config
    assert inf.slow_kv_bytes_per_position(cfg) == 147456
    inf.check_serve_kv_fits(64, 8192, cfg, 80 * 10 ** 9)  # 77.3 GB fits in 80
    with pytest.raises(ValueError, match="FSB_SERVE_KV_LEN"):
        inf.check_serve_kv_fits(64, 8192, cfg, 70 * 10 ** 9)
    inf.check_serve_kv_fits(64, 4096, cfg, 70 * 10 ** 9)


def test_serve_slots_clamp_to_64_and_kv_check(monkeypatch):
    seen = []
    monkeypatch.setattr(inf, "init_model", lambda *a, **k: (_S2ProSizedModel(), inf.decode_one_token_ar))
    monkeypatch.setattr(inf, "serve_requests", lambda model, q, slots: seen.append((slots, model.caches)))
    monkeypatch.setenv("FSB_SERVE_SLOTS", "100")
    monkeypatch.setenv("FSB_SERVE_KV_LEN", "1024")
    inf.launch_thread_safe_queue("ckpt", "cpu", torch.bfloat16)
    for _ in range(200):
        if seen:
            break
        time.sleep(0.01)
    assert seen and seen[0][0] == 64 and seen[0][1]["max_batch_size"] == 64 and seen[0][1]["max_seq_len"] == 1024

    # on a CUDA device the worker first checks that the slots' slow KV caches fit in free memory
    monkeypatch.setenv("FSB_SERVE_SLOTS", "64")
    monkeypatch.setenv("FSB_SERVE_KV_LEN", "8192")
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (40 * 10 ** 9, 80 * 10 ** 9))
    with pytest.raises(ValueError, match="FSB_SERVE_KV_LEN"):
        inf.launch_thread_safe_queue("ckpt", "cuda", torch.bfloat16)
    assert len(seen) == 1
