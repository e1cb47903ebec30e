"""Parking and resuming requests between frames on the GPU (fsb_lm_slot_save / fsb_lm_slot_restore, LmEngine.park_slot /
resume_slot, the pacing policy of scheduler.ContinuousBatcher).

The contract is the scheduler's: a request returns EXACTLY the tokens `generate` returns for it alone, however often it
was taken out of its slot, whichever slots it continued in, and whatever its neighbours did meanwhile."""
import pytest
import torch

from fish_speech_b200.engine import kv_pages_for
from oracle import lm_oracle as O
from tests.lm_util import make_prompt
from tests.test_paged_kv_gpu import _paged_model, _s2pro_model, _s2pro_prompt, _s2pro_small
from tests.test_scheduler_gpu import _alone, _grown_prompt

pytestmark = pytest.mark.gpu

GREEDY = dict(temperature=0.7, top_p=0.7, top_k=1)
SAMPLED = dict(temperature=0.9, top_p=0.9, top_k=30)
_models = {}


def _tiny(rows, kv_pages=None, max_seq_len=128, seed=77):
    """One tiny model per engine size; <|im_end|> is never sampled, so every request runs to its budget."""
    key = (rows, kv_pages, max_seq_len, seed)
    if kv_pages is None:  # parked requests keep their pages: room for eight of them beside the slots
        kv_pages = (rows + 8) * kv_pages_for(max_seq_len)
    if key not in _models:
        cfg = O.tiny_config(max_seq_len=max_seq_len)
        w = O.make_weights(cfg, seed=seed, head_gain=2.5)
        w["embeddings.weight"][cfg.im_end_id] = 0
        _models[key] = (cfg, _paged_model(cfg, w, kv_pages=kv_pages, max_batch=rows))
    return _models[key]


def _submit(b, prompt, n, seed, kw, **extra):
    from fish_speech_b200.scheduler import SlotRequest

    return b.submit(SlotRequest(prompt=prompt.cuda(), max_new_tokens=n, seed=seed, **kw, **extra))


def _park_and_resume_elsewhere(model, probe, k, others, spoil_ras=False, frames_per_poll=1):
    """Run `probe` = (prompt, n, seed, kw) in slot 0 of three for k frames, park it, hand slot 0 to another request, and
    resume it in slot 1 once that slot's short request is done. others: three (prompt, n, seed, kw);
    the first one's budget decides how long the probe stays parked. Returns (probe request, other requests, window)."""
    from fish_speech_b200.scheduler import ContinuousBatcher

    b = ContinuousBatcher(model, max_slots=3, frames_per_poll=frames_per_poll, max_live=4)
    eng = model.engine
    r = _submit(b, *probe)
    short, long_ = _submit(b, *others[0]), _submit(b, *others[1])
    b._schedule()  # the prefill: frame 1 of all three
    for _ in range(k - 1):
        b.step()
    assert (r.slot, short.slot, long_.slot) == (0, 1, 2) and not r.done.is_set()
    assert int(eng.buffer("n_out")[0]) == k
    b._park(r)
    b.parked.remove(r)  # held back by hand: the policy would give an unpaced request the first free slot
    assert int(eng.buffer("slot_state")[0]) == 0 and int(eng.buffer("pos")[0]) == -1
    late = _submit(b, *others[2])
    while not short.done.is_set():
        b.step()
    b.parked.append(r)
    b.step()  # resumes it in the slot that has just become free, and runs one frame
    window = eng.buffer("ras_window")[r.slot].cpu().tolist()
    if spoil_ras:
        eng.buffer("ras_window")[r.slot] = 0
    b.run()
    b.close()
    assert late.slot == 0 and r.slot == 1 and (r.parks, r.resumes) == (1, 1)
    return r, [short, long_, late], window


def _others(cfg, k, kw):
    return [(make_prompt(cfg, 301, 9), k + 3, 11, kw), (make_prompt(cfg, 302, 17), 40, 12, kw),
            (make_prompt(cfg, 303, 6), 30, 13, kw)]


@pytest.mark.parametrize("rows", [3, 40], ids=["rows32", "rows64"])
@pytest.mark.parametrize("kw", [GREEDY, SAMPLED], ids=["greedy", "sampled"])
@pytest.mark.parametrize("k", [1, 12, 23], ids=["after1", "mid", "last"])
def test_parked_request_resumes_in_another_slot_with_the_same_tokens(rows, kw, k):
    cfg, model = _tiny(rows)
    assert model.engine.row_tile == (32 if rows <= 32 else 64)
    T, n = 11, 24
    probe = (make_prompt(cfg, 300, T), n, 4242, kw)
    others = _others(cfg, k, kw)
    solo = _alone(model, probe[0], n, seed=probe[2], **kw)
    solo_others = [_alone(model, p, m, seed=s, **kw) for p, m, s, _ in others]
    assert solo.shape[1] == T + n
    r, rest, window = _park_and_resume_elsewhere(model, probe, k, others)
    assert torch.equal(r.result.cpu(), solo), (r.result.cpu() != solo).nonzero()[:4].tolist()
    for q, a in zip(rest, solo_others):
        assert torch.equal(q.result.cpu(), a)
    # the RAS window came along: the slow tokens of the decode frames so far (the prefill's frame is not part of it),
    # one frame after the resume
    seen = solo[0, T + 1: T + k + 1].tolist()
    assert window == ([0] * 10 + seen)[-10:]


def test_tokens_after_the_resume_depend_on_the_restored_ras_window():
    """Sampled requests whose later frames hit repetition-aware sampling: with the window lost at the resume the
    tokens change, with the window restored (the test above) they do not."""
    cfg, model = _tiny(3)
    changed = 0
    for seed in (1, 2, 3, 4):
        probe = (make_prompt(cfg, 310 + seed, 11), 60, seed, SAMPLED)
        solo = _alone(model, probe[0], 60, seed=seed, **SAMPLED)
        others = [(make_prompt(cfg, 301, 9), 15, 11, SAMPLED), (make_prompt(cfg, 302, 17), 40, 12, SAMPLED),
                  (make_prompt(cfg, 303, 6), 30, 13, SAMPLED)]
        r, _, _ = _park_and_resume_elsewhere(model, probe, 12, others, spoil_ras=True)
        assert torch.equal(r.result.cpu()[:, :11 + 13], solo[:, :11 + 13])
        changed += not torch.equal(r.result.cpu(), solo)
    assert changed >= 1


def test_parked_request_at_s2pro_layer_geometry_in_a_64_row_engine():
    cfg, w = _s2pro_small(2048)
    model = _s2pro_model(cfg, w, 64)
    kw = dict(temperature=0.8, top_p=0.9, top_k=30)
    probe = (_s2pro_prompt(cfg, 1, 70), 20, 99, kw)
    others = [(_s2pro_prompt(cfg, 2, 30), 12, 5, kw), (_s2pro_prompt(cfg, 3, 90), 30, 6, kw),
              (_s2pro_prompt(cfg, 4, 12), 20, 7, kw)]
    solo = _alone(model, probe[0], 20, seed=99, **kw)
    solo_others = [_alone(model, p, m, seed=s, **kw) for p, m, s, _ in others]
    r, rest, _ = _park_and_resume_elsewhere(model, probe, 9, others)
    assert torch.equal(r.result.cpu(), solo)
    for q, a in zip(rest, solo_others):
        assert torch.equal(q.result.cpu(), a)


def test_parked_pages_survive_reclaim_and_stay_shared_in_a_small_pool():
    """9 pages. The probe (3 pages) shares its 130-row prefix with a running request; while it is parked, requests
    come and go and the pool reclaims retired slots for them. Nothing of the probe's K/V is copied or lost."""
    from fish_speech_b200.scheduler import ContinuousBatcher

    cfg, model = _tiny(3, kv_pages=9, max_seq_len=1024, seed=78)
    _, ref = _tiny(3, kv_pages=None, max_seq_len=1024, seed=78)
    kw = GREEDY
    shared = make_prompt(cfg, 500, 130)
    specs = dict(probe=(_grown_prompt(cfg, shared, shared[:, :0], 501, 11), 30, 1),
                 sharer=(_grown_prompt(cfg, shared, shared[:, :0], 502, 10), 60, 2),
                 f1=(make_prompt(cfg, 503, 70), 6, 3), f2=(make_prompt(cfg, 504, 70), 6, 4),
                 f3=(make_prompt(cfg, 505, 130), 6, 5))
    solo = {name: _alone(ref, p, n, seed=s, **kw) for name, (p, n, s) in specs.items()}
    eng = model.engine
    reclaimed = []
    forget = eng.kv_pool.on_reclaim
    eng.kv_pool.on_reclaim = lambda s: (reclaimed.append(s), forget(s))
    # the probe is paced against a clock that stands still: once parked it is never short of frames, so it waits
    # for a slot nobody else wants
    b = ContinuousBatcher(model, max_slots=3, frames_per_poll=2, max_live=4, clock=lambda: 0.0)
    sub = lambda name, **kw2: _submit(b, *specs[name][:2], specs[name][2], kw, reuse_prefix=True, tag=name, **kw2)
    probe = sub("probe", pace=1.0)
    b.step()
    sharer = sub("sharer")
    b.step()
    pool = eng.kv_pool
    assert pool.table[0, :2].tolist() == pool.table[1, :2].tolist() and pool.ref[pool.table[0, :2]].tolist() == [2, 2]
    pages = pool.table[0, :3].tolist()
    before = eng.buffer("k_slow")[:, pages].clone()
    b._park(probe)
    assert pool.ref[pages].tolist() == [2, 2, 1] and eng.kv_pages_available() == 9 - 5
    fillers = [sub("f1"), sub("f2"), sub("f3")]
    while not probe.resumes:
        b.step()
        assert pool.ref[pages].tolist() == [2, 2, 1]
    assert reclaimed and probe.slot != 0 and not sharer.done.is_set()
    assert pool.table[probe.slot, :3].tolist() == pages  # the same pages, mapped again: nothing was copied
    n_prompt = specs["probe"][0].size(1)
    assert torch.equal(eng.buffer("k_slow")[:, pages, :, :1], before[:, :, :, :1]) and n_prompt > 128
    b.run()
    b.close()
    assert pool.peak <= 9 and not pool.detached
    for r in [probe, sharer] + fillers:
        assert torch.equal(r.result.cpu(), solo[r.tag]), r.tag


def test_paced_streams_on_three_slots_are_parked_repeatedly_and_equal_generate():
    """Eight paced two-chunk streams and an unpaced request on three slots, with a clock under which every stream runs
    ahead of its listener and is parked at least twice."""
    from fish_speech_b200.scheduler import ContinuousBatcher, StreamClock

    cfg, model = _tiny(3, max_seq_len=256, seed=79)
    _, ref = _tiny(1, max_seq_len=256, seed=79)
    N, n1, n2 = 8, 40, 40
    first = [make_prompt(cfg, 600 + i, 8 + i) for i in range(N)]
    solo1 = [_alone(ref, first[i], n1, seed=10 + i, **SAMPLED) for i in range(N)]
    second = [_grown_prompt(cfg, first[i], solo1[i][:, first[i].size(1):-1], 700 + i, 5) for i in range(N)]
    solo2 = [_alone(ref, second[i], n2, seed=50 + i, **SAMPLED) for i in range(N)]
    lone_p = make_prompt(cfg, 650, 20)
    solo_lone = _alone(ref, lone_p, 120, seed=5, **GREEDY)

    clk = [0.0]
    b = ContinuousBatcher(model, max_slots=3, frames_per_poll=2, max_live=N + 1, clock=lambda: clk[0])
    pieces = {(i, c): [] for i in range(N) for c in (0, 1)}
    chunk2 = {}

    def next_chunk(r):
        i, clock = r.tag
        T = first[i].size(1)
        grown = _grown_prompt(cfg, first[i], r.result.cpu()[:, T:-1], 700 + i, 5)
        chunk2[i] = _submit(b, grown, n2, 50 + i, SAMPLED, pace=1.0, stream=clock, reuse_prefix=True, tag=(i, 1),
                            on_frames=lambda q, c: pieces[q.tag].append(c))

    chunk1 = [_submit(b, first[i], n1, 10 + i, SAMPLED, pace=1.0, stream=StreamClock(), reuse_prefix=True,
                      on_frames=lambda q, c: pieces[q.tag[0], 0].append(c), on_done=next_chunk) for i in range(N)]
    for i, r in enumerate(chunk1):
        r.tag = (i, r.stream)
    lone = _submit(b, lone_p, 120, 5, GREEDY)
    while not b.idle():
        b.step()
        clk[0] += 0.5  # a poll makes 2 frames per running stream; the 8 listeners play 4 between them
        assert len(b.active) <= 3
    b.close()
    assert torch.equal(lone.result.cpu(), solo_lone) and lone.parks == 0
    for i in range(N):
        a, c = chunk1[i], chunk2[i]
        assert torch.equal(a.result.cpu(), solo1[i]) and torch.equal(c.result.cpu(), solo2[i]), i
        assert a.parks + c.parks >= 2 and a.parks + c.parks == a.resumes + c.resumes, (i, a.parks, c.parks)
        assert torch.equal(torch.cat(pieces[i, 0], dim=1), a.result.cpu()[1:, first[i].size(1):-1].to(torch.int32))
        assert torch.equal(torch.cat(pieces[i, 1], dim=1), c.result.cpu()[1:, second[i].size(1):-1].to(torch.int32))
        assert a.stream is c.stream and a.stream.frames == n1 - 1 + n2 - 1


def test_cancel_frees_the_slot_and_pages_for_the_next_request():
    from fish_speech_b200.scheduler import Cancelled, ContinuousBatcher

    cfg, model = _tiny(2, kv_pages=6, max_seq_len=1024, seed=80)
    _, ref = _tiny(1, max_seq_len=1024, seed=80)
    specs = [(make_prompt(cfg, 800, 100), 60, 1), (make_prompt(cfg, 801, 40), 50, 2), (make_prompt(cfg, 802, 150), 30, 3)]
    solo = [_alone(ref, p, n, seed=s, **SAMPLED) for p, n, s in specs]
    done = []
    b = ContinuousBatcher(model, max_slots=2, frames_per_poll=4)
    r0, r1 = [_submit(b, p, n, s, SAMPLED, on_done=lambda r: done.append(r)) for p, n, s in specs[:2]]
    b.step()
    b.step()
    r2 = _submit(b, *specs[2][:2], specs[2][2], SAMPLED)
    b.step()
    assert r2.slot == -1 and model.engine.kv_pages_available() == 6 - 3 - 2  # 3 pages needed, 1 there
    assert b.cancel(r0) and isinstance(r0.error, Cancelled) and r0.result is None and done == [r0]
    assert model.engine.kv_pages_available() == 6 - 2
    b.step()
    assert r2.slot == 0 and not b.cancel(r0)
    b.run()
    b.close()
    assert torch.equal(r1.result.cpu(), solo[1]) and torch.equal(r2.result.cpu(), solo[2])
    assert done == [r0, r1]


def test_slot_save_and_restore_reject_bad_arguments():
    from fish_speech_b200 import _lib

    cfg, model = _tiny(3)
    eng = model.engine
    lib = eng.lib
    blob = torch.empty(int(lib.fsb_lm_slot_blob_bytes(eng.h)), dtype=torch.uint8, device="cuda")
    C1 = cfg.num_codebooks + 1
    assert blob.numel() >= 4 * (20 + C1 + C1 * eng.max_frames)
    eng.set_slot_control(False)
    for call in (lib.fsb_lm_slot_save, lib.fsb_lm_slot_restore):
        with pytest.raises(_lib.FsbError, match="slot control"):
            _lib.check(call(eng.h, 0, blob.data_ptr(), None))
    eng.set_slot_control(True)
    try:
        for call in (lib.fsb_lm_slot_save, lib.fsb_lm_slot_restore):
            for slot in (-1, 3, 64):
                with pytest.raises(_lib.FsbError, match="slot="):
                    _lib.check(call(eng.h, slot, blob.data_ptr(), None))
            with pytest.raises(_lib.FsbError, match="null blob"):
                _lib.check(call(eng.h, 0, None, None))
            with pytest.raises(_lib.FsbError, match="aligned"):
                _lib.check(call(eng.h, 0, blob.data_ptr() + 4, None))
        state = {k: eng.buffer(k).clone() for k in ("slot_state", "n_out", "pos", "out_tokens")}
        torch.cuda.synchronize()
        assert all(torch.equal(eng.buffer(k), v) for k, v in state.items())  # no rejected call launched anything
    finally:
        eng.set_slot_control(False)
