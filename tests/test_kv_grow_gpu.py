"""KV growth on the GPU (ContinuousBatcher(kv_growth=True)): requests map pages as they decode, wait parked for pages
on a small pool, and still return exactly the tokens `generate` returns for each alone. The decode attention records a
live row that meets an unmapped page in "kv_miss"."""
import pytest
import torch

from fish_speech_b200.engine import kv_pages_for
from oracle import lm_oracle as O
from tests.lm_util import build_model, make_prompt
from tests.test_paged_kv_gpu import _gen, _paged_model, _s2pro_model, _s2pro_prompt, _s2pro_small

pytestmark = pytest.mark.gpu

GREEDY = dict(temperature=0.7, top_p=0.7, top_k=1)
SAMPLED = dict(temperature=0.9, top_p=0.9, top_k=30)


def _setup(geometry, rows, pages):
    """(model under test, solo model, prompt maker). <|im_end|> is never sampled: requests run to their budgets."""
    if geometry == "tiny":
        cfg = O.tiny_config(max_seq_len=1024)
        w = O.make_weights(cfg, seed=31, head_gain=2.5)
        w["embeddings.weight"][cfg.im_end_id] = 0
        model = _paged_model(cfg, w, kv_pages=pages, max_batch=rows, max_rows=1024, scramble=3)
        return model, build_model(cfg, w, debug=False), lambda seed, T: make_prompt(cfg, seed, T)
    cfg, w = _s2pro_small(1024)
    return (_s2pro_model(cfg, w, rows, kv_pages=pages, max_rows=1024), _s2pro_model(cfg, w, 1),
            lambda seed, T: _s2pro_prompt(cfg, seed, T))


def _specs(make, n, prefix=None):
    out = []
    for i in range(n):
        T = 40 + (29 * i) % 90
        p = make(500 + i, T)
        if prefix is not None:
            p = torch.cat([prefix, p], 1)
        kw = dict(GREEDY if i % 2 == 0 else SAMPLED)
        out.append((p, 120 + (37 * i) % 80, dict(kw, seed=700 + i)))
    return out


def _run(model, specs, slots, fpp=8, reuse=False, **kw):
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    b = ContinuousBatcher(model, max_slots=slots, frames_per_poll=fpp, kv_growth=True, **kw)
    assert b.kv_growth
    reqs = [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=n, reuse_prefix=reuse, **k)) for p, n, k in specs]
    peak = 0
    while not b.idle():
        b.step()
        peak = max(peak, model.engine.kv_pool.in_use())
    assert peak <= model.engine.kv_pool.n_pages
    assert not model.engine.buffer("kv_miss").any()
    b.close()
    return b, reqs


def _check_solo(solo, specs, reqs):
    for i, ((p, n, kw), r) in enumerate(zip(specs, reqs)):
        assert r.error is None, r.error
        assert torch.equal(r.result.cpu(), _gen(solo, p, n, **kw)), f"request {i} != its solo run"


@pytest.mark.parametrize("geometry,rows", [("tiny", 6), ("tiny", 40), ("s2pro", 6)],
                         ids=["tiny-rows32", "tiny-rows64", "s2pro-rows32"])
def test_small_pool_parks_for_pages_with_the_same_tokens(geometry, rows):
    """12 requests, greedy and sampled with their own seeds, on a pool of about two worst cases: running requests
    are parked for pages mid-utterance, and every result equals `generate` of that request alone."""
    probe = _specs(lambda s, T: torch.zeros(1, T), 12)
    worst = max(kv_pages_for(p.shape[1] + n) for p, n, _ in probe)
    model, solo, make = _setup(geometry, rows, 2 * worst)
    specs = _specs(make, 12)
    b, reqs = _run(model, specs, min(rows, 12))
    assert sum(r.page_parks for r in reqs) > 0
    _check_solo(solo, specs, reqs)


def test_shared_prefix_with_growth():
    """Requests that share a live donor's 200-row prefix (whole pages mapped by reference, the partial page copied at
    admission) grow their own pages; tokens match solo runs and every reference is gone after release_kv."""
    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=32, head_gain=2.5)
    w["embeddings.weight"][cfg.im_end_id] = 0
    prefix = make_prompt(cfg, 77, 200)
    specs = _specs(lambda s, T: make_prompt(cfg, s, T), 8, prefix=prefix)
    worst = max(kv_pages_for(p.shape[1] + n) for p, n, _ in specs)
    model = _paged_model(cfg, w, kv_pages=2 * worst, max_batch=8, max_rows=2048)
    b, reqs = _run(model, specs, 8, reuse=True)
    assert model.engine.rows_reused > 0
    _check_solo(build_model(cfg, w, debug=False), specs, reqs)
    eng = model.engine
    eng.release_kv()
    assert eng.kv_pool.in_use() == 0 and not eng.kv_pool.ref.any()


def test_paced_streams_and_cancel_while_parked_for_pages():
    """More live paced streams than slots (max_live > max_slots) with growth, and a request cancelled while it is
    parked for pages: the others match their solo runs."""
    from fish_speech_b200.scheduler import Cancelled, ContinuousBatcher, SlotRequest

    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=33, head_gain=2.5)
    w["embeddings.weight"][cfg.im_end_id] = 0
    specs = _specs(lambda s, T: make_prompt(cfg, s, T), 10)
    worst = max(kv_pages_for(p.shape[1] + n) for p, n, _ in specs)
    model = _paged_model(cfg, w, kv_pages=2 * worst, max_batch=4, max_rows=1024)
    clk = [0.0]
    b = ContinuousBatcher(model, max_slots=4, frames_per_poll=8, max_live=7, kv_growth=True, clock=lambda: clk[0])
    reqs = [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=n, pace=400.0 if i % 2 else None, **k))
            for i, (p, n, k) in enumerate(specs)]
    victim = None
    while not b.idle():
        b.step()
        clk[0] += 0.01
        if victim is None and b.short:
            victim = b.short[-1]
            assert b.cancel(victim)
    assert victim is not None and isinstance(victim.error, Cancelled)
    assert not model.engine.buffer("kv_miss").any()
    b.close()
    solo = build_model(cfg, w, debug=False)
    for (p, n, k), r in zip(specs, reqs):
        if r is not victim:
            assert r.error is None and torch.equal(r.result.cpu(), _gen(solo, p, n, **k))


@pytest.mark.parametrize("geometry", ["tiny", "s2pro"])
def test_kv_miss_records_the_row_that_meets_an_unmapped_page(geometry):
    """One live row's next page-table entry is set to -1 (unmapped): the decode attention skips it, records
    1 + its position in kv_miss, and the other rows' tokens equal their solo runs."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    model, solo, make = _setup(geometry, 3, None)
    specs = [(make(41, 37), 20, dict(SAMPLED, seed=1)), (make(42, 64), 20, dict(GREEDY)),
             (make(43, 90), 20, dict(SAMPLED, seed=3))]
    b = ContinuousBatcher(model, max_slots=3, frames_per_poll=1)
    reqs = [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=n, **k)) for p, n, k in specs]
    eng = model.engine
    b._schedule()  # prefill: row 1 has written positions [0, 64); its next frame writes position 64, on page 1
    assert reqs[1].slot == 1 and int(eng.kv_pool.table[1, 1]) >= 0
    eng.buffer("kv_page")[1, 1] = -1
    b.step()
    assert eng.buffer("kv_miss").cpu().tolist() == [0, 65, 0]
    b.run()
    b.close()
    for i in (0, 2):
        assert torch.equal(reqs[i].result.cpu(), _gen(solo, *specs[i][:2], **specs[i][2]))
