"""A 64-slot engine on the 32-row step (csrc/lm_engine.cu frame_tile / frame_plans, scheduler compact_rows).

An engine of 33..64 slots holds the step GEMM plans of both row tiles and runs a frame of <= 32 rows on the 32-row
ones. Every output element is the same sum of the same MMAs at either tile, so a request's tokens and logits must be
bitwise those of the same engine forced onto the 64-row tile and of a 32-slot engine; these tests check that from the
tiny geometry up to full S2-Pro frames, across tile switches, slot moves, parking, KV growth and split attention, and
that a switch between tiles replays a captured graph instead of capturing a new one.
"""
from __future__ import annotations

import pytest
import torch

from oracle import lm_oracle as O
from tests.lm_util import build_model, make_prompt

pytestmark = pytest.mark.gpu

KS = (1, 17, 32)


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32)


def _model(cfg, w, max_batch, debug=True, kv_pages=None, attn_split=0):
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from tests.lm_util import model_args

    m = DualARTransformer(model_args(cfg), w, device="cuda", im_end_id=cfg.im_end_id)
    m.debug = debug
    m.max_rows = 2048
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages, attn_split=attn_split)
    m._cache_setup_done = True
    return m


def _batch(model, prompts, n, tile, **sp):
    """generate_batch on `tile` (0 = automatic): tokens and the last frame's debug logits of the batch's rows."""
    from fish_speech_b200.models.text2semantic.inference import generate_batch

    eng = model.engine
    eng.set_decode_tile(tile)
    out = generate_batch(model=model, prompts=[p.cuda() for p in prompts], max_new_tokens=n, **sp)
    torch.cuda.synchronize()
    k = len(prompts)
    used = eng.decode_tile
    eng.set_decode_tile(0)
    return ([o.cpu() for o in out], eng.buffer("slow_logits")[:k].clone().cpu(),
            eng.buffer("fast_logits")[:, :k].clone().cpu(), used)


def _same(a, b, what):
    ta, sa, fa, _ = a
    tb, sb, fb, _ = b
    for i, (x, y) in enumerate(zip(ta, tb)):
        assert torch.equal(x, y), f"{what}: sequence {i} tokens differ"
    assert torch.equal(_bits(sa), _bits(sb)), f"{what}: slow logits differ"
    assert torch.equal(_bits(fa), _bits(fb)), f"{what}: fast logits differ"


# ---------------------------------------------------------------------------------------------------------------------
# the two tiles of one engine, and a 32-slot engine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sp", [dict(temperature=0.7, top_p=0.7, top_k=1, seed=1),
                                dict(temperature=0.8, top_p=0.9, top_k=30, seed=77)], ids=["greedy", "sampled"])
def test_tiny_k_rows_on_the_32_row_tile_equal_the_64_row_tile_and_a_32_slot_engine(sp):
    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=41, head_gain=2.5)
    m64 = build_model(cfg, w, max_batch=64)
    m32 = build_model(cfg, w, max_batch=32)
    assert m64.engine.row_tile == 64 and m32.engine.row_tile == 32
    for k in KS:
        prompts = [make_prompt(cfg, 900 + 3 * i + k, 4 + (5 * i) % 19) for i in range(k)]
        auto = _batch(m64, prompts, 10, 0, **sp)
        forced = _batch(m64, prompts, 10, 64, **sp)
        one = _batch(m32, prompts, 10, 0, **sp)
        assert (auto[3], forced[3], one[3]) == (32, 64, 32)
        _same(auto, forced, f"k={k}: 32-row vs 64-row tile")
        _same(auto, one, f"k={k}: 64-slot engine vs 32-slot engine")
    # more rows than the 32-row tile holds: automatic is the 64-row tile, and forcing 32 is refused
    from fish_speech_b200 import _lib

    prompts = [make_prompt(cfg, 50 + i, 6) for i in range(33)]
    assert _batch(m64, prompts, 2, 0, **sp)[3] == 64
    with pytest.raises(_lib.FsbError, match="forced 32-row tile"):
        _batch(m64, prompts, 2, 32, **sp)
    with pytest.raises(_lib.FsbError, match="exceeds"):
        m32.engine.set_decode_tile(64)
    with pytest.raises(_lib.FsbError, match="must be 0"):
        m64.engine.set_decode_tile(48)
    m64.engine.close()
    m32.engine.close()


def test_s2pro_k_rows_on_the_32_row_tile_equal_the_64_row_tile_and_a_32_slot_engine():
    """Full S2-Pro geometry (36 slow + 4 fast layers, real vocabulary, synthetic weights), greedy, tokens and debug
    logits bitwise."""
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    dev = torch.device("cuda", 0)
    cfg = s2pro_args(max_seq_len=64)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    g = torch.Generator().manual_seed(9)
    prompts = []
    for i in range(32):
        p = torch.zeros(cfg.num_codebooks + 1, 8 + i % 13, dtype=torch.int32)
        p[0] = torch.randint(0, 151643, (p.shape[1],), generator=g, dtype=torch.int32)
        prompts.append(p)
    sp = dict(temperature=0.7, top_p=0.7, top_k=1, seed=1)
    results = {}
    for slots in (64, 32):
        model = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        model.debug = True
        model.max_rows = 64 * 24
        model.setup_caches(max_batch_size=slots, max_seq_len=cfg.max_seq_len)
        assert model.engine.row_tile == slots
        for k in KS:
            results[(slots, k, 0)] = _batch(model, prompts[:k], 4, 0, **sp)
            if slots == 64:
                results[(slots, k, 64)] = _batch(model, prompts[:k], 4, 64, **sp)
        model.engine.close()
        del model
    del w
    for k in KS:
        assert (results[(64, k, 0)][3], results[(64, k, 64)][3]) == (32, 64)
        _same(results[(64, k, 0)], results[(64, k, 64)], f"S2-Pro k={k}: 32-row vs 64-row tile")
        _same(results[(64, k, 0)], results[(32, k, 0)], f"S2-Pro k={k}: 64-slot vs 32-slot engine")


def test_switching_tiles_replays_captured_graphs():
    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=43, head_gain=2.5)
    m = build_model(cfg, w, max_batch=64)
    eng = m.engine
    sp = dict(temperature=0.7, top_p=0.7, top_k=1, seed=1)
    few = [make_prompt(cfg, 10 + i, 7) for i in range(20)]
    many = [make_prompt(cfg, 40 + i, 7) for i in range(40)]
    seen = []
    for prompts in (few, many, few, many, few):
        first = _batch(m, prompts, 6, 0, **sp)
        seen.append((first[3], eng.graph_captures))
    assert [t for t, _ in seen] == [32, 64, 32, 64, 32]
    caps = [c for _, c in seen]
    assert caps[1] > caps[0] >= 1 and caps[2:] == [caps[1]] * 3, caps  # the second round captured nothing
    # the same bits as before the switches
    again = _batch(m, few, 6, 0, **sp)
    assert all(torch.equal(a, b) for a, b in zip(again[0], _batch(m, few, 6, 64, **sp)[0]))
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# the scheduler: sampled requests with their own seeds, tile switches, moves, parking and KV growth
# ---------------------------------------------------------------------------------------------------------------------
def _specs(cfg, n, seed0, budget=(6, 30)):
    g = torch.Generator().manual_seed(seed0)
    out = []
    for i in range(n):
        greedy = i % 3 == 0
        lo, hi = budget
        out.append(dict(prompt=make_prompt(cfg, seed0 + i, 3 + (7 * i) % 29),
                        max_new_tokens=int(torch.randint(lo, hi + 1, (1,), generator=g)),
                        temperature=0.8, top_p=0.9, top_k=1 if greedy else 30, seed=seed0 * 100 + 13 * i))
    return out


def _serve(model, waves, tile=0, polls_between=2, **kw):
    """Submit the request specs of each wave, run `polls_between` polls, then the next wave; run to the end. Returns
    the requests, the tile of every poll, and the batcher."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    eng = model.engine
    eng.set_decode_tile(tile)
    b = ContinuousBatcher(model, max_slots=model.engine.max_batch, frames_per_poll=4, **kw)
    reqs, tiles = [], []
    for wave in waves:
        reqs += [b.submit(SlotRequest(**{**s, "prompt": s["prompt"].cuda()})) for s in wave]
        for _ in range(polls_between):
            if b.active or b.waiting:
                b.step()
                tiles.append(eng.decode_tile)
    while not b.idle():
        b.step()
        tiles.append(eng.decode_tile)
    b.close()
    eng.set_decode_tile(0)
    return reqs, tiles, b


def _check_same(ra, rb, what):
    for i, (a, b) in enumerate(zip(ra, rb)):
        assert a.error is None and b.error is None, (what, i, a.error, b.error)
        assert torch.equal(a.result.cpu(), b.result.cpu()), f"{what}: request {i} (slots {a.slot} / {b.slot}) differs"


@pytest.mark.parametrize("paged,split", [(False, 0), (True, 0), (True, 64)], ids=["contiguous", "paged", "split"])
def test_sampled_requests_on_the_32_row_tile_equal_the_64_row_tile_and_a_32_slot_engine(paged, split):
    """k <= 32 sampled and greedy requests with their own seeds: compact rows put every frame on <= 32 rows, which the
    64-slot engine runs on its 32-row tile (or forced onto the 64-row tile), the same engine without compact rows on
    all 64 rows, and a 32-slot engine."""
    cfg = O.tiny_config(max_seq_len=1024 if split else 256)
    w = O.make_weights(cfg, seed=45, head_gain=2.5)
    pages = 64 * 4 if paged else None  # 64 slots share 256 pages of the 1024 the slots could map
    m64 = _model(cfg, w, 64, debug=False, kv_pages=pages, attn_split=split)
    m32 = _model(cfg, w, 32, debug=False, kv_pages=pages and 128, attn_split=split)
    for k in KS:
        specs = _specs(cfg, k, 60 + k, budget=(6, 40))
        if split:  # contexts past the span, so the split kernels run
            for s in specs:
                s["prompt"] = make_prompt(cfg, s["seed"] % 1000, 70 + s["prompt"].shape[1])
        auto, t_auto, _ = _serve(m64, [specs], compact_rows=True)
        forced, t_forced, _ = _serve(m64, [specs], tile=64, compact_rows=True)
        full, t_full, _ = _serve(m64, [specs])
        one, _, _ = _serve(m32, [specs])
        assert set(t_auto) == {32} and set(t_forced) == {64} and set(t_full) == {64}
        _check_same(auto, forced, f"k={k}: 32-row vs 64-row tile")
        _check_same(auto, full, f"k={k}: compact rows vs all 64 rows")
        _check_same(auto, one, f"k={k}: 64-slot vs 32-slot engine")
    m64.engine.close()
    m32.engine.close()


def _ramp_waves(cfg, seed0):
    """Load above 32, down to a few, above 32 again: a long request admitted first keeps running through every phase,
    requests arrive into slots >= 32 after a run of 32-row frames, and the scheduler moves high ones down."""
    probe = _specs(cfg, 1, seed0, budget=(90, 90))
    w1 = _specs(cfg, 39, seed0 + 1, budget=(3, 10))
    w2 = _specs(cfg, 5, seed0 + 2, budget=(40, 60))
    w3 = _specs(cfg, 40, seed0 + 3, budget=(6, 30))
    return [probe + w1, [], [], w2, [], [], [], w3]


@pytest.mark.parametrize("mode", ["plain", "kv_growth", "parking"])
def test_requests_keep_their_bits_across_tile_switches_moves_and_admissions(mode):
    """The same load-varying queue with compact rows on and off. On, frames switch 64 -> 32 -> 64 rows while requests
    run, requests sitting in slots >= 32 are moved down, and requests are admitted into slots >= 32 after 32-row
    frames; every request returns the tokens of the run with compact rows off (all 64 rows, nobody moved). With KV
    growth the requests share a page pool too small for all of them at full length; with parking every request is a
    paced stream and the last wave brings more of them than there are slots, so streams far enough ahead are parked
    (the clock stands still: a stream's lead is the frames it was handed) and resumed into free slots."""
    cfg = O.tiny_config(max_seq_len=256)
    w = O.make_weights(cfg, seed=47, head_gain=2.5)
    w["embeddings.weight"][cfg.im_end_id] = 0  # <|im_end|> is never sampled: every request runs to its budget
    m = _model(cfg, w, 64, debug=False, kv_pages=72 if mode == "kv_growth" else None)
    waves = _ramp_waves(cfg, 300)
    kw = {}
    if mode == "kv_growth":
        kw = dict(kv_growth=True)
    if mode == "parking":
        waves[-1] += _specs(cfg, 40, 307, budget=(20, 40))
        for wave in waves:
            for s in wave:
                s["pace"] = 20.0
        kw = dict(max_live=128, clock=lambda: 0.0)
    runs = {compact: _serve(m, waves, compact_rows=compact, **kw) for compact in (True, False)}
    on, tiles, b_on = runs[True]
    off, tiles_off, b_off = runs[False]
    assert set(tiles_off) == {64} and b_off.moves == 0
    # 64 -> 32 -> 64 while the probe (the first request) ran
    first32 = tiles.index(32)
    assert tiles[0] == 64 and 64 in tiles[first32:], tiles
    assert b_on.moves > 0 and any(r.moves for r in on)
    assert any(r.slot >= 32 or r.moves for r in on[45:]), "no request was admitted into a slot >= 32 after 32-row frames"
    if mode == "parking":
        assert any(r.parks for r in on) and any(r.parks for r in off)
    if mode == "kv_growth":
        assert b_on.kv_growth
    _check_same(on, off, f"{mode}: compact rows on vs off")
    m.engine.close()
