"""Fused admission (LmEngine.prefill defer_first_frame, ContinuousBatcher fused_admission) on the GPU.

A deferred prefill stages each new sequence's last prompt row per slot and parks the slot at position -1; the next decode
frame splices the staged row into its own residual stream after the slow stack (csrc/lm_kernels.cu
first_frame_splice_kernel) and samples a row whose slot has produced no frame yet by the prefill's rule
(sample_first_frame_kernel). The step GEMMs are batch-invariant and a request's random stream is keyed by its own seed
and frame index, so the work must be bitwise the work of today's order: a decode frame over the running rows, then a
prefill with its own first frame. These tests check that for the whole engine state, then for requests through the
scheduler against `generate` alone and the oracle.
"""
from __future__ import annotations

import random

import pytest
import torch

from oracle import lm_oracle as O
from tests.lm_util import build_model, make_prompt

pytestmark = pytest.mark.gpu

STATE = ("cur_tok", "out_tokens", "n_out", "pos", "ras_window", "finished", "slot_state", "kv_page", "k_fast",
         "v_fast", "k_slow", "v_slow")


def _bits(t: torch.Tensor) -> torch.Tensor:
    t = t.contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def _model(cfg, w, max_batch, max_rows=2048, debug=True, kv_pages=None):
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from tests.lm_util import model_args

    m = DualARTransformer(model_args(cfg), w, device="cuda", im_end_id=cfg.im_end_id)
    m.debug = debug
    m.max_rows = max_rows
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages)
    m._cache_setup_done = True
    return m


def _s2pro_model(w, cfg, max_batch):
    from fish_speech_b200.configs import S2PRO_IM_END_ID
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    m = DualARTransformer(cfg, w, device=torch.device("cuda", 0), im_end_id=S2PRO_IM_END_ID)
    m.debug = True
    m.max_rows = 512
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len)
    return m


def _params(eng, specs):
    """Slot-control parameters of new requests: (slot, limit, temperature, top_p, top_k, seed)."""
    from fish_speech_b200.engine import bf16_round

    for s, limit, t, p, k, seed in specs:
        eng.buffer("slot_limit")[s] = limit
        eng.buffer("slot_temperature")[s] = bf16_round(t)
        eng.buffer("slot_top_p")[s] = bf16_round(p)
        eng.buffer("slot_top_k")[s] = k
        eng.buffer("slot_seed")[s] = seed
        eng.buffer("n_out")[s] = 0
        eng.buffer("ras_window")[s] = 0
        eng.buffer("slot_state")[s] = 1


def _two_orders(make, running, new, sampled, reuse=False, frames_before=3):
    """The same work in two orders on two engines built alike: (a) a deferred prefill of `new`, then one decode frame;
    (b) one decode frame with the new slots idle, then today's prefill with its own first frame. `running`, `new`:
    lists of (slot, prompt). Returns the state buffers of both engines and the debug logits."""
    out = []
    for order in ("fused", "today"):
        m = make()
        eng = m.engine
        B = eng.max_batch
        eng.reset()
        eng.release_kv()
        eng.set_slot_control(True)
        eng.buffer("pos").fill_(-1)
        eng.set_context_bound_exact(eng.kv_len)

        def spec(i, slot):
            greedy = not sampled or i % 3 == 0
            return (slot, 40, 0.7 if greedy else 0.8, 0.7 if greedy else 0.9, 1 if greedy else 30, 7919 * (i + 1))

        def prefill(pairs, defer):
            prompts = [p.cuda() for _, p in pairs]
            slots = [s for s, _ in pairs]
            kv_end = [p.shape[1] + 48 for p in prompts]
            kw = dict(defer_first_frame=True) if defer else {}
            if reuse:
                eng.prefill_reusing(prompts, slots, None, do_sample=True, kv_end=kv_end, **kw)
            else:
                eng.prefill(prompts, slots, None, do_sample=True, kv_end=kv_end, **kw)

        _params(eng, [spec(i, s) for i, (s, _) in enumerate(running)])
        prefill(running, False)
        eng.decode(B, frames_before, None)
        new_specs = [spec(100 + i, s) for i, (s, _) in enumerate(new)]
        if order == "fused":
            _params(eng, new_specs)
            prefill(new, True)
            eng.decode(B, 1, None)
        else:
            eng.decode(B, 1, None)
            _params(eng, new_specs)
            prefill(new, False)
        torch.cuda.synchronize()
        st = {k: eng.buffer(k).clone() for k in STATE}
        st["slow_logits"] = eng.buffer("slow_logits").clone()
        st["fast_logits"] = eng.buffer("fast_logits").clone()
        out.append(st)
        eng.close()
        del m, eng
        torch.cuda.empty_cache()
    return out


def _assert_same(a, b, running, new, what):
    for k in a:
        if k in ("slow_logits", "fast_logits"):
            continue
        assert torch.equal(_bits(a[k]), _bits(b[k])), f"{what}: {k} differs"
    for s, _ in running + new:  # the logits of every live row (idle rows keep whatever they held)
        assert torch.equal(_bits(a["slow_logits"][s]), _bits(b["slow_logits"][s])), f"{what}: slow logits of slot {s}"
        assert torch.equal(_bits(a["fast_logits"][:, s]), _bits(b["fast_logits"][:, s])), f"{what}: fast logits {s}"
    # the work happened: the new slots made their first frame, the running ones one more
    for s, p in new:
        assert int(a["n_out"][s]) == 1 and int(a["pos"][s]) == p.shape[1], (what, s)
    for s, _ in running:
        assert int(a["n_out"][s]) >= 2, (what, s)


TINY_CASES = {
    # engine slots, running slots, new slots
    "tiny32": (32, [1, 5, 18, 30], [0, 17, 31]),
    "tiny64": (64, [1, 5, 18, 30, 40, 50], [0, 17, 31, 33, 63]),
}


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
@pytest.mark.parametrize("case", list(TINY_CASES))
def test_tiny_deferred_prefill_then_frame_equals_frame_then_prefill(case, sampled):
    cfg = O.tiny_config(max_seq_len=512)
    w = O.make_weights(cfg, seed=23, head_gain=2.5)
    slots, run_slots, new_slots = TINY_CASES[case]
    running = [(s, make_prompt(cfg, 300 + s, 5 + (7 * s) % 23)) for s in run_slots]
    new = [(s, make_prompt(cfg, 500 + s, 3 + (11 * s) % 29)) for s in new_slots]
    a, b = _two_orders(lambda: _model(cfg, w, slots), running, new, sampled)
    _assert_same(a, b, running, new, f"{case}/{'sampled' if sampled else 'greedy'}")


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_tiny_split_prompt_longer_than_max_rows_defers_like_one_pass(sampled):
    """max_rows = 64: a new prompt of 150 rows is prefilled in three passes, the last one deferred."""
    cfg = O.tiny_config(max_seq_len=512)
    w = O.make_weights(cfg, seed=29, head_gain=2.5)
    running = [(2, make_prompt(cfg, 31, 9)), (9, make_prompt(cfg, 32, 20))]
    new = [(0, make_prompt(cfg, 33, 150)), (17, make_prompt(cfg, 34, 12))]
    a, b = _two_orders(lambda: _model(cfg, w, 32, max_rows=64), running, new, sampled)
    _assert_same(a, b, running, new, "split prompt")


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_tiny_prefill_reusing_a_shared_prefix_defers_like_a_full_prefill(sampled):
    """New prompts share a 70-row prefix with a running slot: whole pages are mapped by reference, the partly shared
    page is copied, and the rest is prefilled with the first frame deferred."""
    cfg = O.tiny_config(max_seq_len=512)
    w = O.make_weights(cfg, seed=31, head_gain=2.5)
    base = make_prompt(cfg, 41, 90)
    running = [(3, base), (6, make_prompt(cfg, 42, 15))]
    new = [(0, torch.cat([base[:, :70], make_prompt(cfg, 43, 9)], 1)),
           (31, torch.cat([base[:, :70], make_prompt(cfg, 44, 25)], 1))]
    a, b = _two_orders(lambda: _model(cfg, w, 32), running, new, sampled, reuse=True)
    _assert_same(a, b, running, new, "prefill_reusing")


@pytest.mark.parametrize("sampled", [False, True], ids=["greedy", "sampled"])
def test_s2pro_layers_deferred_prefill_then_frame_equals_frame_then_prefill(sampled):
    """The S2-Pro geometry (real vocabulary, 2560-wide stacks, 10 codebooks) with 3 slow and 4 fast layers."""
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import s2pro_args

    cfg = s2pro_args(max_seq_len=256, n_layer=3)
    w = synthetic.lm_state_dict(cfg, torch.device("cuda", 0))
    g = torch.Generator().manual_seed(5)

    def prompt(T):
        p = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.int32)
        p[0] = torch.randint(0, 151643, (T,), generator=g, dtype=torch.int32)
        return p

    running = [(s, prompt(6 + s)) for s in (2, 9, 20)]
    new = [(s, prompt(4 + s % 13)) for s in (0, 17, 31)]
    a, b = _two_orders(lambda: _s2pro_model(w, cfg, 32), running, new, sampled)
    _assert_same(a, b, running, new, "S2-Pro layers")


def test_refusals():
    from fish_speech_b200 import _lib

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=3, head_gain=2.5)
    m = _model(cfg, w, 4)
    eng = m.engine
    eng.reset()
    eng.release_kv()
    p = make_prompt(cfg, 1, 6).cuda()
    with pytest.raises(ValueError, match="slot control"):
        eng.prefill([p], [0], eng.sampling(0.7, 0.7, 1), defer_first_frame=True)
    eng.slot_control = True  # the library still has it off: its own check refuses
    with pytest.raises(_lib.FsbError, match="slot control"):
        eng.prefill([p], [0], eng.sampling(0.7, 0.7, 1), defer_first_frame=True)
    eng.set_slot_control(True)
    _params(eng, [(1, 8, 0.7, 0.7, 1, 5)])
    eng.prefill([p], [1], None, defer_first_frame=True)
    with pytest.raises(_lib.FsbError, match="deferred first frame"):
        eng.park_slot(1, 8)
    with pytest.raises(_lib.FsbError, match="outside the batch"):
        eng.decode(1, 1, None)  # slot 1 is pending: a batch of one row does not reach it
    eng.decode(2, 1, None)
    parked = eng.park_slot(1, 8)  # served: the slot can be parked now
    eng.resume_slot(1, parked)
    torch.cuda.synchronize()
    assert int(eng.buffer("n_out")[1]) == 1
    eng.close()


# ---------------------------------------------------------------------------------------------------------------------
# the scheduler
# ---------------------------------------------------------------------------------------------------------------------
def _alone(model, prompt, n, **kw):
    from fish_speech_b200.models.text2semantic.inference import generate

    return generate(model=model, prompt=prompt.cuda(), max_new_tokens=n, **kw).cpu()


def _im_end_weights(cfg, seed, prompt, at_frame, total):
    """Weights for which a greedy run of `prompt` emits <|im_end|> at generated frame `at_frame`."""
    w = O.make_weights(cfg, seed=seed, head_gain=8.0)
    free = O.generate(O.setup(cfg, w), prompt, total, temperature=0.7, top_p=0.7, top_k=1, noise=False)
    T = prompt.size(1)
    w["embeddings.weight"][cfg.im_end_id] = (w["embeddings.weight"][int(free[0, T + at_frame])].float() * 1.5).bfloat16()
    return w


@pytest.mark.parametrize("at_frame", [0, 1], ids=["im_end_at_frame0", "im_end_at_frame1"])
def test_fused_scheduled_requests_equal_generate_alone_and_the_oracle(at_frame):
    """A ragged queue through 3 slots with fused admission. Request 0 draws <|im_end|> at frame 0 (not a stop: it runs
    on) or at frame 1 (a stop); one request has a budget of 1 frame. Every result equals `generate` alone; the greedy
    ones also equal the oracle."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config()
    p0 = make_prompt(cfg, 61, 10)
    w = _im_end_weights(cfg, 61, p0, at_frame=at_frame, total=6)
    st = O.setup(cfg, w)
    specs = [dict(prompt=p0, n=12, temperature=0.7, top_p=0.7, top_k=1, seed=5)]
    for i, (T, n, k) in enumerate([(7, 9, 1), (23, 17, 30), (12, 1, 1), (31, 12, 30), (9, 25, 1), (16, 2, 30),
                                   (5, 14, 30), (40, 8, 1), (3, 1, 30)]):
        specs.append(dict(prompt=make_prompt(cfg, 100 + i, T), n=n, temperature=0.7 if k == 1 else 0.9,
                          top_p=0.7 if k == 1 else 0.85, top_k=k, seed=1000 + 17 * i))
    model = build_model(cfg, w, max_batch=3, debug=False)
    alone = [_alone(model, s["prompt"], s["n"], temperature=s["temperature"], top_p=s["top_p"], top_k=s["top_k"],
                    seed=s["seed"]) for s in specs]
    T0 = p0.size(1)
    assert alone[0][0, T0 + at_frame].item() == cfg.im_end_id
    assert (alone[0].shape[1] == T0 + 2) if at_frame == 1 else (alone[0].shape[1] > T0 + 1)
    for s, a in zip(specs, alone):
        if s["top_k"] == 1:
            ref = O.generate(st, s["prompt"], s["n"], temperature=s["temperature"], top_p=s["top_p"], top_k=1,
                             noise=False)
            assert torch.equal(a.to(torch.int32), ref.to(torch.int32))
    b = ContinuousBatcher(model, max_slots=3, frames_per_poll=4, fused_admission=True)
    reqs = [b.submit(SlotRequest(prompt=s["prompt"].cuda(), max_new_tokens=s["n"], temperature=s["temperature"],
                                 top_p=s["top_p"], top_k=s["top_k"], seed=s["seed"])) for s in specs[:5]]
    b.step()
    b.step()
    reqs += [b.submit(SlotRequest(prompt=s["prompt"].cuda(), max_new_tokens=s["n"], temperature=s["temperature"],
                                  top_p=s["top_p"], top_k=s["top_k"], seed=s["seed"])) for s in specs[5:]]
    b.run()
    b.close()
    for i, (r, a) in enumerate(zip(reqs, alone)):
        assert r.error is None and torch.equal(r.result.cpu(), a), (i, r.result.shape, a.shape)


def test_a_repeated_first_token_is_not_in_the_ras_window_of_frame_1():
    """Sampled requests whose frame-1 token equals their frame-0 token: had frame 0 pushed its token into the RAS
    window, frame 1 would have been re-drawn. Fused admission must give `generate`'s tokens for them."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=87, head_gain=1.0)
    model = build_model(cfg, w, max_batch=4, debug=False)
    specs, alone = [], []
    for i in range(80):
        s = dict(prompt=make_prompt(cfg, 700 + i, 4 + i % 9), n=6, temperature=0.5, top_p=0.95, top_k=30, seed=31 + i)
        a = _alone(model, s["prompt"], s["n"], temperature=s["temperature"], top_p=s["top_p"], top_k=s["top_k"],
                   seed=s["seed"])
        T = s["prompt"].size(1)
        if a.shape[1] >= T + 2 and a[0, T] == a[0, T + 1]:
            specs.append(s)
            alone.append(a)
        if len(specs) == 6:
            break
    assert specs, "no sampled request repeats its first token"
    b = ContinuousBatcher(model, max_slots=4, frames_per_poll=3, fused_admission=True)
    reqs = [b.submit(SlotRequest(prompt=s["prompt"].cuda(), max_new_tokens=s["n"], temperature=s["temperature"],
                                 top_p=s["top_p"], top_k=s["top_k"], seed=s["seed"])) for s in specs]
    b.run()
    b.close()
    for r, a in zip(reqs, alone):
        assert torch.equal(r.result.cpu(), a)


def test_64_slot_engine_with_compact_rows_switching_tiles():
    """The load-varying queue of the compact-rows tests (64 -> 32 -> 64 rows, moves, admissions into slots >= 32):
    fused admission on gives every request the tokens of the run with it off."""
    from tests.test_decode_rows_gpu import _check_same, _ramp_waves, _serve

    cfg = O.tiny_config(max_seq_len=256)
    w = O.make_weights(cfg, seed=47, head_gain=2.5)
    w["embeddings.weight"][cfg.im_end_id] = 0
    m = _model(cfg, w, 64, debug=False)
    waves = _ramp_waves(cfg, 300)
    on, tiles, b_on = _serve(m, waves, compact_rows=True, fused_admission=True)
    off, _, _ = _serve(m, waves, compact_rows=True)
    assert 32 in tiles and 64 in tiles and b_on.moves > 0
    _check_same(on, off, "fused admission on vs off")
    m.engine.close()


def test_kv_growth_small_pool_paced_parking_and_cancel():
    """Pages granted as requests decode from a pool too small for all of them, paced streams parked and resumed, and a
    cancel right after a poll: fused on and off give the same tokens to every other request."""
    from fish_speech_b200.scheduler import Cancelled, ContinuousBatcher, SlotRequest

    cfg = O.tiny_config(max_seq_len=256)
    w = O.make_weights(cfg, seed=53, head_gain=2.5)
    w["embeddings.weight"][cfg.im_end_id] = 0
    rnd = random.Random(4)
    specs = [dict(prompt=make_prompt(cfg, 900 + i, rnd.randint(3, 40)), max_new_tokens=rnd.randint(4, 60),
                  temperature=0.8, top_p=0.9, top_k=1 if i % 3 == 0 else 30, seed=77 + i) for i in range(30)]
    specs[11]["max_new_tokens"] = 60  # still running after its first poll in either mode, when it is cancelled
    runs = {}
    for fused in (False, True):
        m = _model(cfg, w, 8, debug=False, kv_pages=14)
        b = ContinuousBatcher(m, max_slots=8, frames_per_poll=4, kv_growth=True, max_live=12, clock=lambda: 0.0,
                              fused_admission=fused)
        reqs = []
        for i, s in enumerate(specs):
            r = SlotRequest(**{**s, "prompt": s["prompt"].cuda()}, pace=20.0)
            reqs.append(b.submit(r))
            if i % 6 == 5:
                b.step()
            if i == 11:
                assert b.cancel(reqs[11])  # admitted by the poll just run, if a slot was free
        while not b.idle():
            b.step()
        b.close()
        assert b.kv_growth and any(r.page_parks or r.parks for r in reqs)
        runs[fused] = reqs
        m.engine.close()
    for i, (a, b_) in enumerate(zip(runs[False], runs[True])):
        if i == 11:
            assert isinstance(a.error, Cancelled) and isinstance(b_.error, Cancelled)
            continue
        assert a.error is None and b_.error is None and torch.equal(a.result.cpu(), b_.result.cpu()), i
