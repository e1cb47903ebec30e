"""The split decode attention (fsb_lm_config.attn_split; csrc/lm_kernels.cu attn_decode_split_kernel, attn_span_kernel,
attn_combine_kernel): a slow-stack row whose context is longer than T = attn_split positions has its history cut into
spans of T positions at absolute positions, one CTA each, merged in ascending order by a kernel of its own.

What must hold, and what each test checks through the handle's own launch sequence (fsb_lm_test_layer_attn) or end to
end:
  * long rows against float64: the reference, the brackets and the wrong references of tests/test_decode_attn_gpu.py
    (the case harness of tests/decode_attn_case.py).
    The tolerance is that module's bound for the unsplit kernel, unchanged: it counts ceil(L / 8) + 9 fp32
    accumulations of the weighted values and ceil(L / 32) + 8 of the sum of exponentials, and the split does fewer of
    each per span (ceil(T / 8) + 8, ceil(T / 32) + 5) plus one product with exp(m_s - M) (expf's 2 ulp, already in
    rho) and one addition per span in the merge, L / T <= L / 64 of them. A reordered fp32 sum moves last bits only,
    and nothing here needs more room than that. The K/V append and every untouched cache bit are checked exactly.
  * rows of at most T positions keep the bits of an engine without the split, beside long rows and on their own;
  * a long row's bits depend on its history only: not on the slot, the neighbours, the context bound's bucket, the
    score chunk, or the run;
  * requests whose context crosses T give the same tokens alone and in a batch, parked and resumed, from shared
    prefix pages, and with the frames replayed from a graph or launched one by one.
"""
from __future__ import annotations

import math
import random

import pytest
import torch

from oracle import lm_oracle as O
from tests.decode_attn_case import TEETH, Geom, State, _check_case, _report_teeth
from tests.kernel_ref import PAGE
from tests.lm_util import _bits, _lib, attn_configs, make_prompt, model_args

pytestmark = pytest.mark.gpu

_ENG: dict = {}


def _split_configs():
    """name -> (config, slots, T). test_decode_attn_gpu's geometries and the default tiny one, slow (64, 4)."""
    out = {name: (cfg, slots, 2048 if cfg.max_seq_len > 16384 else 128)
           for name, (cfg, slots) in attn_configs().items()}
    out["tiny-e"] = (O.tiny_config(max_seq_len=1024), 32, 128)
    return out


def _engine(name, split):
    """(cfg, attention weights, engine) with attn_split = `split` (0: off); the engines of one configuration at a time."""
    if (name, split) not in _ENG:
        from fish_speech_b200.engine import LmEngine

        if any(k[0] != name for k in _ENG):
            _close_engines()
        cfg, slots, _ = _split_configs()[name]
        w = O.make_weights(cfg, seed=59)
        rt = 32 if slots <= 32 else 64
        pages = math.ceil(cfg.max_seq_len / PAGE) - 1 + rt + 8
        eng = LmEngine(cfg, w, "cuda", cfg.im_end_id, max_batch=slots, kv_len=cfg.max_seq_len, max_rows=128,
                       max_frames=4, kv_pages=pages, attn_split=split)
        _ENG[(name, split)] = (cfg, {k: v.cuda() for k, v in w.items() if ".attention" in k}, eng)
    return _ENG[(name, split)]


def _close_engines():
    for _, _, e in _ENG.values():
        e.close()
    _ENG.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _free_engines():
    yield
    _close_engines()


def _edge_positions(S, T, rows, rng, long):
    """Positions (L = position + 1) around T, the span edges k T - 1, k T, k T + 1, page edges inside a span, the
    capacity's last, (S2-Pro) beyond 16 384, and a few short rows among them."""
    pos = [T - 1, T, T + 1, 2 * T - 2, 2 * T - 1, 2 * T, 3 * T - 1, 3 * T, 2 * T + 63, 2 * T + 64, 2 * T + 65, S - 1,
           S - T - 1, S - T, 5, T // 2]
    if long:
        pos += [16384, 16447, 16448, 19999, 8 * T - 1, 8 * T]
    pos = pos[:rows] + [rng.randrange(S) for _ in range(rows - len(pos))]
    rng.shuffle(pos)
    return pos


@pytest.mark.parametrize("name", list(_split_configs()))
def test_long_rows_match_fp64(name):
    """Every (head_dim, group) instance: 13 or 32 rows of a 32-slot engine, 33 or 64 of a 64-slot one; one row parked
    at -1 and one long row with an unmapped page (nothing written, nothing attended); kv_only (append only)."""
    _, _, T = _split_configs()[name]
    cfg, w, eng = _engine(name, T)
    g = Geom(cfg, 0)
    long = cfg.max_seq_len > 16384
    rng = random.Random(sum(map(ord, name)))
    teeth = {k: [] for k in TEETH}
    n_long = 0
    for n, rows in enumerate((13, 32) if eng.max_batch <= 32 else (33, 64)):
        layer = n % g.nl
        pos = _edge_positions(g.S, T, rows, rng, long)
        pos[7] = max(pos[7], 3 * T + 5)  # the row with an unmapped page is a long one
        st = State(eng, g, rows, pos, seed=2000 * n + rows, parked=(3,), unmapped=(7,))
        _check_case(cfg, w, g, layer, st, f"{name} split {T} layer {layer} rows={rows}", teeth)
        n_long += sum(st.pos[i] + 1 > T for i in st.live())
    assert n_long >= 16
    _report_teeth(teeth, f"{name} split {T}", 0)


def _run_with_bound(st, eng, bound, layer=0):
    """State.run with the context bound forced to `bound` instead of the longest row."""
    orig = st.load

    def load():
        orig()
        eng.set_context_bound_exact(bound)

    st.load = load
    try:
        return st.run(layer)
    finally:
        st.load = orig


@pytest.mark.parametrize("name", ["tiny-a", "s2pro"])  # a 32-row and a 64-row engine
def test_short_rows_keep_the_bits_of_the_unsplit_engine(name):
    _, _, T = _split_configs()[name]
    cfg, _, on = _engine(name, T)
    _, _, off = _engine(name, 0)
    g = Geom(cfg, 0)
    rt = on.row_tile
    rng = random.Random(17)
    mixed = [rng.randrange(T) if i % 3 else rng.randrange(T, g.S) for i in range(rt)]
    mixed[:4] = [T - 1, T, 0, g.S - 1]
    alone = [rng.randrange(T) for _ in range(rt)]
    alone[:2] = [T - 1, 0]
    for what, pos, bound in (("beside long rows", mixed, None), ("short rows only", alone, g.S)):
        runs = []
        for eng in (on, off):
            st = State(eng, g, rt, pos, seed=31, parked=(5,))
            runs.append(st.run(0) if bound is None else _run_with_bound(st, eng, bound))
        (a1, k1, v1), (a0, k0, v0) = runs
        assert torch.equal(_bits(k1), _bits(k0)) and torch.equal(_bits(v1), _bits(v0)), f"{name} {what}: K/V differ"
        short = [i for i in range(rt) if 0 <= st.pos[i] < T]
        assert len(short) >= rt // 2
        assert torch.equal(_bits(a1[short]), _bits(a0[short])), f"{name} {what}: attn of short rows differs"
        if bound is None:  # and the others did go through the spans: same values up to the summation order
            longs = [i for i in range(rt) if st.pos[i] >= T]
            assert float(on.buffer("attn_span_ws").abs().sum()) > 0
            assert (a1[longs].float() - a0[longs].float()).abs().max() < 0.01


@pytest.mark.parametrize("name,P", [("tiny-a", 700), ("s2pro", 19000), ("s2pro", 4096)])
def test_long_row_is_deterministic_and_slot_invariant(name, P):
    """The same row (operand, position, history) in slot 0 alone and in the last slot among the others, under every
    context bound bucket above it, a forced score chunk, and twice: one set of bits."""
    _, _, T = _split_configs()[name]
    cfg, _, eng = _engine(name, T)
    g = Geom(cfg, 0)
    rt = eng.row_tile
    rng = random.Random(P)
    pos = [rng.randrange(g.S) for _ in range(rt)]
    pos[0] = pos[rt - 1] = P
    st = State(eng, g, rt, pos, seed=P)
    st.x[rt - 1], st.ssq[rt - 1] = st.x[0], st.ssq[0]
    for c in (st.k0, st.v0):  # the page the row appends to: the same content before the append
        c[:, st.private[rt - 1]] = c[:, st.private[0]]
    full = st.run(0)
    want = full[0][0]
    assert torch.equal(_bits(full[0][rt - 1]), _bits(want)), "last slot among the others != slot 0"
    assert torch.equal(_bits(st.run(0)[0][0]), _bits(want)), "second run"
    st.rows = 1
    assert torch.equal(_bits(st.run(0)[0][0]), _bits(want)), "alone in slot 0"
    for bound in (P + 1, P + 1 + 1024, g.S):
        assert torch.equal(_bits(_run_with_bound(st, eng, bound)[0][0]), _bits(want)), f"context bound {bound}"
    L = _lib()
    try:
        for chunk in (32, 4096):
            L.check(L.lib().fsb_op_attn_score_chunk(chunk))
            st.rows = rt
            got = st.run(0)
            assert torch.equal(_bits(got[0]), _bits(full[0])), f"score chunk {chunk}"
    finally:
        L.lib().fsb_op_attn_score_chunk(0)


# ---------------------------------------------------------------------------------------------------------------------
# end to end: tiny model, T = 128, contexts that cross T while they decode
# ---------------------------------------------------------------------------------------------------------------------
T_E2E = 128
KW = dict(temperature=0.8, top_p=0.9, top_k=30)


def _model(cfg, w, max_batch, attn_split, kv_pages=None):
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    m = DualARTransformer(model_args(cfg), w, device="cuda", im_end_id=cfg.im_end_id)
    m.setup_caches(max_batch_size=max_batch, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages, attn_split=attn_split)
    m._cache_setup_done = True
    assert m.engine.attn_split == attn_split
    return m


def _alone(model, prompt, n, **kw):
    from fish_speech_b200.models.text2semantic.inference import generate

    return generate(model=model, prompt=prompt.cuda(), max_new_tokens=n, **kw).cpu()


@pytest.fixture(scope="module")
def tiny():
    _close_engines()
    cfg = O.tiny_config(max_seq_len=1024)
    w = O.make_weights(cfg, seed=77, head_gain=2.5)
    w["embeddings.weight"][cfg.im_end_id] = 0  # <|im_end|> is never sampled: every request runs to its budget
    return cfg, w, _model(cfg, w, 1, T_E2E)


def test_batch_equals_alone_across_the_threshold(tiny):
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg, w, solo = tiny
    # (prompt rows, frames): crosses T mid-utterance; long from the first frame; two that never reach T; crosses 2 T
    shapes = [(100, 60), (300, 24), (20, 30), (9, 50), (250, 20), (127, 8), (60, 100)]
    specs = [dict(prompt=make_prompt(cfg, 500 + i, t), max_new_tokens=n, seed=40 + i) for i, (t, n) in enumerate(shapes)]
    model = _model(cfg, w, 8, T_E2E)
    b = ContinuousBatcher(model, max_slots=8, frames_per_poll=4)
    reqs = [b.submit(SlotRequest(**{**s, "prompt": s["prompt"].cuda()}, **KW)) for s in specs]
    b.run()
    b.close()
    model.engine.close()
    off = _model(cfg, w, 1, 0)
    for i, (s, r) in enumerate(zip(specs, reqs)):
        one = _alone(solo, s["prompt"], s["max_new_tokens"], seed=s["seed"], **KW)
        assert torch.equal(r.result.cpu(), one), f"request {i} {shapes[i]} != its solo run with the split on"
        if sum(shapes[i]) <= T_E2E:  # never longer than T: the tokens of an engine without the split
            assert torch.equal(one, _alone(off, s["prompt"], s["max_new_tokens"], seed=s["seed"], **KW)), i
    off.engine.close()


def test_graph_replay_equals_eager(tiny, monkeypatch):
    from fish_speech_b200.engine import LmEngine

    cfg, _, solo = tiny
    prompt = make_prompt(cfg, 611, 110)
    graph = _alone(solo, prompt, 40, seed=5, **KW)
    decode = LmEngine.decode
    monkeypatch.setattr(LmEngine, "decode", lambda self, batch, n, sp, use_graph=True: decode(self, batch, n, sp, False))
    assert torch.equal(_alone(solo, prompt, 40, seed=5, **KW), graph)


def test_park_and_resume_across_the_threshold(tiny):
    from fish_speech_b200.engine import kv_pages_for
    from tests.test_live_sched_gpu import _park_and_resume_elsewhere

    cfg, w, solo = tiny
    model = _model(cfg, w, 3, T_E2E, kv_pages=11 * kv_pages_for(400))
    probe = (make_prompt(cfg, 620, 100), 60, 4242, KW)  # parked at 110 positions, resumed, then past T
    others = [(make_prompt(cfg, 621, 9), 13, 11, KW), (make_prompt(cfg, 622, 140), 40, 12, KW),
              (make_prompt(cfg, 623, 6), 30, 13, KW)]
    r, rest, _ = _park_and_resume_elsewhere(model, probe, 10, others)
    model.engine.close()
    assert torch.equal(r.result.cpu(), _alone(solo, probe[0], 60, seed=4242, **KW))
    for q, (p, n, seed, _) in zip(rest, others):
        assert torch.equal(q.result.cpu(), _alone(solo, p, n, seed=seed, **KW))


def test_shared_prefix_pages_equal_a_fresh_prefill(tiny):
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg, w, solo = tiny
    prefix = make_prompt(cfg, 5, 200)  # 3 whole pages shared, the 4th copied; every sharer is long from its first frame
    prompts = [torch.cat([prefix, make_prompt(cfg, 630 + i, 24)], dim=1) for i in range(4)]
    model = _model(cfg, w, 4, T_E2E)
    b = ContinuousBatcher(model, max_slots=4, frames_per_poll=4)
    r0 = b.submit(SlotRequest(prompt=prompts[0].cuda(), max_new_tokens=9, reuse_prefix=True, seed=0, **KW))
    b.step()
    rs = [r0] + [b.submit(SlotRequest(prompt=p.cuda(), max_new_tokens=40, reuse_prefix=True, seed=i, **KW))
                 for i, p in enumerate(prompts[1:], 1)]
    b.run()
    b.close()
    assert model.engine.rows_reused >= 3 * 192
    model.engine.close()
    for i, r in enumerate(rs):
        assert torch.equal(r.result.cpu(), _alone(solo, prompts[i], r.max_new_tokens, seed=i, **KW)), i
