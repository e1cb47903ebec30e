"""The launches of a decode frame around its two stacks (csrc/lm_engine.cu frame_stage, through fsb_lm_test_frame_stage)
against float64 references and exact models: the decode embed, the first-frame splice, the restricted slow head, the fast
pass 0 input (norm_fastlayer_input, fast_project_in), the fast embed and head of passes p >= 1, and the frame end. Each
test writes its stage's inputs itself (teacher forcing), so an error in one stage cannot reach the next; the fast
stack's layers are covered by test_step_gemm_gpu.py and test_decode_attn_gpu.py. The helpers live in tests/frame_ref.py
(rehearsed on the CPU by test_frame_tail_cpu.py) and tests/kernel_ref.py.

Heads. logits = rbf(W X'), X' = norm(x) normalised on load (the final `norm` for the slow head, `fast_norm` for the
codebook heads) with the sums of squares the test wrote. norm_operand brackets X' over rsqrtf's 2 ulp; the step GEMM's
accumulation is within C_AMB |W| |X'| of float64 (test_step_gemm_gpu.py keeps C_AMB 4x above what it measures). Each
logit must lie inside rbf(v -+ E), bit-identical where that bracket is one value, and differ from rbf(v) in < 1 % of
the logits a test checks (pooled over its row sets: one row of 96 codes cannot show a share below 1 %). The
slow head's W is built here from the checkpoint: the semantic rows, then <|im_end|>, of the tied embedding or the untied
output.weight.

Fast input. A plain copy is bit-exact; the norm lies in the rbf(rbf(x r) w) bracket; fast_project_in is rbf(y + b) of
the kernel's own hidden row, with no residual (the test leaves random values in x_fast for a stale residual to pick up).

Every stage: rows at and past `rows`, sums-of-squares tiles past the row's, logits of slots outside the row set and the
columns of cur_tok a stage does not own keep the sentinel or NaN they were given; dead rows of fp32 inputs are NaN.
"""
from __future__ import annotations

import math

import pytest
import torch

from tests import frame_ref as F
from tests.kernel_ref import (C_AMB, bracket_bf16, check_bracket, check_ssq, check_tally, embed_ref, norm_operand,
                              normed_gemm, rbf, tile_ssq)
from tests.lm_util import _bits, _gen

pytestmark = pytest.mark.gpu

SENTINEL = -12288.0  # exact in bf16
T_CAP = 8


def _configs():
    from oracle import lm_oracle as O

    return {
        # tied head, norm_fastlayer_input, no fast_project_in, codebook scaling, 32 slots
        "tied": (O.tiny_config(), 32),
        # the fast input as a plain copy of the slow row
        "plain": (O.tiny_config(norm_fastlayer_input=False), 32),
        # untied output.weight, fast_project_in without the norm, no scaling, 64 slots (both row tiles)
        "untied-proj": (O.tiny_config(tie_word_embeddings=False, fast_dim=384, norm_fastlayer_input=False,
                                      scale_codebook_embeddings=False), 64),
        # fast_project_in after the norm into a fast_dim whose last sum-of-squares tile is partial
        "proj-192": (O.tiny_config(fast_dim=192), 32),
        # S2-Pro head geometry (4097 head rows: the last 128-wide tile holds one), 4096 codes, 10 codebooks, 64 slots;
        # the reduced vocabulary test_lm_gpu.py uses
        "s2pro": (O.LMConfig(n_layer=1, n_fast_layer=1, vocab_size=8192, max_seq_len=256, semantic_begin_id=4000,
                             semantic_end_id=8095, im_end_id=3999), 64),
    }


NAMES = list(_configs())
_ENG: dict = {}


def _engine(name):
    """(cfg, weights on the device, debug engine)."""
    if name not in _ENG:
        from fish_speech_b200.engine import LmEngine
        from oracle import lm_oracle as O

        cfg, slots = _configs()[name]
        w = O.make_weights(cfg, seed=83)
        eng = LmEngine(cfg, w, "cuda", cfg.im_end_id, max_batch=slots, kv_len=cfg.max_seq_len, max_rows=128,
                       max_frames=T_CAP, debug=True)
        _ENG[name] = (cfg, {k: v.cuda() for k, v in w.items() if not k.startswith(("layers.", "fast_layers."))}, eng)
    return _ENG[name]


@pytest.fixture(scope="module", autouse=True)
def _free_engines():
    yield
    for e in _ENG.values():
        e[2].close()
    _ENG.clear()


def _rows(eng):
    return (1, 13, 32) + ((33, 64) if eng.max_batch == 64 else ())


def _row_slots(eng, rows, permuted, seed):
    """None (row i is slot i) or distinct scrambled slots in [0, max_batch)."""
    if not permuted:
        return None
    return torch.randperm(eng.max_batch, generator=_gen(seed), device="cuda")[:rows].int()


def _tile(eng, rows):
    return 32 if rows <= 32 else 64


def _same(a, b):
    return torch.equal(_bits(a.contiguous()), _bits(b.contiguous()))


def _resid_rows(eng, D, rows, seed):
    """Residual rows [RT, D] of different scales, NaN past `rows`, and their per-tile sums of squares [RT, 32], NaN past
    the row's tiles and past `rows`."""
    RT = eng.row_tile
    scale = torch.tensor([2.0 ** (j % 7 - 3) for j in range(RT)], device="cuda")[:, None]
    x = (torch.randn(RT, D, generator=_gen(seed), device="cuda") * scale).bfloat16()
    x[rows:] = float("nan")
    ssq = torch.full((RT, 32), float("nan"), device="cuda")
    ssq[:rows, : math.ceil(D / 128)] = tile_ssq(x[:rows]).float()
    return x, ssq


def _head_bracket(x, ssq, norm_w, W, eps):
    """(lo, hi, mid) of rbf(W X') with X' = norm(x) normalised on load (module docstring)."""
    v, E = normed_gemm(x, ssq, norm_w, eps, W)
    return *bracket_bf16(v, E), rbf(v)


# ---------------------------------------------------------------------------------------------------------------------
# embed
# ---------------------------------------------------------------------------------------------------------------------
def _edge_tokens(cfg, n, seed):
    """cur_tok [n][C+1]: the semantic range's edges, tokens outside [0, vocab), codes outside [0, codebook_size)."""
    g = torch.Generator().manual_seed(seed)
    C, cs, sb, se, V = cfg.num_codebooks, cfg.codebook_size, cfg.semantic_begin_id, cfg.semantic_end_id, cfg.vocab_size
    t = torch.randint(0, cs, (n, C + 1), generator=g)
    special = [sb - 1, sb, se, se + 1, -1, -1000, V, V + 77, V - 1, 0, cfg.im_end_id]
    t[:, 0] = torch.where(torch.rand(n, generator=g) < 0.5, sb + torch.randint(0, se - sb + 1, (n,), generator=g),
                          torch.randint(0, V, (n,), generator=g))
    t[: min(n, len(special)), 0] = torch.tensor(special[:n])
    bad_codes = torch.tensor([-1, cs, cs + 5, -7, 2 ** 30])
    for i in range(1, n, 3):  # every third row: a code outside [0, cs) in one codebook, on a semantic token
        t[i, 1 + (i // 3) % C] = bad_codes[(i // 3) % len(bad_codes)]
        if i >= len(special):
            t[i, 0] = sb + i % (se - sb + 1)
    return t.int().cuda()


@pytest.mark.parametrize("name", NAMES)
def test_decode_embed(name):
    """x_slow bit-exact against the fp32 emulation, inside the float64 bracket of oracle.embed; ssq_slow of x_slow."""
    from oracle import lm_oracle as O

    cfg, w, eng = _engine(name)
    C, D, RT = cfg.num_codebooks, cfg.dim, eng.row_tile
    xb, sb, ct = eng.buffer("x_slow"), eng.buffer("ssq_slow"), eng.buffer("cur_tok")
    emb, cb = w["embeddings.weight"], w["codebook_embeddings.weight"]
    tally = [0, 0]
    for rows in _rows(eng):
        what = f"{name} embed rows={rows}"
        tok = _edge_tokens(cfg, eng.max_batch, rows)
        ct.copy_(tok)
        xb.fill_(SENTINEL)
        sb.fill_(float("nan"))
        eng.test_frame_stage("embed", rows, tile=_tile(eng, rows))
        x = xb[:rows].float()
        want = F.embed_emul(tok[:rows], emb, cb, C, cfg.codebook_size, cfg.semantic_begin_id, cfg.semantic_end_id,
                            cfg.scale_codebook_embeddings)
        bad = x != want
        assert not bad.any(), f"{what}: {int(bad.sum())} elements differ from the emulation, first {bad.nonzero()[0]}"
        lo, hi, mid, x64 = embed_ref(tok[:rows], emb, cb, C, cfg.codebook_size, cfg.semantic_begin_id,
                                     cfg.semantic_end_id, cfg.scale_codebook_embeddings)
        check_bracket(x, lo, hi, what, mid, tally=tally)
        # the bracket's float64 centre is oracle.embed on the clamped ids (the clamps keep each row's semantic flag)
        clamped = tok[:rows].long().clone()
        clamped[:, 0] = clamped[:, 0].clamp(0, cfg.vocab_size - 1)
        clamped[:, 1:] = clamped[:, 1:].clamp(0, cfg.codebook_size - 1)
        st = O.LMState(cfg, {k: emb.double() if k == "embeddings.weight" else cb.double()
                             for k in ("embeddings.weight", "codebook_embeddings.weight")})
        ref = O.embed(st, clamped[:, :, None])[:, 0]
        assert torch.allclose(ref, x64, rtol=0, atol=1e-12), f"{what}: embed_ref's centre is not oracle.embed"
        check_ssq(sb[:rows], xb[:rows], what, nan_past=True)
        assert (xb[rows:].float() == SENTINEL).all() and torch.isnan(sb[rows:]).all(), f"{what}: rows past rows written"
        assert torch.equal(ct, tok), f"{what}: cur_tok written"
    check_tally(tally, f"{name} embed")


# ---------------------------------------------------------------------------------------------------------------------
# slow head
# ---------------------------------------------------------------------------------------------------------------------
def _sp(eng):
    return eng.sampling(1.0, 1.0, 1, 0)  # greedy: the token is the first maximum of the kernel's own logits


@pytest.mark.parametrize("name", NAMES)
def test_slow_head(name):
    cfg, w, eng = _engine(name)
    C = cfg.num_codebooks
    xb, sb, ct, lg = eng.buffer("x_slow"), eng.buffer("ssq_slow"), eng.buffer("cur_tok"), eng.buffer("slow_logits")
    W = F.restricted_head(w, cfg)
    assert W.shape[0] == eng.head_rows
    tally = [0, 0]
    for rows in _rows(eng):
        for permuted in (False, True):
            what = f"{name} head rows={rows} permuted={permuted}"
            rs = _row_slots(eng, rows, permuted, rows)
            slots = rs.long() if rs is not None else torch.arange(rows, device="cuda")
            x, ssq = _resid_rows(eng, cfg.dim, rows, 3 * rows + permuted)
            lo, hi, mid = _head_bracket(x[:rows], ssq[:rows], w["norm.weight"], W, cfg.norm_eps)
            tok0 = torch.randint(0, 50, (eng.max_batch, C + 1), generator=_gen(rows), device="cuda").int()
            tiles = (32, 64) if (eng.max_batch == 64 and rows <= 32) else (_tile(eng, rows),)
            first = None
            for tile in tiles:
                xb.copy_(x)
                sb.copy_(ssq)
                ct.copy_(tok0)
                lg.fill_(float("nan"))
                eng.test_frame_stage("head", rows, tile=tile, row_slot=rs, sp=_sp(eng))
                got = lg[slots]
                check_bracket(got, lo, hi, f"{what} tile={tile}", mid, tally=tally)
                others = torch.ones(eng.max_batch, dtype=torch.bool, device="cuda")
                others[slots] = False
                assert torch.isnan(lg[others]).all(), f"{what}: logits of slots outside the rows written"
                e = got.argmax(1)
                n_sem = eng.head_rows - 1
                want0 = torch.where(e < n_sem, cfg.semantic_begin_id + e, torch.full_like(e, cfg.im_end_id))
                want1 = (want0 - cfg.semantic_begin_id).clamp(0, cfg.codebook_size - 1)
                assert torch.equal(ct[slots, 0].long(), want0) and torch.equal(ct[slots, 1].long(), want1), \
                    f"{what}: sampled token is not the first maximum of the logits"
                assert torch.equal(ct[slots, 2:], tok0[slots, 2:]) and torch.equal(ct[others], tok0[others]), \
                    f"{what}: cur_tok written outside the slow head's columns"
                if first is None:
                    first = got.clone()
                else:
                    assert _same(got, first), f"{what}: the 32- and 64-row tiles differ"
    check_tally(tally, f"{name} slow head")


# ---------------------------------------------------------------------------------------------------------------------
# fast pass 0 input
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_fast_input(name):
    cfg, w, eng = _engine(name)
    D, fD, RT = cfg.dim, cfg.fast_dim, eng.row_tile
    proj, norm = cfg.has_fast_project_in, cfg.norm_fastlayer_input
    xb, sb, xf, sf = eng.buffer("x_slow"), eng.buffer("ssq_slow"), eng.buffer("x_fast"), eng.buffer("ssq_fast")
    hid = eng.buffer("fast_hidden")
    tally = [0, 0]
    for rows in _rows(eng):
        what = f"{name} fast input (proj={proj}, norm={norm}) rows={rows}"
        x, ssq = _resid_rows(eng, D, rows, 5 * rows)
        stale = (torch.randn(RT, fD, generator=_gen(rows + 1), device="cuda")).bfloat16()  # a stale residual
        stale[rows:] = SENTINEL
        xb.copy_(x)
        sb.copy_(ssq)
        xf.copy_(stale)
        sf.fill_(float("nan"))
        hid.fill_(SENTINEL)
        eng.test_frame_stage("fast_in", rows, tile=_tile(eng, rows))
        h = (hid[: rows * D].view(rows, D) if proj else xf[:rows]).float()
        if norm:
            mid, lo, hi = norm_operand(x[:rows], ssq[:rows], w["norm.weight"], cfg.norm_eps, D)
            check_bracket(h, lo, hi, f"{what}: normed hidden", mid, tally=tally)
        else:
            assert _same(h.bfloat16(), x[:rows]), f"{what}: the plain copy is not bit-exact"
        if proj:
            assert (hid[rows * D:].float() == SENTINEL).all(), f"{what}: fast_hidden written past rows"
            Wp, b = w["fast_project_in.weight"], w["fast_project_in.bias"]
            hb = hid[: rows * D].view(rows, D)
            # rbf(y + b) with no residual: the finalize's rounding of y + b may go either way within C_AMB |W||h|
            v = hb.double() @ Wp.double().T + b.double()[None, :]
            y_lo, y_hi = bracket_bf16(v, C_AMB * (hb.double().abs() @ Wp.double().abs().T))
            check_bracket(xf[:rows].float(), y_lo, y_hi, f"{what}: fast_project_in", rbf(v), tally=tally)
        check_ssq(sf[:rows], xf[:rows], what, nan_past=True)
        assert (xf[rows:].float() == SENTINEL).all() and torch.isnan(sf[rows:]).all(), f"{what}: rows past rows written"
    check_tally(tally, f"{name} fast input")


def test_fast_input_covers_every_variant():
    seen = {(c.has_fast_project_in, c.norm_fastlayer_input) for c, _ in _configs().values()}
    assert seen == {(False, False), (False, True), (True, False), (True, True)}
    assert any(c.fast_dim % 128 != 0 and c.has_fast_project_in and c.norm_fastlayer_input for c, _ in
               _configs().values())


# ---------------------------------------------------------------------------------------------------------------------
# fast passes p >= 1: embed and head
# ---------------------------------------------------------------------------------------------------------------------
def _codes(cfg, eng, seed):
    """cur_tok with a different in-range code in every column, so that a wrong column or slot is visible."""
    C = cfg.num_codebooks
    t = torch.randint(0, cfg.codebook_size, (eng.max_batch, C + 1), generator=_gen(seed), device="cuda")
    t[:, 0] = cfg.semantic_begin_id
    return t.int()


@pytest.mark.parametrize("name", NAMES)
def test_fast_embed(name):
    cfg, w, eng = _engine(name)
    C, fD = cfg.num_codebooks, cfg.fast_dim
    xf, sf, ct = eng.buffer("x_fast"), eng.buffer("ssq_fast"), eng.buffer("cur_tok")
    fe = w["fast_embeddings.weight"]
    for rows in _rows(eng):
        for permuted in (False, True):
            rs = _row_slots(eng, rows, permuted, 7 * rows)
            slots = rs.long() if rs is not None else torch.arange(rows, device="cuda")
            for p in (1, C - 1):
                what = f"{name} fast embed p={p} rows={rows} permuted={permuted}"
                tok = _codes(cfg, eng, rows + p)
                ct.copy_(tok)
                xf.fill_(SENTINEL)
                sf.fill_(float("nan"))
                eng.test_frame_stage("fast_embed", rows, tile=_tile(eng, rows), p=p, row_slot=rs)
                want = fe[tok[slots, p].long()]
                assert _same(xf[:rows], want), f"{what}: x_fast is not fast_embeddings[cur_tok[slot][p]]"
                check_ssq(sf[:rows], xf[:rows], what, nan_past=True)
                assert (xf[rows:].float() == SENTINEL).all() and torch.isnan(sf[rows:]).all(), \
                    f"{what}: rows past rows written"
                assert torch.equal(ct, tok), f"{what}: cur_tok written"


@pytest.mark.parametrize("name", NAMES)
def test_fast_head(name):
    cfg, w, eng = _engine(name)
    C, B = cfg.num_codebooks, eng.max_batch
    xf, sf, ct, lg = eng.buffer("x_fast"), eng.buffer("ssq_fast"), eng.buffer("cur_tok"), eng.buffer("fast_logits")
    W = w["fast_output.weight"]
    tally = [0, 0]
    for rows in _rows(eng):
        for permuted in (False, True):
            rs = _row_slots(eng, rows, permuted, 11 * rows)
            slots = rs.long() if rs is not None else torch.arange(rows, device="cuda")
            x, ssq = _resid_rows(eng, cfg.fast_dim, rows, 13 * rows + permuted)
            lo, hi, mid = _head_bracket(x[:rows], ssq[:rows], w["fast_norm.weight"], W, cfg.norm_eps)
            for p in (1, C - 1):
                what = f"{name} fast head p={p} rows={rows} permuted={permuted}"
                tok = _codes(cfg, eng, rows + 2 * p)
                xf.copy_(x)
                sf.copy_(ssq)
                ct.copy_(tok)
                lg.fill_(float("nan"))
                eng.test_frame_stage("fast_head", rows, tile=_tile(eng, rows), p=p, row_slot=rs, sp=_sp(eng))
                got = lg[p - 1, slots]
                check_bracket(got, lo, hi, what, mid, tally=tally)
                written = torch.zeros(C, B, dtype=torch.bool, device="cuda")
                written[p - 1, slots] = True
                assert torch.isnan(lg[~written]).all(), f"{what}: logits written outside [p - 1][slots]"
                want = tok.clone()
                want[slots, p + 1] = got.argmax(1).int()
                assert torch.equal(ct, want), f"{what}: cur_tok is not the old one with [slot][p + 1] = argmax"
    check_tally(tally, f"{name} fast head")


# ---------------------------------------------------------------------------------------------------------------------
# frame end and first-frame splice: exact models
# ---------------------------------------------------------------------------------------------------------------------
def _frame_state(cfg, eng, rows, slots, seed, slot_control):
    """Random per-slot state that reaches every branch of frame_end_kernel."""
    g = torch.Generator().manual_seed(seed)
    B, C1 = eng.max_batch, cfg.num_codebooks + 1
    cur = torch.randint(0, 5000, (B, C1), generator=g).int()
    out = torch.randint(-9, 0, (B, C1, T_CAP), generator=g).int()
    state = torch.randint(0, 4, (B,), generator=g).int()
    n_out = torch.randint(0, T_CAP - 1, (B,), generator=g).int()
    limit = n_out + 1 + torch.randint(0, 4, (B,), generator=g).int()  # some slots reach their limit with this frame
    edges = [T_CAP - 1, T_CAP, T_CAP + 3, 0]
    for k, s in enumerate(slots[: 2 * len(edges)].tolist()):  # n_out at T_cap - 1, T_cap and past it
        n_out[s] = edges[k % len(edges)]
        limit[s] = T_CAP + 10 if k < len(edges) else n_out[s] + 1
        state[s] = 1 if k % 2 == 0 else 3
    pos = torch.randint(0, 200, (eng.row_tile,), generator=g).int()
    parked = slots[len(slots) // 2]  # a parked row: state 0, position -1
    state[parked] = 0
    pos[parked] = -1
    step = torch.tensor([int(torch.randint(0, 1000, (1,), generator=g))], dtype=torch.int64)
    return dict(cur=cur, out=out, n_out=n_out, pos=pos, state=state, limit=limit, step=step)


def _write_state(eng, s):
    eng.buffer("cur_tok").copy_(s["cur"])
    eng.buffer("out_tokens").copy_(s["out"])
    eng.buffer("n_out").copy_(s["n_out"])
    eng.buffer("pos").copy_(s["pos"])
    eng.buffer("slot_state").copy_(s["state"])
    eng.buffer("slot_limit").copy_(s["limit"])
    eng.buffer("step").copy_(s["step"])


@pytest.mark.parametrize("name", ["tied", "untied-proj"])
def test_frame_end(name):
    cfg, w, eng = _engine(name)
    try:
        for slot_control in (False, True):
            eng.set_slot_control(slot_control)
            for rows in _rows(eng):
                for permuted in (False, True):
                    for prefill_tail in (False, True):
                        what = f"{name} frame end ctl={slot_control} rows={rows} permuted={permuted} " \
                               f"prefill_tail={prefill_tail}"
                        seed = rows * 8 + 4 * slot_control + 2 * permuted + prefill_tail
                        rs = _row_slots(eng, rows, permuted, seed)
                        slots = rs.cpu() if rs is not None else torch.arange(rows, dtype=torch.int32)
                        s = _frame_state(cfg, eng, rows, slots, seed, slot_control)
                        spr = rps = None
                        if prefill_tail:
                            g = torch.Generator().manual_seed(seed)
                            rps = torch.randint(0, 100, (rows + 5,), generator=g).int()
                            spr = torch.randperm(rows + 5, generator=g)[:rows].int()
                        _write_state(eng, s)
                        eng.test_frame_stage("end", rows, tile=_tile(eng, rows), row_slot=rs, set_pos_rows=spr,
                                             row_pos_src=rps)
                        out, n_out, pos, state, step = F.frame_end_model(
                            s["cur"], s["out"], s["n_out"], s["pos"], s["state"], s["limit"], s["step"], rows,
                            slots, slot_control, spr, rps)
                        for key, want in (("out_tokens", out), ("n_out", n_out), ("pos", pos),
                                          ("slot_state", state), ("step", step), ("cur_tok", s["cur"])):
                            got = eng.buffer(key).cpu()
                            assert torch.equal(got, want.to(got.dtype)), f"{what}: {key} differs from the model"
    finally:
        eng.set_slot_control(False)


def test_frame_end_model_reaches_its_branches():
    """The random states of test_frame_end freeze, advance, skip and store past T_cap."""
    cfg, slots = _configs()["tied"]

    class E:
        max_batch, row_tile = slots, 32

    hit = set()
    for seed in range(16):
        sl = torch.arange(13, dtype=torch.int32)
        s = _frame_state(cfg, E, 13, sl, seed, True)
        out, n_out, pos, state, _ = F.frame_end_model(s["cur"], s["out"], s["n_out"], s["pos"], s["state"],
                                                      s["limit"], s["step"], 13, sl, True)
        for i in range(13):
            if int(s["state"][i]) not in (1, 3):
                hit.add("skip")
            elif int(state[i]) == 2:
                hit.add("freeze-im-end" if int(s["state"][i]) == 3 else "freeze-limit")
            else:
                hit.add("advance")
            if int(s["n_out"][i]) >= T_CAP and int(n_out[i]) > int(s["n_out"][i]):
                hit.add("past-cap")
    assert hit == {"skip", "freeze-im-end", "freeze-limit", "advance", "past-cap"}


@pytest.mark.parametrize("name", ["tied", "untied-proj"])
def test_first_frame_splice(name):
    cfg, w, eng = _engine(name)
    B, D, RT = eng.max_batch, cfg.dim, eng.row_tile
    bufs = {k: eng.buffer(k) for k in ("x_slow", "ssq_slow", "pos", "first_frame_pending", "slot_state",
                                       "first_frame_x", "first_frame_ssq", "first_frame_pos")}
    for rows in _rows(eng):
        what = f"{name} splice rows={rows}"
        g = _gen(17 * rows)
        x = torch.randn(RT, D, generator=g, device="cuda").bfloat16()
        ssq = torch.randn(RT, 32, generator=g, device="cuda")
        pos = torch.randint(-1, 300, (RT,), generator=g, device="cuda").int()
        # every (pending, state) pair among the rows, and pending slots past the rows
        pending = (torch.arange(B, device="cuda") // 4 % 2).int()
        state = (torch.arange(B, device="cuda") % 4).int()
        sx = torch.randn(B, D, generator=g, device="cuda").bfloat16()
        sssq = torch.randn(B, 32, generator=g, device="cuda")
        spos = torch.randint(0, 300, (B,), generator=g, device="cuda").int()
        for k, v in (("x_slow", x), ("ssq_slow", ssq), ("pos", pos), ("first_frame_pending", pending),
                     ("slot_state", state), ("first_frame_x", sx), ("first_frame_ssq", sssq),
                     ("first_frame_pos", spos)):
            bufs[k].copy_(v)
        eng.test_frame_stage("splice", rows, tile=_tile(eng, rows))
        wx, wssq, wpos, wpend = F.splice_model(x, ssq, pos, pending, state, sx, sssq, spos, rows)
        assert _same(bufs["x_slow"], wx), f"{what}: x_slow differs from the model"
        assert _same(bufs["ssq_slow"], wssq), f"{what}: ssq_slow differs from the model"
        assert torch.equal(bufs["pos"], wpos), f"{what}: pos differs from the model"
        assert torch.equal(bufs["first_frame_pending"], wpend), f"{what}: pending differs from the model"
        for k, v in (("slot_state", state), ("first_frame_x", sx), ("first_frame_ssq", sssq), ("first_frame_pos", spos)):
            assert _same(bufs[k], v), f"{what}: {k} written"
        if rows >= 8:  # every (pending, state) pair
            assert len({(int(a), int(b)) for a, b in zip(pending[:rows], state[:rows])}) == 8
        assert pending[rows:].any() or rows == B, f"{what}: no pending slot past the rows"
    bufs["first_frame_pending"].zero_()


# ---------------------------------------------------------------------------------------------------------------------
# the hook runs what a frame runs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,rows", [("tied", 13), ("untied-proj", 13), ("untied-proj", 40)])
def test_head_stage_reproduces_a_decode_frame(name, rows):
    """One eager fsb_lm_decode frame, then the slow head stage on the x_slow / ssq_slow it left: the same logits."""
    from tests.lm_util import make_prompt

    cfg, w, eng = _engine(name)
    eng.reset()
    eng.release_kv()
    sp = eng.sampling(0.7, 0.8, 30, 5)
    eng.prefill([make_prompt(cfg, 40 + s, 9 + s % 5) for s in range(rows)], list(range(rows)), sp)
    eng.decode(rows, 1, sp, use_graph=False)
    torch.cuda.synchronize()
    lg = eng.buffer("slow_logits")
    frame = lg[:rows].clone()
    assert torch.isfinite(frame).all()
    lg.fill_(float("nan"))
    eng.test_frame_stage("head", rows, tile=eng.decode_tile, sp=sp)
    assert _same(lg[:rows], frame), f"{name} rows={rows}: the head stage does not reproduce the frame's logits"
    eng.reset()
    eng.release_kv()


def test_frame_stage_rejects_bad_arguments():
    from fish_speech_b200 import _lib

    cfg, w, eng = _engine("tied")
    C = cfg.num_codebooks
    with pytest.raises(_lib.FsbError, match="stage"):
        _lib.check(eng.lib.fsb_lm_test_frame_stage(eng.h, 7, 32, 1, 0, None, None, None, 0, None, None))
    for kw, match in ((dict(stage="head", rows=0), "rows"), (dict(stage="head", rows=33), "rows"),
                      (dict(stage="head", rows=1, tile=64), "tile"), (dict(stage="fast_embed", rows=1, p=0), "p="),
                      (dict(stage="fast_head", rows=1, p=C), "p="),
                      (dict(stage="embed", rows=2, row_slot=torch.tensor([1, 0])), "row_slot"),
                      (dict(stage="end", rows=1, set_pos_rows=torch.tensor([0])), "together"),
                      (dict(stage="fast_in", rows=1, first_frame=True), "first_frame"),
                      (dict(stage="head", rows=1), "sampling")):
        with pytest.raises(_lib.FsbError, match=match):
            eng.test_frame_stage(**kw)
    _, _, e64 = _engine("untied-proj")
    with pytest.raises(_lib.FsbError, match="rows"):
        e64.test_frame_stage("end", 33, tile=32)
