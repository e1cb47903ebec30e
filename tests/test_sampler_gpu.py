"""The LM sampler (csrc/lm_kernels.cu sample_kernel) on its own, through fsb_lm_test_sample, against the exact
emulation of tests/test_sampler_cpu.py (its docstring lists the kernel's steps and the brackets). The hook stages
fp32 logits as the single partial of a step GEMM, so the kernel's logit is exactly rbf(logit), and runs the sampler
with the arguments a decode frame gives it; everything else is the engine's own state.

Decisions. Every draw's bracket comes from the arithmetic: differences of bf16 values, divisions, rbf and the running
sum of the rounded probabilities are emulated exactly in fp32; expf carries 2 ulp and logf 1 ulp (CUDA Math API, no
fast-math); fp32 sums of d positive terms carry d * 2^-24 relative (d = ceil(n / 1024) + 37 for the softmax denominator
over the candidates, ceil(ns / 32) + 5 for the survivors' warp sum). A draw is determined when no cum bracket straddles
its top_p and the winner's lowest score beats every other survivor's highest score: the kernel must return exactly that
token. Otherwise it must return one of the candidates the emulation names, and the share of such draws must stay below
AMBIGUOUS_MAX = 1 %. Observed on an H100 80GB HBM3 (700 W power limit): 3 of 4 320 draws, 0.07 % (at most 2 of 720, 0.28
%, on one head), each inside its named candidates. The grid: n in {97, 96 (tiny), 4097 (S2-Pro slow head), 4096 (its
codebooks), 8192 (both heads at the largest size the engine accepts)}; top_k in {2, 30, 255, 256, 300, n}; top_p in bf16
{0.1, 0.7, 0.8, 0.95, 1.0}; temperature in bf16 {1e-6 (clipped to 1e-5), 0.3, 0.7, 1.0, 1.5}; peaky, flat (the 256 cap
binds), tied (a plateau of min(300, n / 3) equal logits across the top-k edge with <|im_end|>, the last candidate, in
it: the tie rule ranks it last, so on the 4097- and 8192-candidate heads it falls past the 256-rank cap and is never
drawn) and |logit| ~ 60 rows, all from fp32 values bf16 cannot represent, some exactly halfway between two bf16 values.
Up to 64 rows per launch through a scrambled row -> slot map, per-slot parameters (slot control) and per-call ones.

Bookkeeping, checked on every row whatever the draw: the slow head's token and code (clamped to the codebook), the RAS
substitution (only when the main token is in the window AND semantic), the window shift, `finished`, state 3 only from a
request's second frame on (the grid draws <|im_end|> rarely and only on the tiny head, so
test_im_end_stops_a_request_from_its_second_frame_and_is_never_replaced makes it the main draw of 64 rows on every slow
head, half at n_out = 0, with a RAS draw that would replace it by a semantic token in 37 of them); the fast head writes
cur_tok column cb_index + 1 only; the logits copy is rbf(logit) bit for bit; idle (0) and frozen (2) slots keep every
bit of cur_tok, ras_window, finished and the logits copy; a request's tokens do not depend on its slot or its
neighbours; top_k above 256 gives the bits of 256.

Parity with the reference's RNG stream: with fsb_lm_set_sampler_noise on slot 0, the kernel's choice must be the
oracle's argmax(logits_to_probs / -log(U)) in torch bf16, except where the oracle's own decision is a near-tie (the two
best scores within 2 bf16 ulp, a cum within 2 bf16 ulp of top_p, or equal logits on both sides of the top-k cut, which
torch.sort orders in no fixed way). U = 0 entries score 0, as in the reference. Peaky and flat rows only: the exact ties
of the other kinds are pinned to the kernel's rules instead (test_ties_are_pinned).

Distribution: 64 slots with their own seeds x 256 frame counters = 16 384 Philox draws per case at n = 4097, chi-square
against float64 logits_to_probs at the 1e-6 upper quantile; no draw outside the survivor set.

Teeth: each deliberately wrong emulation must disagree with the kernel on at least TEETH[name] of the decisions both
determine (among the rows it can affect): temperature before the cut, >= at top_p, top-k one short, the RAS draw with
the request's top_p or temperature, draw and r swapped in the counter, the lane ignored per call, u without the + 0.5.
Observed shares on the S2-Pro-sized engine, slow head / fast codebook 1 (the asserted least shares are about half):
temperature before the cut 15.3 % / 4.9 %, top-k one short 2.9 % / 5.2 %, RAS with the request's top_p 3.9 % and
temperature 12.3 % (slow only), draw and r swapped 79.7 % / 50.3 %, lane ignored 96.8 % / 34.5 % of the per-call rows.
">=" at top_p (0.14 % / 0 %) and u without the + 0.5 (0 %) almost never change a grid decision, so test_targeted_teeth
builds a row where each must. The whole file runs in about 36 s on that H100.

The two fixes: a per-slot or per-call top_k of 0 or -1 gives the top_k = 1 token (before, the draw read ranks nothing
wrote); fsb_lm_create refuses more than 8192 candidates (tests/test_sampler_cpu.py).
"""
from __future__ import annotations

import itertools

import numpy as np
import pytest
import torch

from tests import test_sampler_cpu as E

pytestmark = pytest.mark.gpu

AMBIGUOUS_MAX = 0.01
# least share of the decisions both determine on which each wrong emulation must disagree with the kernel, slow / fast
# head of the S2-Pro-sized engine (about half the observed share, module docstring). ">=" at top_p and u without the
# + 0.5 change a grid decision too rarely to count there: test_targeted_teeth builds rows where they must.
TEETH = {"temp-before-cut": (0.07, 0.02), "top-k-1": (0.012, 0.025), "ras-top-p": (0.015, None),
         "ras-temp": (0.05, None), "swap-counter": (0.35, 0.25), "lane-ignored": (0.45, 0.15)}
SENT_TOK, SENT_LOGIT, SENT_WIN = -7, -12345.0, -3
TOP_P = [0.10009765625, 0.69921875, 0.80078125, 0.94921875, 1.0]  # bf16 of 0.1, 0.7, 0.8, 0.95, 1.0
TEMP = [9.98377799987793e-07, 0.30078125, 0.69921875, 1.0, 1.5]  # bf16 of 1e-6, 0.3, 0.7, 1.0, 1.5
KINDS = ("peaky", "flat", "tied", "large")


def _engine_cfgs():
    from oracle import lm_oracle as O

    base = dict(n_layer=1, n_fast_layer=1, max_seq_len=64)
    return {
        "tiny": O.tiny_config(**base),  # slow 97, fast 96
        "s2": O.tiny_config(vocab_size=8192, codebook_size=4096, semantic_begin_id=4000, semantic_end_id=8095,
                            im_end_id=3999, **base),  # slow 4097, fast 4096
        "wide": O.tiny_config(vocab_size=16384, codebook_size=8192, semantic_begin_id=8000, semantic_end_id=16190,
                              im_end_id=7999, **base),  # slow 8192, fast 8192
    }


_ENG: dict = {}


def _engine(name):
    if name not in _ENG:
        from fish_speech_b200.engine import LmEngine
        from oracle import lm_oracle as O

        for e in _ENG.values():
            e.close()
        _ENG.clear()
        cfg = _engine_cfgs()[name]
        eng = LmEngine(cfg, O.make_weights(cfg, seed=11), "cuda", cfg.im_end_id, max_batch=64, kv_len=64, max_rows=128,
                       max_frames=4, debug=True)
        eng.cfg_oracle = cfg
        _ENG[name] = eng
    return _ENG[name]


@pytest.fixture(scope="module", autouse=True)
def _free_engines():
    yield
    for e in _ENG.values():
        e.close()
    _ENG.clear()


# ---------------------------------------------------------------------------------------------------------------------
# rows
# ---------------------------------------------------------------------------------------------------------------------
def make_logits(kind, n, rng):
    x = rng.standard_normal(n)
    if kind == "peaky":
        v = x * 3.0
        # a few values exactly halfway between two bf16 values: round to even
        k = rng.choice(n, size=min(8, n), replace=False)
        v[k] = np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 2 + 2 ** -7, 0.5 + 2 ** -10, -3 - 3 * 2 ** -7,
                         4 + 2 ** -6, -0.25 - 2 ** -11])[: k.size]
    elif kind == "flat":
        v = x * 0.02
    elif kind == "tied":
        v = x * 1.5
        plat = min(300, n // 3)
        k = rng.choice(n - 1, size=plat - 1, replace=False)
        v[np.append(k, n - 1)] = 5.0 + rng.uniform(0, 2 ** -9, size=plat)  # one bf16 value after rounding
    else:  # large
        v = np.where(rng.random(n) < 0.5, 60.0, -60.0) + x * 2.0
    return v.astype(np.float32)


class Row:
    def __init__(self, logits, req, slot, state=1, window=None):
        self.logits, self.req, self.slot, self.state, self.window = logits, req, slot, state, window


class Head:
    """A head of an engine: n candidates, token ids, draw id."""

    def __init__(self, eng, cb):
        c = eng.cfg_oracle
        self.eng, self.cb = eng, cb
        self.slow = cb == 0
        self.n = eng.head_rows if self.slow else c.codebook_size
        self.keys = E.slow_keys(self.n, c.semantic_begin_id, c.im_end_id) if self.slow else np.arange(self.n)
        self.entry_of = {int(t): e for e, t in enumerate(self.keys)}
        self.c = c

    def token(self, entry):
        return int(self.keys[entry])


def grid_rows(head, kind, seed, per_slot, nrows=64, idle=6):
    """nrows rows in scrambled slots cycling through the (top_k, top_p, T) grid; `idle` of the slots are idle (0) or
    frozen (2)."""
    rng = np.random.default_rng(seed)
    n = head.n
    combos = list(itertools.product([2, 30, 255, 256, 300, n], TOP_P, TEMP))
    start = int(rng.integers(len(combos)))
    slots = rng.permutation(64)[:nrows]
    rows = []
    for i in range(nrows):
        k, p, t = combos[(start + i * 7) % len(combos)]
        lg = make_logits(kind, n, rng)
        seed_i = int(rng.integers(0, 2 ** 63)) * 2 + 1
        off = int(rng.integers(0, 6))
        state = 1 if i >= idle else (0 if i % 2 else 2)
        req = E.Request(t, p, k, seed_i, off, 0)
        win = None
        if head.slow:
            top = np.argsort(-E.rbf(lg), kind="stable")[:5]
            win = np.array([head.token(e) for e in top] + [head.c.im_end_id] +
                           [head.token(int(e)) for e in rng.integers(0, n, 4)])
            rng.shuffle(win)
        rows.append(Row(lg, req, int(slots[i]), state, win))
    return rows


# ---------------------------------------------------------------------------------------------------------------------
# one launch
# ---------------------------------------------------------------------------------------------------------------------
class Observed:
    def __init__(self, eng):
        self.cur_tok = eng.buffer("cur_tok").cpu().numpy().copy()
        self.ras_window = eng.buffer("ras_window").cpu().numpy().copy()
        self.finished = eng.buffer("finished").cpu().numpy().copy()
        self.state = eng.buffer("slot_state").cpu().numpy().copy()
        self.slow_logits = eng.buffer("slow_logits").cpu().numpy().view(np.int32).copy()
        self.fast_logits = eng.buffer("fast_logits").cpu().numpy().view(np.int32).copy()


def launch(head, rows, per_slot, use_ras, sp=None, step=0, full=True):
    """Writes every slot's state (sentinels where the kernel must not write), runs the hook, returns (before, after);
    full=False: (None, cur_tok) only."""
    eng = head.eng
    dev = eng.device
    B, C1 = eng.max_batch, head.c.num_codebooks + 1
    rng = np.random.default_rng(len(rows) * 7919 + rows[0].slot)
    eng.set_slot_control(per_slot)
    state = np.zeros(B, np.int32)
    temp, top_p, top_k = np.ones(B, np.float32), np.ones(B, np.float32), np.ones(B, np.int32)
    seed, n_out = np.zeros(B, np.int64), rng.integers(0, 6, B).astype(np.int32)
    win = np.full((B, 10), SENT_WIN, np.int32)
    for r in rows:
        state[r.slot] = r.state
        temp[r.slot], top_p[r.slot], top_k[r.slot] = r.req.T, r.req.top_p, r.req.top_k
        seed[r.slot] = np.array(r.req.seed, dtype=np.uint64).view(np.int64)
        if per_slot:
            n_out[r.slot] = r.req.off
        if r.window is not None:
            win[r.slot] = r.window
    bufs = {"slot_state": state, "slot_temperature": temp, "slot_top_p": top_p, "slot_top_k": top_k,
            "slot_seed": seed, "n_out": n_out, "ras_window": win, "finished": np.zeros(B, np.int32),
            "cur_tok": np.full((B, C1), SENT_TOK, np.int32), "step": np.array([step], np.int64)}
    for name, v in bufs.items():
        eng.buffer(name).copy_(torch.from_numpy(v).to(dev))
    if full:
        eng.buffer("slow_logits").fill_(SENT_LOGIT)
        eng.buffer("fast_logits").fill_(SENT_LOGIT)
    before = Observed(eng) if full else None
    logits = torch.from_numpy(np.stack([r.logits for r in rows]))
    rs = torch.tensor([r.slot for r in rows], dtype=torch.int32)
    eng.test_sample(logits, sp, codebook=head.cb, row_slot=rs, use_ras=use_ras)
    return before, (Observed(eng) if full else eng.buffer("cur_tok").cpu().numpy().copy())


# ---------------------------------------------------------------------------------------------------------------------
# checks
# ---------------------------------------------------------------------------------------------------------------------
class Tally:
    def __init__(self):
        self.decisions = 0
        self.ambiguous = 0
        self.teeth = {w: [0, 0] for w in E.WRONG}  # [disagreements, decisions both determine]


def expected(head, row, per_slot, use_ras, wrong=None, noise=None):
    """(determined final entry or None, possible final entries) of one row by the emulation."""
    two = head.slow and use_ras
    d0, d1 = E.emulate(row.logits, row.req, head.keys, 0 if head.slow else head.cb, two, noise=noise, wrong=wrong)
    if not two:
        return d0.entry, d0.cands
    win = set(int(t) for t in row.window)

    def hit(e):
        tok = head.token(e)
        return tok in win and tok != head.c.im_end_id

    final = set()
    for e in d0.cands:
        final |= d1.cands if hit(e) else {e}
    if d0.determined and (not hit(d0.entry) or d1.determined):
        return (d1.entry if hit(d0.entry) else d0.entry), final
    return None, final


def check_launch(head, rows, before, after, per_slot, use_ras, tally=None, teeth=False):
    c = head.c
    live = [r for r in rows if r.state in (1, 3)]
    for r in rows:
        s = r.slot
        if r.state not in (1, 3):  # idle / frozen: every bit as it was
            assert (after.cur_tok[s] == before.cur_tok[s]).all() and (after.ras_window[s] == before.ras_window[s]).all()
            assert after.finished[s] == before.finished[s] and after.state[s] == before.state[s]
            assert (after.slow_logits[s] == before.slow_logits[s]).all()
            assert (after.fast_logits[:, s] == before.fast_logits[:, s]).all()
            continue
        bits = E.rbf(r.logits).view(np.int32)
        if head.slow:
            assert (after.slow_logits[s] == bits).all(), "logits copy is not rbf(logit)"
        else:
            assert (after.fast_logits[head.cb - 1, s] == bits).all(), "logits copy is not rbf(logit)"
            others = [k for k in range(c.num_codebooks) if k != head.cb - 1]
            assert (after.fast_logits[others, s] == before.fast_logits[others, s]).all()
    for r in live:
        s = r.slot
        req = r.req
        if not per_slot:
            r.req = req = E.Request(req.T, req.top_p, req.top_k, req.seed, req.off, s)
        det, cands = expected(head, r, per_slot, use_ras)
        got_cols = after.cur_tok[s]
        if head.slow:
            tok = int(got_cols[0])
            assert tok in head.entry_of, f"slot {s}: token {tok} is no candidate"
            entry = head.entry_of[tok]
            assert got_cols[1] == min(max(tok - c.semantic_begin_id, 0), c.codebook_size - 1)
            assert (got_cols[2:] == before.cur_tok[s][2:]).all()
            if use_ras:
                assert after.ras_window[s].tolist() == list(r.window[1:]) + [tok]
            else:
                assert (after.ras_window[s] == before.ras_window[s]).all()
            assert after.finished[s] == (1 if tok == c.im_end_id else before.finished[s])
            n_out = req.off if per_slot else None
            want_state = 3 if (per_slot and tok == c.im_end_id and n_out >= 1) else before.state[s]
            assert after.state[s] == want_state, f"slot {s}: state {after.state[s]} want {want_state}"
        else:
            entry = int(got_cols[head.cb + 1])
            keep = [k for k in range(c.num_codebooks + 1) if k != head.cb + 1]
            assert (got_cols[keep] == before.cur_tok[s][keep]).all(), "the fast head wrote another column"
            assert after.finished[s] == before.finished[s] and (after.ras_window[s] == before.ras_window[s]).all()
        what = f"slot {s} T={req.T} top_p={req.top_p} top_k={req.top_k} off={req.off}"
        if det is not None:
            assert entry == det, f"{what}: kernel chose {entry}, the emulation determines {det}"
        else:
            assert entry in cands, f"{what}: kernel chose {entry}, outside the possible winners {sorted(cands)}"
        if tally is None:
            continue
        tally.decisions += 1
        tally.ambiguous += det is None
        if not teeth or det is None:
            continue
        for w in E.WRONG:
            if w.startswith("ras-") and not (head.slow and use_ras and req.top_k > 1):
                continue
            if w == "lane-ignored" and (per_slot or r.slot == 0):
                continue
            wd, _ = expected(head, r, per_slot, use_ras, wrong=w)
            if wd is not None:
                tally.teeth[w][0] += wd != entry
                tally.teeth[w][1] += 1


HEADS = [("tiny", 0), ("tiny", 2), ("s2", 0), ("s2", 1), ("wide", 0), ("wide", 3)]


@pytest.mark.parametrize("name,cb", HEADS)
def test_decisions_match_the_emulation(name, cb):
    head = Head(_engine(name), cb)
    tally = Tally()
    teeth = name == "s2"
    for i, kind in enumerate(KINDS):
        for j, per_slot in enumerate((True, True, False)):
            seed = 1000 * (HEADS.index((name, cb)) + 1) + 10 * i + j
            rows = grid_rows(head, kind, seed, per_slot, idle=6 if per_slot else 0)
            use_ras = head.slow and j != 1
            sp = None
            step = 0
            if not per_slot:
                r0 = rows[0].req
                sp = head.eng.sampling(r0.T, r0.top_p, r0.top_k, seed=r0.seed)
                step = (3 << 32) + 5 + j
                for r in rows:
                    r.req = E.Request(sp.temperature, sp.top_p, sp.top_k, sp.seed, step, r.slot)
            before, after = launch(head, rows, per_slot, use_ras, sp=sp, step=step)
            check_launch(head, rows, before, after, per_slot, use_ras, tally, teeth)
    share = tally.ambiguous / tally.decisions
    print(f"{name} cb={cb}: {tally.decisions} decisions, {tally.ambiguous} ambiguous ({100 * share:.2f} %)")
    assert share <= AMBIGUOUS_MAX
    if teeth:
        for w, (bad, tot) in tally.teeth.items():
            sh = bad / max(tot, 1)
            print(f"  teeth {w}: {bad} / {tot} = {sh:.4f}")
            least = TEETH.get(w, (None, None))[0 if head.slow else 1]
            if least is not None:
                assert tot > 0 and sh >= least, f"{w}: the wrong emulation disagrees on only {sh:.4f}"


def test_top_k_above_the_cap_gives_the_bits_of_256():
    head = Head(_engine("s2"), 0)
    rows = grid_rows(head, "flat", 77, True, idle=0)
    outs = []
    for k in (256, 300, head.n):
        for r in rows:
            r.req.top_k = k
        outs.append(launch(head, rows, True, True)[1])
    for o in outs[1:]:
        assert (o.cur_tok == outs[0].cur_tok).all() and (o.ras_window == outs[0].ras_window).all()
        assert (o.finished == outs[0].finished).all() and (o.state == outs[0].state).all()


def test_a_request_does_not_depend_on_its_slot_or_neighbours():
    head = Head(_engine("s2"), 0)
    rows = grid_rows(head, "peaky", 91, True, idle=0, nrows=32)
    a = launch(head, rows, True, True)[1]
    rng = np.random.default_rng(5)
    moved = rng.permutation(64)
    others = grid_rows(head, "flat", 92, True, idle=0, nrows=32)
    rows2 = [Row(r.logits, r.req, int(moved[i]), r.state, r.window) for i, r in enumerate(rows)]
    free = [s for s in range(64) if s not in set(moved[:32].tolist())]
    for i, r in enumerate(others):
        r.slot = free[i]
    b = launch(head, rows2 + others, True, True)[1]
    for r, r2 in zip(rows, rows2):
        assert (a.cur_tok[r.slot] == b.cur_tok[r2.slot]).all()
        assert (a.ras_window[r.slot] == b.ras_window[r2.slot]).all()


@pytest.mark.parametrize("name,cb", [("s2", 0), ("s2", 1), ("tiny", 0)])
def test_ties_are_pinned(name, cb):
    """Ranks tie toward the lower candidate index (so <|im_end|>, the last candidate, loses a tie at the top-k edge);
    the draw ties toward the lower token id (so <|im_end|>, whose id is below the semantic ids, wins a tied score)."""
    head = Head(_engine(name), cb)
    n = head.n
    rng = np.random.default_rng(3)
    # a plateau of 8 equal logits, <|im_end|> / the last code among them; top_k 4: the 4 lowest indices survive
    plat = np.sort(np.append(rng.choice(n - 1, 7, replace=False), n - 1))
    rows = []
    for i in range(64):
        lg = (rng.standard_normal(n) - 4).astype(np.float32)
        lg[plat] = 3.0
        rows.append(Row(lg, E.Request(1.0, 1.0, 4, 1000 + i, i % 4, 0), i, 1,
                        np.full(10, SENT_WIN) if head.slow else None))
    _, after = launch(head, rows, True, False)
    got = after.cur_tok[:, 0] if head.slow else after.cur_tok[:, cb + 1]
    allowed = set(head.token(int(e)) for e in plat[:4]) if head.slow else set(int(e) for e in plat[:4])
    assert set(got.tolist()) <= allowed and len(set(got.tolist())) > 1
    # equal scores through the noise hook (slot 0): equal logits and equal U
    lg = (rng.standard_normal(n) - 4).astype(np.float32)
    lo = 5
    lg[[lo, n - 1]] = 3.0
    eng = head.eng
    U = torch.full((1, 2 * head.c.num_codebooks, max(eng.head_rows, head.c.codebook_size)), 0.5)
    eng.set_sampler_noise(U.cuda())
    try:
        row = Row(lg, E.Request(1.0, 1.0, 2, 0, 0, 0), 0, 1, np.full(10, SENT_WIN) if head.slow else None)
        _, after = launch(head, [row], False, False, sp=eng.sampling(1.0, 1.0, 2))
    finally:
        eng.set_sampler_noise(None)
    want = (head.c.im_end_id if head.c.im_end_id < head.token(lo) else head.token(lo)) if head.slow else lo
    got = after.cur_tok[0, 0] if head.slow else after.cur_tok[0, cb + 1]
    assert got == want


@pytest.mark.parametrize("name", ["tiny", "s2", "wide"])
def test_im_end_stops_a_request_from_its_second_frame_and_is_never_replaced(name):
    """<|im_end|> is the main draw of every row: it leads the other two candidates by 1/16 and 1/8, and top_p = 0.1
    keeps rank 0 only. The RAS draw (top_p 0.9) keeps <|im_end|> and the next candidate, so it picks a semantic token
    in about half the rows, and <|im_end|> is in every window: the token must still be <|im_end|> (it is not semantic).
    finished is set in every row; slot control turns the state to 3 only for requests past their first frame
    (n_out >= 1), since the reference does not test the prefill's token (inference.py:336-352)."""
    head = Head(_engine(name), 0)
    c, n = head.c, head.n
    im_end = n - 1
    lg = np.full(n, -200.0, np.float32)
    lg[[im_end, 7, 8]] = [5.0, 4.9375, 4.875]
    win = np.array([head.token(7), c.im_end_id, head.token(8)] + [SENT_WIN] * 7)
    rows = [Row(lg, E.Request(1.0, TOP_P[0], 30, 4242 + 31 * i, 0 if i < 32 else 1 + i % 5, 0), (i * 37) % 64, 1, win)
            for i in range(64)]
    ras_semantic = 0
    for r in rows:
        d0, d1 = E.emulate(lg, r.req, head.keys, 0, True)
        assert d0.entry == im_end and d1.determined and d1.entry in (im_end, 7)
        ras_semantic += d1.entry == 7
    assert ras_semantic >= 16, "the RAS draw must offer a semantic replacement often enough to test the guard"
    before, after = launch(head, rows, True, True)
    check_launch(head, rows, before, after, True, True)
    for r in rows:
        s = r.slot
        assert after.cur_tok[s, 0] == c.im_end_id and after.cur_tok[s, 1] == 0
        assert after.ras_window[s].tolist() == list(win[1:]) + [c.im_end_id]
        assert after.finished[s] == 1
        assert after.state[s] == (1 if r.req.off == 0 else 3), f"n_out={r.req.off}: state {after.state[s]}"


def _oracle_choice(lg32, T, top_p, top_k, U):
    """The reference's draw in torch bf16 (oracle logits_to_probs, then argmax(probs / -log(U))); also whether that
    decision is a near-tie (best two scores within 2 bf16 ulp, or a cum within 2 ulp of top_p)."""
    from oracle import lm_oracle as O

    logits = torch.from_numpy(lg32).bfloat16()
    t, p = torch.tensor(T, dtype=torch.bfloat16), torch.tensor(top_p, dtype=torch.bfloat16)
    rec = []
    probs = O.logits_to_probs(logits, t, p, top_k, rec)
    q = -torch.log(U.bfloat16())
    score = (probs / q).float()
    top2 = torch.topk(score, 2).values
    ulp = float(top2[0].abs()) * 2 ** -7
    cum, top = rec
    near = float(top2[0] - top2[1]) <= 2 * ulp or bool(((cum - float(p)).abs() <= 2 * float(p) * 2 ** -7).any())
    return int(torch.argmax(score)), near or (top.numel() > top_k and bool(top[top_k - 1] == top[top_k]))


@pytest.mark.parametrize("name,cb", [("s2", 0), ("s2", 1)])
def test_noise_hook_matches_the_reference_stream(name, cb):
    head = Head(_engine(name), cb)
    eng, c = head.eng, head.c
    rng = np.random.default_rng(17 + cb)
    gen = torch.Generator().manual_seed(17 + cb)
    ld = max(eng.head_rows, c.codebook_size)
    compared = tolerated = ras = 0
    for i in range(96):
        kind = ("peaky", "flat")[i % 2]  # torch.sort breaks exact ties in no fixed order: the tied rows are elsewhere
        lg = make_logits(kind, head.n, rng)
        T, p, k = TEMP[1 + i % 4], TOP_P[1 + (i // 4) % 4], [2, 30, 256, head.n][(i // 16) % 4]
        # drawn in bf16 like the reference's (inference.py:43-46): an fp32 draw rounded to bf16 could give U = 1
        U = torch.rand((1, 2 * c.num_codebooks, ld), generator=gen, dtype=torch.bfloat16).float()
        U[0, :, rng.integers(0, head.n, 4).tolist()] = 0.0  # -log(0) = inf: that candidate scores 0
        top = np.argsort(-E.rbf(lg), kind="stable")[:3]
        U[0, :, int(top[i % 3])] = 0.0
        dr = 0 if head.slow else 2 * cb
        want, near = _oracle_choice(lg, T, p, k, U[0, dr, : head.n])
        win = np.full(10, SENT_WIN)
        use_ras = head.slow and i % 2 == 1
        if use_ras and want < head.n - 1:  # put the main token in the window: the RAS draw decides
            win[3] = head.token(want)
            want, near2 = _oracle_choice(lg, 1.0, 0.9, k, U[0, 1, : head.n])
            near = near or near2
            ras += 1
        eng.set_sampler_noise(U.cuda())
        try:
            row = Row(lg, E.Request(T, p, k, 0, 0, 0), 0, 1, win if head.slow else None)
            _, after = launch(head, [row], False, use_ras, sp=eng.sampling(T, p, k))
        finally:
            eng.set_sampler_noise(None)
        got = after.cur_tok[0, 0] if head.slow else after.cur_tok[0, cb + 1]
        compared += 1
        if got != head.token(want):
            assert near, f"case {i}: kernel {got}, reference {head.token(want)} (no near-tie)"
            tolerated += 1
    print(f"{name} cb={cb}: {compared} draws, {tolerated} near-tie differences, {ras} RAS draws")
    assert tolerated <= compared // 10


@pytest.mark.parametrize("kind,top_k", [("peaky", 30), ("flat", 256), ("peaky", 256), ("flat", 30)])
def test_distribution_of_philox_draws(kind, top_k):
    head = Head(_engine("s2"), 0)
    lg = E.dist_logits(kind)
    T, p = 0.69921875, 0.94921875
    probs, cum = E.logits_to_probs64(E.rbf(lg), T, p, top_k)
    st = E.RowStage1(lg, top_k)
    assert np.abs(cum[: st.kcap] - p).min() > 0.01  # the float64 cut is the kernel's
    counts = np.zeros(head.n, np.int64)
    rows = [Row(lg, E.Request(T, p, top_k, 0x9E3779B97F4A7C15 ^ (s * 1000003), 0, 0), s, 1, np.full(10, SENT_WIN))
            for s in range(64)]
    for ctr in range(256):
        for r in rows:
            r.req.off = ctr
        _, cur_tok = launch(head, rows, True, False, full=False)
        toks = cur_tok[:64, 0]
        entries = np.where(toks == head.c.im_end_id, head.n - 1, toks - head.c.semantic_begin_id)
        np.add.at(counts, entries, 1)
    stat, df, pv = E.chi2_pvalue(counts, probs)
    print(f"{kind} top_k={top_k}: chi2 {stat:.1f} on {df} degrees of freedom, p = {pv:.3g}")
    assert pv > 1e-6


@pytest.mark.parametrize("name,cb", [("s2", 0), ("s2", 1), ("tiny", 0)])
def test_top_k_below_one_is_greedy(name, cb):
    head = Head(_engine(name), cb)
    rng = np.random.default_rng(23)
    rows = [Row(make_logits(KINDS[i % 4], head.n, rng), E.Request(0.7, 0.8, [0, -1, 1][i % 3], 5 + i, 1, 0), i, 1,
                np.array([head.token(e) for e in range(10)]) if head.slow else None) for i in range(48)]
    _, after = launch(head, rows, True, head.slow)
    col = 0 if head.slow else cb + 1
    for r in rows:
        want = int(np.argmax(E.rbf(r.logits)))
        assert after.cur_tok[r.slot, col] == head.token(want), f"top_k={r.req.top_k}"
    # the per-call parameters accept it too
    for k in (0, -1):
        _, after = launch(head, rows[:8], False, head.slow, sp=head.eng.sampling(0.7, 0.8, k, seed=3))
        for r in rows[:8]:
            assert after.cur_tok[r.slot, col] == head.token(int(np.argmax(E.rbf(r.logits))))


def test_hook_refuses_bad_arguments():
    from fish_speech_b200 import _lib

    eng = _engine("tiny")
    lg = torch.zeros(4, eng.head_rows, device="cuda")
    sp = eng.sampling(1.0, 1.0, 2)
    L, before = eng.lib, _lib.launch_count()
    for fast, cb, rows, ras, msg in ((0, 1, 4, 0, "cb_index"), (1, 0, 4, 0, "cb_index"), (1, 4, 4, 0, "cb_index"),
                                     (1, 1, 4, 1, "RAS"), (0, 0, 0, 0, "rows"), (0, 0, 65, 0, "rows")):
        rc = L.fsb_lm_test_sample(eng.h, fast, cb, rows, None, lg.data_ptr(), ras, sp, 0)
        assert rc != 0 and msg in L.fsb_last_error().decode()
    assert _lib.launch_count() == before


def test_targeted_teeth():
    """Rows where the two rare wrong emulations must disagree with the kernel.
    u without the + 0.5: seed 0x5EED, frame 12454404 gives rank 1 of draw 0 the word 0xffffff07, so u rounds to 1 and
    that rank sits the draw out (score -inf); without the + 0.5 its score would be pr * 2^24 and it would win.
    >= at top_p: four equal logits and nothing else (exp underflows to 0): every cum is exact, 0.25, 0.5, ...; at
    top_p = 0.5 rank 1 survives (0.5 > 0.5 is false) and wins about half the draws, with >= it never would."""
    head = Head(_engine("s2"), 0)
    n = head.n
    lg = np.full(n, -200.0, np.float32)
    lg[[10, 20]] = 0.0
    row = Row(lg, E.Request(1.0, 1.0, 2, 0x5EED, 12454404, 0), 7, 1, np.full(10, SENT_WIN))
    x0 = E.philox4x32(0x5EED, 0, 12454404, 0, 0, 1)[0]
    assert int(x0) == 0xFFFFFF07 and E.uniform_from_word(x0) == 1.0
    right, _ = expected(head, row, True, False)
    wrong, _ = expected(head, row, True, False, wrong="no-half")
    assert (right, wrong) == (10, 20)
    _, after = launch(head, [row], True, False)
    assert after.cur_tok[7, 0] == head.token(10)

    lg = np.full(n, -200.0, np.float32)
    lg[[3, 9, 30, 31]] = 0.0
    rows = [Row(lg, E.Request(1.0, 0.5, 30, 77 + i, i, 0), i, 1, np.full(10, SENT_WIN)) for i in range(64)]
    _, after = launch(head, rows, True, False)
    got = after.cur_tok[:64, 0]
    assert set(got.tolist()) == {head.token(3), head.token(9)}
    for r in rows:
        right, _ = expected(head, r, True, False)
        wrong, _ = expected(head, r, True, False, wrong="ge-top-p")
        assert wrong == 3 and right == head.entry_of[int(after.cur_tok[r.slot, 0])]
