"""The decode attention (csrc/lm_kernels.cu attn_decode_kernel) against float64 references built from the same bf16
operands: the qkv step GEMM's fix-up (slot-ordered partial sums, bias, bf16 rounding, per-head nn.RMSNorm, interleaved
RoPE), the K/V append into the paged slow cache or the contiguous fast cache, and the attention over the row's history
read through the page table. The copy-on-write kernels of the paged cache (fsb_lm_copy_kv_page, fsb_lm_copy_kv) are
checked against a torch copy at the end.

fsb_lm_test_layer_attn runs one layer's qkv GEMM (no finalize in front of it: its operand is x_* as the test wrote it,
normalised on load with ssq_*) and the attention with the arguments decode gives them. Each test fills the whole cache
with random bf16 K/V and builds a scrambled page table itself: the pages of full history are shared between the rows,
the page a row appends to is private to it, as KvPagePool guarantees. The whole-model tests only compare tokens; these
compare every appended element, every attention output, and every bit of the caches that must not change.

Fix-up. v = rbf(W X' + b) with X' the operand normalised on load. Where the float64 value of W X' + b lies within
E = C_AMB * (|W| |X'|^T) + (X'_hi - X'_lo) |W|^T of a bf16 rounding boundary (test_step_gemm_gpu: the accumulation
bound, plus the rsqrtf ambiguity of X'), v may round either way: v in [rbf(y - E), rbf(y + E)]. Every later step is
monotone in each input, so it maps the corners of its inputs' brackets to a bracket of its output:
  * qk-norm, x * rsqrtf(sum(v^2) / Dh + eps) * w with one rounding: the squares of bf16 values are exact in fp32, the
    sum takes at most 5 + Dh/32 roundings of partial sums no larger than the total, then the +eps, rsqrtf (2 ulp) and
    two products: at most 11.5 * 2^-24 relative in all, bounded by RN_HEAD = 2^-20. The bracket is the extremes of
    v * r * w over v in {lo, hi} and r in [rsqrt(max sum / Dh + eps) (1 - RN_HEAD),
    rsqrt(min sum / Dh + eps) (1 + RN_HEAD)].
  * RoPE, fp32 products and one fp32 difference / sum (__fmul_rn, __fsub_rn, __fadd_rn) of the bf16 table, then bf16:
    the reference evaluates exactly those fp32 operations at the four corners of each rotary pair (RoPE is not monotone
    in the pair as a whole, but it is in each element of it).
Each appended element must lie in its bracket (and so be bit-identical to the reference wherever the bracket holds one
value), and fewer than 1 % of the elements may differ from the float64 value's rounding.

Slow attention (fp32). The reference is o = softmax(q k^T / sqrt(Dh)) v in float64 over positions [0, pos] read
through the page table from the cache the kernel left, with q the reference q (the kernel's q stays in shared memory).
The kernel's arithmetic: a score is 8 fp32 products summed per lane plus log2(Dh / 8) <= 4 shuffle additions and one
product with the scale, so |ds_p| <= 14 * 2^-24 * scale * (|q| |k_p|); exp(s_p - m) adds the rounding of s_p - m
(2^-24 |s_p - m|) and expf's 2 ulp; the sum of exponentials has at most ceil(L / 32) + 5 roundings, the division one.
With eps_s the largest score error, each probability is off by a factor within 1 +- rho,
    rho = e^(2 eps_s) - 1 + 2 * 2^-22 + (ceil(L / 32) + 8) * 2^-24,
and the weighted sum of values has at most ceil(L / 8) fp32 accumulations per warp plus 8 across warps, so
    |o_kernel - o(q_kernel)| <= (rho + g (1 + rho)) * sum_p p_p |v_p|,   g = (ceil(L / 8) + 9) * 2^-24.
q's own ambiguity (its bracket's width dq) moves each score by at most ds = scale * dq . |k_p|; a softmax whose scores
move by at most ds changes every probability by a factor within e^(+-2 ds), and since sum_p (p'_p - p_p) = 0,
    |o(q_kernel) - o(q_ref)| <= (e^(2 ds) - 1) * sum_p p_p |v_p - o| <= (e^(2 ds) - 1) * (sum_p p_p |v_p| + |o|).
The output must lie in [rbf(o - E), rbf(o + E)] with E the sum of the two bounds (the first one scaled by e^(2 ds)).

Fast attention (bf16_math, llama.py:948-976, oracle.lm_oracle._eq_sdpa): the scores, the scaled scores, the
probabilities and the output are each rounded to bf16. The reference carries a bracket through each rounding: the
score from q's corners and the fp32 bound above, the probability from the softmax's monotonicity (p_j rises with s_j
and falls with every other score) and the fp32 bound, the output from the probabilities' brackets plus the accumulation
bound. Contexts are at most num_codebooks long, so nearly every bracket holds one value and the bits are checked.

The bounds have teeth: for each attention check a stated share (TEETH) of the rows must fall outside the bound
around a reference with one history position dropped or counted twice (histories up to SHORT positions: in a longer
one a single position carries less weight than the worst-case bound), q rotated at pos + 1, the next KV head's K/V,
or the first page's content replaced by another page's.

The case harness (state, run, checks, TEETH) lives in tests/decode_attn_case.py, the references in tests/kernel_ref.py
(rehearsed on the CPU by test_kernel_ref_cpu.py).
"""
from __future__ import annotations

import math
import random

import pytest
import torch

from tests.decode_attn_case import TEETH, Geom, State, _check_case, _report_teeth
from tests.kernel_ref import PAGE
from tests.lm_util import _bits, _lib, attn_configs

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# engines: every (head_dim, group) instance of the kernel in one stack or the other
# ---------------------------------------------------------------------------------------------------------------------
_ENG: dict = {}


def _engine(name):
    """(cfg, weights, engine) of one configuration; one engine on the device at a time. The slow pool holds every full
    history page once, a private page per slot and 8 pages nobody maps."""
    if name not in _ENG:
        from fish_speech_b200.engine import LmEngine
        from oracle import lm_oracle as O

        for _, _, e in _ENG.values():
            e.close()
        _ENG.clear()
        torch.cuda.empty_cache()
        cfg, slots = attn_configs()[name]
        w = O.make_weights(cfg, seed=59)
        rt = 32 if slots <= 32 else 64
        pages = math.ceil(cfg.max_seq_len / PAGE) - 1 + rt + 8
        eng = LmEngine(cfg, w, "cuda", cfg.im_end_id, max_batch=slots, kv_len=cfg.max_seq_len, max_rows=128,
                       max_frames=4, kv_pages=pages)
        _ENG[name] = (cfg, {k: v.cuda() for k, v in w.items() if ".attention" in k}, eng)  # attention_norm too
    return _ENG[name]


@pytest.fixture(scope="module", autouse=True)
def _free_engines():
    yield
    for _, _, e in _ENG.values():
        e.close()
    _ENG.clear()


def _positions(g: Geom, n, rng, long):
    """n positions: the edges first (page and score-chunk boundaries, the capacity's last), then random ones."""
    if g.fast:
        edges, draw = [0, 1, g.S - 1], (lambda: rng.randrange(g.S))
    else:
        edges = [0, 1, 63, 64, 65, 127, 128, g.S - 1]
        if long:  # page-table entries past the 256 the kernel loads before its dependency wait
            edges += [16384, 16447, 16448, 16449, 19999]
        draw = (lambda: rng.randrange(16385, 20001)) if long else (lambda: rng.randrange(g.S))
    if n < len(edges):
        return rng.sample(edges, n)
    out = edges + [draw() for _ in range(n - len(edges))]
    rng.shuffle(out)
    return out


def _tag(name, fast):
    return f"{name}-{'fast' if fast else 'slow'}"


CASES = [pytest.param(name, fast, id=_tag(name, fast)) for name in attn_configs() for fast in (0, 1)
         if not (name == "s2pro-g8" and fast)]


@pytest.mark.parametrize("name,fast", CASES)
def test_decode_attn_matches_fp64(name, fast):
    """Every (Dh, G) instance in one stack or the other; rows 1 / 13 / 32 of a 32-slot engine or 33 / 64 of a 64-slot
    one; one row parked at -1 and (slow) one whose history has an unmapped page; kv_only; positions at the page edges,
    the capacity's last and (S2-Pro) beyond 16 384."""
    cfg, w, eng = _engine(name)
    g = Geom(cfg, fast)
    long = cfg.max_seq_len > 16384
    rng = random.Random(sum(map(ord, name)) + fast)
    teeth = {k: [] for k in TEETH}
    singles = total = 0
    for n, rows in enumerate((1, 13, 32) if eng.max_batch <= 32 else (33, 64)):
        layer = n % g.nl
        pos = _positions(g, rows, rng, long)
        parked, unmapped = ((3,), (() if g.fast else (7,))) if rows >= 13 else ((), ())
        if unmapped:
            pos[7] = max(pos[7], 3 * PAGE + 5)
        st = State(eng, g, rows, pos, seed=1000 * n + rows, parked=parked, unmapped=unmapped)
        s, t = _check_case(cfg, w, g, layer, st, f"{_tag(name, fast)} layer {layer} rows={rows}", teeth)
        singles += s
        total += t
    print(f"{_tag(name, fast)}: {singles} of {total} attention outputs have a one-value bracket (checked bit for bit)")
    _report_teeth(teeth, _tag(name, fast), fast)


@pytest.mark.parametrize("name", ["s2pro-g8", "s2pro"])
def test_decode_attn_chunks_are_bit_identical(name):
    """A context bound below the positions, or a forced score chunk of 32, 64 or 4096 positions, walks the history in
    chunks: the outputs and the appends keep the bits of the automatic chunk."""
    cfg, w, eng = _engine(name)
    g = Geom(cfg, 0)
    L = _lib()
    rows = 13
    rng = random.Random(5)
    pos = [rng.randrange(16385, 20001) for _ in range(rows - 2)] + [g.S - 1, 700]
    st = State(eng, g, rows, pos, seed=77)
    base = st.run(0)
    runs = {}
    orig_load = st.load

    def load_low_bound():
        orig_load()
        eng.set_context_bound_exact(1024)  # rounded to a 1024-position bucket, far below the positions

    st.load = load_low_bound
    runs["bound 1024"] = st.run(0)
    st.load = orig_load
    try:
        for chunk in (32, 64, 4096):
            L.check(L.lib().fsb_op_attn_score_chunk(chunk))
            runs[f"chunk {chunk}"] = st.run(0)
    finally:
        L.lib().fsb_op_attn_score_chunk(0)
    for k, r in runs.items():
        for a, b, what in zip(r, base, ("attn", "K", "V")):
            assert torch.equal(_bits(a), _bits(b)), f"{name} {k}: {what} differs from the automatic chunk"


@pytest.mark.parametrize("name,fast", [pytest.param(n, f, id=_tag(n, f)) for n, f in
                                       (("tiny-a", 0), ("tiny-c", 1), ("s2pro", 0), ("s2pro", 1))])
def test_decode_attn_rows_are_independent(name, fast):
    """A row's append and attention output keep their bits whatever the other rows hold (NaN, +-1e30), wherever they
    sit, and however many rows run."""
    cfg, w, eng = _engine(name)
    g = Geom(cfg, fast)
    rt = eng.row_tile
    rng = random.Random(3)
    pos = _positions(g, rt, rng, cfg.max_seq_len > 16384)
    st = State(eng, g, rt, pos, seed=11)
    x0, ssq0, pos0, table0 = st.x.clone(), st.ssq.clone(), list(st.pos), None if st.table is None else st.table.clone()
    attn, kc, vc = st.run(0)
    for j in (0, 12, rt - 1):
        want = (attn[j], kc[st.slot_index(0, j)], vc[st.slot_index(0, j)])
        for other in ("nan", "1e30", "-1e30", "moved", "fewer rows"):
            st.x, st.ssq, st.pos, st.rows = x0.clone(), ssq0.clone(), list(pos0), rt
            others = [i for i in range(rt) if i != j]
            if other in ("nan", "1e30", "-1e30"):
                st.x[others] = float(other)
                st.ssq[others] = float("nan") if other == "nan" else 1e38
            elif other == "moved":
                for i in others:
                    st.pos[i] = rng.randrange(g.S)
                if table0 is not None:  # the moved rows append to their own private pages
                    st.table = table0.clone()
                    for i in others:
                        p = st.pos[i]
                        st.table[i] = -1
                        st.table[i, : p // PAGE] = torch.tensor(st.shared[: p // PAGE], dtype=torch.int32)
                        st.table[i, p // PAGE] = st.private[i]
            else:
                st.rows = j + 1
            a, k, v = st.run(0)
            got = (a[j], k[st.slot_index(0, j)], v[st.slot_index(0, j)])
            for x, y, what in zip(got, want, ("attn", "appended k", "appended v")):
                assert torch.equal(_bits(x), _bits(y)), f"{_tag(name, fast)} row {j}: {what} changed ({other})"
            if table0 is not None:
                st.table = table0.clone()


# ---------------------------------------------------------------------------------------------------------------------
# copy-on-write: fsb_lm_copy_kv_page and fsb_lm_copy_kv against a torch copy
# ---------------------------------------------------------------------------------------------------------------------
def test_copy_kv_page_and_copy_kv():
    """Exactly positions [0, n_pos) of every layer and KV head are copied; the rest of the destination page and every
    other page keep their bits; unmapped and identical pages are skipped."""
    L = _lib()
    cfg, _, eng = _engine("tiny-b")  # two layers, two KV heads
    kc, vc = eng.buffer("k_slow"), eng.buffer("v_slow")
    n_pages = kc.shape[1]
    gen = torch.Generator(device="cuda").manual_seed(123)

    def fill():
        kc.copy_(torch.randn(kc.shape, generator=gen, device="cuda").bfloat16())
        vc.copy_(torch.randn(vc.shape, generator=gen, device="cuda").bfloat16())
        torch.cuda.synchronize()
        return kc.clone(), vc.clone()

    def same(want_k, want_v, what):
        torch.cuda.synchronize()
        for got, want, name in ((kc, want_k, "K"), (vc, want_v, "V")):
            bad = _bits(got) != _bits(want)
            assert not bad.any(), f"{what}: {int(bad.sum())} {name} elements differ, first at {bad.nonzero()[0].tolist()}"

    for n_pos in (0, 1, 63, 64):
        k0, v0 = fill()
        src, dst = 5, n_pages - 3
        L.check(L.lib().fsb_lm_copy_kv_page(eng.h, src, dst, n_pos, _stream()))
        k0[:, dst, :, :n_pos], v0[:, dst, :, :n_pos] = k0[:, src, :, :n_pos], v0[:, src, :, :n_pos]
        same(k0, v0, f"copy_kv_page n_pos={n_pos}")
    k0, v0 = fill()
    L.check(L.lib().fsb_lm_copy_kv_page(eng.h, 9, 9, 64, _stream()))
    same(k0, v0, "copy_kv_page onto itself")

    # through the page table: 6 entries (n_pos = 5 pages + 17), one unmapped in the source, one in the destination,
    # one page both slots map
    pps = eng.kv_pool.pages_per_slot
    table = torch.full((eng.max_batch, pps), -1, dtype=torch.int32)
    table[2, :6] = torch.tensor([11, -1, 13, 14, 15, 16], dtype=torch.int32)
    table[40, :6] = torch.tensor([21, 22, -1, 14, 25, 26], dtype=torch.int32)
    table[40, 6:9] = torch.tensor([27, 28, 29], dtype=torch.int32)  # past n_pos: not copied
    table[2, 6:9] = torch.tensor([17, 18, 19], dtype=torch.int32)
    eng.buffer("kv_page").copy_(table)
    n_pos = 5 * PAGE + 17
    for src_slot, dst_slot in ((2, 40), (40, 2)):
        k0, v0 = fill()
        L.check(L.lib().fsb_lm_copy_kv(eng.h, src_slot, dst_slot, n_pos, _stream()))
        for j in range(math.ceil(n_pos / PAGE)):
            sp, dp = int(table[src_slot, j]), int(table[dst_slot, j])
            n = min(PAGE, n_pos - j * PAGE)
            if sp >= 0 and dp >= 0 and sp != dp:
                k0[:, dp, :, :n], v0[:, dp, :, :n] = k0[:, sp, :, :n], v0[:, sp, :, :n]
        same(k0, v0, f"copy_kv {src_slot} -> {dst_slot}")
