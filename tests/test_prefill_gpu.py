"""The LM prefill layer stage by stage (csrc/lm_engine.cu prefill_stage, through fsb_lm_test_prefill_stage) against
float64 references built from the same bf16 operands. Each stage reads inputs the test wrote itself (teacher forcing),
so an error in one stage cannot reach the next: embed + attention_norm_0, the qkv GEMM + qkv_prep_row_kernel (bias,
per-head qk-norm, RoPE, K/V append through the page table), attn_tile_kernel over the page table, wo + residual + norm,
w1|w3 + SwiGLU, w2 + residual + the next layer's norm. The hand-off to decode (rows_kernel, frame_end_kernel) is checked
after a whole fsb_lm_prefill. The helpers live in tests/kernel_ref.py (rehearsed on the CPU by test_prefill_cpu.py).

Rows. One pass holds sequences of 1, 63, 64, 65, 200 and 333 rows in scrambled slots, starting at positions 0, 100
(mid-page), 128 (page edge) and, with S2-Pro's 32 768 positions, 16 400; several sequences share each 64-row tile.
The page table is scrambled; the history pages below each start are shared between the sequences and full of random
K/V, so are the positions after each row's own (a causal-mask leak reads them). One more sequence of 10 rows at 120
has page 1 unmapped: its attention output is zero and nothing is written at positions 120..127.

Embed. s = fp32 sum of the C codebook rows rounded once to bf16, x = rbf(e + s), semantic rows / sqrtf(C + 1) once
more when the model scales them. An fp32 sum of C terms is within (C - 1) 2^-24 sum |terms| of its float64 value in any
order, which brackets s; the rest is monotone. The unrounded chain equals oracle.lm_oracle.embed on float64 weights.

Norms. rbf(rbf(x r) w), r = rsqrtf(sum(x^2) / D + eps). The block sum adds at most 25 fp32 partial sums of positive
terms (16 per thread, 5 warp and 4 block levels), then / D, + eps and rsqrtf's 2 ulp: r is within 17.5 * 2^-24 < 2^-19
(RN_ROW) of its float64 value. The per-head qk-norm sums 4 values per lane over a warp: 2^-20 (RN_HEAD).

GEMMs. ws_prefill against float64 W X with |ws - W X| <= C_CONV |W| |X|, C_CONV = 2^-18: the same gemm_tc kernel,
whose accumulation error test_codec_ops_gpu measures and keeps at least 4x inside C_CONV. Rows common to a launch below
and above the narrow / wide switch of launch_rows_of (computed from the SM count) must match bit for bit.

Consumers. Each is checked twice: bit-exact (inside a bracket that holds one value almost everywhere) against an fp32
emulation of the kernel's rounding points evaluated on the kernel's own ws_prefill -- bias add, rbf, the per-head
RMSNorm over the rsqrtf bracket, RoPE with fp32 products and one add, SwiGLU over expf's 2 ulp, residual add and norm
--, and against the float64 chain from the stage's operand, inside its bracket and off its rounding in < 1 %.

Attention (attn_tile_kernel, fp32 path). o = softmax(q k^T / sqrt(Dh)) v over [0, pos] in float64, with q, K, V the
bf16 values the test wrote. The kernel:
  * scores: Dh/16 mma.sync m16n8k16 steps (bf16 products exact, fp32 accumulation). CUDA does not document the
    accumulation's rounding; each instruction is allowed MU = 2^-21 of the sum of the magnitudes it adds, so
    |ds_p| <= (Dh/16) MU |q||k_p| scale;
  * the score times the fp32 constant log2(e) / sqrt(Dh) (3 roundings in the constant, one in the product), the
    subtraction of the running maximum and exp2f (2 ulp): 2^-24 (3 |s| + 3 |s - m|) + 2^-22 in the log domain;
  * one online rescale per 64-position tile: exp2f of a difference of maxima and a product, kappa = 2^-22 + 2^-23 |s|
    per tile, at most T = pos / 64 + 1 tiles (masked tiles add exact zeros);
  so every weight is within e^(+-eta) of its float64 value, eta = max_p |ds_p| + log-domain terms + T kappa, and each
  probability within e^(+-2 eta);
  * p as a bf16 hi + lo pair: lo = p - rbf(p) is exact in fp32 and its bf16 rounding costs 2^-8 |lo| <= 2^-16 p;
  * P V: 8 mma.sync per tile (4 k-steps, hi and lo) into one fp32 accumulator: (8 T + 1) MU sum_p p |v_p|;
  * the row sum: 16 + 2 fp32 adds per tile plus the rescale: (20 T + 2) 2^-24; one division and one product.
  E = (e^(2 eta) - 1 + 2^-16 + (8 T + 1) MU e^(2 eta) + (20 T + 2) 2^-24) sum_p p_p |v_p|, and the output must lie in
  [rbf(o - E), rbf(o + E)]. MU is an allowance, not a documented figure: the test asserts every output also lies
  inside the bracket of E / 4 (MARGIN), so the measured error stays at least 4x inside it.
The bound has teeth: each wrong reference below puts at least TEETH[k] of the checked rows outside the bracket of E
around it (a dropped or doubled position only for histories up to SHORT positions, where one position weighs more
than the worst-case bound): a dropped or a doubled position, position pos + 1 included (causal leak), q rotated at
pos + 1, the next KV head's K/V, the first page read from a page nobody maps, the preceding sequence's history (a
run-boundary mistake in a shared tile), and p rounded to one bf16. Shares seen on an H100 80GB HBM3 (132 SMs, 700 W
power limit): 100 % for every wrong reference in the tiny engines (the pos + 1 rotation and the single-bf16 p
each miss two rows); in both S2-Pro engines 100 % except the causal leak (75 %) and the single-bf16 p
(72 %), whose effect on a 16 400-position history can stay inside the bound.

Bits. A sequence's q, K/V, attention, x and h keep their bits in one pass, split at any row (the first piece writes
K/V, the second attends over it), shifted by any number of rows next to other sequences, and under a context bound
just above its length or at capacity.
"""
from __future__ import annotations

import ctypes
import dataclasses
import math
import random

import pytest
import torch

from tests import kernel_ref as R
from tests.kernel_ref import PAGE, rbf
from tests.lm_util import _bits, _lib, _randn, _sms, attn_configs

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0
SHORT = 1024
MARGIN = 0.25
LONG_START = 16400
# least share of the checked rows each wrong reference must put outside the bound (module docstring). With S2-Pro's
# 16 400-position histories one extra position, or p's lost low bits, can stay inside the bound: 'leak' and
# 'p-hi-only' are rejected for 75 % and 72 % of the rows there, for every row but two in the other engines.
TEETH = {"drop": 0.9, "double": 0.9, "leak": 0.6, "rope+1": 0.9, "next-head": 0.9, "page": 0.9, "prev-seq": 0.9,
         "p-hi-only": 0.6}
LENS = (1, 63, 64, 65, 200, 333)


def wide_from(n_out: int) -> int:
    """Fewest rows that launch_rows_of gives the 256-row plan (lm_engine.cu): >= 512 rows and two waves of tiles."""
    tiles = math.ceil(n_out / 128)
    return max(512, 256 * (math.ceil(2 * _sms() / tiles) - 1) + 1)


# ---------------------------------------------------------------------------------------------------------------------
# engines: the decode attention matrix, wo bias in two of them, and one intermediate size that is not a multiple of 64
# ---------------------------------------------------------------------------------------------------------------------
def _configs():
    from oracle import lm_oracle as O

    out = {}
    for name, (cfg, slots) in attn_configs().items():
        if name == "tiny-b":
            cfg = dataclasses.replace(cfg, attention_o_bias=True)
        out[name] = (cfg, slots)
    out["tiny-pad"] = (O.tiny_config(max_seq_len=1024, intermediate_size=528, attention_o_bias=True,
                                     attention_qkv_bias=True, scale_codebook_embeddings=False), 32)
    return out


NAMES = list(_configs())
_ENG: dict = {}


class Geom:
    def __init__(self, cfg):
        self.D, self.H, self.Hkv, self.Dh, self.I = cfg.dim, cfg.n_head, cfg.n_local_heads, cfg.head_dim, \
            cfg.intermediate_size
        self.G, self.S, self.nl = self.H // self.Hkv, cfg.max_seq_len, cfg.n_layer
        self.Nqkv = (self.H + 2 * self.Hkv) * self.Dh
        self.n13 = math.ceil(self.I / 64) * 128
        self.scale = float(torch.tensor(1.0) / torch.sqrt(torch.tensor(float(self.Dh))))


def _engine(name):
    """(cfg, weights on the device, engine, geometry); one engine on the device at a time."""
    if name not in _ENG:
        from fish_speech_b200.engine import LmEngine
        from oracle import lm_oracle as O

        for e in _ENG.values():
            e[2].close()
        _ENG.clear()
        torch.cuda.empty_cache()
        cfg, slots = _configs()[name]
        g = Geom(cfg)
        w = O.make_weights(cfg, seed=61)
        max_rows = max(wide_from(g.Nqkv), wide_from(g.n13), sum(LENS) + 10)
        pages = math.ceil(cfg.max_seq_len / PAGE) + 64
        eng = LmEngine(cfg, w, "cuda", cfg.im_end_id, max_batch=slots, kv_len=cfg.max_seq_len, max_rows=max_rows,
                       max_frames=4, kv_pages=pages)
        dw = {k: v.cuda() for k, v in w.items() if not k.startswith("fast")}
        _ENG[name] = (cfg, dw, eng, g)
    return _ENG[name]


@pytest.fixture(scope="module", autouse=True)
def _free_engines():
    yield
    for e in _ENG.values():
        e[2].close()
    _ENG.clear()


# ---------------------------------------------------------------------------------------------------------------------
# a pass: sequences (slot, start, rows, unmapped page), the page table and random caches
# ---------------------------------------------------------------------------------------------------------------------
class Pass:
    def __init__(self, eng, g: Geom, seqs, seed):
        """seqs: [(slot, start, n, unmapped page or None)] in row order."""
        self.eng, self.g, self.seqs = eng, g, list(seqs)
        rng = random.Random(seed)
        pps = eng.kv_pool.pages_per_slot
        kc = eng.buffer("k_slow")
        n_pages = kc.shape[1]
        perm = list(range(n_pages))
        rng.shuffle(perm)
        n_shared = max(s0 // PAGE for _, s0, _, _ in seqs)
        self.shared, free = perm[:n_shared], perm[n_shared:]
        table = torch.full((eng.max_batch, pps), -1, dtype=torch.int32)
        for slot, s0, n, un in seqs:
            table[slot, : s0 // PAGE] = torch.tensor(self.shared[: s0 // PAGE], dtype=torch.int32)
            for j in range(s0 // PAGE, (s0 + n - 1) // PAGE + 1):
                table[slot, j] = free.pop()
            if un is not None:
                table[slot, un] = -1
        self.spare = free
        self.table = table.cuda()
        self.row_seq = torch.cat([torch.full((n,), slot, dtype=torch.int32) for slot, _, n, _ in seqs]).cuda()
        self.row_pos = torch.cat([torch.arange(s0, s0 + n, dtype=torch.int32) for _, s0, n, _ in seqs]).cuda()
        self.rows = int(self.row_seq.numel())
        self.first = [sum(n for _, _, n, _ in seqs[:k]) for k in range(len(seqs))]
        gen = torch.Generator(device="cuda").manual_seed(seed)
        self.k0 = torch.randn(kc.shape, generator=gen, device="cuda").bfloat16()
        self.v0 = torch.randn(kc.shape, generator=gen, device="cuda").bfloat16()

    def load(self, bound=None):
        e = self.eng
        e.buffer("kv_page").copy_(self.table)
        e.buffer("k_slow").copy_(self.k0)
        e.buffer("v_slow").copy_(self.v0)
        e.set_context_bound_exact(bound or int(self.row_pos.max()) + 1)
        torch.cuda.synchronize()

    def padded(self, rows):
        """row_seq / row_pos for `rows` rows: the pass, then rows without a position (pos -1: no K/V written)."""
        extra = rows - self.rows
        if extra <= 0:
            return self.row_seq[:rows], self.row_pos[:rows]
        z = torch.zeros(extra, dtype=torch.int32, device="cuda")
        return torch.cat([self.row_seq, z]), torch.cat([self.row_pos, z - 1])

    def mapped(self):
        """(row index, page, offset) of every row whose own position is mapped."""
        out = []
        seq, pos = self.row_seq.tolist(), self.row_pos.tolist()
        tab = self.table.tolist()
        for i, (s, p) in enumerate(zip(seq, pos)):
            if p >= 0 and tab[s][p // PAGE] >= 0:
                out.append((i, tab[s][p // PAGE], p % PAGE))
        return out

    def unmapped_rows(self):
        out = []
        for k, (slot, s0, n, un) in enumerate(self.seqs):
            if un is not None:
                out += list(range(self.first[k], self.first[k] + n))
        return out


def _main_pass(eng, g, seed, with_unmapped=True):
    rng = random.Random(seed)
    slots = rng.sample(range(eng.max_batch), len(LENS) + 1)
    far = LONG_START if g.S > LONG_START + 400 else 300
    starts = (100, 128, 0, 100, far, 0)
    seqs = [(slots[k], starts[k], n, None) for k, n in enumerate(LENS)]
    if with_unmapped:
        seqs.insert(3, (slots[-1], 120, 10, 1))
    return Pass(eng, g, seqs, seed)


# ---------------------------------------------------------------------------------------------------------------------
# embed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny-a", "tiny-pad", "s2pro"])
def test_prefill_embed(name):
    """Codebook sum, semantic-range edges, the / sqrt(C+1) scale (on, and off in tiny-pad), attention_norm_0."""
    from oracle import lm_oracle as O

    cfg, w, eng, g = _engine(name)
    C, cs = cfg.num_codebooks, cfg.codebook_size
    rows = 300
    gen = torch.Generator().manual_seed(7)
    tok = torch.randint(0, cfg.vocab_size, (rows, C + 1), generator=gen)
    tok[:, 1:] = torch.randint(0, cs, (rows, C), generator=gen)
    sb, se = cfg.semantic_begin_id, cfg.semantic_end_id
    edges = [sb - 1, sb, se, se + 1, cfg.im_end_id, 0]
    tok[: 6 * 8, 0] = torch.tensor(edges).repeat(8)
    tok[100:200, 0] = torch.randint(sb, se + 1, (100,), generator=gen)
    xb, nb = eng.buffer("x_prefill"), eng.buffer("xn_prefill")
    xb.fill_(SENTINEL)
    nb.fill_(SENTINEL)
    eng.test_prefill_stage("embed", rows, tokens=tok.int())
    x, xn = xb[:rows].float(), nb[:rows].float()
    lo, hi, mid, x64 = R.embed_ref(tok.cuda(), w["embeddings.weight"], w["codebook_embeddings.weight"], C, cs, sb, se,
                                   cfg.scale_codebook_embeddings)
    R.check_bracket(x, lo, hi, f"{name} embed x", mid)
    sem = (tok[:, 0] >= sb) & (tok[:, 0] <= se)
    assert sem[:48].tolist() == [e in (sb, se) for e in edges] * 8
    # the unrounded chain is the oracle's embedding, evaluated in float64
    st = O.LMState(cfg, {k: v.double().cpu() for k, v in w.items() if "embeddings" in k})
    want = O.embed(st, tok.t()[None].long())[0]
    assert torch.allclose(x64.cpu(), want, rtol=1e-12, atol=1e-15), f"{name}: embed reference differs from the oracle"
    nlo, nhi, nmid = R.row_norm(x, w["layers.0.attention_norm.weight"], cfg.norm_eps)
    R.check_bracket(xn, nlo, nhi, f"{name} embed attention_norm_0", nmid)
    for b, what in ((xb, "x"), (nb, "xn")):
        assert (b[rows:].float() == rbf(torch.tensor(SENTINEL))).all(), f"{name}: {what}_prefill written past rows"


# ---------------------------------------------------------------------------------------------------------------------
# GEMM stages and their consumers
# ---------------------------------------------------------------------------------------------------------------------
def _check_gemm(ws, x, W, what):
    y, a = R.fp64_gemm(x, W)
    err = (ws.double() - y).abs()
    bad = ~(err <= R.C_CONV * a)
    assert not bad.any(), (f"{what}: {int(bad.sum())} GEMM outputs off, first at {bad.nonzero()[0].tolist()}, max "
                           f"err / |W||X| = 2^{math.log2(float((err / a).max())):.2f}")


def _freqs(cfg, g):
    from fish_speech_b200.engine import rope_table

    return rope_table(g.S, g.Dh, cfg.rope_base).cuda()


def _qkv_stage(cfg, w, eng, g, ps: Pass, layer, xn, rows):
    ps.load()
    eng.buffer("xn_prefill")[:rows].copy_(xn[:rows])
    eng.buffer("q_prefill").fill_(SENTINEL)
    seq, pos = ps.padded(rows)
    eng.test_prefill_stage("qkv", rows, layer, row_seq=seq, row_pos=pos)
    ws = eng.buffer("ws_prefill")[: rows * g.Nqkv].view(rows, g.Nqkv).clone()
    return ws, eng.buffer("q_prefill")[:rows].clone(), eng.buffer("k_slow").clone(), eng.buffer("v_slow").clone()


@pytest.mark.parametrize("name", NAMES)
def test_prefill_qkv(name):
    """qkv GEMM (128- and 256-row plans) against float64; q and the appended K/V against the fp32 emulation (bits) and
    the float64 chain; every other cache element, and the unmapped rows' positions, untouched."""
    cfg, w, eng, g = _engine(name)
    ps = _main_pass(eng, g, seed=sum(map(ord, name)))
    layer = g.nl - 1
    pre = f"layers.{layer}.attention"
    W, b = w[f"{pre}.wqkv.weight"], w.get(f"{pre}.wqkv.bias")
    qn, kn = w.get(f"{pre}.q_norm.weight") if cfg.attention_qk_norm else None, \
        w.get(f"{pre}.k_norm.weight") if cfg.attention_qk_norm else None
    thr = wide_from(g.Nqkv)
    n_wide = max(thr, ps.rows)
    xn = _randn((n_wide, g.D), seed=3)
    ws_n, *_ = _qkv_stage(cfg, w, eng, g, ps, layer, xn, thr - 1)
    ws, q, kc, vc = _qkv_stage(cfg, w, eng, g, ps, layer, xn, n_wide)
    common = min(thr - 1, n_wide)
    assert torch.equal(_bits(ws_n[:common]), _bits(ws[:common])), f"{name}: narrow and wide qkv plans differ"
    _check_gemm(ws, xn, W, f"{name} qkv")

    n = ps.rows
    cs = _freqs(cfg, g)[ps.row_pos.long()].float()
    emul = R.qkv_emul(ws[:n], b, g.H, g.Hkv, g.Dh, qn, kn, cfg.norm_eps, cs)
    ref = R.qkv_ref64(xn[:n], W, b, g.H, g.Hkv, g.Dh, qn, kn, cfg.norm_eps, cs)
    R.check_bracket(q[:n].float(), emul[0][0], emul[0][1], f"{name} q (emulation)")
    R.check_bracket(q[:n].float(), ref[0][0], ref[0][1], f"{name} q (float64)", ref[0][2])
    # the appends: mapped rows only; every other element of both caches keeps its bits
    idx = ps.mapped()
    rows = torch.tensor([i for i, _, _ in idx], device="cuda")
    for j, (cache, c0, what) in enumerate(((kc, ps.k0, "k"), (vc, ps.v0, "v"))):
        got = torch.stack([cache[layer, pg, :, off] for _, pg, off in idx]).float()
        e, r = emul[1 + j], ref[1 + j]
        R.check_bracket(got, e[0][rows], e[1][rows], f"{name} appended {what} (emulation)")
        R.check_bracket(got, r[0][rows], r[1][rows], f"{name} appended {what} (float64)", r[2][rows])
        want = c0.clone()
        for _, pg, off in idx:
            want[layer, pg, :, off] = cache[layer, pg, :, off]
        bad = _bits(cache) != _bits(want)
        assert not bad.any(), f"{name}: {int(bad.sum())} {what} cache elements written outside the appends, first at " \
                              f"{bad.nonzero()[0].tolist()}"
    assert len(idx) == n - 8, "the unmapped sequence appends exactly its two mapped rows"


@pytest.mark.parametrize("name", NAMES)
def test_prefill_w13_swiglu(name):
    """w1|w3 GEMM in w13_gate_row order (128- and 256-row plans, padding columns exactly 0) and SwiGLU."""
    cfg, w, eng, g = _engine(name)
    from fish_speech_b200.engine import interleave_w13

    layer = g.nl - 1
    w1, w3 = w[f"layers.{layer}.feed_forward.w1.weight"], w[f"layers.{layer}.feed_forward.w3.weight"]
    thr = wide_from(g.n13)
    n_wide = max(thr, sum(LENS))
    xn = _randn((n_wide, g.D), seed=5)
    hb = eng.buffer("h_prefill")
    out = []
    for rows in (thr - 1, n_wide):
        eng.buffer("xn_prefill")[:rows].copy_(xn[:rows])
        hb.fill_(SENTINEL)
        eng.test_prefill_stage("w13", rows, layer)
        out.append((eng.buffer("ws_prefill")[: rows * g.n13].view(rows, g.n13).clone(), hb.clone()))
    (ws_n, h_n), (ws, h) = out
    assert torch.equal(_bits(ws_n), _bits(ws[: thr - 1])), f"{name}: narrow and wide w1|w3 plans differ"
    assert torch.equal(_bits(h_n[: thr - 1]), _bits(h[: thr - 1])), f"{name}: h differs between the plans"
    _check_gemm(ws, xn, interleave_w13(w1, w3), f"{name} w1|w3")
    Ip = math.ceil(g.I / 64) * 64
    if Ip > g.I:
        pad = R.gate_row(torch.arange(g.I, Ip, device="cuda"))
        assert (ws[:, pad] == 0).all() and (ws[:, pad + 16] == 0).all(), f"{name}: w1|w3 padding columns not 0"
    n = sum(LENS)
    lo, hi, _ = R.swiglu_emul(ws[:n], g.I)
    R.check_bracket(h[:n].float(), lo, hi, f"{name} h (emulation)")
    lo, hi, mid = R.swiglu_ref64(xn[:n], w1, w3)
    R.check_bracket(h[:n].float(), lo, hi, f"{name} h (float64)", mid)
    assert (h[n_wide:].float() == rbf(torch.tensor(SENTINEL))).all(), f"{name}: h_prefill written past rows"


@pytest.mark.parametrize("name", NAMES)
def test_prefill_wo_w2_residual(name):
    """wo (+ bo) + residual + ffn_norm, w2 + residual + the next layer's attention_norm (none on the last layer)."""
    cfg, w, eng, g = _engine(name)
    n = sum(LENS)
    xb, nb = eng.buffer("x_prefill"), eng.buffer("xn_prefill")
    for layer in sorted({0, g.nl - 1}):
        pre = f"layers.{layer}"
        for stage in ("wo", "w2"):
            what = f"{name} layer {layer} {stage}"
            x0 = _randn((n, g.D), seed=layer * 10 + len(stage))
            if stage == "wo":
                a = _randn((n, g.H * g.Dh), seed=layer * 10 + 1, scale=0.5)
                eng.buffer("attn_prefill")[:n].copy_(a)
                W, b, norm = w[f"{pre}.attention.wo.weight"], w.get(f"{pre}.attention.wo.bias"), \
                    w[f"{pre}.ffn_norm.weight"]
            else:
                a = _randn((n, g.I), seed=layer * 10 + 2, scale=0.1)
                eng.buffer("h_prefill")[:n].copy_(a)
                W, b = w[f"{pre}.feed_forward.w2.weight"], None
                norm = w[f"layers.{layer + 1}.attention_norm.weight"] if layer + 1 < g.nl else None
            xb.fill_(SENTINEL)
            xb[:n].copy_(x0)
            nb.fill_(SENTINEL)
            eng.test_prefill_stage(stage, n, layer)
            ws = eng.buffer("ws_prefill")[: n * g.D].view(n, g.D)
            _check_gemm(ws, a, W, what)
            x = xb[:n].float()
            assert torch.equal(x, R.resid_emul(x0, ws, b)), f"{what}: x differs from the emulation"
            lo, hi, mid = R.resid_ref64(x0, a, W, b)
            R.check_bracket(x, lo, hi, f"{what}: x (float64)", mid)
            if norm is None:
                assert (nb.float() == rbf(torch.tensor(SENTINEL))).all(), f"{what}: xn written on the last layer"
            else:
                lo, hi, mid = R.row_norm(x, norm, cfg.norm_eps)
                R.check_bracket(nb[:n].float(), lo, hi, f"{what}: xn", mid)
                assert (nb[n:].float() == rbf(torch.tensor(SENTINEL))).all(), f"{what}: xn written past rows"
            assert (xb[n:].float() == rbf(torch.tensor(SENTINEL))).all(), f"{what}: x written past rows"


# ---------------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------------
def _attn_run(eng, g, ps: Pass, layer, q, bound=None):
    ps.load(bound)
    eng.buffer("q_prefill")[: ps.rows].copy_(q)
    ab = eng.buffer("attn_prefill")
    ab.fill_(SENTINEL)
    eng.test_prefill_stage("attn", ps.rows, layer, row_seq=ps.row_seq, row_pos=ps.row_pos)
    return ab.clone()


def _caught(got, lo, hi):
    return ((got < lo) | (got > hi)).flatten(1).any(1)


@pytest.mark.parametrize("name", NAMES)
def test_prefill_attention(name):
    """attn_tile_kernel over the scrambled page table against the float64 softmax over [0, pos]; zeros for the
    sequence with an unmapped history page; a 4x margin inside the bound; and the wrong references it must reject."""
    cfg, w, eng, g = _engine(name)
    ps = _main_pass(eng, g, seed=sum(map(ord, name)) + 1)
    layer = g.nl - 1
    q = _randn((ps.rows, g.H, g.Dh), seed=9)
    out = _attn_run(eng, g, ps, layer, q)
    n = ps.rows
    assert (out[n:].float() == rbf(torch.tensor(SENTINEL))).all(), f"{name}: attention written past rows"
    un = ps.unmapped_rows()
    assert (out[un] == 0).all(), f"{name}: a row whose history has an unmapped page attended to something"
    kc, vc = ps.k0[layer], ps.v0[layer]
    cs1 = _freqs(cfg, g)[1].float()
    teeth = {k: [] for k in TEETH}
    singles = total = 0
    for k, (slot, s0, cnt, unm) in enumerate(ps.seqs):
        if unm is not None:
            continue
        L = min(s0 + cnt + 1, g.S)
        K, V = R.paged_history(kc, ps.table[slot], L), R.paged_history(vc, ps.table[slot], L)
        prev = ps.seqs[k - 1][0] if k > 0 else None
        for c0 in range(0, cnt, 32):
            rows = list(range(ps.first[k] + c0, ps.first[k] + min(cnt, c0 + 32)))
            pos = ps.row_pos[rows].long()
            qq = q[rows].double().view(len(rows), g.Hkv, g.G, g.Dh)
            got = out[rows].float().view(len(rows), g.Hkv, g.G, g.Dh)
            o, E = R.attn_ref64(qq, K, V, pos, g.scale)
            lo, hi = rbf(o - E), rbf(o + E)
            R.check_bracket(got, lo, hi, f"{name} attention seq {k} rows {rows[0]}..{rows[-1]}")
            R.check_bracket(got, rbf(o - MARGIN * E), rbf(o + MARGIN * E),
                            f"{name} attention seq {k} (E / {1 / MARGIN:.0f}: less than 4x margin)")
            singles += int((lo == hi).sum())
            total += lo.numel()

            def caught(o2):
                return _caught(got, rbf(o2 - E), rbf(o2 + E)).tolist()

            short = (pos >= 1) & (pos < SHORT)  # a history of one position has nothing left to drop
            if short.any():
                sel = short.nonzero().flatten()[::4]  # every 4th short row: one float64 softmax per row
                for kind, mult in (("drop", 0.0), ("double", 2.0)):
                    # weight of position pos // 2 set to 0 or 2 for each short row
                    o2 = []
                    for i in sel.tolist():
                        h = int(pos[i]) // 2
                        keep = [p for p in range(int(pos[i]) + 1) if p != h] + ([h, h] if mult == 2.0 else [])
                        o2.append(R.attn_ref64(qq[i: i + 1], K[:, keep], V[:, keep],
                                               torch.tensor([len(keep) - 1]), g.scale)[0])
                    teeth[kind] += _caught(got[sel], rbf(torch.cat(o2) - E[sel]), rbf(torch.cat(o2) + E[sel])).tolist()
            if L > int(pos.max()) + 1:
                teeth["leak"] += caught(R.attn_ref64(qq, K, V, pos + 1, g.scale)[0])
            teeth["rope+1"] += caught(R.attn_ref64(R.rotate_by(qq, cs1), K, V, pos, g.scale)[0])
            if g.Hkv >= 2:
                teeth["next-head"] += caught(R.attn_ref64(qq, K.roll(-1, 0), V.roll(-1, 0), pos, g.scale)[0])
            K2, V2 = K.clone(), V.clone()
            K2[:, :PAGE] = kc[ps.spare[0]].double()[:, : min(PAGE, L)]
            V2[:, :PAGE] = vc[ps.spare[0]].double()[:, : min(PAGE, L)]
            teeth["page"] += caught(R.attn_ref64(qq, K2, V2, pos, g.scale)[0])
            if prev is not None:
                Kp, Vp = R.paged_history(kc, ps.table[prev], L), R.paged_history(vc, ps.table[prev], L)
                teeth["prev-seq"] += caught(R.attn_ref64(qq, Kp, Vp, pos, g.scale)[0])
            teeth["p-hi-only"] += caught(R.attn_ref64(qq, K, V, pos, g.scale, p_hi_only=True)[0])
    print(f"{name}: {singles} of {total} attention outputs have a one-value bracket")
    for kind, v in teeth.items():
        if v:
            share = sum(v) / len(v)
            print(f"{name}: wrong reference '{kind}' rejected for {sum(v)} of {len(v)} rows ({share:.0%})")
            assert share >= TEETH[kind], f"{name}: the bound accepts a wrong reference ({kind}) for {len(v) - sum(v)} " \
                                         f"of {len(v)} rows"


# ---------------------------------------------------------------------------------------------------------------------
# bits: one pass, split, shifted, context bound
# ---------------------------------------------------------------------------------------------------------------------
def _chain(eng, g, ps: Pass, layer, xn_rows, x_rows, bound=None):
    """qkv -> attention -> wo -> w1|w3 -> w2 of one pass; returns per-row q, attn, h, x and the caches."""
    n = ps.rows
    ps.load(bound)
    eng.buffer("xn_prefill")[:n].copy_(xn_rows)
    eng.buffer("x_prefill")[:n].copy_(x_rows)
    eng.test_prefill_stage("qkv", n, layer, row_seq=ps.row_seq, row_pos=ps.row_pos)
    q = eng.buffer("q_prefill")[:n].clone()
    eng.test_prefill_stage("attn", n, layer, row_seq=ps.row_seq, row_pos=ps.row_pos)
    a = eng.buffer("attn_prefill")[:n].clone()
    for stage in ("wo", "w13", "w2"):
        eng.test_prefill_stage(stage, n, layer)
    return dict(q=q, attn=a, h=eng.buffer("h_prefill")[:n].clone(), x=eng.buffer("x_prefill")[:n].clone())


@pytest.mark.parametrize("name", ["tiny-a", "tiny-d", "s2pro"])
def test_prefill_bits_split_shifted_bounded(name):
    """A 200-row sequence starting at 100: its q, K/V, attention, h and x keep their bits in one pass, split at any
    row (the first piece writes K/V, the second attends over it), shifted next to the rows of another sequence, and
    under a context bound just above its length or at capacity."""
    cfg, w, eng, g = _engine(name)
    layer = g.nl - 1
    s0, cnt = 100, 200
    base = Pass(eng, g, [(3, 0, 100, None), (7, s0, cnt, None)], seed=13)  # slot 3: the filler, slot 7: the sequence
    pages = base.table[7, : (s0 + cnt - 1) // PAGE + 1].long()
    xn_all, x_all = _randn((cnt, g.D), seed=21), _randn((cnt, g.D), seed=22)

    def run(pieces, bound=None):
        """pieces: [(filler rows in front, first row, end row)], run one after the other on the caches left."""
        res = {key: [] for key in ("q", "attn", "h", "x")}
        k0, v0 = base.k0, base.v0
        for d, a, b in pieces:
            p = Pass(eng, g, ([(3, 0, d, None)] if d else []) + [(7, s0 + a, b - a, None)], seed=13)
            p.table, p.k0, p.v0 = base.table, k0, v0
            xn, x = xn_all[a:b], x_all[a:b]
            if d:
                xn, x = torch.cat([_randn((d, g.D), seed=d), xn]), torch.cat([_randn((d, g.D), seed=d + 1), x])
            r = _chain(eng, g, p, layer, xn, x, bound)
            k0, v0 = eng.buffer("k_slow").clone(), eng.buffer("v_slow").clone()
            for key in res:
                res[key].append(r[key][d:])
        res = {key: torch.cat(v) for key, v in res.items()}
        res["k"], res["v"] = k0[layer, pages], v0[layer, pages]
        return res

    want = run([(0, 0, cnt)])
    cases = {f"split at {s}": ([(0, 0, s), (0, s, cnt)], None) for s in (1, 28, 37, 64, 100, 199)}
    cases.update({f"shifted by {d}": ([(d, 0, cnt)], None) for d in (1, 17, 64, 100)})
    cases.update({f"bound {b}": ([(0, 0, cnt)], b) for b in (s0 + cnt + 1, g.S)})
    for what, (pieces, bound) in cases.items():
        got = run(pieces, bound)
        for key in want:
            assert torch.equal(_bits(got[key]), _bits(want[key])), f"{name} {what}: {key} differs from one pass"


# ---------------------------------------------------------------------------------------------------------------------
# hand-off to decode
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny-b", "s2pro"])
def test_prefill_handoff(name):
    """After fsb_lm_prefill with sampling: x_slow[k] == x_prefill[last[k]], ssq_slow its per-128-feature sums of
    squares, pos[slot] == row_pos[last] + 1."""
    cfg, w, eng, g = _engine(name)
    ps = _main_pass(eng, g, seed=5, with_unmapped=False)
    C = cfg.num_codebooks
    gen = torch.Generator().manual_seed(3)
    tok = torch.randint(0, cfg.im_end_id, (ps.rows, C + 1), generator=gen)
    tok[:, 1:] = torch.randint(0, cfg.codebook_size, (ps.rows, C), generator=gen)
    last = [ps.first[k] + n - 1 for k, (_, _, n, _) in enumerate(ps.seqs)]
    slots = [s for s, _, _, _ in ps.seqs]
    eng.reset()
    ps.load()
    eng.buffer("x_slow").fill_(SENTINEL)
    eng.buffer("ssq_slow").fill_(float("nan"))
    d_tok = tok.int().cuda()
    d_last = torch.tensor(last, dtype=torch.int32, device="cuda")
    d_slots = torch.tensor(slots, dtype=torch.int32, device="cuda")
    sp = eng.sampling(0.7, 0.7, 1)
    L = _lib()
    L.check(eng.lib.fsb_lm_prefill(eng.h, d_tok.data_ptr(), ps.row_seq.data_ptr(), ps.row_pos.data_ptr(), ps.rows,
                                   d_last.data_ptr(), d_slots.data_ptr(), len(slots), 1, ctypes.byref(sp),
                                   torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    xp = eng.buffer("x_prefill")[d_last.long()]
    xs = eng.buffer("x_slow")[: len(slots)]
    assert torch.equal(_bits(xs), _bits(xp)), f"{name}: x_slow is not the last rows of x_prefill"
    nt = math.ceil(g.D / 128)
    ssq = eng.buffer("ssq_slow")[: len(slots), :nt].double()
    want = R.tile_ssq(xp)
    rel = float(((ssq - want).abs() / want).max())
    assert rel <= 2.0 ** -16, f"{name}: ssq_slow off by {rel:.3g} (relative)"
    pos = eng.buffer("pos")
    for k, s in enumerate(slots):
        assert int(pos[s]) == int(ps.row_pos[last[k]]) + 1, f"{name}: pos[{s}] = {int(pos[s])}"
