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
    two products: at most 11.5 * 2^-24 relative in all, bounded by DELTA = 2^-20. The bracket is the extremes of
    v * r * w over v in {lo, hi} and r in [rsqrt(max sum / Dh + eps) (1 - DELTA), rsqrt(min sum / Dh + eps) (1 + DELTA)].
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
"""
from __future__ import annotations

import math
import random

import pytest
import torch

from tests.test_step_gemm_gpu import C_AMB, _bracket_bf16, _check_rounded, fp64_gemm, norm_operand, rbf, tile_ssq

pytestmark = pytest.mark.gpu

DELTA = 2.0 ** -20  # relative error bound of the qk-norm's fp32 arithmetic (module docstring)
PAGE = 64
SENTINEL = -12345.0
# least share of the checked rows that each wrong reference must put outside the bound (module docstring). The fast
# stack's positions are below num_codebooks, where most rotary pairs turn by a small fraction of a radian per position.
TEETH = {"drop": 0.9, "double": 0.9, "rope+1": 0.9, "next-head": 0.9, "page": 0.9}
TEETH_FAST = {**TEETH, "rope+1": 0.25}
SHORT = 1024  # histories up to this long are checked for a dropped or doubled position (module docstring)


def _lib():
    from fish_speech_b200 import _lib

    return _lib


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------
# engines: every (head_dim, group) instance of the kernel in one stack or the other
# ---------------------------------------------------------------------------------------------------------------------
def _configs():
    """name -> (config, slots). (Dh, G) per stack in the comments; both row tiles; qk-norm and qkv bias on and off."""
    from oracle import lm_oracle as O

    s2 = dict(vocab_size=8192, semantic_begin_id=4000, semantic_end_id=8095, im_end_id=3999, max_seq_len=32768)
    return {
        # slow (64, 8) norm; fast (128, 2) norm + bias
        "tiny-a": (O.tiny_config(max_seq_len=1024, n_head=8, n_local_heads=1, head_dim=64, fast_n_head=2,
                                 fast_n_local_heads=1, fast_head_dim=128, fast_attention_qk_norm=True,
                                 fast_attention_qkv_bias=True), 32),
        # slow (128, 1) bias; fast (64, 2) plain, behind fast_project_in (fast_dim != dim)
        "tiny-b": (O.tiny_config(max_seq_len=1024, n_head=2, n_local_heads=2, head_dim=128, attention_qk_norm=False,
                                 attention_qkv_bias=True, fast_dim=128, fast_n_head=4, fast_n_local_heads=2,
                                 fast_head_dim=64), 64),
        # slow (64, 1) norm + bias; fast (128, 8) norm
        "tiny-c": (O.tiny_config(max_seq_len=1024, n_head=2, n_local_heads=2, head_dim=64, attention_qkv_bias=True,
                                 fast_n_head=8, fast_n_local_heads=1, fast_head_dim=128, fast_attention_qk_norm=True),
                   32),
        # slow (128, 2) plain; fast (64, 4) bias
        "tiny-d": (O.tiny_config(max_seq_len=1024, n_head=4, n_local_heads=2, head_dim=128, attention_qk_norm=False,
                                 fast_attention_qkv_bias=True), 64),
        # S2-Pro layers: slow (128, 4) norm, fast (128, 4) plain; 32 768 positions per slot
        "s2pro": (O.LMConfig(n_layer=2, n_fast_layer=2, **s2), 64),
        # slow (128, 8) norm: the smallest score buffer per position
        "s2pro-g8": (O.LMConfig(n_layer=2, n_fast_layer=1, n_local_heads=4, **s2), 32),
    }


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
        cfg, slots = _configs()[name]
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


class Geom:
    def __init__(self, cfg, fast):
        self.fast = fast
        if fast:
            self.D, self.H, self.Hkv, self.Dh = cfg.fast_dim, cfg.fast_n_head, cfg.fast_n_local_heads, cfg.fast_head_dim
            self.S, self.nl, self.qk_norm = cfg.num_codebooks, cfg.n_fast_layer, cfg.fast_attention_qk_norm
        else:
            self.D, self.H, self.Hkv, self.Dh = cfg.dim, cfg.n_head, cfg.n_local_heads, cfg.head_dim
            self.S, self.nl, self.qk_norm = cfg.max_seq_len, cfg.n_layer, cfg.attention_qk_norm
        self.G = self.H // self.Hkv
        self.scale32 = float(torch.tensor(1.0) / torch.sqrt(torch.tensor(float(self.Dh))))  # 1.0f / sqrtf(Dh)

    def prefix(self, layer):
        return f"{'fast_layers' if self.fast else 'layers'}.{layer}"


# ---------------------------------------------------------------------------------------------------------------------
# state: operand, positions, page table, caches
# ---------------------------------------------------------------------------------------------------------------------
class State:
    """Everything fsb_lm_test_layer_attn reads, written to the engine's buffers. pos[i] = -1 parks row i; `unmapped`
    rows have one history page unmapped. Rows >= `rows` get a table and positions too: the kernel must not touch them."""

    def __init__(self, eng, g: Geom, rows, pos, seed, parked=(), unmapped=()):
        rt = eng.row_tile
        self.g, self.rows, self.rt = g, rows, rt
        gen = torch.Generator(device="cuda").manual_seed(seed)
        rng = random.Random(seed)
        self.x = torch.randn(rt, g.D, generator=gen, device="cuda").bfloat16()
        self.ssq = torch.full((rt, 32), float("nan"), device="cuda")
        self.ssq[:, : math.ceil(g.D / 128)] = tile_ssq(self.x)
        self.pos = list(pos) + [rng.randrange(g.S) for _ in range(rt - len(pos))]
        for i in parked:
            self.pos[i] = -1
        self.parked, self.unmapped = set(parked), set(unmapped)
        kname, vname = ("k_fast", "v_fast") if g.fast else ("k_slow", "v_slow")
        self.kc, self.vc = eng.buffer(kname), eng.buffer(vname)
        self.k0 = torch.randn(self.kc.shape, generator=gen, device="cuda").bfloat16()
        self.v0 = torch.randn(self.vc.shape, generator=gen, device="cuda").bfloat16()
        self.table = None
        if not g.fast:
            n_pages, pps = self.kc.shape[1], eng.kv_pool.pages_per_slot
            perm = list(range(n_pages))
            rng.shuffle(perm)
            self.shared = perm[: pps - 1]  # the pages of full history, the same for every row
            self.private = perm[pps - 1: pps - 1 + rt]  # the page each row appends to
            self.spare = perm[pps - 1 + rt:]  # mapped by nobody
            t = torch.full((eng.max_batch, pps), -1, dtype=torch.int32)
            for i in range(rt):
                p = self.pos[i]
                if p < 0 or i >= eng.max_batch:
                    continue
                t[i, : p // PAGE] = torch.tensor(self.shared[: p // PAGE], dtype=torch.int32)
                t[i, p // PAGE] = self.private[i]
                if i in self.unmapped:
                    assert p >= PAGE
                    t[i, (p // PAGE) // 2] = -1
            self.table = t.cuda()
        self.eng = eng

    def load(self):
        e = self.eng
        e.buffer("x_fast" if self.g.fast else "x_slow").copy_(self.x)
        e.buffer("ssq_fast" if self.g.fast else "ssq_slow").copy_(self.ssq)
        e.buffer("pos").copy_(torch.tensor(self.pos, dtype=torch.int32))
        if self.table is not None:
            e.buffer("kv_page").copy_(self.table)
            e.set_context_bound_exact(max(self.pos) + 1)
        self.kc.copy_(self.k0)
        self.vc.copy_(self.v0)
        self.attn_buf().fill_(SENTINEL)
        torch.cuda.synchronize()

    def attn_buf(self):
        HD = self.g.H * self.g.Dh
        return self.eng.buffer("attn")[: self.rt * HD].view(self.rt, HD)

    def run(self, layer, kv_only=0):
        """Loads the state, runs the hook; returns (attn rows, K cache, V cache) as the kernel left them."""
        L = _lib()
        self.load()
        L.check(L.lib().fsb_lm_test_layer_attn(self.eng.h, int(self.g.fast), layer, self.rows, kv_only, _stream()))
        torch.cuda.synchronize()
        return self.attn_buf().clone(), self.kc.clone(), self.vc.clone()

    def live(self):
        return [i for i in range(self.rows) if i not in self.parked and i not in self.unmapped]

    def slot_index(self, layer, i):
        """Index of row i's appended position in the K / V cache, minus the head dimension."""
        p = self.pos[i]
        if self.g.fast:
            return (layer, i, slice(None), p)
        return (layer, int(self.table[i, p // PAGE]), slice(None), p % PAGE)

    def history(self, cache, layer, i, L=None):
        """Positions [0, L) of row i through its page table: float64 [Hkv, L, Dh]."""
        L = self.pos[i] + 1 if L is None else L
        if self.g.fast:
            return cache[layer, i, :, :L].double()
        n = (L + PAGE - 1) // PAGE
        pages = self.table[i, :n].long()
        c = cache[layer][pages]  # [n, Hkv, 64, Dh]
        return c.permute(1, 0, 2, 3).reshape(c.shape[1], n * PAGE, -1)[:, :L].double()


# ---------------------------------------------------------------------------------------------------------------------
# the fix-up reference: brackets (lo, hi) and the float64 value's rounding (mid), bf16 values held in fp32
# ---------------------------------------------------------------------------------------------------------------------
def _qk_norm(lo, hi, mid, wn, eps):
    Dh = lo.shape[-1]
    lo64, hi64, mid64, w64 = lo.double(), hi.double(), mid.double(), wn.double()
    straddle = (lo64 <= 0) & (hi64 >= 0)
    sq_lo = torch.where(straddle, 0.0, torch.minimum(lo64 ** 2, hi64 ** 2)).sum(-1, keepdim=True)
    sq_hi = torch.maximum(lo64 ** 2, hi64 ** 2).sum(-1, keepdim=True)
    r_lo = torch.rsqrt(sq_hi / Dh + eps) * (1 - DELTA)
    r_hi = torch.rsqrt(sq_lo / Dh + eps) * (1 + DELTA)
    corners = torch.stack([a * r * w64 for a in (lo64, hi64) for r in (r_lo, r_hi)])
    ref = mid64 * torch.rsqrt((mid64 ** 2).mean(-1, keepdim=True) + eps) * w64
    return rbf(corners.amin(0)), rbf(corners.amax(0)), rbf(ref)


def _rope(lo, hi, mid, cs):
    """[rows, heads, Dh] brackets rotated by cs fp32 [rows, Dh/2, 2] with the kernel's fp32 operations."""
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]

    def rot(x0, x1):
        return rbf(x0 * c - x1 * s), rbf(x1 * c + x0 * s)

    ev = [rot(a[..., 0::2], b[..., 1::2]) for a in (lo, hi) for b in (lo, hi)]
    out = []
    for k in (0, 1):
        vals = torch.stack([e[k] for e in ev])
        out.append((vals.amin(0), vals.amax(0)))
    m0, m1 = rot(mid[..., 0::2], mid[..., 1::2])

    def weave(a, b):
        return torch.stack([a, b], -1).flatten(-2)

    return weave(out[0][0], out[1][0]), weave(out[0][1], out[1][1]), weave(m0, m1)


class Fixup:
    """Brackets of q (after RoPE; before it too, for the pos + 1 teeth), of the appended k and of v, for rows `idx`."""

    def __init__(self, cfg, w, g: Geom, layer, st: State, idx, freqs):
        pre = g.prefix(layer)
        W = w[f"{pre}.attention.wqkv.weight"]
        b = w.get(f"{pre}.attention.wqkv.bias")
        mid, lo, hi = norm_operand(st.x[idx], st.ssq[idx], w[f"{pre}.attention_norm.weight"], cfg.norm_eps, g.D)
        y, _ = fp64_gemm(W, mid)
        E = C_AMB * fp64_gemm(W, torch.maximum(lo.abs(), hi.abs()))[1] + (hi - lo).double() @ W.double().abs().T
        if b is not None:
            y = y + b.double()[None, :]
        n, H, Hkv, Dh = len(idx), g.H, g.Hkv, g.Dh

        def split(t):
            return (t[:, : H * Dh].view(n, H, Dh), t[:, H * Dh: (H + Hkv) * Dh].view(n, Hkv, Dh),
                    t[:, (H + Hkv) * Dh:].view(n, Hkv, Dh))

        (qlo, klo, self.vlo), (qhi, khi, self.vhi) = (split(t) for t in _bracket_bf16(y, E))
        qm, km, self.vmid = split(rbf(y))
        if g.qk_norm:
            qlo, qhi, qm = _qk_norm(qlo, qhi, qm, w[f"{pre}.attention.q_norm.weight"].float(), cfg.norm_eps)
            klo, khi, km = _qk_norm(klo, khi, km, w[f"{pre}.attention.k_norm.weight"].float(), cfg.norm_eps)
        self.q_pre = (qlo, qhi, qm)
        self.freqs = freqs
        cs = freqs[torch.tensor([st.pos[i] for i in idx], device="cuda").long()].float()
        self.q = _rope(qlo, qhi, qm, cs)
        self.k = _rope(klo, khi, km, cs)

    def q_at(self, j, p, shape):
        """(lo, hi, mid) of row j's q rotated at position p, float64 in `shape`."""
        qt = _rope(*(t[j: j + 1] for t in self.q_pre), self.freqs[p: p + 1].float())
        return tuple(t[0].double().view(shape) for t in qt)


# ---------------------------------------------------------------------------------------------------------------------
# attention references
# ---------------------------------------------------------------------------------------------------------------------
def _attn_fp32(q, qd, K, V, scale):
    """q, qd (its bracket width) float64 [Hkv, G, Dh]; K, V [Hkv, L, Dh] -> (o, E) [Hkv, G, Dh] (module docstring)."""
    L = K.shape[1]
    Kt = K.transpose(1, 2)
    s = scale * (q @ Kt)
    p = torch.softmax(s, -1)
    o = p @ V
    absdot = scale * ((q.abs() + qd) @ Kt.abs())
    eps_s = (14 * 2.0 ** -24 * absdot).amax(-1, keepdim=True) + 2.0 ** -24 * (
        s.amax(-1, keepdim=True) - s.amin(-1, keepdim=True))
    rho = torch.expm1(2 * eps_s) + 2 * 2.0 ** -22 + (math.ceil(L / 32) + 8) * 2.0 ** -24
    gacc = (math.ceil(L / 8) + 9) * 2.0 ** -24
    pv = p @ V.abs()
    ds = (scale * (qd @ Kt.abs())).amax(-1, keepdim=True)
    E = (rho + gacc * (1 + rho)) * pv * torch.exp(2 * ds) + torch.expm1(2 * ds) * (pv + o.abs())
    return o, E


def _attn_bf16(qlo, qhi, qm, K, V, scale32):
    """The fast stack's all-bf16 attention: brackets (lo, hi) and the float64 rounding chain (mid), [Hkv, G, Dh]."""
    L = K.shape[1]
    Kt = K.transpose(1, 2)  # [Hkv, Dh, L]
    a, b = qlo[..., None] * Kt[:, None], qhi[..., None] * Kt[:, None]  # [Hkv, G, Dh, L]
    gam = 13 * 2.0 ** -24 * (torch.maximum(qlo.abs(), qhi.abs()) @ Kt.abs())
    dlo, dhi = torch.minimum(a, b).sum(-2) - gam, torch.maximum(a, b).sum(-2) + gam

    def sc(d):  # rbf(rbf(d) * scale): the fp32 product of a bf16 value and the fp32 scale
        return rbf(rbf(d) * scale32).double()

    slo, shi, sm = sc(dlo), sc(dhi), sc(qm @ Kt)
    M = shi.amax(-1, keepdim=True)
    elo, ehi = torch.exp(slo - M), torch.exp(shi - M)
    rho = (L + 8) * 2.0 ** -24 + 2 * 2.0 ** -22
    plo = rbf(elo / (elo + ehi.sum(-1, keepdim=True) - ehi) * (1 - rho)).double()
    phi = rbf(ehi / (ehi + elo.sum(-1, keepdim=True) - elo) * (1 + rho)).double()
    pm = rbf(torch.softmax(sm, -1)).double()
    ua, ub = plo[..., None] * V[:, None], phi[..., None] * V[:, None]  # [Hkv, G, L, Dh]
    gacc = (math.ceil(L / 8) + 9) * 2.0 ** -24 * (phi @ V.abs())
    return rbf(torch.minimum(ua, ub).sum(-2) - gacc), rbf(torch.maximum(ua, ub).sum(-2) + gacc), rbf(pm @ V)


# ---------------------------------------------------------------------------------------------------------------------
# one case: run, then check the append, the untouched bits, the attention and the skipped rows
# ---------------------------------------------------------------------------------------------------------------------
def _check_case(cfg, w, g: Geom, layer, st: State, what, teeth):
    attn, kc, vc = st.run(layer)
    # kv_only: the same append, no attention output
    attn_kv, kc_kv, vc_kv = st.run(layer, kv_only=1)
    assert torch.equal(_bits(kc_kv), _bits(kc)) and torch.equal(_bits(vc_kv), _bits(vc)), f"{what}: kv_only append"
    assert (_bits(attn_kv) == _bits(torch.tensor(SENTINEL).bfloat16())).all(), f"{what}: kv_only wrote attn"

    live = st.live()
    from fish_speech_b200.engine import rope_table

    freqs = rope_table(g.S, g.Dh, cfg.rope_base).cuda()
    fx = Fixup(cfg, w, g, layer, st, live, freqs)
    Hkv, G, Dh = g.Hkv, g.G, g.Dh

    # fix-up and append
    idx = [st.slot_index(layer, i) for i in live]
    got_k = torch.stack([kc[ix] for ix in idx]).float()
    got_v = torch.stack([vc[ix] for ix in idx]).float()
    _check_rounded(got_k, fx.k[0], fx.k[1], fx.k[2], f"{what}: appended k")
    _check_rounded(got_v, fx.vlo, fx.vhi, fx.vmid, f"{what}: appended v")

    # nothing else written: every other element of both caches keeps its bits
    for got, before, name in ((kc, st.k0, "K"), (vc, st.v0, "V")):
        want = before.clone()
        for ix in idx:
            want[ix] = got[ix]
        bad = _bits(got) != _bits(want)
        assert not bad.any(), f"{what}: {int(bad.sum())} {name} cache elements written outside the appends, first at " \
                              f"{bad.nonzero()[0].tolist()}"

    # skipped rows and rows past `rows`: attn row untouched
    sent = _bits(torch.tensor(SENTINEL).bfloat16())
    for i in range(st.rt):
        if i not in live:
            assert (_bits(attn[i]) == sent).all(), f"{what}: row {i} (pos {st.pos[i]}) wrote attn"

    # attention, and the wrong references it must reject
    singles = total = 0
    for j, i in enumerate(live):
        p = st.pos[i]
        K, V = st.history(kc, layer, i), st.history(vc, layer, i)
        got = attn[i].float().view(Hkv, G, Dh)
        qt = tuple(t[j].double().view(Hkv, G, Dh) for t in fx.q)
        rw = f"{what}: row {i} pos {p}"
        if g.fast:
            lo, hi, mid = _attn_bf16(*qt, K, V, g.scale32)

            def bracket(q2, K2, V2):
                return _attn_bf16(*q2, K2, V2, g.scale32)[:2]
        else:
            o, E = _attn_fp32(qt[2], qt[1] - qt[0], K, V, g.scale32)
            lo, hi, mid = rbf(o - E), rbf(o + E), rbf(o)

            def bracket(q2, K2, V2):  # the same bound around a wrong float64 value
                o2 = _attn_fp32(q2[2], q2[1] - q2[0], K2, V2, g.scale32)[0]
                return rbf(o2 - E), rbf(o2 + E)
        inside = (got >= lo) & (got <= hi)
        assert inside.all(), (f"{rw}: attention off at {(~inside).nonzero()[0].tolist()} ({int((~inside).sum())} of "
                              f"{got.numel()}): got {float(got[~inside][0])} want {float(mid[~inside][0])}")
        singles += int((lo == hi).sum())
        total += lo.numel()

        def caught(q2=qt, K2=K, V2=V):
            l2, h2 = bracket(q2, K2, V2)
            return bool(((got < l2) | (got > h2)).any())

        if 1 <= p < SHORT:
            h = p // 2
            keep = [q for q in range(p + 1) if q != h]
            teeth["drop"].append(caught(K2=K[:, keep], V2=V[:, keep]))
            twice = list(range(p + 1)) + [h]
            teeth["double"].append(caught(K2=K[:, twice], V2=V[:, twice]))
        if p + 1 < g.S:
            teeth["rope+1"].append(caught(q2=fx.q_at(j, p + 1, (Hkv, G, Dh))))
        if Hkv >= 2:
            teeth["next-head"].append(caught(K2=K.roll(-1, 0), V2=V.roll(-1, 0)))
        if not g.fast:  # the first page read from a page nobody maps
            n0 = min(p + 1, PAGE)
            K2, V2 = K.clone(), V.clone()
            K2[:, :n0] = kc[layer, st.spare[0], :, :n0].double()
            V2[:, :n0] = vc[layer, st.spare[0], :, :n0].double()
            teeth["page"].append(caught(K2=K2, V2=V2))
    return singles, total


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


def _report_teeth(teeth, what, fast):
    for k, v in teeth.items():
        if v:
            print(f"{what}: wrong reference '{k}' rejected for {sum(v)} of {len(v)} rows")
            assert sum(v) >= (TEETH_FAST if fast else TEETH)[k] * len(v), (f"{what}: the bound accepts a wrong reference ({k}) for "
                                                 f"{len(v) - sum(v)} of {len(v)} rows")


def _tag(name, fast):
    return f"{name}-{'fast' if fast else 'slow'}"


CASES = [pytest.param(name, fast, id=_tag(name, fast)) for name in _configs() for fast in (0, 1)
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
