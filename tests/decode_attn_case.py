"""One case of the decode attention (csrc/lm_kernels.cu attn_decode_kernel and the split kernels behind it), shared by
tests/test_decode_attn_gpu.py and tests/test_attn_split_gpu.py: the engine state fsb_lm_test_layer_attn reads
(operand, positions, page table, caches), one run of the hook, and the checks of its append, of the cache bits it
must not change, of its attention output and of the wrong references the bound must reject. The bounds and the TEETH
shares are derived in the test_decode_attn_gpu docstring; the references live in tests/kernel_ref.py."""
from __future__ import annotations

import math
import random

import torch

from tests import kernel_ref as R
from tests.kernel_ref import PAGE, check_bracket, rbf, tile_ssq
from tests.lm_util import _bits, _lib

SENTINEL = -12345.0
# least share of the checked rows that each wrong reference must put outside the bound (test_decode_attn_gpu
# docstring). The fast stack's positions are below num_codebooks, where most rotary pairs turn by a small fraction of a
# radian per position.
TEETH = {"drop": 0.9, "double": 0.9, "rope+1": 0.9, "next-head": 0.9, "page": 0.9}
TEETH_FAST = {**TEETH, "rope+1": 0.25}
SHORT = 1024  # histories up to this long are checked for a dropped or doubled position (test_decode_attn_gpu docstring)


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
        self.ssq[:, : math.ceil(g.D / 128)] = tile_ssq(self.x).float()
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
        L.check(L.lib().fsb_lm_test_layer_attn(self.eng.h, int(self.g.fast), layer, self.rows, kv_only,
                                                torch.cuda.current_stream().cuda_stream))
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

    def history(self, cache, layer, i):
        """Positions [0, pos] of row i (through its page table in the slow stack): float64 [Hkv, pos + 1, Dh]."""
        L = self.pos[i] + 1
        if self.g.fast:
            return cache[layer, i, :, :L].double()
        return R.paged_history(cache[layer], self.table[i], L)


class Fixup:
    """Brackets of q (after RoPE; before it too, for the pos + 1 teeth), of the appended k and of v, for rows `idx`."""

    def __init__(self, cfg, w, g: Geom, layer, st: State, idx, freqs):
        pre = g.prefix(layer)
        qn, kn = ((w[f"{pre}.attention.q_norm.weight"], w[f"{pre}.attention.k_norm.weight"]) if g.qk_norm
                  else (None, None))
        self.q_pre, k, (self.vlo, self.vhi, self.vmid) = R.fixup_ref64(
            st.x[idx], st.ssq[idx], w[f"{pre}.attention_norm.weight"], w[f"{pre}.attention.wqkv.weight"],
            w.get(f"{pre}.attention.wqkv.bias"), g.H, g.Hkv, g.Dh, qn, kn, cfg.norm_eps)
        self.freqs = freqs
        cs = freqs[torch.tensor([st.pos[i] for i in idx], device="cuda").long()].float()
        self.q = R.rope_bracket(*self.q_pre, cs)
        self.k = R.rope_bracket(*k, cs)

    def q_at(self, j, p, shape):
        """(lo, hi, mid) of row j's q rotated at position p, float64 in `shape`."""
        qt = R.rope_bracket(*(t[j: j + 1] for t in self.q_pre), self.freqs[p: p + 1].float())
        return tuple(t[0].double().view(shape) for t in qt)


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
    check_bracket(got_k, fx.k[0], fx.k[1], f"{what}: appended k", fx.k[2])
    check_bracket(got_v, fx.vlo, fx.vhi, f"{what}: appended v", fx.vmid)

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
            lo, hi, mid = R.attn_decode_bf16(*qt, K, V, g.scale32)

            def bracket(q2, K2, V2):
                return R.attn_decode_bf16(*q2, K2, V2, g.scale32)[:2]
        else:
            o, E = R.attn_decode_fp32(qt[2], qt[1] - qt[0], K, V, g.scale32)
            lo, hi, mid = rbf(o - E), rbf(o + E), rbf(o)

            def bracket(q2, K2, V2):  # the same bound around a wrong float64 value
                o2 = R.attn_decode_fp32(q2[2], q2[1] - q2[0], K2, V2, g.scale32)[0]
                return rbf(o2 - E), rbf(o2 + E)
        check_bracket(got, lo, hi, f"{rw}: attention")
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


def _report_teeth(teeth, what, fast):
    for k, v in teeth.items():
        if v:
            print(f"{what}: wrong reference '{k}' rejected for {sum(v)} of {len(v)} rows")
            assert sum(v) >= (TEETH_FAST if fast else TEETH)[k] * len(v), (f"{what}: the bound accepts a wrong reference ({k}) for "
                                                 f"{len(v) - sum(v)} of {len(v)} rows")
