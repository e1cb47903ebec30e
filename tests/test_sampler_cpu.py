"""An exact emulation of the LM sampler (csrc/lm_kernels.cu sample_kernel), checked on its own: Philox4x32-10 against
the Random123 known-answer vectors, the kernel's counter layout and uniform, and the distribution of the emulated
exponential race against float64 logits_to_probs. tests/test_sampler_gpu.py holds the kernel to this emulation.

The kernel, for one row of n candidates (logit l_e = rbf(fp32 logit), token id key_e):
  1. m = max l, z = fp32 sum of expf(l_e - m) over every candidate (per-thread strided sums, then a block reduction).
  2. Ranks one at a time (largest logit first, ties toward the lower candidate index), at most
     kcap = min(top_k, n, 256):
     pr_r = rbf(expf(v_r - m) / z), cum_r = rbf(fp32 running sum of pr). Survivors: rank 0, and rank r >= 1 while
     cum_r <= top_p. top_k <= 1 is the greedy argmax (and no RAS draw).
  3. Per draw w (0: the request's temperature / top_p; 1, the slow head's RAS re-draw: T = 1.0, top_p = 0.9):
     Tc = max(T, 1e-5), t_r = rbf(v_r / Tc), pr2_r = rbf(expf(t_r - t_0) / zz), zz the warp sum over the survivors.
  4. The exponential race: score_r = pr2_r / -logf(u_r), the winner the largest score, ties toward the lower token id.
     u_r = ((x0 >> 8) + 0.5) / 2^24 in fp32, x0 the first word of Philox4x32-10 with key (seed lo, seed hi) and counter
     (off lo, off hi, lane, draw * 256 + r): off = the frame counter "step" and lane = slot with per-call parameters,
     off = n_out[slot] and lane = 0 with slot control; draw = 2 * draw_id + w, draw_id 0 on the slow head and p on fast
     codebook p. With the noise hook (slot 0 only) the score is rbf(pr2_r / rbf(-logf(U_e))) instead.

Every step is emulated in fp32 exactly where the kernel's arithmetic is exact (differences of bf16 values, divisions,
rbf, the running sum of pr), and with a bracket where it is not: expf <= 2 ulp and logf <= 1 ulp (CUDA Math API, no
fast-math in the build), fp32 sums of d terms of one sign within d * 2^-24 of their float64 value. A quantity is an
interval [lo, hi]; every later step is monotone in it and maps the corners. A draw is *determined* when no cum bracket
straddles its top_p and the winner's lowest score beats every other survivor's highest score; otherwise the emulation
names the candidates that can win.

Distribution: the emulated race over 2^17 (seed, counter) pairs at n = 4097 against float64 logits_to_probs, chi-square
at the 1e-6 upper quantile, on peaky and flat logits at top_k 30 and 256. The float64 reference cuts where the
emulation does (the test checks that no cum lies near top_p), so what remains is the bf16 rounding of pr2: a relative
error up to 2^-9 per probability, far below what 2^17 draws resolve.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import pytest
import torch

SEL_CAP = 256
RAS_T, RAS_TOP_P = 1.0, 0.9
_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_S32 = np.uint64(32)
U24 = np.float32(2.0 ** -24)
EXP_REL = 2.0 ** -22 + 2.0 ** -50  # expf: 2 ulp <= 2 * 2^-23 relative (+ the float64 arithmetic of the bracket)
LOG_REL = 2.0 ** -23 + 2.0 ** -50  # logf: 1 ulp


# ---------------------------------------------------------------------------------------------------------------------
# Philox4x32-10 and the kernel's uniform
# ---------------------------------------------------------------------------------------------------------------------
def philox4x32(k0, k1, c0, c1, c2, c3):
    """Philox4x32-10 (Salmon et al., SC'11; Random123) on arrays, in uint64 arithmetic."""
    k0, k1, c0, c1, c2, c3 = (np.asarray(v, dtype=np.uint64) & _MASK for v in (k0, k1, c0, c1, c2, c3))
    for _ in range(10):
        p0, p1 = _M0 * c0, _M1 * c2
        c0, c1, c2, c3 = (p1 >> _S32) ^ c1 ^ k0, p1 & _MASK, (p0 >> _S32) ^ c3 ^ k1, p0 & _MASK
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return c0, c1, c2, c3


def uniform_from_word(x0, half=True):
    """u = ((x0 >> 8) + 0.5) * 2^-24 in fp32 (the sum rounds to even above 2^23); half=False drops the + 0.5."""
    v = (np.asarray(x0, dtype=np.uint64) >> np.uint64(8)).astype(np.float32)
    return ((v + np.float32(0.5)) if half else v) * U24


def philox_uniform(seed, off, lane, draw, r, half=True, swap=False):
    """The uniform of rank r of draw `draw`; swap=True exchanges draw and r in the counter (a wrong layout)."""
    seed, off = int(seed), int(off)
    r = np.asarray(r, dtype=np.uint64)
    word = r * np.uint64(SEL_CAP) + np.uint64(draw) if swap else np.uint64(draw * SEL_CAP) + r
    x0 = philox4x32(seed & 0xFFFFFFFF, seed >> 32, off & 0xFFFFFFFF, off >> 32, lane, word)[0]
    return uniform_from_word(x0, half)


# ---------------------------------------------------------------------------------------------------------------------
# fp32 helpers
# ---------------------------------------------------------------------------------------------------------------------
def rbf(x) -> np.ndarray:
    """fp32 -> bf16 (round to nearest even) -> fp32."""
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).bfloat16().float().numpy()


def down32(a) -> np.ndarray:
    a = np.asarray(a, dtype=np.float64)
    f = a.astype(np.float32)
    return np.where(f.astype(np.float64) > a, np.nextafter(f, np.float32(-np.inf)), f)


def up32(a) -> np.ndarray:
    a = np.asarray(a, dtype=np.float64)
    f = a.astype(np.float32)
    return np.where(f.astype(np.float64) < a, np.nextafter(f, np.float32(np.inf)), f)


def _exp_bracket(d32):
    """expf of fp32 differences d (exact): [lo, hi] in float64."""
    e = np.exp(d32.astype(np.float64))
    return e * (1 - EXP_REL), e * (1 + EXP_REL) + 2.0 ** -148


def _div_bracket_bf16(a_lo, a_hi, b_lo, b_hi):
    """rbf(RN(a / b)) for a, b in brackets (b > 0)."""
    return rbf(down32(a_lo / b_hi)), rbf(up32(a_hi / b_lo))


def _sum_gamma(depth):
    return depth * 2.0 ** -24 * 1.01


# ---------------------------------------------------------------------------------------------------------------------
# the emulation
# ---------------------------------------------------------------------------------------------------------------------
class Draw:
    """One draw's outcome: `entry` when determined (else None), `cands` the entries that can win."""

    def __init__(self, entry, cands):
        self.entry, self.cands = entry, cands

    @property
    def determined(self):
        return self.entry is not None


class RowStage1:
    """Steps 1-2 of the module docstring for one row: ranks, their logits and the cum brackets."""

    def __init__(self, logits32, top_k, n_ranks_cap=SEL_CAP, rank_logits=None):
        lg = rbf(logits32)
        self.lg = lg
        n = lg.shape[0]
        self.kcap = max(1, min(int(top_k), n, n_ranks_cap))
        key = lg if rank_logits is None else rank_logits
        order = np.argsort(-key, kind="stable")[: self.kcap]  # ties toward the lower candidate index
        self.idx = order
        self.v = lg[order]
        kv = key[order]
        m = np.float32(key.max())
        e_lo, e_hi = _exp_bracket((key - m).astype(np.float32))
        g = _sum_gamma(math.ceil(n / 1024) + 5 + 32)
        z_lo, z_hi = e_lo.sum() * (1 - g), e_hi.sum() * (1 + g)
        r_lo, r_hi = _exp_bracket((kv - m).astype(np.float32))
        pr_lo, pr_hi = _div_bracket_bf16(r_lo, r_hi, z_lo, z_hi)
        self.cum_lo = rbf(np.cumsum(pr_lo, dtype=np.float32))
        self.cum_hi = rbf(np.cumsum(pr_hi, dtype=np.float32))

    def survivors(self, tp, ge=False):
        """(ns_early, ns_late): the survivor count with every cum at its high / low end."""
        tp = np.float32(tp)

        def first(cum):
            cut = (cum[1:] >= tp) if ge else (cum[1:] > tp)
            hit = np.flatnonzero(cut)
            return int(hit[0]) + 1 if hit.size else self.kcap

        return first(self.cum_hi), first(self.cum_lo)


def draw(st: RowStage1, T, tp, keys, uniforms=None, noise=None, ge=False):
    """Steps 3-4 for one draw. uniforms(ranks) -> fp32 u of those ranks (Philox); noise: fp32 U per candidate."""
    ns_e, ns_l = st.survivors(tp, ge)
    Tc = np.float32(max(np.float32(T), np.float32(1e-5)))
    t = rbf((st.v[:ns_l] / Tc).astype(np.float32))
    d = (t - t[0]).astype(np.float32)
    x_lo, x_hi = _exp_bracket(d)
    zz_lo = x_lo[:ns_e].sum() * (1 - _sum_gamma(math.ceil(ns_e / 32) + 5))
    zz_hi = x_hi[:ns_l].sum() * (1 + _sum_gamma(math.ceil(ns_l / 32) + 5))
    p_lo, p_hi = _div_bracket_bf16(x_lo, x_hi, zz_lo, zz_hi)
    p_lo, p_hi = p_lo.astype(np.float64), p_hi.astype(np.float64)
    ent = st.idx[:ns_l]
    if noise is None:
        u = np.asarray(uniforms(np.arange(ns_l)), dtype=np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            L = -np.log(u)  # u = 1: -0, and the score is -inf (test_uniform_rounds_like_fp32)
            s_lo = np.where(np.isinf(L), 0.0, down32(p_lo / (L * (1 + LOG_REL))))
            s_hi = np.where(np.isinf(L), 0.0, up32(p_hi / (L * (1 - LOG_REL))))
    else:
        U = noise[ent].astype(np.float64)
        with np.errstate(divide="ignore"):
            L = -np.log(U)
        q_lo, q_hi = rbf(down32(L * (1 - LOG_REL))).astype(np.float64), rbf(up32(L * (1 + LOG_REL))).astype(np.float64)
        with np.errstate(divide="ignore", invalid="ignore"):
            s_lo = np.where(np.isinf(q_hi), 0.0, rbf(down32(p_lo / q_hi)))
            s_hi = np.where(np.isinf(q_lo), 0.0, rbf(up32(p_hi / q_lo)))
    s_lo, s_hi = s_lo.astype(np.float64), s_hi.astype(np.float64)
    order_key = keys[ent].astype(np.int64) * SEL_CAP + np.arange(ns_l)  # ties toward the lower token id
    # the candidate that wins with every score at its low end, tie-broken like the kernel
    best = int(np.lexsort((order_key[:ns_e], -s_lo[:ns_e]))[0])
    cands = set(int(e) for e in ent[s_hi >= s_lo[best]])
    cands.add(int(ent[best]))
    point_tie = (s_lo == s_hi) & (s_lo == s_lo[best]) & (s_lo[best] == s_hi[best]) & (order_key[best] < order_key)
    beaten = (s_lo[best] > s_hi) | point_tie
    beaten[best] = True
    det = ns_e == ns_l and bool(beaten.all())
    return Draw(int(ent[best]) if det else None, cands)


def greedy(logits32):
    lg = rbf(logits32)
    return Draw(int(np.argmax(lg)), {int(np.argmax(lg))})  # np.argmax: the first maximum


class Request:
    """What the sampler reads for one row: parameters and its RNG stream."""

    def __init__(self, T, top_p, top_k, seed, off, lane):
        self.T, self.top_p, self.top_k, self.seed, self.off, self.lane = (
            np.float32(T), np.float32(top_p), int(top_k), int(seed), int(off), int(lane))


WRONG = ("temp-before-cut", "ge-top-p", "top-k-1", "ras-top-p", "ras-temp", "swap-counter", "lane-ignored", "no-half")


def emulate(logits32, req: Request, keys, draw_id, two, noise=None, wrong=None):
    """[main draw, RAS draw or None] of one row. keys: token id per candidate; two: the slow head's RAS re-draw.
    wrong: one of WRONG, a deliberately wrong emulation."""
    if req.top_k <= 1:
        g = greedy(logits32)
        return [g, g if two else None]
    Tc = np.float32(max(req.T, np.float32(1e-5)))
    rank_logits = rbf((rbf(logits32) / Tc).astype(np.float32)) if wrong == "temp-before-cut" else None
    top_k = req.top_k - 1 if wrong == "top-k-1" else req.top_k
    st = RowStage1(logits32, top_k, rank_logits=rank_logits)
    out = []
    for w in range(2 if two else 1):
        T, tp = (req.T, req.top_p) if w == 0 else (RAS_T, RAS_TOP_P)
        if w == 1 and wrong == "ras-top-p":
            tp = req.top_p
        if w == 1 and wrong == "ras-temp":
            T = req.T
        lane = 0 if wrong == "lane-ignored" else req.lane
        dr = 2 * draw_id + w

        def uni(ranks, dr=dr, lane=lane):
            return philox_uniform(req.seed, req.off, lane, dr, ranks, half=wrong != "no-half",
                                  swap=wrong == "swap-counter")

        out.append(draw(st, T, tp, keys, uniforms=uni, noise=None if noise is None else noise[dr],
                        ge=wrong == "ge-top-p"))
    return out + [None] * (2 - len(out))


def slow_keys(n, sem_begin, im_end_id):
    """Token id of each slow-head candidate: semantic ids in order, then <|im_end|>."""
    k = np.arange(n, dtype=np.int64) + sem_begin
    k[n - 1] = im_end_id
    return k


# ---------------------------------------------------------------------------------------------------------------------
# float64 reference (inference.py:54-67 logits_to_probs)
# ---------------------------------------------------------------------------------------------------------------------
def logits_to_probs64(logits, T, top_p, top_k):
    lg = np.asarray(logits, dtype=np.float64)
    order = np.argsort(-lg, kind="stable")
    s = lg[order]
    p = np.exp(s - s[0])
    cum = np.cumsum(p / p.sum())
    remove = (cum > top_p) | (np.arange(lg.size) >= top_k)
    remove[0] = False
    keep = order[~remove]
    out = np.zeros(lg.size)
    x = lg[keep] / max(float(T), 1e-5)
    e = np.exp(x - x.max())
    out[keep] = e / e.sum()
    return out, cum


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_matches_the_random123_known_answers(ctr, key, want):
    got = philox4x32(key[0], key[1], *ctr)
    assert tuple(int(x) for x in got) == want


def test_philox_vectorises_over_counters():
    c3 = np.arange(300, dtype=np.uint64)
    many = philox4x32(7, 9, 1, 2, 3, c3)
    for i in (0, 1, 255, 299):
        one = philox4x32(7, 9, 1, 2, 3, i)
        assert all(int(a[i]) == int(b) for a, b in zip(many, one))


def test_counter_layout():
    seed, off, lane = 0x0123456789ABCDEF, (5 << 32) | 17, 9
    for dr, r in ((0, 0), (1, 3), (19, 255)):
        x0 = philox4x32(0x89ABCDEF, 0x01234567, 17, 5, lane, dr * 256 + r)[0]
        assert philox_uniform(seed, off, lane, dr, r) == uniform_from_word(x0)
    # draw and r are not interchangeable, nor are the lanes
    assert philox_uniform(seed, off, lane, 1, 3) != philox_uniform(seed, off, lane, 3, 1)
    assert philox_uniform(seed, off, lane, 1, 3) == philox_uniform(seed, off, lane, 3, 1, swap=True)
    assert philox_uniform(seed, off, lane, 1, 3) != philox_uniform(seed, off, 0, 1, 3)


def test_uniform_rounds_like_fp32():
    w = np.array([0, 0xFF, 0x100, 0x7FFFFF00, 0x80000000, 0xFFFFFE00, 0xFFFFFF00, 0xFFFFFFFF], dtype=np.uint64)
    u = uniform_from_word(w)
    assert u.dtype == np.float32 and (u > 0).all() and (u <= 1).all()
    assert u[0] == u[1] == np.float32(2.0 ** -25)
    assert u[2] == np.float32(1.5 * 2.0 ** -24)
    # from 2^23 on, (x >> 8) + 0.5 is not an fp32 value and rounds to even: 0xFFFFFE + 0.5 down, 0xFFFFFF + 0.5 up
    # to 2^24, so u = 1 exactly once in 2^24 words. Then -logf(u) = -0 and the score is -inf: that rank sits the
    # draw out (a chance of 2^-24 per rank, which the emulation reproduces rather than corrects).
    assert u[5] == np.float32(1 - 2.0 ** -23)
    assert u[6] == u[7] == np.float32(1.0)
    assert uniform_from_word(w, half=False)[0] == 0


def test_rbf_rounds_to_nearest_even():
    x = np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 1 + 2 ** -8 + 2 ** -20], dtype=np.float32)
    assert rbf(x).tolist() == [1.0, 1 + 2 ** -6, -1.0, 1 + 2 ** -7]


def test_tie_rules_of_the_emulation():
    # four equal logits at the top, top_k 2: the two lowest candidate indices are the survivors
    lg = np.full(40, -3.0, dtype=np.float32)
    lg[[5, 7, 20, 39]] = 2.0
    st = RowStage1(lg, 2)
    assert st.idx.tolist() == [5, 7]
    # the draw: equal scores (equal probability, equal noise) -> the lower token id, <|im_end|> (entry 39, token 3) wins
    keys = slow_keys(40, 100, 3)
    st = RowStage1(lg, 4)
    d = draw(st, 1.0, 1.0, keys, noise=np.full(40, 0.5, dtype=np.float32))
    assert d.determined and d.entry == 39


def _race_counts(logits, T, top_p, top_k, n_draws, seed0=1):
    """Winners of the emulated race for n_draws (seed, counter) pairs; every survivor decision must be determined."""
    st = RowStage1(logits, top_k)
    ns_e, ns_l = st.survivors(np.float32(top_p))
    assert ns_e == ns_l, "the test's logits put a cum next to top_p"
    Tc = np.float32(max(np.float32(T), np.float32(1e-5)))
    t = rbf((st.v[:ns_e] / Tc).astype(np.float32))
    x = np.exp((t - t[0]).astype(np.float32).astype(np.float64))
    pr2 = rbf((x / x.sum()).astype(np.float32)).astype(np.float64)
    counts = np.zeros(logits.size, dtype=np.int64)
    per = 256
    ranks = np.arange(ns_e, dtype=np.uint64)
    for s in range(n_draws // per):
        off = np.arange(per, dtype=np.uint64)[:, None]
        x0 = philox4x32(seed0 + s, 0, off, 0, 0, ranks[None, :])[0]
        u = uniform_from_word(x0).astype(np.float64)
        win = np.argmax(pr2[None, :] / -np.log(u), axis=1)
        np.add.at(counts, st.idx[win], 1)
    return counts, st


def chi2_pvalue(counts, probs):
    """Pearson chi-square of counts against probs (bins with an expected count below 5 merged)."""
    from scipy.stats import chi2

    N = counts.sum()
    exp = probs * N
    assert counts[probs == 0].sum() == 0, "a draw outside the survivor set"
    big = exp >= 5
    o = np.append(counts[big], counts[~big].sum())
    e = np.append(exp[big], exp[~big].sum())
    if e[-1] == 0:
        o, e = o[:-1], e[:-1]
    stat = float(((o - e) ** 2 / e).sum())
    return stat, len(o) - 1, float(chi2.sf(stat, len(o) - 1))


def dist_logits(kind, n=4097, seed=3):
    rng = np.random.default_rng(seed)
    if kind == "peaky":
        return (rng.standard_normal(n) * 2.5).astype(np.float32)
    return (rng.standard_normal(n) * 0.02).astype(np.float32)  # flat: the 256 cap binds


@pytest.mark.parametrize("kind", ["peaky", "flat"])
@pytest.mark.parametrize("top_k", [30, 256])
def test_emulated_race_follows_logits_to_probs(kind, top_k):
    lg = dist_logits(kind)
    T, top_p = 0.69921875, 0.94921875  # bf16(0.7), bf16(0.95)
    counts, st = _race_counts(lg, T, top_p, top_k, 1 << 17)
    p, cum = logits_to_probs64(rbf(lg), T, top_p, top_k)
    # the float64 cut is the emulation's: no cum within 1 % of top_p over the ranks that count
    assert np.abs(cum[: st.kcap] - top_p).min() > 0.01
    stat, df, pv = chi2_pvalue(counts, p)
    assert pv > 1e-6, f"chi2 {stat:.1f} on {df} degrees of freedom, p = {pv:.2e}"


def test_chi_square_has_teeth():
    """The same race with the probabilities of top_k - 1 survivors (one rank too few) must fail the test."""
    lg = dist_logits("peaky")
    T, top_p, top_k = 0.69921875, 0.94921875, 30
    counts, _ = _race_counts(lg, T, top_p, top_k - 1, 1 << 15)
    p, _ = logits_to_probs64(rbf(lg), T, top_p, top_k)
    assert chi2_pvalue(counts, p)[2] < 1e-6


# ---------------------------------------------------------------------------------------------------------------------
# fsb_lm_create refuses a head or a codebook the sampler cannot hold (before any device is looked for)
# ---------------------------------------------------------------------------------------------------------------------
def _create(head_rows, codebook_size):
    from fish_speech_b200 import _lib

    K = _lib.LmConfig()
    K.dim, K.n_layer, K.n_head, K.n_kv_head, K.head_dim, K.intermediate = 256, 1, 4, 1, 128, 512
    K.fast_dim, K.n_fast_layer, K.fast_n_head, K.fast_n_kv_head = 256, 1, 4, 1
    K.fast_head_dim, K.fast_intermediate = 64, 512
    K.vocab_size, K.codebook_size, K.num_codebooks = 20000, codebook_size, 4
    K.semantic_begin_id, K.semantic_end_id, K.im_end_id = 1000, 1000 + head_rows - 2, 999
    K.max_batch, K.kv_len, K.max_rows, K.max_frames = 1, 128, 128, 4
    W = _lib.LmWeights()
    W.head_rows = head_rows
    h = C.c_void_p()
    L = _lib.lib()
    rc = L.fsb_lm_create(C.byref(K), C.byref(W), C.byref(h))
    msg = L.fsb_last_error().decode()
    if rc == 0:
        L.fsb_lm_destroy(h)
    return rc, msg, h.value


@pytest.mark.parametrize("head_rows,codebook_size", [(8193, 4096), (4097, 8193), (16384, 16384)])
def test_create_refuses_more_candidates_than_the_sampler_holds(head_rows, codebook_size):
    rc, msg, h = _create(head_rows, codebook_size)
    assert rc != 0 and h is None
    assert f"head_rows={head_rows}" in msg and f"codebook_size={codebook_size}" in msg and "8192" in msg


def test_create_accepts_8192_candidates():
    if torch.cuda.is_available():
        pytest.skip("on a GPU this would build an engine; tests/test_sampler_gpu.py runs one at 8192")
    rc, msg, h = _create(8192, 8192)
    assert rc != 0 and "8192" not in msg  # past the check: the next failure is the missing device


def test_test_sample_hook_is_bound():
    from fish_speech_b200 import _lib

    assert "fsb_lm_test_sample" in _lib.exported_symbols()
    assert len(_lib.lib().fsb_lm_test_sample.argtypes) == 9
