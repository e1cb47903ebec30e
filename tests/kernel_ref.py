"""Float64 references, rounding brackets and fp32 emulations of the LM and codec kernels, shared by their GPU tests. The
GPU test module that uses a bound derives it in its docstring; each function here names that module. Plain torch on
whatever device the inputs live on; tests/test_prefill_cpu.py and tests/test_kernel_ref_cpu.py rehearse them on the
CPU.

Every bracket is a pair (lo, hi) of bf16 values held in fp32: the kernel's output must lie in [lo, hi], and where
lo == hi it is fixed bit for bit. `mid` is the reference value rounded the way the float64 value would be."""
from __future__ import annotations

import math

import torch

PAGE = 64
C_AMB = 2.0 ** -19  # step GEMM accumulation, relative to |W| |X| (test_step_gemm_gpu docstring, which measures it)
C_CONV = 2.0 ** -18  # gemm_tc accumulation, relative to |W| |X| (test_codec_ops_gpu docstring, which measures it)
RN_ROW = 2.0 ** -19  # relative error of a row RMSNorm's rsqrt over a block sum (test_prefill_gpu docstring)
RN_HEAD = 2.0 ** -20  # the same for the per-head qk-norm over a warp sum (test_prefill_gpu, test_decode_attn_gpu)
EXP_ULP = 2.0 ** -22  # expf: 2 ulp
MU = 2.0 ** -21  # mma.sync accumulation allowance per instruction, relative to the sum of magnitudes


def rbf(t: torch.Tensor) -> torch.Tensor:
    """Round to bf16 the way the kernels do: to fp32 first (a no-op for fp32 input), then to bf16."""
    return t.float().bfloat16().float()


def bf16_key(t: torch.Tensor) -> torch.Tensor:
    """Integers ordered like the bf16 values of t, one apart for neighbouring values (ulp distance)."""
    b = t.bfloat16().view(torch.int16).int()
    return torch.where(b < 0, -(b & 0x7FFF), b)


def bracket_bf16(v, E):
    """The bf16 values between which the kernel's rbf(fp32 accumulation) of the float64 value v lies when the
    accumulation is off by at most E (rounding to fp32, then to bf16, is monotone)."""
    return rbf(v - E), rbf(v + E)


def check_bracket(got, lo, hi, what, mid=None, share=0.01, tally=None):
    """got inside [lo, hi] (bit-identical where lo == hi). With mid, the elements that differ from it: fewer than
    `share` of them, or, with a tally [differ, total], counted into it for check_tally to bound over a whole test."""
    inside = (got >= lo) & (got <= hi)
    if not bool(inside.all()):
        bad = (~inside).nonzero()[0].tolist()
        at = tuple(bad)
        raise AssertionError(f"{what}: {int((~inside).sum())} of {got.numel()} off, first at {bad}: got "
                             f"{float(got[at])} in [{float(lo[at])}, {float(hi[at])}]"
                             + ("" if mid is None else f", float64 rounds to {float(mid[at])}"))
    if mid is None:
        return
    if tally is not None:
        tally[0] += int((got != mid).sum())
        tally[1] += got.numel()
        return
    diff = float((got != mid).double().mean())
    assert diff < share, f"{what}: {diff:.2%} of the elements differ from the float64 value's rounding"


def check_tally(tally, what):
    """Fewer than 1 % of the elements check_bracket counted into tally differ from the float64 value's rounding."""
    assert tally[0] == 0 or tally[0] < 0.01 * tally[1], f"{what}: {tally[0]} of {tally[1]} elements differ from float64"


def gate_row(i: torch.Tensor) -> torch.Tensor:
    """Column of gate feature i in the interleaved w1|w3 result (lm_gemm.cuh w13_gate_row); up is 16 further."""
    return (i >> 6) * 128 + ((i >> 4) & 3) * 32 + (i & 15)


def fp64_gemm(x: torch.Tensor, w: torch.Tensor):
    """x [rows, K], w [n, K] -> (x w^T, |x| |w|^T) in float64."""
    x64, w64 = x.double(), w.double()
    return x64 @ w64.T, x64.abs() @ w64.abs().T


def acc_bound(absprod, K, parts):
    """The step GEMM's worst-case accumulation error, (ACC) in the test_step_gemm_gpu docstring."""
    return (K / 16 + parts + 1) * 2.0 ** -23 * absprod


def gemm_bracket(x, w, bias=None):
    """(lo, hi, mid) of rbf(x w^T + bias) when the fp32 accumulation is within C_CONV |x||w| of the float64 value."""
    y, a = fp64_gemm(x, w)
    if bias is not None:
        y = y + bias.double()[None, :]
    return *bracket_bf16(y, C_CONV * a), rbf(y)


# ---------------------------------------------------------------------------------------------------------------------
# sums of squares and normalise-on-load (the step GEMM's operand)
# ---------------------------------------------------------------------------------------------------------------------
def tile_ssq(x: torch.Tensor) -> torch.Tensor:
    """Per-128-feature sums of squares [rows, ceil(D/128)] in float64."""
    rows, D = x.shape
    nt = math.ceil(D / 128)
    xp = torch.zeros(rows, nt * 128, dtype=torch.float64, device=x.device)
    xp[:, :D] = x.double() ** 2
    return xp.view(rows, nt, 128).sum(-1)


def check_ssq(ssq, x, what, nan_past=False):
    """The fp32 sums of squares ssq a kernel left for its rows x: within 2^-16 (relative) of tile_ssq(x) in fp32; with
    nan_past, NaN in the tiles past the row's."""
    nt = math.ceil(x.shape[1] / 128)
    want = tile_ssq(x).float().double()
    rel = ((ssq[:, :nt].double() - want).abs() / want).max()
    assert rel <= 2.0 ** -16, f"{what}: sums of squares off by {float(rel):.3g} (relative)"
    if nan_past:
        assert torch.isnan(ssq[:, nt:]).all(), f"{what}: sums of squares written past the row's {nt} tiles"


def norm_operand(x, ssq, norm_w, eps, K):
    """X' = rbf(rbf(x * r) * w) in the kernel's order (tile sums added in tile order in fp32, / K, + eps, rsqrt) for
    r and for r * (1 -+ 2^-21): rsqrtf may be off by 2 ulp (2^-22 relative). Returns (mid, lo, hi), fp32 [rows, K];
    lo / hi bracket every X' a 2-ulp rsqrtf can give."""
    nt = math.ceil(K / 128)
    tot = torch.zeros(ssq.shape[0], dtype=torch.float32, device=ssq.device)
    for t in range(nt):
        tot = tot + ssq[:, t]
    v = tot / torch.tensor(float(K), dtype=torch.float32) + torch.tensor(eps, dtype=torch.float32)
    r = (1.0 / torch.sqrt(v.double())).float()

    def apply(rr):
        return rbf(rbf(x.float() * rr[:, None]) * norm_w.float()[None, :])

    mid = apply(r)
    a, b = apply((r.double() * (1 - 2.0 ** -21)).float()), apply((r.double() * (1 + 2.0 ** -21)).float())
    return mid, torch.minimum(a, b), torch.maximum(a, b)


def normed_gemm(x, ssq, norm_w, eps, W):
    """(v, E) of the step GEMM W X' normalised on load: v the float64 product with X' = norm_operand's mid, E the
    accumulation allowance C_AMB |W| |X'| plus the width of X''s bracket through |W| (test_decode_attn_gpu docstring).
    The kernel's rbf(W X') lies in bracket_bf16(v, E)."""
    mid, lo, hi = norm_operand(x, ssq, norm_w, eps, x.shape[1])
    v, _ = fp64_gemm(mid, W)
    E = C_AMB * fp64_gemm(torch.maximum(lo.abs(), hi.abs()), W)[1] + (hi - lo).double() @ W.double().abs().T
    return v, E


# ---------------------------------------------------------------------------------------------------------------------
# embedding
# ---------------------------------------------------------------------------------------------------------------------
def embed_ref(tokens, emb, cb_emb, C, cs, sem_begin, sem_end, scale):
    """tokens int [rows][C+1] -> (lo, hi, mid, x64). The kernel: s = fp32 sum of the C codebook rows (codebook order),
    one bf16 rounding; x = rbf(e + s); semantic rows with `scale`: rbf(x / sqrtf(C + 1)). An fp32 sum of C terms is off
    by at most (C - 1) 2^-24 sum |terms| whatever its order, which brackets s. x64 is the float64 value of the same
    expression without the roundings (oracle.lm_oracle.embed on float64 weights)."""
    tok = tokens[:, 0].long()
    sem = (tok >= sem_begin) & (tok <= sem_end)
    codes = tokens[:, 1:].long().clamp(0, cs - 1) + torch.arange(C, device=tokens.device)[None, :] * cs
    terms = cb_emb.double()[codes]  # [rows, C, D]
    S = terms.sum(1)
    E = (C - 1) * 2.0 ** -24 * terms.abs().sum(1)
    e = emb.double()[tok.clamp(0, emb.shape[0] - 1)]
    m = sem[:, None].double()
    div = torch.tensor(float(C + 1), dtype=torch.float32).sqrt().to(tokens.device)

    def chain(s):
        x = rbf(e + s * m)
        if scale:
            x = torch.where(sem[:, None], rbf(x / div), x)
        return x

    lo, hi, mid = chain(rbf(S - E)), chain(rbf(S + E)), chain(rbf(S))
    x64 = e + S * m
    if scale:
        x64 = torch.where(sem[:, None], x64 / math.sqrt(C + 1), x64)
    return torch.minimum(lo, hi), torch.maximum(lo, hi), mid, x64


# ---------------------------------------------------------------------------------------------------------------------
# RMSNorm of a row (resid_norm4_kernel) and of a head (qkv_prep_row_kernel, the decode qkv fix-up)
# ---------------------------------------------------------------------------------------------------------------------
def _r_corners(ss, n, eps, rel):
    r = 1.0 / torch.sqrt(ss / n + eps)
    return [(r * f).float() for f in (1 - rel, 1.0, 1 + rel)]


def row_norm(x, w, eps):
    """rbf(rbf(x r) w) with r = rsqrtf(sum(x^2) / D + eps): (lo, hi, mid) over r within RN_ROW of its float64 value.
    x fp32 [rows, D] holding bf16 values."""
    r_lo, r_mid, r_hi = _r_corners((x.double() ** 2).sum(-1, keepdim=True), x.shape[-1], eps, RN_ROW)
    wf = w.float()[None, :]
    a, b, mid = (rbf(rbf(x.float() * r) * wf) for r in (r_lo, r_hi, r_mid))
    return torch.minimum(a, b), torch.maximum(a, b), mid


def _rot(x0, x1, c, s):
    """The kernel's RoPE of one pair: fp32 products, one fp32 difference / sum, then bf16."""
    return rbf(x0 * c - x1 * s), rbf(x1 * c + x0 * s)


def rope_bracket(lo, hi, mid, cs):
    """[rows, heads, Dh] brackets rotated by cs fp32 [rows, Dh/2, 2] with the kernel's fp32 operations, over the four
    corners of each rotary pair (RoPE is monotone in each element of a pair, not in the pair)."""
    c, s = cs[:, None, :, 0], cs[:, None, :, 1]
    ev = [_rot(a[..., 0::2], b[..., 1::2], c, s) for a in (lo, hi) for b in (lo, hi)]
    m0, m1 = _rot(mid[..., 0::2], mid[..., 1::2], c, s)

    def weave(a, b):
        return torch.stack([a, b], -1).flatten(-2)

    out = []
    for k in (0, 1):
        vals = torch.stack([e[k] for e in ev])
        out.append((vals.amin(0), vals.amax(0)))
    return weave(out[0][0], out[1][0]), weave(out[0][1], out[1][1]), weave(m0, m1)


def head_norm_emul(v, w, eps):
    """qk-norm of bf16 values v fp32 [rows, heads, Dh]: rbf(v * r * w) in fp32 with r within RN_HEAD."""
    Dh = v.shape[-1]
    r_lo, r_mid, r_hi = _r_corners((v.double() ** 2).sum(-1, keepdim=True), Dh, eps, RN_HEAD)
    wf = w.float()
    a, b, mid = (rbf(v * r * wf) for r in (r_lo, r_hi, r_mid))
    return torch.minimum(a, b), torch.maximum(a, b), mid


def head_norm64(lo, hi, mid, w, eps):
    """The same over a bracket of v, in float64 (the reference q / k of the float64 chain)."""
    Dh = lo.shape[-1]
    lo64, hi64, mid64, w64 = lo.double(), hi.double(), mid.double(), w.double()
    straddle = (lo64 <= 0) & (hi64 >= 0)
    sq_lo = torch.where(straddle, 0.0, torch.minimum(lo64 ** 2, hi64 ** 2)).sum(-1, keepdim=True)
    sq_hi = torch.maximum(lo64 ** 2, hi64 ** 2).sum(-1, keepdim=True)
    r_lo = torch.rsqrt(sq_hi / Dh + eps) * (1 - RN_HEAD)
    r_hi = torch.rsqrt(sq_lo / Dh + eps) * (1 + RN_HEAD)
    corners = torch.stack([a * r * w64 for a in (lo64, hi64) for r in (r_lo, r_hi)])
    ref = mid64 * torch.rsqrt((mid64 ** 2).mean(-1, keepdim=True) + eps) * w64
    return rbf(corners.amin(0)), rbf(corners.amax(0)), rbf(ref)


def qkv_split(t, H, Hkv, Dh):
    n = t.shape[0]
    return (t[:, : H * Dh].reshape(n, H, Dh), t[:, H * Dh: (H + Hkv) * Dh].reshape(n, Hkv, Dh),
            t[:, (H + Hkv) * Dh:].reshape(n, Hkv, Dh))


def qkv_norm(lo, hi, mid, H, Hkv, Dh, q_norm, k_norm, eps, norm_fn):
    """q, k (after the qk-norm, before RoPE) and v brackets from brackets of the biased, rounded qkv row."""
    (ql, kl, vl), (qh, kh, vh), (qm, km, vm) = (qkv_split(t, H, Hkv, Dh) for t in (lo, hi, mid))
    if q_norm is not None:
        ql, qh, qm = norm_fn(ql, qh, qm, q_norm, eps)
        kl, kh, km = norm_fn(kl, kh, km, k_norm, eps)
    return (ql, qh, qm), (kl, kh, km), (vl, vh, vm)


def qkv_chain(lo, hi, mid, H, Hkv, Dh, q_norm, k_norm, eps, cs, norm_fn):
    """q, k (after qk-norm and RoPE) and v brackets from brackets of the biased, rounded qkv row."""
    q, k, v = qkv_norm(lo, hi, mid, H, Hkv, Dh, q_norm, k_norm, eps, norm_fn)
    return rope_bracket(*q, cs), rope_bracket(*k, cs), v


def qkv_emul(ws, bias, H, Hkv, Dh, q_norm, k_norm, eps, cs):
    """qkv_prep_row_kernel on the kernel's own fp32 GEMM result ws [rows, Nqkv]: rbf(ws + bias), qk-norm (rsqrtf
    bracket), RoPE. Returns ((lo, hi, mid) of q, of k, of v)."""
    v = ws.float()
    if bias is not None:
        v = v + bias.float()[None, :]
    v = rbf(v)

    def norm(lo, hi, mid, w, e):
        a = head_norm_emul(lo, w, e)
        return a[0], a[1], a[2]

    return qkv_chain(v, v, v, H, Hkv, Dh, q_norm, k_norm, eps, cs, norm)


def qkv_ref64(xn, W, bias, H, Hkv, Dh, q_norm, k_norm, eps, cs):
    """The float64 chain of the prefill qkv stage from its operand xn."""
    lo, hi, mid = gemm_bracket(xn, W, bias)
    return qkv_chain(lo, hi, mid, H, Hkv, Dh, q_norm, k_norm, eps, cs, head_norm64)


def fixup_ref64(x, ssq, norm_w, W, bias, H, Hkv, Dh, q_norm, k_norm, eps):
    """The float64 chain of the decode qkv step GEMM and its fix-up from the operand x normalised on load with ssq:
    brackets of q and k after the qk-norm, before RoPE, and of v (test_decode_attn_gpu docstring)."""
    y, E = normed_gemm(x, ssq, norm_w, eps, W)
    if bias is not None:
        y = y + bias.double()[None, :]
    return qkv_norm(*bracket_bf16(y, E), rbf(y), H, Hkv, Dh, q_norm, k_norm, eps, head_norm64)


# ---------------------------------------------------------------------------------------------------------------------
# residual add + norm, SwiGLU
# ---------------------------------------------------------------------------------------------------------------------
def resid_emul(x, ws, bias):
    """rbf(x + rbf(ws + bias)) in fp32 (resid_norm4_kernel before the norm)."""
    y = ws.float()
    if bias is not None:
        y = y + bias.float()[None, :]
    return rbf(x.float() + rbf(y))


def resid_ref64(x, a, W, bias):
    """(lo, hi, mid) of the residual add from the GEMM operand a in float64."""
    ylo, yhi, ymid = gemm_bracket(a, W, bias)
    xf = x.float()
    return rbf(xf + ylo), rbf(xf + yhi), rbf(xf + ymid)


def _silu(g, f):
    """rbf(g / (1 + expf(-g))) with the add and the division in fp32 as the kernels do; f = 1 -+ EXP_ULP brackets an
    expf that is off by up to 2 fp32 ulp."""
    ef = (torch.exp(-g.double()) * f).float()
    return rbf(g / (1.0 + ef))


def swiglu_from(g_lo, g_hi, g_mid, u_lo, u_hi, u_mid):
    """h = rbf(rbf(silu(g)) u) with expf within 2 ulp: the extremes over the corners of g, u and expf."""
    corners = torch.stack([rbf(_silu(g, f) * u) for g in (g_lo, g_hi) for f in (1 - EXP_ULP, 1 + EXP_ULP)
                           for u in (u_lo, u_hi)])
    return corners.amin(0), corners.amax(0), rbf(_silu(g_mid, 1.0) * u_mid)


def swiglu_emul(ws, I):
    """swiglu4_kernel (interleaved) on the kernel's own fp32 result ws [rows, n13]."""
    gi = gate_row(torch.arange(I, device=ws.device))
    g, u = rbf(ws[:, gi]), rbf(ws[:, gi + 16])
    return swiglu_from(g, g, g, u, u, u)


def swiglu_ref64(xn, w1, w3):
    g = gemm_bracket(xn, w1)
    u = gemm_bracket(xn, w3)
    return swiglu_from(g[0], g[1], g[2], u[0], u[1], u[2])


# ---------------------------------------------------------------------------------------------------------------------
# attention over [0, pos]
# ---------------------------------------------------------------------------------------------------------------------
def attn_ref64(q, K, V, pos, scale, tiles=None, p_hi_only=False):
    """q float64 [n, Hkv, G, Dh]; K, V float64 [Hkv, L, Dh]; pos int [n] (each < L). Returns (o, E) [n, Hkv, G, Dh]:
    the float64 softmax(q k^T scale) v over positions [0, pos] and the bound of attn_tile_kernel's arithmetic around
    it (test_prefill_gpu docstring). tiles [n]: 64-position tiles the kernel walks for each row (pos // 64 + 1).
    p_hi_only: a wrong reference whose probabilities are single bf16 values (the hi + lo split dropped)."""
    n, Hkv, G, Dh = q.shape
    L = K.shape[1]
    pos = pos.to(q.device).long()
    tiles = (pos // PAGE + 1) if tiles is None else tiles.to(q.device)
    kp = torch.arange(L, device=q.device)
    mask = (kp[None, :] <= pos[:, None])[:, None, None, :]  # [n, 1, 1, L]
    s = scale * torch.einsum("nhgd,hld->nhgl", q, K)
    s = s.masked_fill(~mask, -math.inf)
    m = s.amax(-1, keepdim=True)
    w = torch.exp(s - m)
    l = w.sum(-1, keepdim=True)
    if p_hi_only:
        o = torch.einsum("nhgl,hld->nhgd", rbf(w).double(), V) / l
    else:
        o = torch.einsum("nhgl,hld->nhgd", w, V) / l
    p = w / l
    pv = torch.einsum("nhgl,hld->nhgd", p, V.abs())
    absqk = scale * torch.einsum("nhgd,hld->nhgl", q.abs(), K.abs()).masked_fill(~mask, 0.0)
    sf = s.masked_fill(~mask, 0.0)
    smax = sf.abs().amax(-1, keepdim=True)
    T = tiles.double()[:, None, None, None]
    KS = Dh // 16
    spread = (sf - m).masked_fill(~mask, 0.0).abs().amax(-1, keepdim=True)
    eps_s = (KS * MU * absqk).amax(-1, keepdim=True) + 2.0 ** -24 * (3 * smax + 3 * spread) + 2 * EXP_ULP
    kappa = 2 * EXP_ULP + 2.0 ** -23 * smax
    eta = eps_s + T * kappa
    rel = torch.expm1(2 * eta) + 2.0 ** -16 + (8 * T + 1) * MU * torch.exp(2 * eta) + (20 * T + 2) * 2.0 ** -24
    return o, rel * pv


def attn_decode_fp32(q, qd, K, V, scale):
    """attn_decode_kernel's fp32 path (the slow stack): q, qd (its bracket width) float64 [Hkv, G, Dh]; K, V
    [Hkv, L, Dh] -> (o, E) [Hkv, G, Dh], the float64 softmax(q k^T scale) v and the bound around it
    (test_decode_attn_gpu docstring)."""
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


def attn_decode_bf16(qlo, qhi, qm, K, V, scale32):
    """attn_decode_kernel's all-bf16 path (the fast stack): brackets (lo, hi) and the float64 rounding chain (mid),
    [Hkv, G, Dh] (test_decode_attn_gpu docstring)."""
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


def rotate_by(q, cs1):
    """q float64 [..., Dh] rotated by one more position: cs1 float [Dh/2, 2] (the table's row 1)."""
    c, s = cs1[:, 0].double(), cs1[:, 1].double()
    x0, x1 = q[..., 0::2], q[..., 1::2]
    return torch.stack([x0 * c - x1 * s, x1 * c + x0 * s], -1).flatten(-2)


def paged_history(cache_layer, table_row, L):
    """Positions [0, L) of one sequence through its page-table row: float64 [Hkv, L, Dh]. Unmapped pages read zero."""
    n = (L + PAGE - 1) // PAGE
    pages = table_row[:n].long()
    c = cache_layer[pages.clamp(min=0)].double()  # [n, Hkv, 64, Dh]
    c[pages < 0] = 0.0
    return c.permute(1, 0, 2, 3).reshape(c.shape[1], n * PAGE, -1)[:, :L]
