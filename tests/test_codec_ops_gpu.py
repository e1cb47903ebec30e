"""The codec's kernels (csrc/codec_kernels.cu, the fused epilogues of csrc/gemm_tc.cu) one layer at a time, against
float64 references built from the same operands the GPU reads.

Each kernel runs through its C-ABI entry point on the packed buffers of a real DAC (tiny_config() and full_config()
of oracle.codec_oracle, weights from make_weights), so a test covers the kernel and the load-time packing together.
The reference for each layer is the oracle's own function for it (causal_conv, causal_conv_transpose, snake, the
pieces of convnext, _vq_from_codes, _vq_encode) evaluated in float64 on weights rounded the way DAC._pack rounds
them: weight norm folded in fp32, bf16 for GEMM weights, fp32 for the depthwise conv, LayerNorm, gamma, bias, Snake
alpha and the VQ tables. Whole-waveform SNR cannot see an error confined to a few samples (a tile edge, a causal pad,
a batch boundary) or a small change of every sample (an eps, a GELU variant); these checks see both.

Bounds. u = 2^-24 is the unit roundoff of fp32. For each op an fp32 error bound E of the value before its bf16
store is derived from the kernel's arithmetic, and every bf16 output must lie in [rbf(v - E), rbf(v + E)], v the
float64 value: bit-identical wherever that bracket holds one value. Fewer than 1 % of the outputs may differ from
rbf(v). Terms of order u^2 are dropped where stated; every such bound is multiplied by SECOND_ORDER = 1 + 2^-10.
  * GEMM accumulation (fsb_conv_gemm): |acc - v| <= C_CONV * (|W| |X|), C_CONV = 2^-18. The worst case of the fp32
    accumulation, (K / 16 + 1) 2^-23 (|W| |X|) (test_step_gemm_gpu), would leave most bf16 roundings undecided at
    K = 4096, so, as C_AMB there, this is a measured error with at least 4x margin (below).
  * Epilogue, in the kernel's order: + bias (one rounding: u |v|); GELU; * gamma (u); + residual (u); bf16 store.
    GELU is 0.5 x (1 + erff(x / sqrt 2)): its error is at most 0.5 |x| G_ERF, where G_ERF = 2^-20 covers erff and the
    three fp32 roundings around it, plus 1.13 (the largest slope of GELU) times the error of its input.
  * Snake, y = v + s^2 / (alpha + 1e-9), s = sin(alpha v): with ds = alpha E_v + u |alpha v| + e_sin the error of s,
    |dy| <= E_v + |1/alpha| (2 |s| ds + ds^2) + 4 u |s^2 / alpha| + 2 u |y|. The epilogue's snake_fast uses __sinf,
    whose error is only documented on [-pi, pi]; the allowance is e_sin = ALLOW_SIN(z) = 2^-19 (1 + |z|) for the
    argument z = alpha v. fsb_first_conv and fsb_snake use sinf, 2 ulp: e_sin = 2^-23.
  * fsb_first_conv: acc = bias + 7 fused multiply-adds: E = 8 u (|b| + sum |w| |x|).
  * fsb_dwconv_ln: conv as above, E_c = (K + 1) u A_c. The mean is a block sum (8 + 5 + 5 roundings) and one
    division: E_m = mean(E_c) + 20 u mean|v|. d_c = v_c - m: E_d = E_c + E_m + u |d_c|. var = sum(d^2) / C:
    E_var = mean(2 |d| E_d) + 21 u var. rsqrtf(var + eps): relative error 0.5 E_var / (var + eps) + 0.5 u + 2^-22.
    y = d r g + b: E_y = |g| r (E_d + |d| (E_r + u)) + u |y|. First order, times SECOND_ORDER.
  * fsb_final_conv_tanh (fp32 out): K C fused multiply-adds, then tanhf (2 ulp, slope <= 1):
    |wav - tanh(v)| <= K C u (|b| + sum |w| |a|) + 2^-23.
  * fsb_snake: the Snake bound with E_v = 0 (the input is bf16) and sinf.
  * fsb_codebook_sum: sum_s tab_s[code_s] with first + (rest in stage order) in fp32: S u sum |tab|, plus the error of
    the fp32 tables folded at load, (cd + 1) u (|codebook| |W_out| + |b_out|) per stage. The kernel's fp32 sum is also
    emulated in torch in the same order, and the bits must be equal.
  * fsb_vq_encode, teacher-forced: after each stage the float64 residual subtracts the table row of the code the GPU
    chose, so each stage is judged on its own. The kernel's in_proj has D / 32 + 6 roundings and reads a residual
    that differs from the float64 one by the fp32 subtractions and table errors of the earlier stages (dres); with
    de = (D / 32 + 6) u (|W_in| |res| + |b_in|) + |W_in| dres, every cosine score is off by at most
    ES = 2 |de| / |e| + (2 cd + 5) u + 2^-22 (normalisation, the fp32 unit codebook, the cd-term dot product, rsqrtf).
    The reference maximises -dist = 2 cos - 2, so the GPU's code must equal the float64 argmax unless the float64 gap
    between them is at most 4 ES (about 1e-5 at the full geometry).

Measured on an H100 80GB HBM3 (SXM, 700 W power limit) by test_conv_gemm_error_allowances, which keeps each at
least 4x inside its allowance:
  * erff in gelu_erf: the worst |gelu_erf(x) - gelu(x)| / (0.5 |x|) over x on the bf16 grid in [-10, 10] is
    2^-22.31, 5x inside G_ERF = 2^-20.
  * __sinf in snake_fast: the worst |__sinf(z) - sin(z)| for |z| up to 300 is 2^-14.86 (it grows about like
    2^-23 |z|); its worst ratio to ALLOW_SIN(z) is 0.124, 8x inside.
  * conv GEMM accumulation: the worst |acc - v| / (|W| |X|) is 2^-20.43 (the dilated conv7, 7 taps x 768 channels;
    pw2 at K = 4096, the stride-8 encoder conv and the stride-8 ConvTranspose: 2^-20.85 .. 2^-20.70), 5.4x inside
    C_CONV.

Teeth. Each op has at least one wrong reference that must fail the bound on a least share (TEETH) of the outputs it
changes; any output outside its bracket already fails the check. The shares seen on the H100 are in brackets:
  * codebook_sum with the semantic stage dropped: test_codebook_sum [99.4 - 99.7 %];
  * dwconv_ln with LayerNorm eps 1e-5, on the rows of variance ~1e-6: test_dwconv_ln [99.5 - 100 %]; the input one
    row late (one tap shifted by one step) [99.9 %]; the window's history zeroed: test_dwconv_ln_window [99.6 % of
    the first 6 rows]. A mean without its "/ C" in dwconv_ln_row fails every test_dwconv_ln case outright;
  * first_conv with the waveform one sample late: test_first_conv [99.9 - 100 %];
  * final_conv_tanh with the halo row before the last tile dropped [16 of 16 outputs], and with batch 0's tail as
    batch 1's history [30 of 30 per C]: test_final_conv_tanh. A "+ K - 1" dropped from final_conv_tanh_kernel's halo
    rows fails it outright;
  * snake with each channel's alpha taken from its neighbour: test_snake [84 - 85 %: inputs go down to |x| ~ 0.01];
  * vq_encode with the second-best code as the reference's answer: test_vq_encode [98.9 - 100 % of the codes];
  * conv_gemm: tanh-approximated GELU in pw1 [4.1 - 6.5 % of all outputs: it moves GELU by at most ~5e-4];
    Snake alphas of a transposed conv in (co, p) order instead of (p, co) [86 - 89 %];
    batch 0's tail as batch 1's causal history [100 %]; the window's history zeroed [99.5 %]: test_conv_gemm_*.
"""
from __future__ import annotations

import ctypes
import math
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from oracle import codec_oracle as CO
from tests.kernel_ref import C_CONV, bf16_key, bracket_bf16, check_bracket, rbf
from tests.lm_util import _bits, _gen, _lib, _randn

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SECOND_ORDER = 1 + 2.0 ** -10
G_ERF = 2.0 ** -20  # GELU allowance, relative to 0.5 |x| (module docstring)
SIN_ACC = 2.0 ** -23  # sinf: 2 ulp of a value below 1


def allow_sin(z):
    """__sinf allowance (absolute) at argument z (module docstring)."""
    return 2.0 ** -19 * (1 + z.abs())


# least share of the outputs a wrong reference changes that must fall outside the bound (module docstring)
TEETH = {"cb-semantic": 0.9, "ln-eps": 0.9, "dw-shift": 0.9, "dw-window": 0.9, "fc-shift": 0.9, "halo": 0.8,
         "batch": 0.8, "snake-alpha": 0.75, "vq-second": 0.9, "gelu-tanh": 0.02, "snake-co-p": 0.8, "leak": 0.9,
         "win": 0.9}


def _L():
    return _lib().lib()


def _check(rc):
    _lib().check(rc)


def _st():
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# the two geometries
# ---------------------------------------------------------------------------------------------------------------------
def _make(name):
    from tests.test_codec_gpu import build

    cfg = CO.tiny_config() if name == "tiny" else CO.full_config()
    w = CO.make_weights(cfg, seed=17)
    return SimpleNamespace(name=name, cfg=cfg, w=w, dac=build(cfg, w))


@pytest.fixture(scope="module")
def tiny():
    return _make("tiny")


@pytest.fixture(scope="module")
def full():
    return _make("full")


def _folded(g, prefix, bf16):
    """The weight the kernel reads, float64 on the GPU: weight norm folded in fp32 as DAC._eff_weight does, rounded
    to bf16 for a GEMM. Returns (W, bias or None)."""
    W = CO._wn_weight(g.w, prefix).float()
    if bf16:
        W = W.bfloat16()
    b = g.w.get(f"{prefix}.bias")
    return W.double().cuda(), (b.double().cuda() if b is not None else None)


def _d(W, b, name="c"):
    return {f"{name}.weight": W, f"{name}.bias": b}


def _alpha(g, prefix):
    return g.w[f"{prefix}.alpha"].reshape(-1).double().cuda()


def _cl(x):
    """[B, C, T] float64 <-> [B, T, C]."""
    return x.transpose(1, 2)


class Teeth:
    def __init__(self):
        self.seen: dict = {}

    def add(self, key, got, lo, hi, mask=None):
        out = (got < lo) | (got > hi)
        if mask is not None:
            out = out[mask]
        n, k = self.seen.get(key, (0, 0))
        self.seen[key] = (n + out.numel(), k + int(out.sum()))

    def report(self, what):
        for key, (n, k) in self.seen.items():
            print(f"{what}: wrong reference '{key}' rejected for {k} of {n} outputs ({100.0 * k / max(n, 1):.1f} %)")
        for key, (n, k) in self.seen.items():
            assert n > 0 and k >= TEETH[key] * n, f"{what}: the bound accepts a wrong reference ({key}): {k} of {n}"


def _snake_ref(v, E, alpha, e_sin):
    """(y, E_y) of Snake over a value v known to +-E (module docstring); alpha broadcasts over the last dim."""
    ia = 1.0 / (alpha + 1e-9)
    z = alpha * v
    s = torch.sin(z)
    y = v + ia * s * s
    ds = alpha.abs() * E + U * z.abs() + e_sin(z)
    Ey = E + ia.abs() * (2 * s.abs() * ds + ds * ds) + 4 * U * (ia * s * s).abs() + 2 * U * y.abs()
    return y, Ey


def _epi(v, absprod, bias=None, gelu=False, gamma=None, resid=None):
    """(value, bound) of the conv GEMM epilogue before the bf16 store (module docstring)."""
    E = C_CONV * absprod
    if bias is not None:
        v = v + bias
        E = E + U * (v.abs() + E)
    if gelu:
        E = 1.13 * E + 0.5 * v.abs() * G_ERF
        v = F.gelu(v)
    if gamma is not None:
        v = v * gamma
        E = E * gamma.abs() + U * (v.abs() + E)
    if resid is not None:
        v = v + resid
        E = E + U * (v.abs() + E)
    return v, E


# ---------------------------------------------------------------------------------------------------------------------
# 1. fsb_codebook_sum
# ---------------------------------------------------------------------------------------------------------------------
def _vq_prefixes(cfg):
    return ["quantizer.semantic_quantizer.quantizers.0"] + [f"quantizer.quantizer.quantizers.{i}"
                                                            for i in range(cfg.n_codebooks)]


def _vq_ref_weights(g):
    """The VQ weights in float64 on the GPU, in_proj / out_proj folded in fp32 like DAC._vq_tables."""
    out = {}
    for p in _vq_prefixes(g.cfg):
        for proj in ("in_proj", "out_proj"):
            W, b = _folded(g, f"{p}.{proj}", bf16=False)
            out[f"{p}.{proj}.weight"], out[f"{p}.{proj}.bias"] = W, b
        out[f"{p}.codebook.weight"] = g.w[f"{p}.codebook.weight"].double().cuda()
    return out


@pytest.mark.parametrize("name", ["tiny", "full"])
def test_codebook_sum(name, request):
    """Both geometries (stages of 4096 / 1024 or 256 / 64 entries, D = 1024 / 256), B = 3, T = 37, codes at 0, at
    size - 1 and above size (clamped like quantizer_decode)."""
    g = request.getfixturevalue(name)
    cfg, dac = g.cfg, g.dac
    B, T, S, D = 3, 37, dac.n_stage, cfg.latent_dim
    sizes = [cfg.semantic_codebook_size] + [cfg.codebook_size] * cfg.n_codebooks
    gen = torch.Generator().manual_seed(3)
    idx = torch.stack([torch.randint(0, n, (B, T), generator=gen) for n in sizes], 1)
    for s, n in enumerate(sizes):
        idx[:, s, 0], idx[:, s, 1], idx[:, s, 2] = 0, n - 1, n + 5 + s
        idx[1, s, 3] = 10 ** 6
    didx = idx.int().cuda().contiguous()
    out = torch.empty(B, T, D, dtype=torch.bfloat16, device="cuda")
    _check(_L().fsb_codebook_sum(didx.data_ptr(), dac.vq_tab_ptrs.data_ptr(), dac.vq_sizes.data_ptr(), S, B, T, D,
                                 out.data_ptr(), _st()))
    torch.cuda.synchronize()
    # the clamp of quantizer_decode (rvq.py:354-359)
    ci = idx.clone()
    ci[:, 0] = ci[:, 0].clamp(max=cfg.semantic_codebook_size - 1)
    ci[:, 1:] = ci[:, 1:].clamp(max=cfg.codebook_size - 1)
    ci = ci.cuda()
    # bits: first + (rest in stage order), fp32, one rounding
    tabs = [t[ci[:, s]] for s, t in enumerate(dac.vq_tabs)]  # [B, T, D] fp32 each
    rest = tabs[1] if S > 1 else torch.zeros_like(tabs[0])
    for t in tabs[2:]:
        rest = rest + t
    emu = (tabs[0] + rest).bfloat16()
    assert torch.equal(_bits(out), _bits(emu)), f"{name}: codebook_sum differs from its fp32 emulation"
    # float64 oracle, from the codebooks and out_proj (the tables are folded at load)
    wr = _vq_ref_weights(g)
    v = _cl(CO._vq_from_codes(wr, "quantizer.semantic_quantizer", ci[:, :1]) +
            CO._vq_from_codes(wr, "quantizer.quantizer", ci[:, 1:]))
    E = 0.0
    tabs64 = []
    for s, p in enumerate(_vq_prefixes(cfg)):
        cb, Wo, bo = wr[f"{p}.codebook.weight"], wr[f"{p}.out_proj.weight"][:, :, 0], wr[f"{p}.out_proj.bias"]
        tab_abs = cb.abs() @ Wo.abs().T + bo.abs()
        t64 = (cb @ Wo.T + bo)[ci[:, s]]
        tabs64.append(t64)
        E = E + (cfg.codebook_dim + 1) * U * tab_abs[ci[:, s]] + S * U * t64.abs()
    check_bracket(out.float(), *bracket_bf16(v, E), f"{name}: codebook_sum", rbf(v))
    teeth = Teeth()
    teeth.add("cb-semantic", out.float(), *bracket_bf16(v - tabs64[0], E))
    teeth.report(f"{name} codebook_sum")


# ---------------------------------------------------------------------------------------------------------------------
# 2. fsb_dwconv_ln
# ---------------------------------------------------------------------------------------------------------------------
def _synthetic_cnx(C, seed):
    """ConvNeXt depthwise conv + LayerNorm parameters of C channels, distributed like make_weights'."""
    gen = torch.Generator().manual_seed(seed)
    w = {"n.dwconv.conv.weight": torch.randn(C, 1, 7, generator=gen) / math.sqrt(7),
         "n.dwconv.conv.bias": torch.randn(C, generator=gen) * 0.02,
         "n.norm.weight": 1 + 0.1 * torch.randn(C, generator=gen), "n.norm.bias": torch.randn(C, generator=gen) * 0.02}
    f = lambda t: t.float().cuda().contiguous()
    cn = dict(dw=f(w["n.dwconv.conv.weight"][:, 0]), dw_b=f(w["n.dwconv.conv.bias"]), ln_w=f(w["n.norm.weight"]),
              ln_b=f(w["n.norm.bias"]), k=7)
    return w, "n", cn


def _dw_case(g, C):
    """(weights dict, prefix, packed convnext dict) of a ConvNeXt with C channels: the DAC's own where it has one."""
    if g is not None and C == g.cfg.latent_dim:
        return g.w, "quantizer.upsample.0.1", g.dac.up[0]["cnx"]
    return _synthetic_cnx(C, C)


def _dw_input(cn, B, T, C, seed):
    """Random bf16 rows, plus designed rows t whose 6 predecessors are zero, so the conv output is bias + w6 x_t:
    rows of variance ~1e-6 (where eps matters) and rows with a common offset of 100 (where a one-pass variance would
    cancel). Returns x and the row masks [B, T]."""
    x = _randn((B, T, C), seed).float()
    tiny_var = torch.zeros(B, T, dtype=torch.bool, device="cuda")
    offset = torch.zeros_like(tiny_var)
    gen = _gen(seed + 1)
    w6, bias = cn["dw"][:, -1].double(), cn["dw_b"].double()
    rows = [(b, t) for b in range(B) for t in ([0] if T < 40 else range(0, T, 40))]
    for n, (b, t) in enumerate(rows):
        x[b, max(0, t - 6): t] = 0
        if n % 3 == 1:
            target = 100 + torch.randn(C, generator=gen, device="cuda", dtype=torch.float64)
            offset[b, t] = True
        else:
            target = 1e-3 * torch.randn(C, generator=gen, device="cuda", dtype=torch.float64)
            tiny_var[b, t] = True
        x[b, t] = ((target - bias) / w6).float()
    return x.bfloat16(), tiny_var, offset


def _dwconv_ln_ref(w, prefix, x, eps=1e-6, shift=0):
    """(y, E) of causal dwconv + LayerNorm in float64 (oracle convnext's first half) over x bf16 [B, T, C]."""
    C = x.shape[-1]
    x64 = _cl(x.double())
    if shift:
        x64 = F.pad(x64, (shift, 0))[..., : x64.shape[-1]]
    Wd = w[f"{prefix}.dwconv.conv.weight"].double().cuda()
    bd = w[f"{prefix}.dwconv.conv.bias"].double().cuda()
    v = _cl(CO.causal_conv(_d(Wd, bd), "c", x64, groups=C))
    A = _cl(CO.causal_conv(_d(Wd.abs(), bd.abs()), "c", x64.abs(), groups=C))
    lw, lb = w[f"{prefix}.norm.weight"].double().cuda(), w[f"{prefix}.norm.bias"].double().cuda()
    y = F.layer_norm(v, (C,), lw, lb, eps)
    K = Wd.shape[-1]
    Ec = (K + 1) * U * A
    m = v.mean(-1, keepdim=True)
    Em = Ec.mean(-1, keepdim=True) + 20 * U * v.abs().mean(-1, keepdim=True)
    d = v - m
    Ed = Ec + Em + U * d.abs()
    var = (d * d).mean(-1, keepdim=True)
    Evar = (2 * d.abs() * Ed).mean(-1, keepdim=True) + 21 * U * var
    r = 1.0 / torch.sqrt(var + eps)
    Er = 0.5 * Evar / (var + eps) + 0.5 * U + 2.0 ** -22
    E = (lw.abs() * r * (Ed + d.abs() * (Er + U)) + U * y.abs()) * SECOND_ORDER
    return y, E, var[..., 0]


DW_CASES = [(C, T) for C in (256, 1024, 2048, 200) for T in (1, 6, 7, 300)]


@pytest.mark.parametrize("C,T", DW_CASES, ids=[f"C{C}-T{T}" for C, T in DW_CASES])
def test_dwconv_ln(C, T, request):
    """C = 256 / 1024 (the DAC's own ConvNeXt), 2048 (8 channels per thread), 200 (a partial last pass); K = 7, B = 2;
    rows of variance ~1e-6 and rows with a large common offset."""
    g = request.getfixturevalue("tiny" if C == 256 else "full") if C in (256, 1024) else None
    w, prefix, cn = _dw_case(g, C)
    B = 2
    x, tiny_var, offset = _dw_input(cn, B, T, C, seed=C + T)
    y = torch.empty(B, T, C, dtype=torch.bfloat16, device="cuda")
    _check(_L().fsb_dwconv_ln(x.data_ptr(), cn["dw"].data_ptr(), cn["dw_b"].data_ptr(), cn["ln_w"].data_ptr(),
                              cn["ln_b"].data_ptr(), B, T, C, cn["k"], 1e-6, y.data_ptr(), _st()))
    torch.cuda.synchronize()
    v, E, var = _dwconv_ln_ref(w, prefix, x)
    got = y.float()
    check_bracket(got, *bracket_bf16(v, E), f"dwconv_ln C={C} T={T}", rbf(v))
    assert tiny_var.any() and offset.any() and (var[tiny_var] < 1e-5).all()
    teeth = Teeth()
    v5 = _dwconv_ln_ref(w, prefix, x, eps=1e-5)[0]
    teeth.add("ln-eps", got, *bracket_bf16(v5, E), mask=tiny_var)
    if T > 1:
        vs = _dwconv_ln_ref(w, prefix, x, shift=1)[0]
        rows = torch.zeros(B, T, dtype=torch.bool, device="cuda")
        rows[:, 1:] = True
        teeth.add("dw-shift", got, *bracket_bf16(vs, E), mask=rows & ~tiny_var & ~offset)
    teeth.report(f"dwconv_ln C={C} T={T}")


def test_dwconv_ln_window(full):
    """fsb_dwconv_ln_window as DecodeStreamPool calls it: rows 0 .. H - 1 of each item are the carried history, only
    the n rows after them are computed, against the float64 conv over the full rows."""
    cn = full.dac.up[1]["cnx"]
    prefix = "quantizer.upsample.1.1"
    B, H, n, C = 2, 6, 37, full.cfg.latent_dim
    x = _randn((B, H + n, C), seed=41)
    y = torch.empty(B, n, C, dtype=torch.bfloat16, device="cuda")
    _check(_L().fsb_dwconv_ln_window(x.data_ptr(), cn["dw"].data_ptr(), cn["dw_b"].data_ptr(), cn["ln_w"].data_ptr(),
                                     cn["ln_b"].data_ptr(), B, H + n, H, n, C, cn["k"], 1e-6, y.data_ptr(), _st()))
    torch.cuda.synchronize()
    v, E, _ = _dwconv_ln_ref(full.w, prefix, x)
    got = y.float()
    check_bracket(got, *bracket_bf16(v[:, H:], E[:, H:]), "dwconv_ln_window", rbf(v[:, H:]))
    x0 = x.clone()
    x0[:, :H] = 0
    v0 = _dwconv_ln_ref(full.w, prefix, x0)[0]
    teeth = Teeth()
    first = torch.zeros(B, n, dtype=torch.bool, device="cuda")
    first[:, : H] = True
    teeth.add("dw-window", got, *bracket_bf16(v0[:, H:], E[:, H:]), mask=first)
    teeth.report("dwconv_ln_window")


# ---------------------------------------------------------------------------------------------------------------------
# 3. fsb_first_conv
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,T,alphas", [("full", 2048 * 3 + 1, "dac"), ("full", 5, "range"),
                                           ("tiny", 2048 * 3 + 1, "range"), ("tiny", 3, "dac")])
def test_first_conv(name, T, alphas, request):
    """C = 64 / 16, K = 7, B = 2, T = 2048 * 3 + 1 and T < K; raw only, Snake only and both; the DAC's alphas or
    alphas from 0.05 to 5."""
    g = request.getfixturevalue(name)
    dac = g.dac
    C, K = dac.enc_in_w.shape
    B = 2
    if alphas == "dac":
        sn = dac.enc_blocks[0]["res"][0]["s0"]
        alpha, inv = sn.alpha, sn.inv
        a64 = _alpha(g, "encoder.block.1.block.0.block.0")
    else:
        alpha = torch.logspace(math.log10(0.05), math.log10(5.0), C, device="cuda").float()
        inv = (alpha + 1e-9).reciprocal()
        a64 = alpha.double()
    wav = (torch.rand(B, T, generator=_gen(T + C), device="cuda") * 2 - 1).float()
    outs = {}
    for mode in ("raw", "act", "both"):
        raw = torch.full((B, T, C), float("nan"), dtype=torch.bfloat16, device="cuda")
        act = torch.full_like(raw, float("nan"))
        _check(_L().fsb_first_conv(wav.data_ptr(), dac.enc_in_w.data_ptr(), dac.enc_in_b.data_ptr(), alpha.data_ptr(),
                                   inv.data_ptr(), B, T, C, K, raw.data_ptr() if mode != "act" else None,
                                   act.data_ptr() if mode != "raw" else None, _st()))
        outs[mode] = (raw, act)
    torch.cuda.synchronize()
    raw, act = outs["both"]
    assert torch.equal(_bits(outs["raw"][0]), _bits(raw)) and torch.equal(_bits(outs["act"][1]), _bits(act))
    assert outs["raw"][1].isnan().all() and outs["act"][0].isnan().all(), "a disabled output was written"
    W, b = _folded(g, "encoder.block.0.conv", bf16=False)

    def ref(shift=0):
        x = wav.double()[:, None]
        if shift:
            x = F.pad(x, (shift, 0))[..., :T]
        v = _cl(CO.causal_conv(_d(W, b), "c", x))
        A = _cl(CO.causal_conv(_d(W.abs(), b.abs()), "c", x.abs()))
        return v, (K + 1) * U * A

    v, E = ref()
    check_bracket(raw.float(), *bracket_bf16(v, E), f"first_conv {name} T={T} raw", rbf(v))
    y, Ey = _snake_ref(v, E, a64, lambda z: SIN_ACC)
    ref_y = _cl(CO.snake(_cl(v), a64[None, :, None]))
    assert torch.allclose(ref_y, y, rtol=0, atol=1e-12)
    check_bracket(act.float(), *bracket_bf16(y, Ey), f"first_conv {name} T={T} act", rbf(y))
    teeth = Teeth()
    vs, _ = ref(shift=1)
    teeth.add("fc-shift", raw.float(), *bracket_bf16(vs, E))
    teeth.report(f"first_conv {name} T={T}")


# ---------------------------------------------------------------------------------------------------------------------
# 4. fsb_final_conv_tanh
# ---------------------------------------------------------------------------------------------------------------------
FC_TILE = 256


@pytest.mark.parametrize("C", [96, 16, 6])
def test_final_conv_tanh(C, request):
    """C = 96 (full) and 16 (tiny) on the 16-byte load path, 6 on the pair-load path; T = 255, 256, 257, 513 and 44100;
    B = 2, batch 1's first samples next to batch 0's tail in memory."""
    if C in (96, 16):
        g = request.getfixturevalue("full" if C == 96 else "tiny")
        n = len(g.cfg.decoder_rates) + 1
        W, b = _folded(g, f"decoder.model.{n + 1}.conv", bf16=False)
        w_dev, bias, K = g.dac.dec_out_w, g.dac.dec_out_b, g.dac.dec_out_k
        assert float(b[0]) == bias
    else:
        gen = torch.Generator().manual_seed(6)
        W = (torch.randn(1, C, 7, generator=gen) * 0.12 / math.sqrt(7 * C)).double().cuda()
        b = torch.tensor([0.01]).double().cuda()  # the fp32 value the kernel is given
        w_dev, bias, K = W[0].t().float().contiguous(), float(b[0]), 7
    B = 2
    teeth = Teeth()
    for T in (255, 256, 257, 513, 44100):
        a = _randn((B, T, C), seed=T + C)
        wav = torch.full((B, T), float("nan"), device="cuda")
        _check(_L().fsb_final_conv_tanh(a.data_ptr(), w_dev.data_ptr(), bias, B, T, C, K, wav.data_ptr(), _st()))
        torch.cuda.synchronize()

        def ref(x):
            v = CO.causal_conv(_d(W, b), "c", _cl(x))[:, 0]
            A = CO.causal_conv(_d(W.abs(), b.abs()), "c", _cl(x).abs())[:, 0]
            return torch.tanh(v), K * C * U * A + 2.0 ** -23

        a64 = a.double()
        v, E = ref(a64)
        err = (wav.double() - v).abs()
        bad = ~(err <= E)
        assert not bad.any(), (f"final_conv C={C} T={T}: {int(bad.sum())} samples off, first at "
                               f"{bad.nonzero()[0].tolist()}: got {float(wav[bad][0])} want {float(v[bad][0])}")
        # the last tile's first K - 1 outputs without the halo row just before the tile
        t0 = (T - 1) // FC_TILE * FC_TILE
        if t0 > 0:
            x2 = a64.clone()
            x2[:, t0 - 1] = 0
            v2, _ = ref(x2)
            m = torch.zeros(B, T, dtype=torch.bool, device="cuda")
            m[:, t0: t0 + K - 1] = True
            teeth.add("halo", wav.double(), v2 - E, v2 + E, mask=m)
        # batch 1 with batch 0's tail as its history
        cat = torch.cat([a64[0], a64[1]], 0)[None]
        v3, _ = ref(cat)
        m = torch.zeros(B, T, dtype=torch.bool, device="cuda")
        m[1, : K - 1] = True
        v3b = torch.stack([v[0], v3[0, T:]])
        teeth.add("batch", wav.double(), v3b - E, v3b + E, mask=m)
    teeth.report(f"final_conv C={C}")


# ---------------------------------------------------------------------------------------------------------------------
# 5. fsb_snake
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["tiny", "full"])
def test_snake(name, request):
    """The encoder's last Snake (C = 256 / 1024, the transformer it follows) over inputs up to |x| ~ 100; n stops 77
    elements into the last row, so n is not a multiple of 256, and nothing past n is written."""
    g = request.getfixturevalue(name)
    sn = g.dac.enc_out_snake
    nb = len(g.cfg.encoder_rates) + 1
    a64 = _alpha(g, f"encoder.block.{nb}")
    C = a64.numel()
    rows = 301
    x = (torch.randn(rows, C, generator=_gen(C), device="cuda") *
         torch.logspace(-2, 2, rows, device="cuda")[:, None]).bfloat16()
    n = rows * C - (C - 77)
    y = torch.full_like(x, 1024.0)
    _check(_L().fsb_snake(x.data_ptr(), sn.alpha.data_ptr(), sn.inv.data_ptr(), n, C, y.data_ptr(), _st()))
    torch.cuda.synchronize()
    assert (y.reshape(-1)[n:].float() == 1024.0).all(), "snake wrote past n"
    v = x.double()
    ys, Ey = _snake_ref(v, torch.zeros_like(v), a64, lambda z: SIN_ACC)
    assert torch.allclose(CO.snake(v.T, a64[:, None]).T, ys, rtol=0, atol=1e-12)
    got = y.reshape(-1)[:n].float()
    ys, Ey = ys.reshape(-1)[:n], Ey.reshape(-1)[:n]
    check_bracket(got, *bracket_bf16(ys, Ey), f"snake {name}", rbf(ys))
    teeth = Teeth()
    yw, _ = _snake_ref(v, torch.zeros_like(v), a64.roll(1), lambda z: SIN_ACC)
    teeth.add("snake-alpha", got, *bracket_bf16(yw.reshape(-1)[:n], Ey))
    teeth.report(f"snake {name}")


# ---------------------------------------------------------------------------------------------------------------------
# 6. fsb_vq_encode
# ---------------------------------------------------------------------------------------------------------------------
def _vq_run(dac, z, S, in_b=None):
    B, T, D = z.shape
    codes = torch.full((B, S, T), -1, dtype=torch.int32, device="cuda")
    _check(_L().fsb_vq_encode(z.data_ptr(), dac.vq_in_w.data_ptr(),
                              (in_b if in_b is not None else dac.vq_in_b).data_ptr(), dac.vq_cbn.data_ptr(),
                              dac.vq_cb_off.data_ptr(), dac.vq_sizes.data_ptr(), dac.vq_tab_ptrs.data_ptr(), S,
                              dac.cfg.codebook_dim, B, T, D, codes.data_ptr(), _st()))
    torch.cuda.synchronize()
    return codes.long()


@pytest.mark.parametrize("name,S", [("tiny", None), ("tiny", 3), ("full", None), ("full", 3)])
def test_vq_encode(name, S, request):
    """Both geometries, every stage and S = 3 (n_quantizers = 2); B = 2, T = 45; the residual chain teacher-forced
    with the GPU's codes, each code equal to the float64 argmax unless the float64 gap is within 4 ES."""
    g = request.getfixturevalue(name)
    cfg, dac = g.cfg, g.dac
    S = dac.n_stage if S is None else S
    B, T, D, cd = 2, 45, cfg.latent_dim, cfg.codebook_dim
    z = _randn((B, T, D), seed=D + S)
    codes = _vq_run(dac, z, S)
    wr = _vq_ref_weights(g)
    res = _cl(z.double())  # [B, D, T]
    dres = torch.zeros_like(res)
    teeth = Teeth()
    exact = total = 0
    for s, p in enumerate(_vq_prefixes(cfg)[:S]):
        scores = []
        CO._vq_encode(wr, p, res, scores)
        sc = scores[0]  # [B, T, K] float64 -dist
        got = codes[:, s]  # [B, T]
        Wi, bi = wr[f"{p}.in_proj.weight"][:, :, 0], wr[f"{p}.in_proj.bias"]
        e = torch.einsum("od,bdt->bot", Wi, res) + bi[None, :, None]
        de = (D / 32 + 6) * U * (torch.einsum("od,bdt->bot", Wi.abs(), res.abs()) + bi.abs()[None, :, None]) + \
            torch.einsum("od,bdt->bot", Wi.abs(), dres)
        ES = 2 * de.norm(dim=1) / e.norm(dim=1) + (2 * cd + 5) * U + 2.0 ** -22  # [B, T]
        gap = sc.amax(-1) - sc.gather(-1, got[..., None])[..., 0]
        ok = gap <= 4 * ES
        assert ok.all(), (f"{name} stage {s}: code off at {(~ok).nonzero()[0].tolist()}: float64 gap "
                          f"{float(gap[~ok][0]):.3g} > bound {float(4 * ES[~ok][0]):.3g}")
        exact += int((got == sc.argmax(-1)).sum())
        total += got.numel()
        second = sc.topk(2, -1).values[..., 1]
        wrong = (sc.amax(-1) - second) > 4 * ES  # the second-best code as the reference's answer is rejected
        n0, k0 = teeth.seen.get("vq-second", (0, 0))
        teeth.seen["vq-second"] = (n0 + wrong.numel(), k0 + int(wrong.sum()))
        # teacher forcing: subtract the table row of the GPU's code
        cb, Wo, bo = wr[f"{p}.codebook.weight"], wr[f"{p}.out_proj.weight"][:, :, 0], wr[f"{p}.out_proj.bias"]
        tab = cb[got] @ Wo.T + bo  # [B, T, D]
        tab_err = (cd + 1) * U * (cb[got].abs() @ Wo.abs().T + bo.abs())
        res = res - _cl(tab)
        dres = dres + _cl(tab_err) + U * res.abs()
    print(f"{name} S={S}: {exact} of {total} codes are the float64 argmax")
    teeth.report(f"vq_encode {name} S={S}")


def test_vq_encode_ties(tiny):
    """Duplicate codewords give the lowest index; an all-zero latent with zero in_b gives code 0 at every stage (every
    dot product is 0 and ties go to the lowest index; the kernel's own contract: float64's (-dist).max(1) would pick
    the codeword whose |c|^2 rounds smallest)."""
    cfg = tiny.cfg
    D, B, T = cfg.latent_dim, 2, 33
    # codebook rows k and k mod 37 equal in every stage: twins in the same thread, warp and in other warps
    w2 = dict(tiny.w)
    for p in _vq_prefixes(cfg):
        cb = w2[f"{p}.codebook.weight"]
        w2[f"{p}.codebook.weight"] = cb[torch.arange(cb.shape[0]) % 37].clone()
    from tests.test_codec_gpu import build

    dup = build(cfg, w2)
    codes = _vq_run(dup, _randn((B, T, D), seed=9), dup.n_stage)
    assert (codes >= 0).all() and (codes < 37).all(), f"a duplicate codeword above the lowest index won: {codes.max()}"
    # zero latent, zero in_b: each stage on its own (S = 1 on that stage's slice of the tables)
    dac = tiny.dac
    z = torch.zeros(B, T, D, dtype=torch.bfloat16, device="cuda")
    zb = torch.zeros_like(dac.vq_in_b)
    cd = cfg.codebook_dim
    for s in range(dac.n_stage):
        codes = torch.full((B, 1, T), -1, dtype=torch.int32, device="cuda")
        _check(_L().fsb_vq_encode(z.data_ptr(), dac.vq_in_w.data_ptr() + 4 * s * cd * D, zb.data_ptr(),
                                  dac.vq_cbn.data_ptr(), dac.vq_cb_off.data_ptr() + 4 * s,
                                  dac.vq_sizes.data_ptr() + 4 * s, dac.vq_tab_ptrs.data_ptr() + 8 * s, 1, cd, B, T, D,
                                  codes.data_ptr(), _st()))
        torch.cuda.synchronize()
        assert (codes == 0).all(), f"stage {s}: zero latent gave codes {codes.unique().tolist()}"


# ---------------------------------------------------------------------------------------------------------------------
# 7. fsb_conv_gemm as the codec calls it
# ---------------------------------------------------------------------------------------------------------------------
def _conv_gemm(cv, x, B, T_in, c_in, T_out, out0=None, out1=None, snake=None, resid=None, gamma=None, act=0,
               row_stride=None, batch_stride=None, shifts=None, c_out=None, out_f32=0, bias="cv"):
    vp = lambda t: None if t is None else t.data_ptr()
    b = cv.bias if bias == "cv" else bias
    _check(_L().fsb_conv_gemm(
        x.data_ptr(), B, T_in, c_in, row_stride or c_in, batch_stride or T_in * (row_stride or c_in), cv.w.data_ptr(),
        c_out or cv.c_out, cv.taps, cv.kpad, shifts or cv.shifts, T_out, vp(b), vp(gamma), vp(resid), act, vp(out0),
        vp(out1), snake.alpha.data_ptr() if snake is not None else None,
        snake.inv.data_ptr() if snake is not None else None, out_f32, _st()))


def _big_batch0(x):
    """Batch 0 scaled up, so that anything of it read into batch 1's causal pad shows."""
    x = x.clone()
    x[0] = (x[0].float() * 64).bfloat16()
    return x


def _leak_teeth(teeth, got, vfn, x64, E, rows):
    """Batch 1 computed with batch 0's tail as its history: the first `rows` outputs of batch 1."""
    cat = torch.cat([x64[0], x64[1]], -1)[None]
    vw = vfn(cat)[..., -vfn(x64[1:]).shape[-1]:]  # batch 1's outputs, [1, C, T_out]
    lo, hi = bracket_bf16(_cl(vw)[0], E[1])
    m = torch.zeros_like(lo, dtype=torch.bool)
    m[:rows] = True
    teeth.add("leak", got[1], lo, hi, mask=m)


@pytest.mark.parametrize("name", ["tiny", "full"])
def test_conv_gemm_convnext_linears(name, request):
    """pw1 (D -> 4D, bias, GELU) and pw2 (4D -> D, bias, gamma, + residual with out0 aliasing it); B = 2, T = 257."""
    g = request.getfixturevalue(name)
    cn = g.dac.up[0]["cnx"]
    prefix = "quantizer.upsample.0.1"
    D = g.cfg.latent_dim
    B, T = 2, 257
    x = _randn((B, T, D), seed=1)
    h = torch.empty(B, T, 4 * D, dtype=torch.bfloat16, device="cuda")
    _conv_gemm(cn["pw1"], x, B, T, D, T, out0=h, act=1)
    torch.cuda.synchronize()
    W1 = g.w[f"{prefix}.pwconv1.weight"].bfloat16().double().cuda()
    b1 = g.w[f"{prefix}.pwconv1.bias"].double().cuda()
    v, E = _epi(F.linear(x.double(), W1), F.linear(x.double().abs(), W1.abs()), bias=b1, gelu=True)
    check_bracket(h.float(), *bracket_bf16(v, E), f"{name} pw1", rbf(v))
    teeth = Teeth()
    vt = F.gelu(F.linear(x.double(), W1, b1), approximate="tanh")
    teeth.add("gelu-tanh", h.float(), *bracket_bf16(vt, E))
    # pw2, in place on the residual stream
    W2 = g.w[f"{prefix}.pwconv2.weight"].bfloat16().double().cuda()
    b2 = g.w[f"{prefix}.pwconv2.bias"].double().cuda()
    gam = g.w[f"{prefix}.gamma"].double().cuda()
    hh = _randn((B, T, 4 * D), seed=2, scale=0.5)
    r = _randn((B, T, D), seed=3)
    r0 = r.clone()
    _conv_gemm(cn["pw2"], hh, B, T, 4 * D, T, out0=r, gamma=cn["gamma"], resid=r)
    torch.cuda.synchronize()
    v, E = _epi(F.linear(hh.double(), W2), F.linear(hh.double().abs(), W2.abs()), bias=b2, gamma=gam,
                resid=r0.double())
    check_bracket(r.float(), *bracket_bf16(v, E), f"{name} pw2", rbf(v))
    teeth.report(f"{name} convnext linears")


def _enc_down_case(g, bi):
    blk = g.dac.enc_blocks[bi]
    s = blk["stride"]
    prefix = f"encoder.block.{bi + 1}.block.4.conv"
    if blk["tfm"] is None:
        nxt = g.dac.enc_blocks[bi + 1]["res"][0]["s0"] if bi + 1 < len(g.dac.enc_blocks) else g.dac.enc_out_snake
        nxt_p = (f"encoder.block.{bi + 2}.block.0.block.0" if bi + 1 < len(g.dac.enc_blocks)
                 else f"encoder.block.{len(g.cfg.encoder_rates) + 1}")
    else:
        nxt, nxt_p = None, None
    return blk["down"], s, prefix, nxt, nxt_p


@pytest.mark.parametrize("name,bi", [("tiny", 0), ("tiny", 2), ("full", 0), ("full", 2)])
def test_conv_gemm_encoder_strided(name, bi, request):
    """Encoder strided convs, stride 2 (block 0) and 8 (block 2): the activation read as [T/s][s c] rows, out0 raw and
    out1 Snake for the next block; B = 2 with batch 0 large, T / s = 129 (a partial second row tile)."""
    g = request.getfixturevalue(name)
    cv, s, prefix, nxt, nxt_p = _enc_down_case(g, bi)
    c = cv.c_in_eff // s
    B, Tn = 2, 129
    T = Tn * s
    x = _big_batch0(_randn((B, T, c), seed=s + c))
    out0 = torch.empty(B, Tn, cv.c_out, dtype=torch.bfloat16, device="cuda")
    out1 = torch.empty_like(out0)
    _conv_gemm(cv, x, B, Tn, s * c, Tn, out0=out0, out1=out1 if nxt else None, snake=nxt)
    torch.cuda.synchronize()
    W, b = _folded(g, prefix, bf16=True)
    x64 = _cl(x.double())
    vfn = lambda xx: CO.causal_conv(_d(W, b), "c", xx, stride=s)
    vraw = _cl(vfn(x64))
    v, E = _epi(_cl(CO.causal_conv(_d(W, None), "c", x64, stride=s)),
                _cl(CO.causal_conv(_d(W.abs(), None), "c", x64.abs(), stride=s)), bias=b)
    assert torch.allclose(v, vraw, rtol=1e-12, atol=1e-9)
    check_bracket(out0.float(), *bracket_bf16(v, E), f"{name} enc{bi} raw", rbf(v))
    if nxt is not None:
        y, Ey = _snake_ref(v, E, _alpha(g, nxt_p), allow_sin)
        check_bracket(out1.float(), *bracket_bf16(y, Ey), f"{name} enc{bi} snake", rbf(y))
    teeth = Teeth()
    _leak_teeth(teeth, out0.float(), vfn, x64, E, 1)
    teeth.report(f"{name} enc{bi}")


@pytest.mark.parametrize("name,bi", [("tiny", 0), ("tiny", 3), ("full", 0), ("full", 3)])
def test_conv_gemm_decoder_transposed(name, bi, request):
    """Decoder ConvTranspose, stride 8 (block 0: full 1536 -> 768, GEMM C_out 6144, BN 256) and stride 2 (block 3:
    full 192 -> 96, C_out 192, BN 192): out0 raw and out1 Snake through _SnakeView in (p, co) order; B = 2 with batch
    0 large, T = 131."""
    g = request.getfixturevalue(name)
    blk = g.dac.dec_blocks[bi]
    cv, s = blk["up"], blk["stride"]
    cin = g.cfg.decoder_dim // 2 ** bi
    cout = cin // 2
    B, T = 2, 131
    x = _big_batch0(_randn((B, T, cin), seed=cin + s))
    out0 = torch.empty(B, T, cv.c_out, dtype=torch.bfloat16, device="cuda")
    out1 = torch.empty_like(out0)
    _conv_gemm(cv, x, B, T, cin, T, out0=out0, out1=out1, snake=blk["up_snake"])
    torch.cuda.synchronize()
    p = f"decoder.model.{bi + 1}.block"
    W, b = _folded(g, f"{p}.1.conv", bf16=True)
    x64 = _cl(x.double())
    vfn = lambda xx: CO.causal_conv_transpose(_d(W, b), "c", xx, s)
    v, E = _epi(_cl(CO.causal_conv_transpose(_d(W, None), "c", x64, s)),
                _cl(CO.causal_conv_transpose(_d(W.abs(), None), "c", x64.abs(), s)), bias=b)  # [B, T*s, cout]
    g0, g1 = out0.view(B, T * s, cout).float(), out1.view(B, T * s, cout).float()
    check_bracket(g0, *bracket_bf16(v, E), f"{name} dec{bi} convT raw", rbf(v))
    alpha = _alpha(g, f"{p}.2.block.0")
    y, Ey = _snake_ref(v, E, alpha, allow_sin)
    assert torch.allclose(_cl(CO.snake(_cl(v), alpha[None, :, None])), y, rtol=0, atol=1e-9)
    check_bracket(g1, *bracket_bf16(y, Ey), f"{name} dec{bi} convT snake", rbf(y))
    teeth = Teeth()
    # alphas in (co, p) order: GEMM channel j = p * cout + co would get alpha[j // s]
    wrong = alpha.repeat_interleave(s).view(s, cout)  # [p, co]
    vv = v.view(B, T, s, cout)
    yw, _ = _snake_ref(vv, E.view(B, T, s, cout), wrong, allow_sin)
    lo, hi = bracket_bf16(yw.view(B, T * s, cout), Ey)
    changed = (wrong != alpha[None, :]).expand(B, T, s, cout).reshape(B, T * s, cout)
    teeth.add("snake-co-p", g1, lo, hi, mask=changed)
    _leak_teeth(teeth, g0, vfn, x64, E, s)
    teeth.report(f"{name} dec{bi}")


def test_conv_gemm_window(full):
    """One call in the shape DecodeStreamPool._gemm_win makes: the dilated (9) conv7 of the last decoder block over a
    window [nb][H + n][C], taps shifted by H = 54, batch_stride (H + n) C, out1 Snake; against float64 over
    [history; new rows]."""
    g = full
    bi = len(g.dac.dec_blocks) - 1
    ru = g.dac.dec_blocks[bi]["res"][2]
    cv, dil = ru["c7"], ru["dil"]
    C = cv.c_in_eff
    H = 6 * dil
    nb, n = 2, 37
    win = _big_batch0(_randn((nb, H + n, C), seed=77))
    out1 = torch.empty(nb, n, C, dtype=torch.bfloat16, device="cuda")
    shifts = (ctypes.c_int * cv.taps)(*[v + H for v in cv.shifts])
    _conv_gemm(cv, win, nb, H + n, C, n, out1=out1, snake=ru["s1"], shifts=shifts)
    torch.cuda.synchronize()
    prefix = f"decoder.model.{bi + 1}.block.4"
    W, b = _folded(g, f"{prefix}.block.1.conv", bf16=True)
    x64 = _cl(win.double())
    v, E = _epi(_cl(CO.causal_conv(_d(W, None), "c", x64, dilation=dil))[:, H:],
                _cl(CO.causal_conv(_d(W.abs(), None), "c", x64.abs(), dilation=dil))[:, H:], bias=b)
    alpha = _alpha(g, f"{prefix}.block.2")
    y, Ey = _snake_ref(v, E, alpha, allow_sin)
    check_bracket(out1.float(), *bracket_bf16(y, Ey), "window conv7", rbf(y))
    teeth = Teeth()
    x0 = x64.clone()
    x0[..., :H] = 0
    v0 = _cl(CO.causal_conv(_d(W, b), "c", x0, dilation=dil))[:, H:]
    y0, _ = _snake_ref(v0, E, alpha, allow_sin)
    m = torch.zeros(nb, n, C, dtype=torch.bool, device="cuda")
    m[:, :H] = True
    teeth.add("win", out1.float(), *bracket_bf16(y0, Ey), mask=m)
    teeth.report("window conv7")


def test_conv_gemm_generic_and_vector_epilogues_agree(tiny):
    """C_out = 100 (rows 100 elements apart: every chunk takes the generic epilogue) against C_out = 104 (the
    vectorised one) on the same first 100 weight rows, with bias, GELU, gamma, residual, out0 and out1: the same
    bits."""
    g = tiny
    cv = g.dac.up[0]["cnx"]["pw1"]
    D = g.cfg.latent_dim
    B, T = 2, 200
    x = _randn((B, T, D), seed=5)
    gam = g.dac.up[0]["cnx"]["gamma"]
    sn = g.dac.enc_out_snake
    r104 = _randn((B, T, 104), seed=6)
    outs = {}
    for c_out in (100, 104):
        r = r104[..., :c_out].contiguous()
        o0 = torch.empty(B, T, c_out, dtype=torch.bfloat16, device="cuda")
        o1 = torch.empty_like(o0)
        _conv_gemm(cv, x, B, T, D, T, out0=o0, out1=o1, snake=sn, resid=r, gamma=gam, act=1, c_out=c_out)
        outs[c_out] = (o0, o1)
    torch.cuda.synchronize()
    for k, what in ((0, "out0"), (1, "out1")):
        a, b = outs[100][k], outs[104][k][..., :100]
        diff = _bits(a) != _bits(b)
        assert not diff.any(), (f"{what}: generic and vectorised epilogues differ at {int(diff.sum())} elements, "
                                f"first at {diff.nonzero()[0].tolist()}; max ulp "
                                f"{int((bf16_key(a.float()) - bf16_key(b.float())).abs().max())}")


def test_conv_gemm_error_allowances(full):
    """The measured worst errors behind C_CONV, G_ERF and ALLOW_SIN (module docstring), each at least 4x inside its
    allowance. fp32 outputs (out_f32) expose the values before the bf16 store."""
    g = full
    ratios = []
    # accumulation at the codec's deepest reductions: pw2 (K = 4096), encoder stride 8 (2 taps x 2048), decoder convT
    # stride 8 (2 taps x 1536), dilated conv7 (7 taps x 768)
    B, T = 2, 257
    cases = [(g.dac.up[0]["cnx"]["pw2"], 4 * g.cfg.latent_dim, 1, None),
             (g.dac.enc_blocks[2]["down"], g.dac.enc_blocks[2]["down"].c_in_eff, 8, "encoder.block.3.block.4.conv"),
             (g.dac.dec_blocks[0]["up"], g.cfg.decoder_dim, -8, "decoder.model.1.block.1.conv"),
             (g.dac.dec_blocks[0]["res"][1]["c7"], g.cfg.decoder_dim // 2, 1, "decoder.model.1.block.3.block.1.conv")]
    for cv, c_in, s, prefix in cases:
        x = _randn((B, T, c_in), seed=c_in + s)
        out = torch.empty(B, T, cv.c_out, device="cuda")
        _conv_gemm(cv, x, B, T, c_in, T, out0=out, out_f32=1, bias=None)
        torch.cuda.synchronize()
        if prefix is None:
            W = g.w["quantizer.upsample.0.1.pwconv2.weight"].bfloat16().double().cuda()
            v, A = F.linear(x.double(), W), F.linear(x.double().abs(), W.abs())
        elif s == -8:
            W, _ = _folded(g, prefix, bf16=True)
            v = _cl(CO.causal_conv_transpose(_d(W, None), "c", _cl(x.double()), 8)).reshape(B, T, -1)
            A = _cl(CO.causal_conv_transpose(_d(W.abs(), None), "c", _cl(x.double()).abs(), 8)).reshape(B, T, -1)
            # [B, T*8, cout] rows -> the GEMM's [B, T, 8*cout] (p, co) rows
        else:
            W, _ = _folded(g, prefix, bf16=True)
            dil = 3 if s == 1 else 1
            # the strided conv reads [T][s * c] rows of the s-times-longer activation
            xx = x.double().reshape(B, T, s, c_in // s).permute(0, 3, 1, 2).reshape(B, c_in // s, T * s) \
                if s > 1 else _cl(x.double())
            v = _cl(CO.causal_conv(_d(W, None), "c", xx, stride=max(s, 1), dilation=dil))
            A = _cl(CO.causal_conv(_d(W.abs(), None), "c", xx.abs(), stride=max(s, 1), dilation=dil))
        ratios.append(float(((out.double() - v).abs() / A.clamp_min(1e-30)).max()))
    acc = max(ratios)
    print(f"conv GEMM accumulation: worst |acc - v| / (|W| |X|) = 2^{math.log2(acc):.2f} per case "
          f"{[round(math.log2(r), 2) for r in ratios]} (C_CONV = 2^-18)")
    # identity GEMMs: out[t][c] = x[t][c % 64] exactly, so the epilogue's own error is what remains
    C_in = 64
    L = _L()

    def eye_conv(c_out):
        w = torch.zeros(c_out, C_in, device="cuda")
        w[torch.arange(c_out), torch.arange(c_out) % C_in] = 1
        return SimpleNamespace(w=w.bfloat16(), bias=None, c_out=c_out, taps=1, kpad=C_in,
                               shifts=(ctypes.c_int * 1)(0))

    # GELU over the bf16 grid in [-10, 10]
    T = 256
    xs = torch.linspace(-10, 10, T * C_in, device="cuda").bfloat16().view(1, T, C_in)
    out = torch.empty(1, T, C_in, device="cuda")
    _conv_gemm(eye_conv(C_in), xs, 1, T, C_in, T, out0=out, act=1, out_f32=1)
    torch.cuda.synchronize()
    x64 = xs.double()
    nz = x64.abs() > 2.0 ** -10
    erf_ratio = float(((out.double() - F.gelu(x64)).abs()[nz] / (0.5 * x64.abs()[nz])).max())
    print(f"gelu_erf: worst |err| / (0.5 |x|) = 2^{math.log2(max(erf_ratio, 2.0 ** -60)):.2f} (G_ERF = 2^-20)")
    # __sinf: alpha v = alpha 2^-k exactly, inv_alpha = 1, so out1 = fl(s^2 + v) and |s| is recovered to ~2^-23
    Cs, T = 4096, 64
    xs = torch.zeros(1, T, C_in, device="cuda")
    xs[0] = (2.0 ** -(2 + torch.arange(T, device="cuda") % 8)).float()[:, None]
    xs = xs.bfloat16()
    alpha = torch.linspace(0.01, 1200.0, Cs, device="cuda").float()
    sn = SimpleNamespace(alpha=alpha, inv=torch.ones(Cs, device="cuda"))
    out = torch.empty(1, T, Cs, device="cuda")
    _conv_gemm(eye_conv(Cs), xs, 1, T, C_in, T, out1=out, snake=sn, out_f32=1)
    torch.cuda.synchronize()
    v = xs.double()[0, :, :1]  # [T, 1]
    z = alpha.double()[None, :] * v  # exact in fp32 too
    s64 = torch.sin(z)
    s_gpu = (out[0].double() - v).clamp_min(0).sqrt()
    big = s64.abs() > 0.25
    sin_err = (s_gpu - s64.abs()).abs()
    sin_ratio = float((sin_err[big] / allow_sin(z)[big]).max())
    print(f"__sinf: worst |err| = 2^{math.log2(float(sin_err[big].max())):.2f} for |z| <= {float(z.abs().max()):.0f}; "
          f"worst |err| / ALLOW_SIN = {sin_ratio:.3f}")
    assert acc <= C_CONV / 4, f"conv GEMM accumulation error 2^{math.log2(acc):.2f} leaves C_CONV less than 4x"
    assert erf_ratio <= G_ERF / 4, f"gelu_erf error 2^{math.log2(erf_ratio):.2f} leaves G_ERF less than 4x"
    assert sin_ratio <= 0.25, f"__sinf error {sin_ratio:.3f} of ALLOW_SIN leaves less than 4x"


# ---------------------------------------------------------------------------------------------------------------------
# 8. rejections: an error message, nothing launched
# ---------------------------------------------------------------------------------------------------------------------
def test_rejections(tiny):
    _l = _lib()
    L = _L()
    dac = tiny.dac
    d = torch.zeros(1 << 20, device="cuda")
    p = d.data_ptr()
    cv = dac.up[0]["cnx"]["pw1"]

    def refused(call, match):
        n0 = _l.launch_count()
        with pytest.raises(_l.FsbError, match=match):
            _check(call())
        assert _l.launch_count() == n0, f"{match}: a kernel was launched"

    refused(lambda: L.fsb_dwconv_ln(p, p, p, p, p, 1, 4, 2049, 7, 1e-6, p, _st()), "C=2049 too large")
    refused(lambda: L.fsb_vq_encode(p, p, p, p, dac.vq_cb_off.data_ptr(), dac.vq_sizes.data_ptr(),
                                    dac.vq_tab_ptrs.data_ptr(), 1, 17, 1, 1, 64, p, _st()), "codebook_dim 17")
    sh = (ctypes.c_int * 9)(*range(9))
    refused(lambda: L.fsb_conv_gemm(p, 1, 8, 64, 64, 512, cv.w.data_ptr(), cv.c_out, 1, 96, sh, 8, None, None, None, 0,
                                    p, None, None, None, 0, _st()), "kpad must be a multiple of 64")
    refused(lambda: L.fsb_conv_gemm(p, 1, 8, 64, 64, 512, cv.w.data_ptr(), cv.c_out, 9, 64, sh, 8, None, None, None, 0,
                                    p, None, None, None, 0, _st()), "taps=9")
    refused(lambda: L.fsb_conv_gemm(p, 1, 8, 64, 64, 512, cv.w.data_ptr(), cv.c_out, 1, 64, sh, 8, None, None, None, 0,
                                    None, p, None, None, 0, _st()), "out1 needs snake parameters")
    refused(lambda: L.fsb_final_conv_tanh(p, p, 0.0, 1, 8, 7, 7, p, _st()), "C=7 not supported")
    refused(lambda: L.fsb_final_conv_tanh(p, p, 0.0, 1, 8, 384, 7, p, _st()), "C=384 not supported")
    torch.cuda.synchronize()
