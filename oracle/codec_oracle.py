"""ORACLE — TEST INFRASTRUCTURE ONLY (never imported by the product path).

CPU restatement of the reference codec ("Firefly VQ-GAN" = modified Descript-DAC) inference algorithm:

  fish_speech/models/dac/modded_dac.py   DAC.encode :874-923, from_indices :925-927, Decoder :760-801,
                                         Encoder :670-709, ResidualUnit :599-620, CausalConvNet :521-560,
                                         CausalTransConvNet :563-588, WindowLimitedTransformer :349-439
  fish_speech/models/dac/rvq.py          DownsampleResidualVectorQuantize.forward :293-343, decode :352-366,
                                         ConvNeXtBlock :129-191
  descript-audio-codec 1.0.0 (third party, NOT in the reference checkout; pinned by uv.lock:864-865):
      dac/nn/layers.py  Snake1d  x + 1/(alpha+1e-9) * sin(alpha x)^2 ; WNConv1d = weight_norm(Conv1d)
      dac/nn/quantize.py VectorQuantize.decode_latents (L2-normalised nearest neighbour),
                         ResidualVectorQuantize.forward / from_codes
    restated from the published algorithm (see oracle/ref_stubs.py for the cross-check source).

Weights are a flat dict in the reference's state_dict naming (weight-norm stored as
parametrizations.weight.original0/1), so the same dict loads into the real reference modules
(oracle/make_golden_codec.py pins this file against them bit for bit).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional

import torch
import torch.nn.functional as F


@dataclass
class TfmConfig:  # modded_dac.ModelArgs as instantiated by configs/modded_dac_vq.yaml
    n_layer: int = 8
    n_head: int = 16
    dim: int = 1024
    intermediate_size: int = 3072
    head_dim: int = 64
    rope_base: float = 10000
    norm_eps: float = 1e-5
    window_size: Optional[int] = 128


@dataclass
class CodecConfig:
    """fish_speech/configs/modded_dac_vq.yaml."""

    sample_rate: int = 44100
    encoder_dim: int = 64
    encoder_rates: tuple = (2, 4, 8, 8)
    decoder_dim: int = 1536
    decoder_rates: tuple = (8, 8, 4, 2)
    encoder_transformer_layers: tuple = (0, 0, 0, 4)
    n_codebooks: int = 9
    codebook_size: int = 1024
    semantic_codebook_size: int = 4096
    codebook_dim: int = 8
    downsample_factor: tuple = (2, 2)
    quant_tfm: TfmConfig = field(default_factory=TfmConfig)  # pre_module / post_module (window 128)
    enc_tfm_window: int = 512  # modded_dac.py:641 getattr(partial, "window_size", 512)

    @property
    def latent_dim(self) -> int:
        return self.encoder_dim * (2 ** len(self.encoder_rates))

    @property
    def hop_length(self) -> int:
        return int(math.prod(self.encoder_rates))

    @property
    def frame_length(self) -> int:  # modded_dac.py:861
        return self.hop_length * 4

    def enc_tfm(self, dim: int, n_layer: int) -> TfmConfig:  # modded_dac.py:642-647
        return TfmConfig(n_layer=n_layer, n_head=dim // 64, dim=dim, intermediate_size=dim * 3, head_dim=64,
                         rope_base=10000, norm_eps=1e-5, window_size=self.enc_tfm_window)


def full_config() -> CodecConfig:
    return CodecConfig()


def tiny_config() -> CodecConfig:
    """Same structure, small channels: latent 256, decoder 256->16, codebooks 3x(64|256) entries."""
    return CodecConfig(encoder_dim=16, decoder_dim=256, n_codebooks=3, codebook_size=64, semantic_codebook_size=256,
                       quant_tfm=TfmConfig(n_layer=2, n_head=4, dim=256, intermediate_size=768, window_size=16),
                       encoder_transformer_layers=(0, 0, 0, 2), enc_tfm_window=32)


# ------------------------------------------------------------------------------------------------
# synthetic weights in the reference's state_dict naming
# ------------------------------------------------------------------------------------------------
def make_weights(cfg: CodecConfig, seed: int = 1234, dtype=torch.float32) -> dict[str, torch.Tensor]:
    """Seeded weights with fan-in scaling so activations stay O(1) through the ~60 layers (the
    reference's trunc_normal(0.02) init is for training, random outputs would saturate/vanish)."""
    g = torch.Generator().manual_seed(seed)
    w: dict[str, torch.Tensor] = {}

    def rn(*shape, std=1.0):
        return (torch.randn(*shape, generator=g) * std).to(dtype)

    def conv(prefix, cout, cin_g, k, wn=True, gain=1.0):
        v = rn(cout, cin_g, k, std=gain / math.sqrt(cin_g * k))
        if wn:
            w[f"{prefix}.parametrizations.weight.original1"] = v
            norm = v.float().flatten(1).norm(dim=1).view(cout, 1, 1)
            w[f"{prefix}.parametrizations.weight.original0"] = (norm * (1 + 0.1 * torch.randn(cout, 1, 1, generator=g))).to(dtype)
        else:
            w[f"{prefix}.weight"] = v
        w[f"{prefix}.bias"] = rn(cout, std=0.02)

    def convT(prefix, cin, cout, k, stride, wn=True):
        # ConvTranspose1d weight [C_in, C_out, k]; every output sample sums k/stride taps of C_in channels
        v = rn(cin, cout, k, std=1.0 / math.sqrt(cin * k / stride))
        if wn:
            w[f"{prefix}.parametrizations.weight.original1"] = v
            norm = v.float().flatten(1).norm(dim=1).view(cin, 1, 1)
            w[f"{prefix}.parametrizations.weight.original0"] = (norm * (1 + 0.1 * torch.randn(cin, 1, 1, generator=g))).to(dtype)
        else:
            w[f"{prefix}.weight"] = v
        w[f"{prefix}.bias"] = rn(cout, std=0.02)

    def snake(prefix, c):
        w[f"{prefix}.alpha"] = (1.0 + 0.3 * torch.randn(1, c, 1, generator=g)).abs().clamp_min(0.2).to(dtype)

    def res_unit(prefix, c):
        snake(f"{prefix}.block.0", c)
        conv(f"{prefix}.block.1.conv", c, c, 7, gain=0.5)
        snake(f"{prefix}.block.2", c)
        conv(f"{prefix}.block.3.conv", c, c, 1, gain=0.5)

    def tfm(prefix, t: TfmConfig):
        for l in range(t.n_layer):
            p = f"{prefix}.layers.{l}"
            w[f"{p}.attention.wqkv.weight"] = rn(3 * t.n_head * t.head_dim, t.dim, std=1 / math.sqrt(t.dim))
            w[f"{p}.attention.wo.weight"] = rn(t.dim, t.n_head * t.head_dim, std=1 / math.sqrt(t.dim))
            w[f"{p}.feed_forward.w1.weight"] = rn(t.intermediate_size, t.dim, std=1 / math.sqrt(t.dim))
            w[f"{p}.feed_forward.w3.weight"] = rn(t.intermediate_size, t.dim, std=1 / math.sqrt(t.dim))
            w[f"{p}.feed_forward.w2.weight"] = rn(t.dim, t.intermediate_size, std=1 / math.sqrt(t.intermediate_size))
            w[f"{p}.ffn_norm.weight"] = (1 + 0.1 * torch.randn(t.dim, generator=g)).to(dtype)
            w[f"{p}.attention_norm.weight"] = (1 + 0.1 * torch.randn(t.dim, generator=g)).to(dtype)
            w[f"{p}.attention_layer_scale.gamma"] = (0.3 + 0.1 * torch.randn(t.dim, generator=g)).to(dtype)
            w[f"{p}.ffn_layer_scale.gamma"] = (0.3 + 0.1 * torch.randn(t.dim, generator=g)).to(dtype)
        w[f"{prefix}.norm.weight"] = (1 + 0.1 * torch.randn(t.dim, generator=g)).to(dtype)

    def convnext(prefix, c):
        w[f"{prefix}.dwconv.conv.weight"] = rn(c, 1, 7, std=1 / math.sqrt(7))
        w[f"{prefix}.dwconv.conv.bias"] = rn(c, std=0.02)
        w[f"{prefix}.norm.weight"] = (1 + 0.1 * torch.randn(c, generator=g)).to(dtype)
        w[f"{prefix}.norm.bias"] = rn(c, std=0.02)
        w[f"{prefix}.pwconv1.weight"] = rn(4 * c, c, std=1 / math.sqrt(c))
        w[f"{prefix}.pwconv1.bias"] = rn(4 * c, std=0.02)
        w[f"{prefix}.pwconv2.weight"] = rn(c, 4 * c, std=1 / math.sqrt(4 * c))
        w[f"{prefix}.pwconv2.bias"] = rn(c, std=0.02)
        w[f"{prefix}.gamma"] = (0.3 + 0.1 * torch.randn(c, generator=g)).to(dtype)

    # ---- encoder (modded_dac.py:670-709) ----
    d = cfg.encoder_dim
    conv("encoder.block.0.conv", d, 1, 7)
    for i, (stride, ntl) in enumerate(zip(cfg.encoder_rates, cfg.encoder_transformer_layers)):
        d *= 2
        p = f"encoder.block.{i + 1}.block"
        for j in range(3):
            res_unit(f"{p}.{j}", d // 2)
        snake(f"{p}.3", d // 2)
        conv(f"{p}.4.conv", d, d // 2, 2 * stride)
        if ntl > 0:
            tfm(f"{p}.5", cfg.enc_tfm(d, ntl))
    nb = len(cfg.encoder_rates) + 1
    snake(f"encoder.block.{nb}", d)
    conv(f"encoder.block.{nb + 1}.conv", cfg.latent_dim, d, 3)

    # ---- quantizer (rvq.py:204-291) ----
    D = cfg.latent_dim

    def vq(prefix, size):
        conv(f"{prefix}.in_proj", cfg.codebook_dim, D, 1)
        conv(f"{prefix}.out_proj", D, cfg.codebook_dim, 1, gain=1.0)
        w[f"{prefix}.codebook.weight"] = rn(size, cfg.codebook_dim)

    vq("quantizer.semantic_quantizer.quantizers.0", cfg.semantic_codebook_size)
    for i in range(cfg.n_codebooks):
        vq(f"quantizer.quantizer.quantizers.{i}", cfg.codebook_size)
    nds = len(cfg.downsample_factor)
    for i, f_ in enumerate(cfg.downsample_factor):
        conv(f"quantizer.downsample.{i}.0.conv", D, D, f_, wn=False)
        convnext(f"quantizer.downsample.{i}.1", D)
    for i, f_ in enumerate(reversed(cfg.downsample_factor)):
        convT(f"quantizer.upsample.{i}.0.conv", D, D, f_, f_, wn=False)
        convnext(f"quantizer.upsample.{i}.1", D)
    tfm("quantizer.pre_module", cfg.quant_tfm)
    tfm("quantizer.post_module", cfg.quant_tfm)

    # ---- decoder (modded_dac.py:760-801) ----
    c = cfg.decoder_dim
    conv("decoder.model.0.conv", c, D, 7)
    for i, stride in enumerate(cfg.decoder_rates):
        cin, cout = cfg.decoder_dim // 2 ** i, cfg.decoder_dim // 2 ** (i + 1)
        p = f"decoder.model.{i + 1}.block"
        snake(f"{p}.0", cin)
        convT(f"{p}.1.conv", cin, cout, 2 * stride, stride)
        for j in range(3):
            res_unit(f"{p}.{2 + j}", cout)
    n = len(cfg.decoder_rates) + 1
    snake(f"decoder.model.{n}", cout)
    conv(f"decoder.model.{n + 1}.conv", 1, cout, 7, gain=0.12)
    return w


# ------------------------------------------------------------------------------------------------
# layers
# ------------------------------------------------------------------------------------------------
def _wn_weight(w: dict, prefix: str) -> torch.Tensor:
    g = w.get(f"{prefix}.parametrizations.weight.original0")
    if g is None:
        return w[f"{prefix}.weight"]
    return torch._weight_norm(w[f"{prefix}.parametrizations.weight.original1"], g, 0)


def snake(x, alpha):
    return x + (alpha + 1e-9).reciprocal() * torch.sin(alpha * x).pow(2)


def causal_conv(w: dict, prefix: str, x, stride=1, dilation=1, groups=1):
    """CausalConvNet.forward (modded_dac.py:546-552): left pad (k_eff - stride), right pad to a whole frame."""
    weight = _wn_weight(w, prefix)
    k_eff = (weight.shape[-1] - 1) * dilation + 1
    pad = k_eff - stride
    length = x.shape[-1]
    n_frames = (length - k_eff + pad) / stride + 1
    extra = (math.ceil(n_frames) - 1) * stride + (k_eff - pad) - length
    x = F.pad(x, (pad, extra))
    return F.conv1d(x, weight, w[f"{prefix}.bias"], stride=stride, dilation=dilation, groups=groups)


def causal_conv_transpose(w: dict, prefix: str, x, stride):
    """CausalTransConvNet.forward (modded_dac.py:574-580): trim k - stride samples on the right."""
    weight = _wn_weight(w, prefix)
    y = F.conv_transpose1d(x, weight, w[f"{prefix}.bias"], stride=stride)
    pad = weight.shape[-1] - stride
    return y[..., : y.shape[-1] - pad] if pad > 0 else y


def residual_unit(w: dict, prefix: str, x, dilation: int):
    y = snake(x, w[f"{prefix}.block.0.alpha"])
    y = causal_conv(w, f"{prefix}.block.1.conv", y, dilation=dilation)
    y = snake(y, w[f"{prefix}.block.2.alpha"])
    y = causal_conv(w, f"{prefix}.block.3.conv", y)
    pad = x.shape[-1] - y.shape[-1]
    if pad > 0:
        x = x[..., :-pad]
    return x + y


_ROPE_CACHE: dict = {}


def _rope_table(n: int, head_dim: int, base: float) -> torch.Tensor:
    key = (n, head_dim, base)
    if key not in _ROPE_CACHE:
        inv = 1.0 / (base ** (torch.arange(0, head_dim, 2)[: head_dim // 2].float() / head_dim))
        ang = torch.outer(torch.arange(n), inv)
        cis = torch.polar(torch.ones_like(ang), ang)
        _ROPE_CACHE[key] = torch.stack([cis.real, cis.imag], dim=-1).to(torch.bfloat16)  # modded_dac.py:442-452
    return _ROPE_CACHE[key]


def _rotary(x, freqs):
    xs = x.float().reshape(*x.shape[:-1], -1, 2)
    fr = freqs.view(1, xs.size(1), 1, xs.size(3), 2)
    out = torch.stack([xs[..., 0] * fr[..., 0] - xs[..., 1] * fr[..., 1],
                       xs[..., 1] * fr[..., 0] + xs[..., 0] * fr[..., 1]], -1)
    return out.flatten(3).type_as(x)


def _rms(x, weight, eps):
    xf = x.float()
    return (xf * torch.rsqrt(torch.mean(xf * xf, dim=-1, keepdim=True) + eps)).type_as(x) * weight


def window_transformer(w: dict, prefix: str, t: TfmConfig, x):
    """WindowLimitedTransformer.forward (modded_dac.py:413-439) for channels_first input [B, C, T]."""
    x = x.transpose(1, 2)
    B, T, _ = x.shape
    idx = torch.arange(T)
    mask = torch.tril(torch.ones(T, T)).bool()
    if t.window_size is not None:
        lo = (idx.view(-1, 1) - t.window_size + 1).clamp(min=0)
        mask = (idx >= lo) & mask
    mask = mask[None, None]
    freqs = _rope_table(T, t.head_dim, t.rope_base)
    H, Dh = t.n_head, t.head_dim
    for l in range(t.n_layer):
        p = f"{prefix}.layers.{l}"
        h_in = _rms(x, w[f"{p}.attention_norm.weight"], t.norm_eps)
        q, k, v = F.linear(h_in, w[f"{p}.attention.wqkv.weight"]).split([H * Dh] * 3, dim=-1)
        q, k, v = (a.view(B, T, H, Dh) for a in (q, k, v))
        q, k = _rotary(q, freqs), _rotary(k, freqs)
        q, k, v = (a.transpose(1, 2) for a in (q, k, v))
        y = F.scaled_dot_product_attention(q, k, v, attn_mask=mask)
        y = y.transpose(1, 2).contiguous().view(B, T, H * Dh)
        h = x + F.linear(y, w[f"{p}.attention.wo.weight"]) * w[f"{p}.attention_layer_scale.gamma"]
        n2 = _rms(h, w[f"{p}.ffn_norm.weight"], t.norm_eps)
        ff = F.linear(F.silu(F.linear(n2, w[f"{p}.feed_forward.w1.weight"])) * F.linear(n2, w[f"{p}.feed_forward.w3.weight"]),
                      w[f"{p}.feed_forward.w2.weight"])
        x = h + ff * w[f"{p}.ffn_layer_scale.gamma"]
    x = _rms(x, w[f"{prefix}.norm.weight"], t.norm_eps)
    return x.transpose(1, 2)


def convnext(w: dict, prefix: str, x):
    """ConvNeXtBlock.forward (rvq.py:173-191)."""
    C = x.shape[1]
    y = causal_conv(w, f"{prefix}.dwconv.conv", x, groups=C)
    y = y.permute(0, 2, 1)
    y = F.layer_norm(y, (C,), w[f"{prefix}.norm.weight"], w[f"{prefix}.norm.bias"], 1e-6)
    y = F.linear(y, w[f"{prefix}.pwconv1.weight"], w[f"{prefix}.pwconv1.bias"])
    y = F.gelu(y)
    y = F.linear(y, w[f"{prefix}.pwconv2.weight"], w[f"{prefix}.pwconv2.bias"])
    y = w[f"{prefix}.gamma"] * y
    return x + y.permute(0, 2, 1)


# ------------------------------------------------------------------------------------------------
# decode path
# ------------------------------------------------------------------------------------------------
def _vq_from_codes(w: dict, prefix: str, codes):
    """ResidualVectorQuantize.from_codes: sum_i out_proj_i(codebook_i[codes_i]) (dac/nn/quantize.py)."""
    z = 0.0
    for i in range(codes.shape[1]):
        p = f"{prefix}.quantizers.{i}"
        e = F.embedding(codes[:, i], w[f"{p}.codebook.weight"]).transpose(1, 2)
        z = z + F.conv1d(e, _wn_weight(w, f"{p}.out_proj"), w[f"{p}.out_proj.bias"])
    return z


def quantizer_decode(w: dict, cfg: CodecConfig, indices, trace: Optional[dict] = None):
    """DownsampleResidualVectorQuantize.decode (rvq.py:352-366). indices [B, 1+n_codebooks, T]."""
    indices = indices.clone()
    indices[:, 0] = torch.clamp(indices[:, 0], max=cfg.semantic_codebook_size - 1)
    indices[:, 1:] = torch.clamp(indices[:, 1:], max=cfg.codebook_size - 1)
    z = _vq_from_codes(w, "quantizer.semantic_quantizer", indices[:, :1]) + \
        _vq_from_codes(w, "quantizer.quantizer", indices[:, 1:])
    if trace is not None:
        trace["z_q"] = z.clone()
    z = window_transformer(w, "quantizer.post_module", cfg.quant_tfm, z)
    if trace is not None:
        trace["post"] = z.clone()
    for i, f_ in enumerate(reversed(cfg.downsample_factor)):
        z = causal_conv_transpose(w, f"quantizer.upsample.{i}.0.conv", z, f_)
        z = convnext(w, f"quantizer.upsample.{i}.1", z)
    if trace is not None:
        trace["z_up"] = z.clone()
    return z


def decoder(w: dict, cfg: CodecConfig, z, trace: Optional[dict] = None):
    """Decoder.forward (modded_dac.py:760-801)."""
    x = causal_conv(w, "decoder.model.0.conv", z)
    for i, stride in enumerate(cfg.decoder_rates):
        p = f"decoder.model.{i + 1}.block"
        x = snake(x, w[f"{p}.0.alpha"])
        x = causal_conv_transpose(w, f"{p}.1.conv", x, stride)
        for j, d in enumerate((1, 3, 9)):
            x = residual_unit(w, f"{p}.{2 + j}", x, d)
        if trace is not None:
            trace[f"dec{i}"] = x.clone()
    n = len(cfg.decoder_rates) + 1
    x = snake(x, w[f"decoder.model.{n}.alpha"])
    x = causal_conv(w, f"decoder.model.{n + 1}.conv", x)
    return torch.tanh(x)


def from_indices(w: dict, cfg: CodecConfig, indices, trace: Optional[dict] = None):
    """DAC.from_indices (modded_dac.py:925-927): [B, 10, T] -> [B, 1, T * frame_length]."""
    return decoder(w, cfg, quantizer_decode(w, cfg, indices, trace), trace)


# ------------------------------------------------------------------------------------------------
# encode path
# ------------------------------------------------------------------------------------------------
def encoder(w: dict, cfg: CodecConfig, x):
    """Encoder.forward (modded_dac.py:670-709)."""
    x = causal_conv(w, "encoder.block.0.conv", x)
    d = cfg.encoder_dim
    for i, (stride, ntl) in enumerate(zip(cfg.encoder_rates, cfg.encoder_transformer_layers)):
        d *= 2
        p = f"encoder.block.{i + 1}.block"
        for j, dil in enumerate((1, 3, 9)):
            x = residual_unit(w, f"{p}.{j}", x, dil)
        x = snake(x, w[f"{p}.3.alpha"])
        x = causal_conv(w, f"{p}.4.conv", x, stride=stride)
        if ntl > 0:
            x = window_transformer(w, f"{p}.5", cfg.enc_tfm(d, ntl), x)
    nb = len(cfg.encoder_rates) + 1
    x = snake(x, w[f"encoder.block.{nb}.alpha"])
    return causal_conv(w, f"encoder.block.{nb + 1}.conv", x)


def _vq_encode(w: dict, prefix: str, z, scores: Optional[list] = None):
    """VectorQuantize.forward (dac/nn/quantize.py): in_proj -> cosine nearest neighbour -> out_proj.
    `scores` (tests): receives -dist [B, T, K], the quantity the reference maximises."""
    z_e = F.conv1d(z, _wn_weight(w, f"{prefix}.in_proj"), w[f"{prefix}.in_proj.bias"])
    B, D, T = z_e.shape
    enc = F.normalize(z_e.permute(0, 2, 1).reshape(B * T, D))
    cb = F.normalize(w[f"{prefix}.codebook.weight"])
    dist = enc.pow(2).sum(1, keepdim=True) - 2 * enc @ cb.t() + cb.pow(2).sum(1, keepdim=True).t()
    idx = (-dist).max(1)[1].reshape(B, T)
    if scores is not None:
        scores.append((-dist).reshape(B, T, -1).clone())
    z_q = F.embedding(idx, w[f"{prefix}.codebook.weight"]).transpose(1, 2)
    z_q = F.conv1d(z_q, _wn_weight(w, f"{prefix}.out_proj"), w[f"{prefix}.out_proj.bias"])
    return z_q, idx


def quantizer_encode(w: dict, cfg: CodecConfig, z, trace: Optional[dict] = None):
    """DownsampleResidualVectorQuantize.forward up to the codes (rvq.py:293-317). The reference goes on
    to run post_module + upsample (rvq.py:318-319), whose result DAC.encode discards."""
    for i, f_ in enumerate(cfg.downsample_factor):
        z = causal_conv(w, f"quantizer.downsample.{i}.0.conv", z, stride=f_)
        z = convnext(w, f"quantizer.downsample.{i}.1", z)
    z = window_transformer(w, "quantizer.pre_module", cfg.quant_tfm, z)
    if trace is not None:
        trace["pre"] = z.clone()
    scores = trace.setdefault("vq_scores", []) if trace is not None else None
    zq, sem = _vq_encode(w, "quantizer.semantic_quantizer.quantizers.0", z, scores)
    residual = z - zq
    codes = [sem]
    for i in range(cfg.n_codebooks):
        zq_i, idx = _vq_encode(w, f"quantizer.quantizer.quantizers.{i}", residual, scores)
        residual = residual - zq_i
        codes.append(idx)
    return torch.stack(codes, dim=1)


def encode(w: dict, cfg: CodecConfig, audio, audio_lengths=None, trace: Optional[dict] = None):
    """DAC.encode (modded_dac.py:874-923): audio [B,1,N] or [B,N] -> (codes [B,10,T], lens [B])."""
    if audio.ndim == 2:
        audio = audio.unsqueeze(1)
    length = audio.shape[-1]
    right_pad = math.ceil(length / cfg.frame_length) * cfg.frame_length - length
    audio = F.pad(audio, (0, right_pad))
    if audio_lengths is None:
        audio_lengths = torch.LongTensor([length + right_pad])
    z = encoder(w, cfg, audio)
    if trace is not None:
        trace["enc"] = z.clone()
    codes = quantizer_encode(w, cfg, z, trace)
    return codes, torch.ceil(audio_lengths / cfg.frame_length).long()
