"""Import the UNMODIFIED reference modules from a checkout of the reference (directory in $FISH_SPEECH_REFERENCE).

Test infrastructure only.  The reference needs three third-party packages that are not installed
here and not vendored in its tree:
  * loralib                       (fish_speech/models/text2semantic/lora.py:3)   — unused at inference
  * descript-audio-codec 1.0.0    (uv.lock:864-865;  modded_dac.py:10-11, rvq.py:8)
  * descript-audiotools 0.7.2     (uv.lock:893-894;  modded_dac.py:8-9)
The stubs below restate the handful of classes the hot path touches, following the published
descript-audio-codec 1.0.0 sources (dac/nn/layers.py, dac/nn/quantize.py, dac/model/base.py); they
were cross-checked against the HF port on this box (transformers/models/dac/modeling_dac.py:85-170,
345-369).  Parity for those third-party pieces is therefore anchored on their published algorithm,
not on an installed copy.
"""
from __future__ import annotations

import math
import os
import sys
import types

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.utils.parametrizations import weight_norm

REF_ROOT = os.environ.get("FISH_SPEECH_REFERENCE", "")


def _snake(x, alpha):
    shape = x.shape
    x = x.reshape(shape[0], shape[1], -1)
    x = x + (alpha + 1e-9).reciprocal() * torch.sin(alpha * x).pow(2)
    return x.reshape(shape)


class Snake1d(nn.Module):  # dac/nn/layers.py
    def __init__(self, channels):
        super().__init__()
        self.alpha = nn.Parameter(torch.ones(1, channels, 1))

    def forward(self, x):
        return _snake(x, self.alpha)


def WNConv1d(*args, **kwargs):
    return weight_norm(nn.Conv1d(*args, **kwargs))


def WNConvTranspose1d(*args, **kwargs):
    return weight_norm(nn.ConvTranspose1d(*args, **kwargs))


class VectorQuantize(nn.Module):  # dac/nn/quantize.py
    def __init__(self, input_dim, codebook_size, codebook_dim):
        super().__init__()
        self.codebook_size = codebook_size
        self.codebook_dim = codebook_dim
        self.in_proj = WNConv1d(input_dim, codebook_dim, kernel_size=1)
        self.out_proj = WNConv1d(codebook_dim, input_dim, kernel_size=1)
        self.codebook = nn.Embedding(codebook_size, codebook_dim)

    def forward(self, z):
        z_e = self.in_proj(z)
        z_q, indices = self.decode_latents(z_e)
        commitment_loss = F.mse_loss(z_e, z_q.detach(), reduction="none").mean([1, 2])
        codebook_loss = F.mse_loss(z_q, z_e.detach(), reduction="none").mean([1, 2])
        z_q = z_e + (z_q - z_e).detach()
        z_q = self.out_proj(z_q)
        return z_q, commitment_loss, codebook_loss, indices, z_e

    def embed_code(self, embed_id):
        return F.embedding(embed_id, self.codebook.weight)

    def decode_code(self, embed_id):
        return self.embed_code(embed_id).transpose(1, 2)

    def decode_latents(self, latents):
        B, D, T = latents.shape
        encodings = latents.permute(0, 2, 1).reshape(B * T, D)
        codebook = self.codebook.weight
        encodings = F.normalize(encodings)
        codebook = F.normalize(codebook)
        dist = (encodings.pow(2).sum(1, keepdim=True) - 2 * encodings @ codebook.t()
                + codebook.pow(2).sum(1, keepdim=True).t())
        indices = (-dist).max(1)[1].reshape(B, T)
        z_q = self.decode_code(indices)
        return z_q, indices


class ResidualVectorQuantize(nn.Module):  # dac/nn/quantize.py
    def __init__(self, input_dim=512, n_codebooks=9, codebook_size=1024, codebook_dim=8, quantizer_dropout=0.0):
        super().__init__()
        if isinstance(codebook_dim, int):
            codebook_dim = [codebook_dim for _ in range(n_codebooks)]
        self.n_codebooks = n_codebooks
        self.codebook_dim = codebook_dim
        self.codebook_size = codebook_size
        self.quantizers = nn.ModuleList(
            [VectorQuantize(input_dim, codebook_size, codebook_dim[i]) for i in range(n_codebooks)])
        self.quantizer_dropout = quantizer_dropout

    def forward(self, z, n_quantizers=None):
        z_q = 0
        residual = z
        commitment_loss = 0
        codebook_loss = 0
        codebook_indices, latents = [], []
        if n_quantizers is None:
            n_quantizers = self.n_codebooks
        for i, quantizer in enumerate(self.quantizers):
            if self.training is False and i >= n_quantizers:
                break
            z_q_i, commitment_loss_i, codebook_loss_i, indices_i, z_e_i = quantizer(residual)
            mask = torch.full((z.shape[0],), fill_value=i, device=z.device) < n_quantizers
            z_q = z_q + z_q_i * mask[:, None, None]
            residual = residual - z_q_i
            commitment_loss = commitment_loss + (commitment_loss_i * mask).mean()
            codebook_loss = codebook_loss + (codebook_loss_i * mask).mean()
            codebook_indices.append(indices_i)
            latents.append(z_e_i)
        codes = torch.stack(codebook_indices, dim=1)
        latents = torch.cat(latents, dim=1)
        return z_q, codes, latents, commitment_loss, codebook_loss

    def from_codes(self, codes):
        z_q = 0.0
        z_p = []
        n_codebooks = codes.shape[1]
        for i in range(n_codebooks):
            z_p_i = self.quantizers[i].decode_code(codes[:, i, :])
            z_p.append(z_p_i)
            z_q_i = self.quantizers[i].out_proj(z_p_i)
            z_q = z_q + z_q_i
        return z_q, torch.cat(z_p, dim=1), codes


class CodecMixin:  # dac/model/base.py (only get_delay is reached: modded_dac.py:859)
    def get_delay(self):
        return 0


class BaseModel(nn.Module):  # audiotools/ml/layers/base.py (only .device is used)
    @property
    def device(self):
        return next(self.parameters()).device


def install() -> None:
    """Register the stub modules and put the reference checkout on sys.path."""
    if "loralib" not in sys.modules:
        sys.modules["loralib"] = types.ModuleType("loralib")

    def mod(name, **attrs):
        m = sys.modules.get(name) or types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        sys.modules[name] = m
        return m

    mod("dac")
    mod("dac.nn")
    mod("dac.nn.layers", Snake1d=Snake1d, WNConv1d=WNConv1d, WNConvTranspose1d=WNConvTranspose1d)
    mod("dac.nn.quantize", ResidualVectorQuantize=ResidualVectorQuantize, VectorQuantize=VectorQuantize)
    mod("dac.model")
    mod("dac.model.base", CodecMixin=CodecMixin)
    mod("audiotools", AudioSignal=object)
    mod("audiotools.ml", BaseModel=BaseModel)
    if not REF_ROOT:
        raise RuntimeError("set FISH_SPEECH_REFERENCE to the directory of a fish-speech checkout")
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)


class FakeTokenizer:
    """The two tokenizer members the decode loop touches (inference.py:207, 320)."""

    def __init__(self, im_end_id, semantic_begin_id):
        self._im_end = im_end_id
        self.semantic_begin_id = semantic_begin_id

    def get_token_id(self, token):
        return self._im_end


def reference_lm(cfg, weights, max_batch=1, assign=False):
    """Build the reference DualARTransformer with the oracle's config/weights (bf16, CPU).
    assign=True (full-size models): construct on the meta device and adopt the given tensors as the parameters
    (nn.Module.load_state_dict(assign=True)) instead of allocating + initialising 4.5 G fp32 parameters first;
    the non-persistent buffers are then rebuilt with the reference's own precompute_freqs_cis."""
    install()
    from fish_speech.models.text2semantic import llama as ref_llama

    args = ref_llama.DualARModelArgs(
        model_type="dual_ar", vocab_size=cfg.vocab_size, n_layer=cfg.n_layer, n_head=cfg.n_head, dim=cfg.dim,
        intermediate_size=cfg.intermediate_size, n_local_heads=cfg.n_local_heads, head_dim=cfg.head_dim,
        rope_base=cfg.rope_base, norm_eps=cfg.norm_eps, max_seq_len=cfg.max_seq_len,
        tie_word_embeddings=cfg.tie_word_embeddings, attention_qkv_bias=cfg.attention_qkv_bias,
        attention_o_bias=cfg.attention_o_bias, attention_qk_norm=cfg.attention_qk_norm,
        codebook_size=cfg.codebook_size, num_codebooks=cfg.num_codebooks,
        semantic_begin_id=cfg.semantic_begin_id, semantic_end_id=cfg.semantic_end_id,
        scale_codebook_embeddings=cfg.scale_codebook_embeddings, n_fast_layer=cfg.n_fast_layer,
        fast_dim=cfg.fast_dim, fast_n_head=cfg.fast_n_head, fast_n_local_heads=cfg.fast_n_local_heads,
        fast_head_dim=cfg.fast_head_dim, fast_intermediate_size=cfg.fast_intermediate_size,
        fast_attention_qkv_bias=cfg.fast_attention_qkv_bias, fast_attention_qk_norm=cfg.fast_attention_qk_norm,
        fast_attention_o_bias=cfg.fast_attention_o_bias, norm_fastlayer_input=cfg.norm_fastlayer_input,
    )
    if assign:
        with torch.device("meta"):
            model = ref_llama.DualARTransformer(args)
    else:
        model = ref_llama.DualARTransformer(args)
    sd = {}
    for k, v in weights.items():
        sd[k] = v
    missing, unexpected = model.load_state_dict(sd, strict=False, assign=assign)
    if assign:
        model.freqs_cis = ref_llama.precompute_freqs_cis(args.max_seq_len, args.head_dim, args.rope_base)
        model.causal_mask = torch.tril(torch.ones(args.max_seq_len, args.max_seq_len, dtype=torch.bool))
        model.fast_freqs_cis = ref_llama.precompute_freqs_cis(args.num_codebooks, args.fast_head_dim, args.rope_base)
    missing = [m for m in missing if "freqs" not in m and "causal" not in m]
    assert not missing and not unexpected, (missing, unexpected)
    model = model.to(dtype=torch.bfloat16).eval()
    model.tokenizer = FakeTokenizer(cfg.im_end_id, cfg.semantic_begin_id)
    model._cache_setup_done = False
    return model
