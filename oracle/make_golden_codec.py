"""Pin oracle/codec_oracle.py against the REAL reference codec classes and write codec fixtures.

Run where a checkout of the reference exists ($FISH_SPEECH_REFERENCE): python -m oracle.make_golden_codec
The reference DAC is instantiated by hand with the values of fish_speech/configs/modded_dac_vq.yaml
(hydra / omegaconf are not installed here); its third-party bases come from oracle/ref_stubs.py.
"""
from __future__ import annotations

import functools
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import codec_oracle as CO  # noqa: E402
from oracle import ref_stubs as R  # noqa: E402

GOLD = ROOT / "tests" / "golden"


def reference_dac(cfg: CO.CodecConfig, weights: dict):
    R.install()
    from fish_speech.models.dac.modded_dac import DAC, ModelArgs, WindowLimitedTransformer
    from fish_speech.models.dac.rvq import DownsampleResidualVectorQuantize

    tgc = functools.partial(ModelArgs, block_size=8192, n_local_heads=-1, head_dim=64, rope_base=10000,
                            norm_eps=1e-5, dropout_rate=0.1, attn_dropout_rate=0.1, channels_first=True)
    if cfg.enc_tfm_window != 512:
        tgc.window_size = cfg.enc_tfm_window  # modded_dac.py:641 reads getattr(partial, "window_size", 512)
    t = cfg.quant_tfm

    def mk():
        return WindowLimitedTransformer(
            causal=True, window_size=t.window_size, input_dim=cfg.latent_dim,
            config=ModelArgs(block_size=2048, n_layer=t.n_layer, n_head=t.n_head, dim=t.dim,
                             intermediate_size=t.intermediate_size, n_local_heads=-1, head_dim=t.head_dim,
                             rope_base=t.rope_base, norm_eps=t.norm_eps, dropout_rate=0.1, attn_dropout_rate=0.1,
                             channels_first=True))

    q = DownsampleResidualVectorQuantize(
        input_dim=cfg.latent_dim, n_codebooks=cfg.n_codebooks, codebook_size=cfg.codebook_size,
        codebook_dim=cfg.codebook_dim, quantizer_dropout=0.5, downsample_factor=tuple(cfg.downsample_factor),
        post_module=mk(), pre_module=mk(), semantic_codebook_size=cfg.semantic_codebook_size)
    dac = DAC(sample_rate=cfg.sample_rate, encoder_dim=cfg.encoder_dim, encoder_rates=list(cfg.encoder_rates),
              decoder_dim=cfg.decoder_dim, decoder_rates=list(cfg.decoder_rates),
              encoder_transformer_layers=list(cfg.encoder_transformer_layers),
              decoder_transformer_layers=[0, 0, 0, 0],  # built but never called by the reference (modded_dac.py:742)
              quantizer=q, transformer_general_config=tgc)
    missing, unexpected = dac.load_state_dict(weights, strict=False)
    assert not missing and not unexpected, (missing[:5], unexpected[:5])
    return dac.eval()


def case(name: str, cfg: CO.CodecConfig, seed: int, B: int, T: int, n_samples: int, store_wave: bool):
    w = CO.make_weights(cfg, seed=seed)
    dac = reference_dac(cfg, w)
    g = torch.Generator().manual_seed(seed)
    codes = torch.stack([torch.randint(0, cfg.semantic_codebook_size, (B, T), generator=g)] +
                        [torch.randint(0, cfg.codebook_size, (B, T), generator=g) for _ in range(cfg.n_codebooks)], dim=1)
    with torch.inference_mode():
        ref_wav = dac.from_indices(codes.clone())
        got_wav = CO.from_indices(w, cfg, codes)
    assert torch.equal(ref_wav, got_wav), f"{name}: decode differs (max {float((ref_wav - got_wav).abs().max())})"
    audio = 0.1 * torch.randn(B, 1, n_samples, generator=g)
    lens = torch.tensor([n_samples] * B)
    with torch.inference_mode():
        ref_codes, ref_lens = dac.encode(audio, lens)
        got_codes, got_lens = CO.encode(w, cfg, audio, lens)
    assert torch.equal(ref_codes, got_codes) and torch.equal(ref_lens, got_lens), f"{name}: encode differs"
    # causality property the reference asserts itself (rvq.py:395-398): a prefix decodes to a prefix
    with torch.inference_mode():
        pre = CO.from_indices(w, cfg, codes[:, :, : T // 2])
    assert torch.allclose(pre, got_wav[..., : pre.shape[-1]], atol=2e-4), f"{name}: decode is not causal"
    out = dict(weight_seed=seed, codes=codes.numpy().astype(np.int32), audio=audio.numpy(), lens=lens.numpy(),
               ref_codes=ref_codes.numpy().astype(np.int32), ref_lens=ref_lens.numpy(),
               wav_rms=float(ref_wav.pow(2).mean().sqrt()))
    if store_wave:
        out["ref_wav"] = ref_wav.numpy().astype(np.float32)
    np.savez_compressed(GOLD / f"{name}.npz", **out)
    print(f"{name}: reference == oracle (decode {tuple(ref_wav.shape)}, rms {out['wav_rms']:.3f}; encode {tuple(ref_codes.shape)})")


def main():
    GOLD.mkdir(parents=True, exist_ok=True)
    case("codec_tiny", CO.tiny_config(), 5, 2, 12, 8192 + 300, True)
    if "--full" in sys.argv:
        # BASELINE config #1: 1 s of 44.1 kHz audio through the real geometry (391 M parameters)
        case("codec_full_1s", CO.full_config(), 6, 1, 22, 44100, True)


if __name__ == "__main__":
    main()
