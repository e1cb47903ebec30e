"""Drop-in surface of fish_speech/models/dac/inference.py: `load_model(config_name, checkpoint_path,
device)` and the wav<->npy CLI (dac/inference.py:23-126).  The codec hyper-parameters come from
`configs/modded_dac_vq.yaml` (same file layout as the reference's; hydra is not needed: the `_target_`
keys are ignored and the YAML anchors resolve natively)."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

from .modded_dac import DAC, CodecConfig, TfmConfig

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("fish_speech_b200")

CONFIG_DIR = Path(__file__).resolve().parent.parent.parent / "configs"
AUDIO_EXTENSIONS = {".mp3", ".wav", ".flac", ".ogg", ".m4a", ".wma", ".aac", ".aiff", ".aif", ".aifc"}


def load_codec_config(config_name: str = "modded_dac_vq") -> CodecConfig:
    import yaml

    path = Path(config_name)
    if not path.exists():
        path = CONFIG_DIR / f"{config_name}.yaml"
    y = yaml.safe_load(path.read_text())
    q = y["quantizer"]
    t = q["post_module"]["config"]
    tfm = TfmConfig(n_layer=t["n_layer"], n_head=t["n_head"], dim=t["dim"], intermediate_size=t["intermediate_size"],
                    head_dim=t["head_dim"], rope_base=t["rope_base"], norm_eps=float(t["norm_eps"]),
                    window_size=q["post_module"].get("window_size"))
    return CodecConfig(
        sample_rate=y["sample_rate"], encoder_dim=y["encoder_dim"], encoder_rates=tuple(y["encoder_rates"]),
        decoder_dim=y["decoder_dim"], decoder_rates=tuple(y["decoder_rates"]),
        encoder_transformer_layers=tuple(y["encoder_transformer_layers"]), n_codebooks=q["n_codebooks"],
        codebook_size=q["codebook_size"], semantic_codebook_size=q["semantic_codebook_size"],
        codebook_dim=q["codebook_dim"], downsample_factor=tuple(q["downsample_factor"]), quant_tfm=tfm,
        enc_tfm_window=y.get("transformer_general_config", {}).get("window_size", 512))


def load_model(config_name, checkpoint_path, device="cuda") -> DAC:
    cfg = load_codec_config(config_name)
    state_dict = torch.load(checkpoint_path, map_location="cpu", mmap=True, weights_only=True)
    if "state_dict" in state_dict:
        state_dict = state_dict["state_dict"]
    if any("generator" in k for k in state_dict):
        state_dict = {k.replace("generator.", ""): v for k, v in state_dict.items() if "generator." in k}
    model = DAC(cfg, state_dict, device=device)
    logger.info("Loaded model (fish_speech_b200 CUDA codec)")
    return model


def write_wav(path: Path, samples: np.ndarray, sample_rate: int, sample_format: str) -> None:
    """A mono WAV file of samples already in `sample_format` (audio.OUTPUT_FORMATS), written as they are."""
    from ...inference_engine.utils import WAVE_OF_FORMAT, wav_chunk_header

    bits, tag = WAVE_OF_FORMAT[sample_format]
    data = np.ascontiguousarray(samples).astype(samples.dtype.newbyteorder("<")).tobytes()
    head = bytearray(wav_chunk_header(sample_rate=sample_rate, bit_depth=bits, format_tag=tag))
    head[4:8] = (len(head) - 8 + len(data)).to_bytes(4, "little")  # RIFF size
    head[40:44] = len(data).to_bytes(4, "little")  # data size
    Path(path).write_bytes(bytes(head) + data)


def main(argv=None):
    import click

    @click.command()
    @click.option("--input-path", "-i", default="test.wav", type=click.Path(exists=True, path_type=Path))
    @click.option("--output-path", "-o", default="fake.wav", type=click.Path(path_type=Path))
    @click.option("--config-name", default="modded_dac_vq")
    @click.option("--checkpoint-path", default="checkpoints/openaudio-s1-mini/codec.pth")
    @click.option("--device", "-d", default="cuda")
    @click.option("--output-sample-rate", type=int, default=None,
                  help="Sample rate of the written audio (default: the codec's), resampled on the device.")
    @click.option("--output-format", type=click.Choice(["float", "pcm16", "mulaw"]), default=None,
                  help="Samples of the written WAV, converted on the device: float (32-bit IEEE), pcm16 (16-bit PCM, "
                       "clipped to [-1, 1] and scaled by 32767) or mulaw (8-bit G.711). Default: the codec's float "
                       "waveform, written by soundfile as before.")
    def _main(input_path, output_path, config_name, checkpoint_path, device, output_sample_rate, output_format):
        import soundfile as sf
        import torchaudio

        from ...audio import convert_out, resample

        model = load_model(config_name, checkpoint_path, device=device)
        if input_path.suffix in AUDIO_EXTENSIONS:
            audio, sr = torchaudio.load(str(input_path))
            if audio.shape[0] > 1:
                audio = audio.mean(0, keepdim=True)
            audios = resample(audio.to(device), sr, model.sample_rate)[None]
            lengths = torch.tensor([audios.shape[2]], device=device, dtype=torch.long)
            indices, _ = model.encode(audios, lengths)
            if indices.ndim == 3:
                indices = indices[0]
            np.save(output_path.with_suffix(".npy"), indices.cpu().numpy())
        elif input_path.suffix == ".npy":
            indices = torch.from_numpy(np.load(input_path)).to(device).long()
            assert indices.ndim == 2, f"Expected 2D indices, got {indices.ndim}"
        else:
            raise ValueError(f"Unknown input type: {input_path}")
        if indices.ndim == 2:
            indices = indices.unsqueeze(0)
        fake = model.from_indices(indices)
        rate = model.sample_rate if output_sample_rate is None else int(output_sample_rate)
        if output_sample_rate is None and output_format is None:
            sf.write(output_path, fake[0, 0].float().cpu().numpy(), model.sample_rate)
        else:
            fmt = {None: "float32", "float": "float32"}.get(output_format, output_format)
            out = convert_out(fake[0, 0].float(), rate, fmt, orig_freq=model.sample_rate).cpu().numpy()
            if output_format is None:  # a rate alone: the float waveform, written by soundfile as before
                sf.write(output_path, out, rate)
            else:
                write_wav(output_path, out, rate, fmt)
        logger.info(f"Saved audio to {output_path}")

    return _main(argv, standalone_mode=False) if argv is not None else _main()


if __name__ == "__main__":
    main()
