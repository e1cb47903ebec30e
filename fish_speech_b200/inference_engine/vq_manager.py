"""Codec side of the TTS engine: the surface of fish_speech/inference_engine/vq_manager.py (`decode_vq_tokens` :16,
`encode_reference` :24) on the CUDA codec, plus the incremental decoder the streaming path uses."""
from typing import Callable, Optional

import torch

from ..models.dac.modded_dac import DAC, DecodeStream

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("fish_speech_b200")


class VQManager:
    decoder_model: DAC
    load_audio: Callable

    def _codec(self) -> DAC:
        if not isinstance(self.decoder_model, DAC):
            raise ValueError(f"Unknown model type: {type(self.decoder_model)}")
        return self.decoder_model

    def decode_vq_tokens(self, codes: torch.Tensor) -> torch.Tensor:
        """codes [C, T] of one utterance -> waveform [T * frame_length]."""
        logger.info(f"VQ features: {codes.shape}")
        return self._codec().from_indices(codes[None])[0].squeeze()

    def open_decode_stream(self, max_frames: int = 4096, **conversion) -> DecodeStream:
        """Incremental decoder for one utterance: `.push(codes[None])` as frames arrive (models/dac/modded_dac.py);
        `sample_rate=` / `sample_format=` convert what it returns (and then `.flush()` ends it)."""
        return self._codec().open_decode_stream(batch=1, max_frames=max_frames, **conversion)

    def encode_reference(self, reference_audio, enable_reference_audio) -> Optional[torch.Tensor]:
        """Reference clip (bytes or path) -> prompt codes [C, T], or None when reference audio is off."""
        if not enable_reference_audio or reference_audio is None:
            logger.info("No reference audio provided")
            return None
        codec = self._codec()
        wav = torch.from_numpy(self.load_audio(reference_audio, codec.sample_rate)).to(codec.device)
        logger.info(f"Loaded audio with {wav.shape[-1] / codec.sample_rate:.2f} seconds")
        lengths = torch.tensor([wav.shape[-1]], device=codec.device, dtype=torch.long)
        codes, code_lens = codec.encode(wav[None, None, :], lengths)
        prompt_tokens = codes[0, :, : int(code_lens[0])]
        logger.info(f"Encoded prompt: {prompt_tokens.shape}")
        return prompt_tokens
