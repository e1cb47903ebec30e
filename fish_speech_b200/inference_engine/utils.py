"""What `TTSInferenceEngine.inference` yields, and the streaming WAV preamble (fish_speech/inference_engine/utils.py:
`InferenceResult`, `wav_chunk_header`)."""
import struct
from dataclasses import dataclass
from typing import Literal, Optional, Tuple

import numpy as np


@dataclass
class InferenceResult:
    """code "header": audio = (sample_rate, header bytes as uint8 array); "segment" / "final": (sample_rate, float
    waveform), or with a request's `sample_rate` / `sample_format` the samples at that rate as float32, int16 (pcm16)
    or uint8 (mulaw); "error": `error` holds the exception."""

    code: Literal["header", "segment", "error", "final"]
    audio: Optional[Tuple[int, np.ndarray]]
    error: Optional[Exception]


# WAVE format tags: integer PCM, IEEE float, G.711 mu-law
WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT, WAVE_FORMAT_MULAW = 1, 3, 7
# the (bit depth, format tag) of each device output format (audio.OUTPUT_FORMATS)
WAVE_OF_FORMAT = {"float32": (32, WAVE_FORMAT_IEEE_FLOAT), "pcm16": (16, WAVE_FORMAT_PCM), "mulaw": (8, WAVE_FORMAT_MULAW)}


def wav_chunk_header(sample_rate: int = 44100, bit_depth: int = 16, channels: int = 1,
                     format_tag: int = WAVE_FORMAT_PCM) -> bytes:
    """The 44 bytes a WAV file starts with, for a stream whose length is not known yet (data size 0): a client
    that receives this and then raw little-endian sample chunks plays the stream. `format_tag` 1 is integer PCM, 3
    IEEE float (bit_depth 32) and 7 G.711 mu-law (bit_depth 8); the 16-byte fmt chunk is the same for all three."""
    frame_bytes = channels * bit_depth // 8
    fmt = struct.pack("<IHHIIHH", 16, format_tag, channels, sample_rate, sample_rate * frame_bytes, frame_bytes,
                      bit_depth)
    return b"RIFF" + struct.pack("<I", 4 + (4 + len(fmt)) + 8) + b"WAVE" + b"fmt " + fmt + b"data" + struct.pack("<I", 0)


def pcm16(waveform: np.ndarray) -> bytes:
    """Float waveform in [-1, 1] -> little-endian 16-bit PCM bytes (what follows `wav_chunk_header` on the wire;
    tools/server/inference.py:32-33 does this per streamed segment)."""
    x = np.clip(np.asarray(waveform, dtype=np.float32), -1.0, 1.0)
    return (x * 32767.0).astype("<i2").tobytes()
