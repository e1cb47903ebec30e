"""Request objects. The wire schema is the reference's (fish_speech/utils/schema.py:81-107, unchanged and
out of scope); when fish_speech is importable its pydantic models are used as-is, otherwise plain
dataclasses with the same fields keep the engine usable stand-alone."""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Optional

try:  # pragma: no cover
    from fish_speech.utils.schema import ServeReferenceAudio, ServeTTSRequest  # type: ignore
except Exception:

    @dataclass
    class ServeReferenceAudio:  # type: ignore[no-redef]
        audio: bytes
        text: str

    @dataclass
    class ServeTTSRequest:  # type: ignore[no-redef]
        text: str
        chunk_length: int = 200
        format: str = "wav"
        latency: str = "normal"
        references: list = field(default_factory=list)
        reference_id: Optional[str] = None
        seed: Optional[int] = None
        use_memory_cache: str = "off"
        normalize: bool = True
        streaming: bool = False
        max_new_tokens: int = 1024
        top_p: float = 0.8
        repetition_penalty: float = 1.1
        temperature: float = 0.8
        # extensions of ours: the audio handed out, converted on the device (audio.convert_out). None: the codec's
        # fp32 at 44.1 kHz, as the reference hands it out
        sample_rate: Optional[int] = None
        sample_format: Optional[str] = None  # "float32", "pcm16" (int16) or "mulaw" (uint8, G.711)
