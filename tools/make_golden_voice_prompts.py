"""Record the first prompts the reference's CPU prompt builder (fish_speech.content_sequence / conversation, unmodified)
produces for two voice-clone requests with one reference and different texts, as
tests/golden/voice_clone_prompts.npz, for tests/test_prefix_cache_cpu.py.

    FISH_SPEECH_REFERENCE=<fish-speech checkout> python tools/make_golden_voice_prompts.py

The CPU test replays these prompts through a stand-in builder (and compares a live builder with them where the
fish-speech package is installed), so that it runs without the reference.
"""
from __future__ import annotations

import os
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))


def main() -> Path:
    ref = os.environ.get("FISH_SPEECH_REFERENCE", "")
    if not (Path(ref) / "fish_speech" / "conversation.py").exists():
        raise SystemExit("set FISH_SPEECH_REFERENCE to the directory of a fish-speech checkout")
    sys.path.insert(0, ref)
    from tests.test_prefix_cache_cpu import voice_clone_prompts

    prompts, _, system_end = voice_clone_prompts()
    path = ROOT / "tests" / "golden" / "voice_clone_prompts.npz"
    np.savez_compressed(path, prompt_0=prompts[0].numpy().astype(np.int32), prompt_1=prompts[1].numpy().astype(np.int32),
                        system_end=np.int32(system_end))
    return path


if __name__ == "__main__":
    print(main())
