"""Record the prompts the reference's CPU prompt builder (fish_speech.content_sequence / conversation, unmodified)
produces for the generate_long scenario of tests/test_engine_cpu.py, as tests/golden/generate_long_prompts.npz.

    FISH_SPEECH_REFERENCE=<fish-speech checkout> python -m oracle.make_golden_frontend

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
    from tests.test_engine_cpu import drive_generate_long_plan

    prompts, _, _ = drive_generate_long_plan()
    arrays = {f"prompt_{i}": p.numpy().astype(np.int32) for i, p in enumerate(prompts)}
    arrays["count"] = np.int32(len(prompts))
    path = ROOT / "tests" / "golden" / "generate_long_prompts.npz"
    np.savez_compressed(path, **arrays)
    return path


if __name__ == "__main__":
    print(main())
