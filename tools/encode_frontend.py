"""Codec input front end: `bulk_encode.encode_files` with the CPU front end (numpy convert + torchaudio resample on the
reader thread) against the device front end (fish_speech_b200.audio), and the encode pool fed at 48 kHz against 44.1 kHz.

S2-Pro codec geometry with synthetic weights.

  (a) Seeded 16-bit WAV files at 16, 22.05, 24, 44.1 and 48 kHz, mono and stereo in turn: --clips clips of 3-15 s and
      one --long-minutes file at 48 kHz stereo. After a warm-up of both front ends on a few clips, `encode_files` over
      all of them with each front end, alternated --rounds times: audio-s/s (audio seconds over the wall time of the
      call, which ends in a device synchronise). Beside it, the CUDA-event time of `audio.load_batch` (upload,
      conversion, resampling, padding) over the same files in batches of --batch-size, per audio-second, and whether the
      two front ends wrote the same codes for the 44.1 kHz files (they must: no resampling runs there).
  (b) --streams streams of --stream-seconds of noise pushed together through one pool, in pieces of --piece-frames
      frames' duration: at 44.1 kHz as whole frames into slots opened without a rate, and at 48 kHz as float32 pieces
      into slots opened with sample_rate=48000 (ended by flush): audio-s/s of each after a warm-up.

    python tools/encode_frontend.py [--clips 2000] [--long-minutes 10] [--rounds 2] [--batch-size 64]
                                    [--streams 64] [--stream-seconds 30] [--piece-frames 32] [--out DIR]

Prints one JSON line with the card's name and power limit. Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
import time
import wave
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from tools.encode_stream import card  # noqa: E402

RATES = [16000, 22050, 24000, 44100, 48000]


def write_clips(root: Path, n_clips: int, long_minutes: float, seed: int) -> list:
    """[(path, rate, channels, frames)]: the long file first, then the clips."""
    rng = np.random.default_rng(seed)
    specs = [(48000, 2, int(long_minutes * 60 * 48000))]
    for i in range(n_clips):
        specs.append((RATES[i % len(RATES)], 1 + (i // len(RATES)) % 2, 0))
    out = []
    for i, (sr, ch, n) in enumerate(specs):
        n = n or int(rng.uniform(3.0, 15.0) * sr)
        pcm = np.clip(rng.standard_normal(n * ch, dtype=np.float32) * 3000.0, -32768, 32767).astype("<i2")
        p = root / f"c{i:05d}_{sr}_{ch}.wav"
        with wave.open(str(p), "wb") as f:
            f.setnchannels(ch)
            f.setsampwidth(2)
            f.setframerate(sr)
            f.writeframes(pcm.tobytes())
        out.append((p, sr, ch, n))
    return out


def run_files(BE, dac, files: list, device_front_end: bool, batch_size: int) -> dict:
    for f in files:
        f.with_suffix(".npy").unlink(missing_ok=True)
    saved = BE._device_front_end
    BE._device_front_end = lambda model: device_front_end
    try:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n, seconds = BE.encode_files(files, dac, batch_size=batch_size)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        BE._device_front_end = saved
    return {"files": n, "audio_s": seconds, "wall_s": wall, "audio_s_per_s": seconds / wall}


def front_end_kernel_time(A, files: list, sr: int, batch_size: int) -> dict:
    pcms = [A.read_pcm(f) for f in files]
    order = sorted(range(len(pcms)), key=lambda i: pcms[i].frames)
    batches = [[pcms[i] for i in order[b: b + batch_size]] for b in range(0, len(order), batch_size)]
    for b in batches[:2]:
        A.load_batch(b, sr, "cuda")  # warm-up: tables, allocator
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    seconds = 0.0
    for b in batches:
        _, lens = A.load_batch(b, sr, "cuda")
        seconds += sum(c.out_length(sr) for c in b) / sr
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    return {"batches": len(batches), "audio_s": seconds, "event_ms": ms, "ms_per_audio_s": ms / seconds,
            "audio_s_per_s": seconds / (ms / 1e3)}


def stream_rate(A, dac, n: int, seconds: float, piece_frames: int, sr: int, seed: int) -> dict:
    FL = dac.frame_length
    frames = int(seconds * dac.sample_rate) // FL
    per_piece = FL * piece_frames if sr == dac.sample_rate else round(FL * piece_frames * sr / dac.sample_rate)
    n_in = frames * FL if sr == dac.sample_rate else round(frames * FL * sr / dac.sample_rate)
    g = torch.Generator().manual_seed(seed)
    clips = [(0.1 * torch.randn(n_in, generator=g)).clamp(-1, 1).cuda() for _ in range(n)]
    pool = dac.open_encode_pool(n, k_max=piece_frames)
    rate = None if sr == dac.sample_rate else sr

    def one_pass(limit: int) -> float:
        slots = [pool.open(sample_rate=rate) for _ in range(n)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for a in range(0, min(limit, n_in), per_piece):
            pool.push({s: clips[i][a: a + per_piece] for i, s in enumerate(slots)})
        if rate is not None:
            for s in slots:
                pool.flush(s)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        for s in slots:
            pool.close(s)
        return wall

    one_pass(4 * per_piece)  # warm-up: workspaces, plans, graphs of the buckets
    one_pass(4 * per_piece)
    wall = one_pass(n_in)
    return {"streams": n, "seconds": n_in / sr, "input_rate": sr, "piece_samples": per_piece,
            "audio_s_per_s": n * n_in / sr / wall, "wall_s": wall}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=2000)
    ap.add_argument("--long-minutes", type=float, default=10.0)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--stream-seconds", type=float, default=30.0)
    ap.add_argument("--piece-frames", type=int, default=32)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/encode_frontend.py needs a GPU")
    from fish_speech_b200 import audio as A
    from fish_speech_b200 import bulk_encode as BE
    from fish_speech_b200 import synthetic
    from fish_speech_b200.models.dac.inference import load_codec_config
    from fish_speech_b200.models.dac.modded_dac import DAC

    ccfg = load_codec_config("modded_dac_vq")
    dac = DAC(ccfg, synthetic.codec_state_dict(ccfg, "cuda"), device="cuda")
    sr = dac.sample_rate
    res = {"card": card(), "geometry": "S2-Pro codec, synthetic weights", "args": vars(args)}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        specs = write_clips(Path(tmp), args.clips, args.long_minutes, args.seed)
        files = [s[0] for s in specs]
        res["files"] = {"count": len(files), "audio_hours": sum(s[3] / s[1] for s in specs) / 3600,
                        "write_s": time.perf_counter() - t0}
        print(json.dumps(res["files"]), file=sys.stderr, flush=True)
        warm = files[1: 1 + 2 * len(RATES)]
        run_files(BE, dac, warm, False, args.batch_size)
        run_files(BE, dac, warm, True, args.batch_size)
        rows = []
        native = [s[0] for s in specs if s[1] == sr]
        for r in range(args.rounds):
            for dev in (False, True):
                row = run_files(BE, dac, files, dev, args.batch_size)
                row["front_end"] = "device" if dev else "cpu"
                if r == args.rounds - 1:
                    row["native_rate_npy"] = [f.with_suffix(".npy").read_bytes() for f in native]
                rows.append(row)
                print(json.dumps({k: v for k, v in row.items() if k != "native_rate_npy"}), file=sys.stderr, flush=True)
        cpu_npy, dev_npy = rows[-2].pop("native_rate_npy"), rows[-1].pop("native_rate_npy")
        res["bulk"] = {"runs": rows, "native_rate_codes_identical": cpu_npy == dev_npy,
                       "front_end_kernels": front_end_kernel_time(A, files, sr, args.batch_size)}
        print(json.dumps(res["bulk"]["front_end_kernels"]), file=sys.stderr, flush=True)
    res["stream"] = [stream_rate(A, dac, args.streams, args.stream_seconds, args.piece_frames, rate, 9)
                     for rate in (sr, 48000)]
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "encode_frontend.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
