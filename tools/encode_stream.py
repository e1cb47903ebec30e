"""Streaming encode: EncodeStreamPool throughput, and `bulk_encode` of clips longer than the one-shot encode can hold.

S2-Pro codec geometry with synthetic weights.

  (a) N = 1, 8, 32, 64 concurrent streams of 30 s of seeded noise, pushed together in pieces of 1, 8 and 32 frames
      through one pool of N slots (after a warm-up of three pushes that sizes the workspaces and captures the bucket's graph):
      audio-s/s (N x 30 s over the wall time of all pushes, ended by a device synchronise) and the mean device-event ms
      per push; beside it the one-shot `DAC.encode` pass over the same N clips, as few batches as its launches take
      (warmed up once); and whether every stream's codes equal the one-shot's.
  (b) `bulk_encode.encode_files` on one synthetic clip, as a 16-bit wav file: once at a length the one-shot encode
      handles, run both ways (the one-shot, and the streamed path forced by a free-memory probe that reports 0), and
      once at --long-hours (default 2 h), which the one-shot cannot hold on an 80 GB card and `DAC.encode` routes to the
      streamed path by itself: peak `torch.cuda.max_memory_allocated` over the call, audio-s/s, which path ran, and
      whether the two `.npy` files of the short clip are byte-identical.

    python tools/encode_stream.py [--streams 1 8 32 64] [--pieces 1 8 32] [--seconds 30] [--short-minutes 10]
                                  [--long-hours 2] [--out DIR]

Prints one JSON line with the card's name and power limit. Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import tempfile
import time
import wave
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card() -> dict:
    q = "name,power.limit"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (v.strip() for v in out.split(","))))
    except Exception as e:  # pragma: no cover
        return {"name": torch.cuda.get_device_name(0), "error": repr(e)}


def noise(n: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return (0.1 * torch.randn(n, generator=g)).clamp(-1, 1)


def streams_case(dac, n: int, k: int, clips: list, ref: torch.Tensor) -> dict:
    FL = dac.frame_length
    frames = -(-clips[0].numel() // FL)
    padded = [torch.nn.functional.pad(c, (0, frames * FL - c.numel())).cuda() for c in clips]
    pool = dac.open_encode_pool(n, k_max=k)
    slots = [pool.open() for _ in range(n)]
    for f0 in range(0, 3 * k, k):  # warm-up: workspaces, GEMM plans and the graph of the (n, k) bucket
        pool.push({s: padded[i][f0 * FL: (f0 + k) * FL] for i, s in enumerate(slots)})
    for s in slots:
        pool.close(s)
    slots = [pool.open() for _ in range(n)]
    events, codes = [], [[] for _ in range(n)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for f0 in range(0, frames, k):
        f1 = min(frames, f0 + k)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = pool.push({s: padded[i][f0 * FL: f1 * FL] for i, s in enumerate(slots)})
        e1.record()
        events.append((e0, e1))
        for i, s in enumerate(slots):
            codes[i].append(out[s])
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    got = torch.stack([torch.cat(c, dim=1) for c in codes])
    return {"audio_s_per_s": n * clips[0].numel() / dac.sample_rate / wall, "pushes": len(events),
            "device_ms_per_push": float(np.mean([a.elapsed_time(b) for a, b in events])),
            "codes_equal_one_shot": bool(torch.equal(got, ref)), "state_mb": pool.state_bytes / 2 ** 20}


def write_wav(path: Path, x: torch.Tensor, sr: int) -> None:
    with wave.open(str(path), "wb") as wf:
        wf.setnchannels(1)
        wf.setsampwidth(2)
        wf.setframerate(sr)
        wf.writeframes((x * 32767).round().to(torch.int16).numpy().tobytes())


def bulk_case(dac, path: Path, force_stream: bool) -> dict:
    from fish_speech_b200 import bulk_encode as BE

    path.with_suffix(".npy").unlink(missing_ok=True)
    ran = []
    one_shot, streamed = dac._encode_one_shot, dac._encode_streamed
    dac._encode_one_shot = lambda *a: ran.append("one_shot") or one_shot(*a)
    dac._encode_streamed = lambda *a: ran.append("streamed") or streamed(*a)
    if force_stream:
        dac._free_device_bytes = lambda: 0
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        _, seconds = BE.encode_files([path], dac, batch_size=1)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
    finally:
        del dac._encode_one_shot, dac._encode_streamed
        if force_stream:
            del dac._free_device_bytes
    return {"path": ran, "audio_s": seconds, "audio_s_per_s": seconds / wall, "wall_s": wall,
            "peak_allocated_gb": torch.cuda.max_memory_allocated() / 1e9,
            "peak_above_start_gb": (torch.cuda.max_memory_allocated() - base) / 1e9,
            "npy": path.with_suffix(".npy").read_bytes()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 8, 32, 64])
    ap.add_argument("--pieces", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--seconds", type=float, default=30.0)
    ap.add_argument("--short-minutes", type=float, default=10.0)
    ap.add_argument("--long-hours", type=float, default=2.0)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/encode_stream.py needs a GPU")
    from fish_speech_b200 import synthetic
    from fish_speech_b200.models.dac.inference import load_codec_config
    from fish_speech_b200.models.dac.modded_dac import DAC

    dev = "cuda"
    ccfg = load_codec_config("modded_dac_vq")
    dac = DAC(ccfg, synthetic.codec_state_dict(ccfg, dev), device=dev)
    sr = dac.sample_rate
    res = {"card": card(), "geometry": "S2-Pro codec, synthetic weights", "streams": {}}

    n_samples = int(args.seconds * sr)
    for n in args.streams:
        clips = [noise(n_samples, 100 + i) for i in range(n)]
        batch = torch.stack(clips)[:, None].cuda()
        sub = max(1, DAC.ONE_SHOT_MAX_ROWS // (-(-n_samples // 512)))  # clips per one-shot call it can launch
        one = lambda: torch.cat([dac._encode_one_shot(batch[i: i + sub], None, None)[0] for i in range(0, n, sub)])
        one()  # warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ref = one()
        torch.cuda.synchronize()
        row = {"one_shot_audio_s_per_s": n * args.seconds / (time.perf_counter() - t0), "one_shot_clips_per_call": sub}
        del batch
        for k in args.pieces:
            row[f"pieces_{k}"] = streams_case(dac, n, k, clips, ref)
        res["streams"][str(n)] = row
        print(json.dumps({"streams": n, **row}), file=sys.stderr, flush=True)

    with tempfile.TemporaryDirectory() as tmp:
        short = Path(tmp) / "short.wav"
        write_wav(short, noise(int(args.short_minutes * 60 * sr), 7), sr)
        a = bulk_case(dac, short, force_stream=False)
        b = bulk_case(dac, short, force_stream=True)
        res["bulk_short"] = {"minutes": args.short_minutes, "npy_identical": a.pop("npy") == b.pop("npy"),
                             "default": a, "forced_stream": b}
        print(json.dumps(res["bulk_short"]), file=sys.stderr, flush=True)
        long = Path(tmp) / "long.wav"
        n_long = int(args.long_hours * 3600 * sr)
        write_wav(long, torch.cat([noise(min(1 << 24, n_long - i), i) for i in range(0, n_long, 1 << 24)]), sr)
        c = bulk_case(dac, long, force_stream=False)
        frames = np.load(long.with_suffix(".npy")).shape
        c.pop("npy")
        res["bulk_long"] = {"hours": args.long_hours, "codes_shape": list(frames),
                            "one_shot_bytes_estimate_gb": dac._encode_one_shot_bytes(1, -(-n_long // 2048) * 2048) / 1e9,
                            **c}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "encode_stream.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
