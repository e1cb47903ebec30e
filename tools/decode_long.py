"""Decode of any length: `DAC.from_indices`' one-shot pass against its streamed route, and the ragged batch decode.

S2-Pro codec geometry with synthetic weights, seeded random codes.

  (a) One-shot against streamed at lengths both can run (default 1, 5 and 15 minutes, B = 1 and B = 4; a case whose
      one-shot rows or workspaces do not fit is run streamed only). Per route: the peak `torch.cuda.max_memory_allocated`
      of the first call above what was allocated before it, with the codec's workspaces and graphs dropped first (so it
      counts every workspace the route needs); the wall time of a call after two warm-up calls, ended by a device
      synchronise; and whether the two waveforms are byte-identical. The streamed route is forced by a free-memory probe
      that reports 0.
  (b) The route `from_indices` takes by itself at --long-minutes (default 30 and 120), B = 1: which route, time, peak.
  (c) Pieces of --sweep-frames frames (default 64, 128, 256) per push at 5 minutes, B = 1 and 4: streamed time and peak.
  (d) `bulk_encode.batch_vqgan_decode` on --items utterances of 5-60 s, against one `from_indices` call per utterance
      and against the reference's scheme (every utterance padded to the longest, micro-batches of 8): audio-s/s of a
      call after one warm-up call, and whether every item's samples equal its `from_indices` alone.

    python tools/decode_long.py [--minutes 1 5 15] [--batches 1 4] [--long-minutes 30 120] [--sweep-frames 64 128 256]
                                [--items 64] [--out DIR]

Prints one JSON line with the card's name and power limit. Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
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


def rand_codes(cfg, B: int, T: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randint(0, cfg.semantic_codebook_size, (B, T), generator=g)] +
                       [torch.randint(0, cfg.codebook_size, (B, T), generator=g) for _ in range(cfg.n_codebooks)], 1)


def drop_workspaces(dac) -> None:
    """Forget the codec's workspaces, graphs and decode pool, so the next call allocates what it needs."""
    dac._bufs.clear()
    dac._graphs.clear()
    dac._graph_seen.clear()
    dac._dec_pool = None
    dac._ws_gen += 1
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def run(dac, codes: torch.Tensor, stream: bool, calls: int = 3) -> tuple:
    """(waveform of the last call, peak GB of the first call above its start, seconds of the last call, route)."""
    ran = []
    real = dac._from_indices_streamed
    dac._from_indices_streamed = lambda idx: ran.append("streamed") or real(idx)
    if stream:
        dac._free_device_bytes = lambda: 0
    try:
        drop_workspaces(dac)
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        wav = dac.from_indices(codes.clone())
        torch.cuda.synchronize()
        peak = (torch.cuda.max_memory_allocated() - base) / 1e9
        secs = None
        for _ in range(calls - 1):
            del wav
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            wav = dac.from_indices(codes.clone())
            torch.cuda.synchronize()
            secs = time.perf_counter() - t0
    finally:
        del dac._from_indices_streamed
        if stream:
            del dac._free_device_bytes
    return wav, peak, secs, "streamed" if ran else "one_shot"


def one_shot_fits(dac, B: int, T: int) -> bool:
    drop_workspaces(dac)
    need = dac._decode_one_shot_bytes(B, T)
    return B * T <= dac.ONE_SHOT_MAX_ROWS and need + need // 20 + dac.ONE_SHOT_MARGIN_BYTES <= dac._free_device_bytes()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--minutes", type=float, nargs="+", default=[1, 5, 15])
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 4])
    ap.add_argument("--long-minutes", type=float, nargs="+", default=[30, 120])
    ap.add_argument("--sweep-frames", type=int, nargs="+", default=[64, 128, 256])
    ap.add_argument("--items", type=int, default=64)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/decode_long.py needs a GPU")
    from fish_speech_b200 import bulk_encode as BE
    from fish_speech_b200 import synthetic
    from fish_speech_b200.models.dac.inference import load_codec_config
    from fish_speech_b200.models.dac.modded_dac import DAC

    dev = "cuda"
    ccfg = load_codec_config("modded_dac_vq")
    dac = DAC(ccfg, synthetic.codec_state_dict(ccfg, dev), device=dev)
    fps = dac.sample_rate / dac.frame_length
    res = {"card": card(), "geometry": "S2-Pro codec, synthetic weights", "slots": DAC.DECODE_STREAM_SLOTS,
           "frames_per_push": DAC.DECODE_STREAM_FRAMES, "one_shot_vs_streamed": [], "long": [], "sweep": []}

    def log(row):
        print(json.dumps(row), file=sys.stderr, flush=True)

    for minutes in args.minutes:
        for B in args.batches:
            T = round(minutes * 60 * fps)
            codes = rand_codes(ccfg, B, T, 10 * B + T).to(dev)
            audio_s = B * T / fps
            row = {"minutes": minutes, "B": B, "frames": T}
            ws, wp, st, _ = run(dac, codes, stream=True)
            row["streamed"] = {"peak_gb": wp, "s": st, "audio_s_per_s": audio_s / st}
            if one_shot_fits(dac, B, T):
                wo, op, ot, route = run(dac, codes, stream=False)
                row["one_shot"] = {"peak_gb": op, "s": ot, "audio_s_per_s": audio_s / ot, "route": route}
                row["byte_identical"] = bool(torch.equal(wo, ws))
                del wo
            else:
                row["one_shot"] = "does not fit"
            del ws
            res["one_shot_vs_streamed"].append(row)
            log(row)

    for minutes in args.long_minutes:
        T = round(minutes * 60 * fps)
        codes = rand_codes(ccfg, 1, T, T).to(dev)
        _, peak, secs, route = run(dac, codes, stream=False, calls=2)
        row = {"minutes": minutes, "B": 1, "frames": T, "route": route, "peak_gb": peak, "s": secs,
               "audio_s_per_s": T / fps / secs, "one_shot_estimate_gb": dac._decode_one_shot_bytes(1, T) / 1e9}
        res["long"].append(row)
        log(row)

    for k in args.sweep_frames:
        dac.DECODE_STREAM_FRAMES = k
        for B in args.batches:
            T = round(5 * 60 * fps)
            codes = rand_codes(ccfg, B, T, 7 + B).to(dev)
            _, peak, secs, _ = run(dac, codes, stream=True)
            row = {"frames_per_push": k, "B": B, "minutes": 5, "peak_gb": peak, "s": secs,
                   "audio_s_per_s": B * T / fps / secs}
            res["sweep"].append(row)
            log(row)
    del dac.DECODE_STREAM_FRAMES

    rng = np.random.default_rng(0)
    lengths = [int(round(s * fps)) for s in rng.uniform(5, 60, args.items)]
    items = [rand_codes(ccfg, 1, T, 500 + i)[0] for i, T in enumerate(lengths)]
    audio_s = sum(lengths) / fps
    longest = max(lengths)
    padded = torch.stack([torch.nn.functional.pad(c, (0, longest - c.shape[1])) for c in items]).to(dev)

    def per_item():
        return [dac.from_indices(c[None].to(dev))[0].cpu().numpy() for c in items]

    def micro_batches():
        out = []
        for i in range(0, len(items), 8):
            wav = dac.from_indices(padded[i: i + 8].clone()).cpu()
            out += [w[:, : n * dac.frame_length].numpy() for w, n in zip(wav, lengths[i: i + 8])]
        return out

    ragged = {"items": len(items), "audio_s": audio_s, "frames_min": min(lengths), "frames_max": longest}
    got = {}
    drop_workspaces(dac)
    for name, fn in [("batch_vqgan_decode", lambda: BE.batch_vqgan_decode(dac, items)), ("per_item", per_item),
                     ("padded_micro_batches_of_8", micro_batches)]:
        fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        got[name] = fn()
        torch.cuda.synchronize()
        secs = time.perf_counter() - t0
        ragged[name] = {"s": secs, "audio_s_per_s": audio_s / secs}
    ragged["items_equal_from_indices_alone"] = all(a.tobytes() == b.tobytes()
                                                   for a, b in zip(got["batch_vqgan_decode"], got["per_item"]))
    res["ragged"] = ragged
    log(ragged)
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "decode_long.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
