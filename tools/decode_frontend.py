"""Codec output front end: what converting the decoder's fp32 44.1 kHz output to a client's rate and sample format
(`audio.OutputStream.push_many`, one `fsb_audio_out` launch) costs beside the decode pool push it follows.

S2-Pro codec geometry with synthetic weights, --streams streams of --frames frames per push.

  (a) kernel: CUDA-event time of one fsb_audio_out launch over the streams' windows (history + the push's
      frames * 2048 samples each), for every (rate, format), averaged over --iters launches after a warm-up.
  (b) conversion call: the same, timed around the whole `OutputStream.push_many` (window concatenation, descriptor
      upload, launch), events on the device and the host clock around a synchronise.
  (c) pool push: CUDA-event time of `DecodeStreamPool.push` of every stream's next frames, with slots opened without
      a format (today's output) and with every slot opened at the (rate, format) (the frame pass plus the conversion
      launch), averaged over --iters pushes after the bucket's graph is captured.
  (d) device -> host bytes per second of audio of each format (rate x sample size), and the bytes of one push.

    python tools/decode_frontend.py [--streams 64] [--frames 8] [--iters 50] [--out DIR]

Prints one JSON line with the card's name and power limit. Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

from tools.encode_stream import card  # noqa: E402

RATES = [8000, 16000, 22050, 24000, 44100, 48000]
FORMATS = ["float32", "pcm16", "mulaw"]


def events_ms(fn, iters: int) -> float:
    """Mean device time of fn() over iters calls, after two warm-up calls."""
    for _ in range(2):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernel_case(A, L, n: int, samples: int, rate: int, fmt: str, iters: int) -> dict:
    """One launch over n streams' windows in steady state: each stream's history plus `samples` new samples."""
    sts = [A.OutputStream(rate, fmt, "cuda") for _ in range(n)]
    g = torch.Generator(device="cuda").manual_seed(rate)
    piece = lambda: (0.3 * torch.randn(samples, generator=g, device="cuda")).clamp(-1, 1)
    for _ in range(2):  # fill the histories
        A.OutputStream.push_many([(s, piece()) for s in sts])
    items = [(s, piece()) for s in sts]
    # (b) the whole call: every call advances the streams, as a pool push does
    call_ms = events_ms(lambda: A.OutputStream.push_many(items), iters)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        A.OutputStream.push_many(items)
    torch.cuda.synchronize()
    host_ms = (time.perf_counter() - t0) * 1e3 / iters
    # (a) the launch alone, over the window and descriptors of one such call
    code, dtype = A.OUTPUT_FORMATS[fmt]
    segs, rows, x_off, ob = [], [], 0, 0
    for s, x in items:
        if s.identity:
            segs.append(x)
            rows.append((x_off, 0, samples, 0, ob, samples, None, code))
            n_win, n_out = samples, samples
        else:
            hist = s._hist
            segs += [hist, x]
            n_win = hist.numel() + samples
            r0 = s.counts.received
            tab = s.counts.table
            j0 = tab.ready(r0)
            n_out = tab.ready(r0 + samples) - j0
            rows.append((x_off, s._h0, r0 + samples, j0, ob, n_out, s._tab, code))
        x_off += n_win
        ob += -(-n_out * dtype.itemsize // 16) * 16
    win = torch.cat(segs)
    out = torch.empty(ob, dtype=torch.uint8, device="cuda")
    desc = []
    for xo, xs, xe, j0, oo, no, tab, c in rows:
        w, sp, o, nn = (0, 0, 1, 1) if tab is None else (tab[0].data_ptr(), tab[1].data_ptr(), tab[2], tab[3])
        desc.append([xo, xs, xe, j0, oo, no, w, sp, o, nn, c])
    d = torch.tensor(desc, dtype=torch.int64).cuda()
    max_out = max(r[5] for r in rows)
    stream = torch.cuda.current_stream().cuda_stream

    def launch():
        L.check(L.lib().fsb_audio_out(win.data_ptr(), d.data_ptr(), len(rows), max_out, out.data_ptr(), stream))

    kernel_ms = events_ms(launch, iters)
    n_in, n_outs = sum(samples for _ in rows), sum(r[5] for r in rows)
    return {"rate": rate, "format": fmt, "kernel_ms": kernel_ms, "call_ms": call_ms, "call_host_ms": host_ms,
            "outputs": n_outs, "bytes": 4 * n_in + n_outs * dtype.itemsize,
            "kernel_GBps": (4 * n_in + n_outs * dtype.itemsize) / kernel_ms / 1e6}


def pool_case(dac, n: int, k: int, iters: int, rate, fmt) -> float:
    """Mean CUDA-event time of one pool push of k frames for each of n streams opened at (rate, fmt)."""
    pool = dac.open_stream_pool(n, k_max=k)
    slots = [pool.open() if rate is None else pool.open(rate, fmt) for _ in range(n)]
    g = torch.Generator().manual_seed(1)
    codes = torch.stack([torch.randint(0, 1024, (k,), generator=g)] +
                        [torch.randint(0, 1024, (k,), generator=g) for _ in range(dac.n_stage - 1)])
    pieces = {s: codes for s in slots}
    for _ in range(3):  # eager, capture, replay
        pool.push(pieces)
    return events_ms(lambda: pool.push(pieces), iters)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/decode_frontend.py needs a GPU")
    from fish_speech_b200 import _lib as L
    from fish_speech_b200 import audio as A
    from fish_speech_b200 import synthetic
    from fish_speech_b200.models.dac.inference import load_codec_config
    from fish_speech_b200.models.dac.modded_dac import DAC

    ccfg = load_codec_config("modded_dac_vq")
    dac = DAC(ccfg, synthetic.codec_state_dict(ccfg, "cuda"), device="cuda")
    n, k = args.streams, args.frames
    samples = k * dac.frame_length
    res = {"card": card(), "geometry": "S2-Pro codec, synthetic weights", "args": vars(args)}
    plain_ms = pool_case(dac, n, k, args.iters, None, None)
    res["pool_push_plain_ms"] = plain_ms
    print(json.dumps({"pool_push_plain_ms": plain_ms}), file=sys.stderr, flush=True)
    rows = []
    for rate in RATES:
        for fmt in FORMATS:
            if rate == dac.sample_rate and fmt == "float32":
                continue  # no conversion: the push's own output
            row = kernel_case(A, L, n, samples, rate, fmt, args.iters)
            row["pool_push_ms"] = pool_case(dac, n, k, args.iters, rate, fmt)
            row["kernel_share_of_plain_push"] = row["kernel_ms"] / plain_ms
            row["call_share_of_plain_push"] = row["call_ms"] / plain_ms
            rows.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    res["conversions"] = rows
    res["d2h_bytes_per_audio_s"] = {f"{fmt}@{rate}": rate * A.OUTPUT_FORMATS[fmt][1].itemsize
                                    for rate in RATES for fmt in FORMATS}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "decode_frontend.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
