"""More live streams than slots: time to first frames and underruns with and without parking.

A slot of a 64-slot engine makes frames several times faster than a listener plays them (44100 / 2048 = 21.5 frames/s).
With `max_live = 64` request 65 waits for a whole request to finish; with `max_live = N` the scheduler parks streams that
are far ahead of their listener and runs the ones about to run dry (fish_speech_b200/scheduler.py, schedule_live).
This tool sends N streaming requests at once (S2-Pro geometry, synthetic weights, 64 slots, 64-token prompts, ragged
lengths from a seed, `--chunks` chunks per utterance, each chunk's prompt extending the previous one), simulates every
listener from the real clock, and runs both settings for each N, alternating, in one process.

    python tools/serve_live.py [--n 64 128 192 256] [--chunks 2] [--lo 48] [--hi 128]

Prints one JSON line. Per configuration: time to the first frames (p50 / p99 / max, s), underruns (times a listener
that had started ran dry) and starved seconds summed over streams, frames/s of the whole engine, parks and resumes per
request, mean device and host time of a park and of a resume, and the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

SLOTS = 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[64, 128, 192, 256])
    ap.add_argument("--chunks", type=int, default=2)
    ap.add_argument("--lo", type=int, default=48, help="fewest frames of a chunk")
    ap.add_argument("--hi", type=int, default=128, help="most frames of a chunk")
    ap.add_argument("--text-rows", type=int, default=8, help="prompt rows a later chunk adds")
    args = ap.parse_args()

    from bench import FRAME, SR, T_PROMPT, make_prompts
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.engine import kv_pages_for
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest, StreamClock
    from tools.step_gemm_boundaries import card

    pace = SR / FRAME
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n_max = max(args.n)
    seq = T_PROMPT + args.chunks * (args.hi + args.text_rows)
    cfg = s2pro_args(max_seq_len=seq)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are set by the per-chunk budgets
    model = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
    model.max_rows = SLOTS * T_PROMPT
    # every live request, running or parked, keeps its pages: room for n_max of them at full length
    model.setup_caches(max_batch_size=SLOTS, max_seq_len=seq, kv_pages=max(n_max, SLOTS) * kv_pages_for(seq))
    del w
    eng = model.engine
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(args.lo, args.hi + 1, (n_max, args.chunks), generator=g).tolist()
    prompts = [p.to(dev) for p in make_prompts(cfg, n_max, 42)]
    text = torch.randint(0, 1000, (n_max, args.chunks, args.text_rows), generator=g)

    timed = {"park": [], "resume": []}  # (host s, start event, end event)

    def timed_call(kind, fn):
        def call(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record()
            out = fn(*a, **k)
            e1.record()
            timed[kind].append((time.perf_counter() - t0, e0, e1))
            return out
        return call

    eng.park_slot = timed_call("park", eng.park_slot)
    eng.resume_slot = timed_call("resume", eng.resume_slot)

    def serve(n, max_live):
        for v in timed.values():
            v.clear()
        b = ContinuousBatcher(model, max_slots=SLOTS, frames_per_poll=8, max_live=max_live)
        t0 = time.perf_counter()
        hand = [[] for _ in range(n)]  # per stream: (time, frames) of every hand-out
        reqs = []

        def submit(i, c, prompt, clock):
            def on_frames(r, codes):
                hand[i].append((time.perf_counter() - t0, codes.shape[1]))

            def on_done(r):
                if c + 1 < args.chunks:
                    rows = torch.zeros(prompt.size(0), args.text_rows, dtype=prompt.dtype, device=dev)
                    rows[0] = text[i, c + 1].to(dev)
                    grown = torch.cat([prompt, r.result[:, prompt.size(1):-1].to(prompt.dtype), rows], dim=1)
                    submit(i, c + 1, grown, clock)

            reqs.append(b.submit(SlotRequest(prompt=prompt, max_new_tokens=lens[i][c], temperature=0.7, top_p=0.7,
                                             top_k=1, seed=1, reuse_prefix=True, pace=pace, stream=clock,
                                             on_frames=on_frames, on_done=on_done)))

        for i in range(n):
            submit(i, 0, prompts[i], StreamClock())
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b.run()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        b.close()
        first = sorted(h[0][0] for h in hand)
        underruns, starved = 0, 0.0
        for h in hand:  # a listener plays at `pace` while it holds frames and stalls when it has none
            t_prev, held = h[0][0], float(h[0][1])
            for t, k in h[1:]:
                dry = (t - t_prev) - held / pace
                if dry > 0:
                    underruns += 1
                    starved += dry
                held = max(0.0, held - pace * (t - t_prev)) + k
                t_prev = t
        frames = sum(k for h in hand for _, k in h)
        dev_ms = {k: [e0.elapsed_time(e1) for _, e0, e1 in v] for k, v in timed.items()}
        mean = lambda xs: sum(xs) / len(xs) if xs else None
        return {
            "first_frames_s": {"p50": first[len(first) // 2], "p99": first[min(len(first) - 1, int(0.99 * len(first)))],
                               "max": first[-1]},
            "underruns": underruns, "starved_s": starved, "wall_s": wall, "frames_per_s": frames / wall,
            "parks_per_request": sum(r.parks for r in reqs) / n, "resumes_per_request": sum(r.resumes for r in reqs) / n,
            "park_ms": {"device": mean(dev_ms["park"]), "host": mean([1e3 * h for h, _, _ in timed["park"]])},
            "resume_ms": {"device": mean(dev_ms["resume"]), "host": mean([1e3 * h for h, _, _ in timed["resume"]])},
            "tokens": [r.result for r in reqs],
        }

    serve(SLOTS, SLOTS)  # warm-up: graph capture and first touch of every buffer
    serve(SLOTS + 8, SLOTS + 8)
    out = {"workload": f"{args.chunks}-chunk streaming requests arriving together, {T_PROMPT}-token prompts, "
                       f"{args.lo}..{args.hi} frames per chunk, greedy, LM stage only, S2-Pro geometry, synthetic "
                       f"weights, {SLOTS} slots, listeners at {pace:.1f} frames/s", "card": card(), "runs": []}
    for n in args.n:
        tokens = None
        for max_live in (SLOTS, n):
            if max_live == SLOTS and n == SLOTS and tokens is not None:
                continue
            r = serve(n, max_live)
            # the order of `reqs` follows the schedule; compare per stream through the sorted token tensors' shapes
            toks = sorted((t.shape[1], t.sum().item()) for t in r.pop("tokens"))
            same = tokens is None or toks == tokens
            tokens = toks
            out["runs"].append({"n": n, "max_live": max_live, "same_tokens_as_unparked": bool(same), **r})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
