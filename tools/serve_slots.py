"""Serving throughput with 32 and with 64 slots per engine, on the same ragged queue.

An engine of up to 32 slots runs the 32-row decode step GEMM; 33..64 slots run the 64-row one. A decode frame streams
the same weight bytes whatever the number of rows, so twice the slots should serve more audio per second. This tool
builds one seeded queue in the style of `bench.py --workload serve` (384 requests, 64-token prompts, 64..256 frames
each, greedy, LM stage only, S2-Pro geometry with synthetic weights), runs it through `ContinuousBatcher` with 32 and
with 64 slots, alternating A B A B in one process, and also times decode frames at full occupancy for each engine.

    python tools/serve_slots.py [--requests 384] [--reps 2] [--frames 64]

Prints one JSON line: audio-s/s and ms per decode frame for each slot count, `identical_tokens` (every request returned
the same tokens in every run) and the card's name and power limit. Needs a GPU with room for both engines' KV caches.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

SLOTS = (32, 64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=384)
    ap.add_argument("--reps", type=int, default=2, help="alternated timed runs per slot count")
    ap.add_argument("--frames", type=int, default=64, help="decode frames timed at full occupancy")
    args = ap.parse_args()

    from bench import FRAME, SR, T_PROMPT, make_prompts
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = s2pro_args(max_seq_len=T_PROMPT + 256)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are set by the per-request budgets
    models = {}
    for n in SLOTS:  # both engines share the weight tensors; each owns its KV caches and plans
        m = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        m.max_rows = n * T_PROMPT
        m.setup_caches(max_batch_size=n, max_seq_len=cfg.max_seq_len)
        models[n] = m
    del w
    g = torch.Generator().manual_seed(7)
    lens = torch.randint(64, 257, (args.requests,), generator=g).tolist()
    prompts = [p.to(dev) for p in make_prompts(cfg, args.requests, 42)]
    audio_s = sum(lens) * FRAME / SR

    def serve(n, count):
        b = ContinuousBatcher(models[n], max_slots=n, frames_per_poll=8)
        reqs = [b.submit(SlotRequest(prompt=p, max_new_tokens=k, temperature=0.7, top_p=0.7, top_k=1, seed=1))
                for p, k in zip(prompts[:count], lens[:count])]
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        b.run()
        ev1.record()
        torch.cuda.synchronize()
        occ = b.slot_frames / max(1, b.frames_run * n)
        b.close()
        return ev0.elapsed_time(ev1), [r.result for r in reqs], occ, b.frames_run

    def frame_ms(n):
        """ms per decode frame with every slot live (the frame graph, greedy)."""
        eng = models[n].engine
        sp = eng.sampling(0.7, 0.7, 1, 42)
        eng.reset()
        eng.prefill(prompts[:n], list(range(n)), sp, do_sample=True)
        eng.decode(n, 2, sp, use_graph=True)  # captures the frame graph
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        eng.decode(n, args.frames, sp, use_graph=True)
        ev1.record()
        torch.cuda.synchronize()
        eng.reset()
        return ev0.elapsed_time(ev1) / args.frames

    for n in SLOTS:  # warm-up: graph capture and first-touch of every buffer
        serve(n, 2 * n)
    runs = {n: [] for n in SLOTS}
    results = {n: None for n in SLOTS}
    same = True
    for _ in range(args.reps):
        for n in SLOTS:  # A B A B
            ms, out, occ, frames = serve(n, args.requests)
            runs[n].append({"ms": ms, "occupancy": occ, "frames_run": frames})
            if results[n] is None:
                results[n] = out
            same &= all(torch.equal(a, b) for a, b in zip(results[n], out))
    same &= all(torch.equal(a, b) for a, b in zip(results[SLOTS[0]], results[SLOTS[1]]))
    frames = {n: [] for n in SLOTS}
    for _ in range(args.reps):
        for n in SLOTS:
            frames[n].append(frame_ms(n))

    out = {"workload": f"serve: {args.requests} queued requests, {T_PROMPT}-token prompts, 64..256 frames each "
                       f"(mean {sum(lens) / len(lens):.0f}), greedy, LM stage only, S2-Pro geometry, synthetic weights",
           "card": card(), "identical_tokens": bool(same), "audio_s": audio_s}
    for n in SLOTS:
        out[f"slots_{n}"] = {
            "audio_s_per_s": [audio_s / (r["ms"] / 1e3) for r in runs[n]],
            "ms": [r["ms"] for r in runs[n]],
            "occupancy": runs[n][0]["occupancy"], "decode_frames_run": runs[n][0]["frames_run"],
            "ms_per_frame_full": frames[n],
            "row_tile": models[n].engine.row_tile,
        }
    best = {n: max(out[f"slots_{n}"]["audio_s_per_s"]) for n in SLOTS}
    out["speedup_64_over_32"] = best[64] / best[32]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
