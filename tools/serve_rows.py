"""A 64-slot engine below peak load: the 32-row step at <= 32 live rows, and compact rows in a load-varying queue.

An engine of 33..64 slots runs a frame of at most 32 rows on its 32-row step GEMM plans (same bits as the 64-row
ones). This tool measures, on the S2-Pro geometry with synthetic weights:

  (a) ms per decode frame of one 64-slot engine with k live rows, k in 1, 8, 16, 32, 33, 48, 64: the tile forced to
      64 rows, then automatic (32 rows for k <= 32);
  (b) one seeded queue whose concurrency ramps 8 -> 64 -> 8 (requests are topped up to a target that changes every
      `--phase` polls; 64-token prompts, 64..256 frames each, greedy), served by one 64-slot `ContinuousBatcher` with
      compact rows off and on, alternating A B A B: audio-s/s, mean ms per frame, moves per request, the share of
      frames that ran on the 32-row tile, and `identical_tokens` (every request the same tokens in every run).

    python tools/serve_rows.py [--reps 2] [--frames 64] [--phase 16]

Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

LIVE = (1, 8, 16, 32, 33, 48, 64)
RAMP = (8, 16, 32, 48, 64, 64, 48, 32, 16, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2, help="alternated runs per setting")
    ap.add_argument("--frames", type=int, default=64, help="decode frames timed per live-row count")
    ap.add_argument("--phase", type=int, default=16, help="polls per step of the concurrency ramp")
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
    model = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
    model.max_rows = 64 * T_PROMPT
    model.setup_caches(max_batch_size=64, max_seq_len=cfg.max_seq_len)
    del w
    eng = model.engine
    assert eng.row_tile == 64
    n_req = 64 * 12
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(64, 257, (n_req,), generator=g).tolist()
    prompts = [p.to(dev) for p in make_prompts(cfg, n_req, 43)]

    # ---- (a) ms per frame at k live rows ----
    def frame_ms(k, tile):
        sp = eng.sampling(0.7, 0.7, 1, 42)
        eng.set_decode_tile(tile)
        eng.reset()
        eng.prefill(prompts[:k], list(range(k)), sp, do_sample=True)
        eng.decode(k, 2, sp, use_graph=True)  # captures (or replays) the frame graph
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        eng.decode(k, args.frames, sp, use_graph=True)
        ev1.record()
        torch.cuda.synchronize()
        used = eng.decode_tile
        eng.set_decode_tile(0)
        eng.reset()
        return ev0.elapsed_time(ev1) / args.frames, used

    for k in LIVE:  # warm-up: every graph the timed loop replays
        for tile in (64, 0):
            frame_ms(k, tile)
    frames = {k: {"forced_64": [], "auto": [], "auto_tile": None} for k in LIVE}
    for _ in range(args.reps):
        for k in LIVE:
            for tile, key in ((64, "forced_64"), (0, "auto")):  # A B A B
                ms, used = frame_ms(k, tile)
                frames[k][key].append(ms)
                if tile == 0:
                    frames[k]["auto_tile"] = used

    # ---- (b) a load-varying queue, compact rows off and on ----
    def serve(compact):
        b = ContinuousBatcher(model, max_slots=64, frames_per_poll=8, compact_rows=compact)
        reqs, nxt, polls, tiles = [], 0, 0, {32: 0, 64: 0}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        while True:
            phase = polls // args.phase
            if phase < len(RAMP):  # top up to the phase's concurrency
                while nxt < n_req and len(b.active) + len(b.waiting) < RAMP[phase]:
                    reqs.append(b.submit(SlotRequest(prompt=prompts[nxt], max_new_tokens=lens[nxt], temperature=0.7,
                                                     top_p=0.7, top_k=1, seed=1)))
                    nxt += 1
            elif b.idle():
                break
            before = b.frames_run
            b.step()
            if b.frames_run > before:
                tiles[eng.decode_tile] += b.frames_run - before
            polls += 1
        ev1.record()
        torch.cuda.synchronize()
        occ = b.slot_frames / max(1, b.frames_run * 64)
        out = dict(ms=ev0.elapsed_time(ev1), frames_run=b.frames_run, occupancy=occ, moves=b.moves,
                   requests=len(reqs), frames_on_32=tiles[32] / max(1, b.frames_run),
                   audio_s=sum(int(r.result.shape[1] - r.prompt.shape[1]) for r in reqs) * FRAME / SR)
        b.close()
        return out, [r.result for r in reqs]

    serve(False)  # warm-up: prefill shapes and frame graphs of both settings
    serve(True)
    runs = {False: [], True: []}
    results, same = None, True
    for _ in range(args.reps):
        for compact in (False, True):  # A B A B
            r, toks = serve(compact)
            runs[compact].append(r)
            if results is None:
                results = toks
            same &= len(toks) == len(results) and all(torch.equal(a, b) for a, b in zip(results, toks))

    out = {"workload": "one 64-slot engine, S2-Pro geometry, synthetic weights, greedy, LM stage only",
           "card": card(), "identical_tokens": bool(same),
           "ms_per_frame_by_live_rows": {str(k): frames[k] for k in LIVE},
           "queue": f"{runs[False][0]['requests']} requests, concurrency ramp {list(RAMP)} ({args.phase} polls of 8 "
                    f"frames per step), {T_PROMPT}-token prompts, 64..256 frames each"}
    for compact, key in ((False, "compact_off"), (True, "compact_on")):
        rs = runs[compact]
        out[key] = {
            "audio_s_per_s": [r["audio_s"] / (r["ms"] / 1e3) for r in rs],
            "mean_frame_ms": [r["ms"] / r["frames_run"] for r in rs],
            "frames_run": rs[0]["frames_run"], "occupancy": rs[0]["occupancy"],
            "moves_per_request": rs[0]["moves"] / rs[0]["requests"],
            "frames_on_32_row_tile": rs[0]["frames_on_32"],
        }
    best = {k: max(out[k]["audio_s_per_s"]) for k in ("compact_off", "compact_on")}
    out["speedup_compact"] = best["compact_on"] / best["compact_off"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
