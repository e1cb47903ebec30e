"""What one long context costs the other slots of a decode frame, with the split decode attention off and on.

S2-Pro geometry with synthetic weights, LM stage only, two 64-slot engines of 32 768 positions per slot over the same
weights: attn_split = 0 and attn_split = `--split`. Three parts, one JSON line:

1. frame time. Slots sit at about 256 positions (256 + 3 i mod 64); 0, 1 or 4 of them at 8 192, 16 384 or 32 000
   instead; and one slot alone at those lengths. The state is written directly (positions, page table, a semantic
   token per slot; the K/V pages hold zeros, the kernels read them all the same), every shape is warmed up (graph
   capture included), then `--frames` graph-replayed frames are timed with device events, off and on alternated
   (A B A B, `--reps` each). ms per frame = window / frames.
2. the attention kernels' share of a frame: their time from `torch.profiler` over `--profile-frames` frames launched
   one by one, a run of its own, 64 slots with one at 32 000 positions, over the frame time of part 1.
3. tokens. Six requests through `ContinuousBatcher` on each engine, one of them with an 8 192-row prompt: requests
   whose context stays at or below the split length must return the same tokens from both engines, and the long one
   with the split on must equal `generate` of it alone with the split on.

    python tools/serve_longctx.py [--split 2048] [--frames 200] [--reps 2]

Reads the card's name, power limit and clocks; changes no device setting.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402

SLOTS = 64
KV_LEN = 32768
LONG = (8192, 16384, 32000)
ATTN_KERNELS = ("attn_decode_kernel", "attn_decode_split_kernel", "attn_span_kernel", "attn_combine_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--split", type=int, default=2048)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=8)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--profile-frames", type=int, default=4)
    args = ap.parse_args()

    from fish_speech_b200 import _lib, synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, S2PRO_TEXT_VOCAB, s2pro_args
    from fish_speech_b200.engine import kv_pages_for
    from fish_speech_b200.models.text2semantic.inference import generate, kv_page_bytes
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    if not torch.cuda.is_available():
        raise SystemExit("serve_longctx.py measures on the GPU; there is none")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = s2pro_args(max_seq_len=KV_LEN)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    span = args.frames + args.warmup + 1  # positions a timed run advances
    pages = 4 * kv_pages_for(max(LONG) + span) + SLOTS * kv_pages_for(256 + 64 + span) + 8

    def model(split, slots=SLOTS, kv_pages=pages):
        m = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        m.max_rows = 4096
        m.setup_caches(max_batch_size=slots, max_seq_len=KV_LEN, kv_pages=kv_pages, attn_split=split)
        return m

    models = {"off": model(0), "on": model(args.split)}
    lib = _lib.lib()
    stream = lambda: torch.cuda.current_stream().cuda_stream  # noqa: E731

    def place(eng, pos):
        """Slots [0, len(pos)) at the given positions, pages mapped for the frames of one run."""
        for s in range(SLOTS):
            eng.kv_pool.release(s)
        eng._covered.clear()
        eng._reserve([(s, p + span, 0) for s, p in enumerate(pos)])
        eng.buffer("pos")[: len(pos)].copy_(torch.tensor(pos, dtype=torch.int32))
        eng.buffer("cur_tok").zero_()
        eng.buffer("cur_tok")[:, 0] = cfg.semantic_begin_id + 7
        for name in ("n_out", "finished", "ras_window"):
            eng.buffer(name).zero_()
        eng.set_context_bound_exact(max(pos) + span)

    def frames(eng, batch, n, sp, graph=True):
        _lib.check(lib.fsb_lm_decode(eng.h, batch, n, C.byref(sp), int(graph), stream()))

    def timed(eng, pos, sp):
        place(eng, pos)
        frames(eng, len(pos), args.warmup, sp)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        frames(eng, len(pos), args.frames, sp)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.frames

    short = [256 + (3 * i) % 64 for i in range(SLOTS)]
    scenarios = [("64 slots at ~256", short)]
    for L in LONG:
        for n_long in (1, 4):
            pos = list(short)
            for j in range(n_long):
                pos[5 + 16 * j] = L - 1
            scenarios.append((f"64 slots, {n_long} at {L}", pos))
    scenarios += [(f"1 slot at {L}", [L - 1]) for L in LONG]
    sps = {k: m.engine.sampling(0.7, 0.7, 1, 1) for k, m in models.items()}
    for _, pos in scenarios:  # warm-up of every shape on both engines
        for k, m in models.items():
            place(m.engine, pos)
            frames(m.engine, len(pos), 2, sps[k])
    torch.cuda.synchronize()
    frame_ms = {}
    for name, pos in scenarios:
        runs = {"off": [], "on": []}
        for _ in range(args.reps):
            for k, m in models.items():  # A B A B
                runs[k].append(round(timed(m.engine, pos, sps[k]), 4))
        frame_ms[name] = runs

    # ---- 2. share of the attention kernels (profiler run of its own) --------------------------------------------------
    from torch.profiler import ProfilerActivity, profile

    pos = scenarios[5][1]  # 64 slots, 1 at 32 000
    share = {}
    for k, m in models.items():
        place(m.engine, pos)
        frames(m.engine, SLOTS, 2, sps[k], graph=False)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            frames(m.engine, SLOTS, args.profile_frames, sps[k], graph=False)
            torch.cuda.synchronize()
        total, by = 0.0, {n: 0.0 for n in ATTN_KERNELS}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None)
            t = ev.cuda_time_total if t is None else t
            total += t
            for n in ATTN_KERNELS:
                if f"{n}<" in ev.key:
                    by[n] += t
        # Kernels are launched with programmatic dependent launch: each starts while its predecessor runs and waits
        # inside, so the durations overlap and their sum exceeds the frame. The share is taken against the timed frame.
        attn_ms = sum(by.values()) / 1e3 / args.profile_frames
        frame = sum(frame_ms[scenarios[5][0]][k]) / args.reps
        share[k] = {"scenario": scenarios[5][0],
                    "attention_ms_per_frame": {n: round(t / 1e3 / args.profile_frames, 4) for n, t in by.items() if t},
                    "sum_of_overlapping_kernel_durations_ms_per_frame": round(total / 1e3 / args.profile_frames, 4),
                    "attention_share_of_timed_frame": round(attn_ms / frame, 4)}

    # ---- 3. tokens ----------------------------------------------------------------------------------------------------
    g = torch.Generator().manual_seed(11)

    def prompt(T):
        p = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.int32)
        p[0] = torch.randint(0, S2PRO_TEXT_VOCAB, (T,), generator=g, dtype=torch.int32)
        return p

    sampled = dict(temperature=0.8, top_p=0.9, top_k=30)
    specs = [(prompt(8192), 24, 1000)] + [(prompt(20 + 31 * i), 16 + 8 * i, i) for i in range(5)]
    outs = {}
    for k, m in models.items():
        m.engine.close()
    del models
    torch.cuda.empty_cache()
    tok_pages = kv_pages_for(8192 + 64) * 2 + 64
    for k, split in (("off", 0), ("on", args.split)):
        m = model(split, slots=8, kv_pages=tok_pages)
        b = ContinuousBatcher(m, max_slots=8, frames_per_poll=8)
        reqs = [b.submit(SlotRequest(prompt=p.to(dev), max_new_tokens=n, seed=s, **sampled)) for p, n, s in specs]
        b.run()
        b.close()
        outs[k] = [r.result.cpu() for r in reqs]
        m.engine.close()
    solo = model(args.split, slots=1, kv_pages=tok_pages)
    p, n, s = specs[0]
    alone = generate(model=solo, prompt=p.to(dev), max_new_tokens=n, seed=s, **sampled).cpu()
    solo.engine.close()
    stays_short = [i for i, (p, n, _) in enumerate(specs) if p.shape[1] + n <= args.split]
    tokens = {
        "requests": [[p.shape[1], n] for p, n, _ in specs],
        "identical_tokens_short_requests": bool(all(torch.equal(outs["off"][i], outs["on"][i]) for i in stays_short)),
        "short_requests_checked": stays_short,
        "long_request_split_on_equals_generate_alone": bool(torch.equal(outs["on"][0], alone)),
        "long_request_tokens_equal_split_off": bool(torch.equal(outs["on"][0], outs["off"][0])),
    }
    print(json.dumps({
        "card": card(), "attn_split": args.split, "slots": SLOTS, "kv_len": KV_LEN, "frames_per_window": args.frames,
        "kv_pool_gb_per_engine": round(pages * kv_page_bytes(cfg) / 1e9, 2),
        "workload": "S2-Pro geometry, synthetic weights, LM stage only, greedy frames replayed from the decode graph; "
                    "ms per frame from device events, [rep 1, rep 2, ...] per setting, off and on alternated",
        "frame_ms": frame_ms, "attention_share": share, "tokens": tokens}))


if __name__ == "__main__":
    main()
