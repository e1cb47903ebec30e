"""Serving with the paged slow KV cache: what a 64-slot engine gains from one shared page pool.

Two seeded workloads, S2-Pro geometry with synthetic weights, LM stage only, 64 slots, `ContinuousBatcher`:

1. voice-clone queue: `--requests` requests that share a 384-row prefix (system + reference audio) plus a 64-row
   unique tail, budgets of 64..1024 frames, greedy, `reuse_prefix=True`. Run with the default pool (every slot at full
   capacity) and with a pool of `--pool-gb` GB, alternating A B per rep. Reports audio-s/s, the peak of pages in use,
   KV GB in use at that peak, and `identical_tokens` (every request returned the same tokens in every run).
2. long tail: per-sequence capacity 32 768 positions with a pool of `--tail-gb` GB, 60 short requests and 4 with
   8k..12k-row prompts. Reports the wall time, the pool's peak, and whether sampled requests equal `generate` alone;
   a contiguous cache of 64 x 32 768 positions would need 309 GB.

    python tools/serve_paged.py [--requests 256] [--reps 1] [--pool-gb 4] [--tail-gb 24]

Prints one JSON line with the card's name and power limit.
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

SLOTS = 64
PREFIX, TAIL = 384, 64


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--reps", type=int, default=1, help="alternated timed runs per pool size")
    ap.add_argument("--pool-gb", type=float, default=4.0)
    ap.add_argument("--tail-gb", type=float, default=24.0)
    args = ap.parse_args()

    from bench import FRAME, SR
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, S2PRO_TEXT_VOCAB, s2pro_args
    from fish_speech_b200.models.text2semantic.inference import generate, kv_page_bytes, slow_kv_bytes_per_position
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(11)

    def prompt(cfg, T, gen=g):
        p = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.int32)
        p[0] = torch.randint(0, S2PRO_TEXT_VOCAB, (T,), generator=gen, dtype=torch.int32)
        return p

    def model(cfg, w, slots, kv_pages=None, max_rows=2048):
        m = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        m.max_rows = max_rows
        m.setup_caches(max_batch_size=slots, max_seq_len=cfg.max_seq_len, kv_pages=kv_pages)
        return m

    def serve(m, specs, **kw):
        b = ContinuousBatcher(m, max_slots=SLOTS, frames_per_poll=8)
        reqs = [b.submit(SlotRequest(prompt=p.to(dev), max_new_tokens=n, **kw, **extra)) for p, n, extra in specs]
        pool = m.engine.kv_pool
        pool.peak = 0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b.run()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        b.close()
        return ms, [r.result.cpu() for r in reqs], pool.peak

    # ---- 1. voice-clone queue --------------------------------------------------------------------------------------
    budgets = torch.randint(64, 1025, (args.requests,), generator=g).tolist()
    cfg = s2pro_args(max_seq_len=(PREFIX + TAIL + 1024 + 63) // 64 * 64)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are set by the per-request budgets
    page_b = kv_page_bytes(cfg)
    prefix = prompt(cfg, PREFIX)
    specs = [(torch.cat([prefix, prompt(cfg, TAIL)], dim=1), n, dict(reuse_prefix=True)) for n in budgets]
    pools = {"default": None, f"{args.pool_gb:g}GB": int(args.pool_gb * 1e9 // page_b)}
    models = {k: model(cfg, w, SLOTS, v, max_rows=SLOTS * (PREFIX + TAIL)) for k, v in pools.items()}
    greedy = dict(temperature=0.7, top_p=0.7, top_k=1, seed=1)
    for k in pools:  # warm-up: graph capture, first touch of every buffer
        serve(models[k], specs[: 2 * SLOTS // 8], **greedy)
    audio_s = sum(budgets) * FRAME / SR
    runs = {k: [] for k in pools}
    first, same = None, True
    for _ in range(args.reps):
        for k in pools:  # A B A B
            ms, out, peak = serve(models[k], specs, **greedy)
            runs[k].append({"audio_s_per_s": audio_s / (ms / 1e3), "ms": ms, "peak_pages": peak,
                            "kv_gb_in_use": peak * page_b / 1e9})
            first = first or out
            same &= all(torch.equal(a, b) for a, b in zip(first, out))
    result = {"card": card(), "page_bytes": page_b}
    result["voice_clone"] = {
        "workload": f"{args.requests} requests, {PREFIX}-row shared prefix + {TAIL}-row unique tail, 64..1024 frames "
                    f"(mean {sum(budgets) / len(budgets):.0f}), greedy, reuse_prefix, {SLOTS} slots, S2-Pro geometry, "
                    "synthetic weights, LM stage only",
        "pools": {k: {"kv_pages": models[k].engine.kv_pool.n_pages,
                      "pool_gb": models[k].engine.kv_pool.n_pages * page_b / 1e9, "runs": runs[k]} for k in pools},
        "identical_tokens": bool(same), "audio_s": audio_s,
    }
    for m in models.values():
        m.engine.close()
    del models, w

    # ---- 2. long tail ------------------------------------------------------------------------------------------------
    cfg = s2pro_args(max_seq_len=32768)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    pages = int(args.tail_gb * 1e9 // kv_page_bytes(cfg))
    m = model(cfg, w, SLOTS, pages, max_rows=4096)
    sampled = dict(temperature=0.8, top_p=0.9, top_k=30)
    long_T = [8192, 9500, 10800, 12000]
    specs = [(prompt(cfg, 16 + (7 * i) % 100), 64 + (29 * i) % 192, dict(seed=i)) for i in range(60)]
    specs[5:5] = [(prompt(cfg, T), 96, dict(seed=1000 + j)) for j, T in enumerate(long_T)]
    ms, out, peak = serve(m, specs, **sampled)
    m.engine.close()
    solo = model(cfg, w, 1)
    checked = [5, 6, 7, 8, 0, 30, 63]
    equal = []
    for i in checked:
        p, n, extra = specs[i]
        one = generate(model=solo, prompt=p.to(dev), max_new_tokens=n, **sampled, **extra).cpu()
        equal.append(bool(torch.equal(one, out[i])))
    result["long_tail"] = {
        "workload": f"60 requests of 16..115 prompt rows and 64..255 frames plus 4 with {long_T} prompt rows and 96 "
                    f"frames, sampled, {SLOTS} slots of 32768 positions, S2-Pro geometry, synthetic weights",
        "kv_pages": pages, "pool_gb": pages * kv_page_bytes(cfg) / 1e9, "ms": ms, "peak_pages": peak,
        "kv_gb_in_use": peak * kv_page_bytes(cfg) / 1e9, "completed": len(out) == len(specs),
        "checked_requests": checked, "identical_to_generate_alone": equal,
        "contiguous_64x32768_gb": SLOTS * 32768 * slow_kv_bytes_per_position(cfg) / 1e9,
    }
    print(json.dumps(result))


if __name__ == "__main__":
    main()
