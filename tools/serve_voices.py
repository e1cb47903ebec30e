"""Prefix cache: what keeping voice prefixes in the KV page pool saves a voice-clone serving mix.

A voice-clone request's prompt starts with a system message holding the reference text and codes, identical for every
request with that voice. Without the cache a prefix is reused only while some slot still holds it; with
`setup_caches(prefix_cache=True)` the prompt pages of a finished request stay in the pool until a reservation needs
them (fish_speech_b200/engine.py KvPagePool.insert / lookup). This tool measures it on the S2-Pro geometry with
synthetic weights (<|im_end|> zeroed, so budgets set the lengths), on a 64-slot engine with a bounded pool of `--pool-gb`
GB: `--voices` voices with prefixes of 512..768 rows, each request picking one by a seeded Zipf(1.1), with a tail of
32..96 rows of its own and a budget of 64..256 frames; `--requests` requests arrive together. Cache off and on run
alternated (off, on, off, on) on two engines built alike, in one process, and every request's tokens must be equal.

    python tools/serve_voices.py [--voices 32 128] [--requests 256] [--reps 2] [--pool-gb 16]

Prints one JSON line: the card's name and power limit; per voice count and run: audio seconds per second, prefill
device ms (CUDA events around every prefill call), rows prefilled and reused, cache hits per request and evictions,
host ms per admission of the prefix search and cache insertion, p50 / p99 time to first frames (from the arrival of
the queue to a request's first frames handed out), and `identical_tokens`."""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--voices", type=int, nargs="+", default=[32, 128])
    ap.add_argument("--requests", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2, help="(off, on) pairs per voice count")
    ap.add_argument("--slots", type=int, default=64)
    ap.add_argument("--pool-gb", type=float, default=16.0)
    args = ap.parse_args()

    from bench import FRAME, SR
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.models.text2semantic.inference import kv_page_bytes
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    seq = 768 + 96 + 256 + 8
    cfg = s2pro_args(max_seq_len=seq)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are set by the budgets
    pages = int(args.pool_gb * 1e9 // kv_page_bytes(cfg))
    models = {}
    for cache in (False, True):
        m = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        m.max_rows = 4096
        m.setup_caches(max_batch_size=args.slots, max_seq_len=seq, kv_pages=pages, prefix_cache=cache)
        models[cache] = m
    out = {"workload": f"S2-Pro geometry, synthetic weights, LM stage only, {args.slots} slots, a pool of {pages} KV "
                       f"pages ({args.pool_gb} GB), {args.requests} requests arriving together, voices by Zipf(1.1) with "
                       f"512-768-row prefixes, 32-96-row tails, 64-256-frame budgets, sampled (top-k 30, top-p 0.9, "
                       f"temperature 0.8); cache off / on alternated {args.reps} times",
           "card": card(), "runs": []}

    def queue(n_voices, n, seed):
        g = torch.Generator().manual_seed(seed)
        lens = torch.randint(512, 769, (n_voices,), generator=g).tolist()
        voices = [torch.randint(0, 151643, (ln,), generator=g, dtype=torch.int32) for ln in lens]
        weights = torch.tensor([1.0 / (k + 1) ** 1.1 for k in range(n_voices)])
        picks = torch.multinomial(weights, n, replacement=True, generator=g).tolist()
        reqs = []
        for i, v in enumerate(picks):
            tail = torch.randint(0, 151643, (int(torch.randint(32, 97, (1,), generator=g)),), generator=g,
                                 dtype=torch.int32)
            p = torch.zeros(cfg.num_codebooks + 1, len(voices[v]) + len(tail), dtype=torch.int32)
            p[0] = torch.cat([voices[v], tail])
            reqs.append((p.to(dev), int(torch.randint(64, 257, (1,), generator=g)), 7 + i))
        return reqs

    def serve(cache, reqs):
        model = models[cache]
        eng = model.engine
        timed, host = [], [0.0]
        real_prefill, real_donor, real_insert = eng.prefill, eng._donor, eng.kv_pool.insert

        def prefill(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = real_prefill(*a, **k)
            e1.record()
            timed.append((e0, e1))
            return r

        def timed_host(fn):
            def call(*a, **k):
                t = time.perf_counter()
                r = fn(*a, **k)
                host[0] += time.perf_counter() - t
                return r
            return call

        eng.prefill, eng._donor, eng.kv_pool.insert = prefill, timed_host(real_donor), timed_host(real_insert)
        b = ContinuousBatcher(model, max_slots=args.slots, frames_per_poll=8)
        rows0 = (eng.rows_prefilled, eng.rows_reused, eng.prefix_hits, eng.prefix_evictions)
        results, first = {}, {}
        t0 = [0.0]

        def on_frames(r, codes):
            first.setdefault(r.tag, time.perf_counter() - t0[0])

        for i, (p, n, seed) in enumerate(reqs):
            b.submit(SlotRequest(prompt=p, max_new_tokens=n, temperature=0.8, top_p=0.9, top_k=30, seed=seed,
                                 reuse_prefix=True, tag=i, on_frames=on_frames,
                                 on_done=lambda r: results.__setitem__(r.tag, r.result)))
        torch.cuda.synchronize()
        t0[0] = time.perf_counter()
        b.run()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0[0]
        b.close()
        eng.prefill, eng._donor, eng.kv_pool.insert = real_prefill, real_donor, real_insert
        frames = sum(int(r.shape[1]) - int(p.shape[1]) for (p, _, _), r in zip(reqs, [results[i] for i in
                                                                                      range(len(reqs))]))
        ttff = sorted(first.values())
        pct = lambda q: ttff[min(len(ttff) - 1, int(q * len(ttff)))] * 1e3
        d = [a - b_ for a, b_ in zip((eng.rows_prefilled, eng.rows_reused, eng.prefix_hits, eng.prefix_evictions),
                                     rows0)]
        return {k: v.cpu() for k, v in results.items()}, {
            "prefix_cache": cache, "wall_s": wall, "frames": frames, "audio_s_per_s": frames * FRAME / SR / wall,
            "prefill_device_ms": sum(e0.elapsed_time(e1) for e0, e1 in timed), "prefill_calls": len(timed),
            "rows_prefilled": d[0], "rows_reused": d[1], "hit_rate": d[2] / len(reqs), "evictions": d[3],
            "host_ms_per_admission": host[0] * 1e3 / len(reqs), "ttff_ms_p50": pct(0.5), "ttff_ms_p99": pct(0.99)}

    warm = queue(8, 2 * args.slots, 1)
    for cache in (False, True):  # graph capture and first touch of every buffer, both engines
        serve(cache, warm)
    for n_voices in args.voices:
        reqs = queue(n_voices, args.requests, 100 + n_voices)
        ref, same, runs = None, True, []
        for _ in range(args.reps):
            for cache in (False, True):
                res, r = serve(cache, reqs)
                if ref is None:
                    ref = res
                same &= res.keys() == ref.keys() and all(torch.equal(res[k], ref[k]) for k in ref)
                runs.append(r)
        out["runs"].append({"voices": n_voices, "requests": len(reqs), "identical_tokens": bool(same), "runs": runs})
        assert same, f"{n_voices} voices: tokens differ between cache off and on"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
