"""Serving with KV growth: reserve-at-admission against pages taken as requests decode (ContinuousBatcher kv_growth).

One seeded queue, S2-Pro geometry with synthetic weights, LM stage only, 64 slots: `--requests` requests that share a
384-row prefix (system + reference audio) plus a 64-row unique tail, `reuse_prefix=True`, greedy, each with a declared
budget of 1024 frames (`max_new_tokens`, ServeTTSRequest's default) and an actual length drawn from 64..1024 frames.
The actual length is written into the device-side `slot_limit` after admission, while the host's page accounting keeps
the declared budget: a request then ends before its budget as one that samples <|im_end|> would.

For each pool size (`--pool-gb`, GB of KV pages) the two policies run alternately, A B A B (`--reps` pairs), on the
same engine. Per run: audio-s/s, mean and peak running requests, peak pages in use, parks for pages per request and the
longest wait of a request parked for pages; `identical_tokens` is true when every run returned the same tokens.

    python tools/serve_grow.py [--requests 64] [--reps 2] [--pool-gb 3 6]

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
BUDGET = 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--requests", type=int, default=64)
    ap.add_argument("--reps", type=int, default=2, help="alternated (reserve, grow) pairs per pool size")
    ap.add_argument("--pool-gb", type=float, nargs="+", default=[3.0, 6.0])
    args = ap.parse_args()

    from bench import FRAME, SR
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, S2PRO_TEXT_VOCAB, s2pro_args
    from fish_speech_b200.models.text2semantic.inference import kv_page_bytes
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    class Batcher(ContinuousBatcher):
        """Writes each request's actual length (its `tag`) into slot_limit once it is admitted."""

        def _admit(self, order=None):
            before = set(self.active)
            super()._admit(order)
            for s in set(self.active) - before:
                self._limit[s] = self.active[s].tag

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(11)

    def prompt(cfg, T):
        p = torch.zeros(cfg.num_codebooks + 1, T, dtype=torch.int32)
        p[0] = torch.randint(0, S2PRO_TEXT_VOCAB, (T,), generator=g, dtype=torch.int32)
        return p

    cfg = s2pro_args(max_seq_len=(PREFIX + TAIL + BUDGET + 63) // 64 * 64)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are the drawn ones
    page_b = kv_page_bytes(cfg)
    lengths = torch.randint(64, BUDGET + 1, (args.requests,), generator=g).tolist()
    prefix = prompt(cfg, PREFIX)
    specs = [(torch.cat([prefix, prompt(cfg, TAIL)], dim=1), n) for n in lengths]
    greedy = dict(temperature=0.7, top_p=0.7, top_k=1, seed=1)

    def serve(m, specs, grow):
        b = Batcher(m, max_slots=SLOTS, frames_per_poll=8, kv_growth=grow)
        assert b.kv_growth == grow
        reqs = [b.submit(SlotRequest(prompt=p.to(dev), max_new_tokens=BUDGET, reuse_prefix=True, tag=n, **greedy))
                for p, n in specs]
        pool = m.engine.kv_pool
        pool.peak = 0
        running = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        while not b.idle():
            b.step()
            running.append(len(b.active))
        torch.cuda.synchronize()
        s = time.perf_counter() - t0
        assert not grow or not m.engine.buffer("kv_miss").any()
        b.close()
        out = [r.result.cpu() for r in reqs]
        assert all(o.shape[1] == p.shape[1] + n for o, (p, n) in zip(out, specs))
        return out, {"audio_s_per_s": sum(lengths[:len(specs)]) * FRAME / SR / s, "s": s,
                     "mean_running": sum(running) / len(running), "peak_running": max(running),
                     "peak_pages": pool.peak, "page_parks_per_request": sum(r.page_parks for r in reqs) / len(reqs),
                     "longest_page_wait_s": max(r.page_wait for r in reqs)}

    result = {"card": card(), "page_bytes": page_b, "worst_case_pages": -(-(PREFIX + TAIL + BUDGET) // 64),
              "workload": f"{args.requests} requests, {PREFIX}-row shared prefix + {TAIL}-row unique tail, budget "
                          f"{BUDGET} frames, actual 64..{BUDGET} (mean {sum(lengths) / len(lengths):.0f}), greedy, "
                          f"reuse_prefix, {SLOTS} slots, S2-Pro geometry, synthetic weights, LM stage only",
              "pools": {}}
    first, same = None, True
    for gb in args.pool_gb:
        pages = int(gb * 1e9 // page_b)
        m = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        m.max_rows = SLOTS * (PREFIX + TAIL)
        m.setup_caches(max_batch_size=SLOTS, max_seq_len=cfg.max_seq_len, kv_pages=pages)
        for grow in (False, True):  # warm-up: graph capture, first touch of every buffer
            serve(m, specs[: SLOTS // 4], grow)
        runs = {"reserve": [], "grow": []}
        for _ in range(args.reps):
            for grow in (False, True):  # A B A B
                out, r = serve(m, specs, grow)
                runs["grow" if grow else "reserve"].append(r)
                print(f"{gb:g} GB {'grow' if grow else 'reserve'}: {r}", file=sys.stderr, flush=True)
                first = first or out
                same &= all(torch.equal(a, b) for a, b in zip(first, out))
        result["pools"][f"{gb:g}GB"] = {"kv_pages": pages, "runs": runs}
        m.engine.close()
        del m
    result["identical_tokens"] = bool(same)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
