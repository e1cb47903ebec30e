"""Fused admission: what running an admitted request's first frame inside the running decode frame saves.

Without it every admission costs a prefill pass plus a frame over the new rows alone, which streams the head and all
ten fast passes' weights (8.28 of a frame's 15.55 GB at the S2-Pro geometry) and delays every running stream's next
frame. With `ContinuousBatcher(fused_admission=True)` the prefill stops after the slow stack and the new rows take their
first frame as rows of the poll's first decode frame (fish_speech_b200/scheduler.py, include/fishb200.h
fsb_lm_prefill_deferred). This tool measures it on the S2-Pro geometry with synthetic weights, on 32- and 64-slot
engines, for two seeded queues: 64-token prompts with budgets of `--lo`..`--hi` frames, and two-chunk streams of
`--slo`..`--shi` frames per chunk (each chunk's prompt extends the previous one, as tools/serve_live.py), each queue
holding `--load` x slots requests that arrive together. Fused admission runs off and on alternated (off, on, off, on)
in one process.

    python tools/serve_admit.py [--slots 32 64] [--load 2] [--reps 2]

Prints one JSON line: per engine and queue, audio seconds per second of each run, device ms of an admission step
(prefill with its first frame / prefill alone, summed over the run and per call), `identical_tokens` (every request's
tokens equal with the mode off and on); per engine, device ms of one decode frame with and without the splice node
(all rows live, CUDA events around single-frame decodes); and the card's name and power limit."""
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
    ap.add_argument("--slots", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--load", type=int, default=2, help="requests per queue, in multiples of the slot count")
    ap.add_argument("--reps", type=int, default=2, help="(off, on) pairs per queue")
    ap.add_argument("--lo", type=int, default=64)
    ap.add_argument("--hi", type=int, default=256)
    ap.add_argument("--slo", type=int, default=48)
    ap.add_argument("--shi", type=int, default=128)
    ap.add_argument("--frames", type=int, default=24, help="timed single-frame decodes per kind")
    args = ap.parse_args()

    from bench import FRAME, SR, T_PROMPT, make_prompts
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.engine import bf16_round
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    text_rows = 8
    seq = T_PROMPT + max(args.hi, 2 * (args.shi + text_rows)) + args.frames + 8
    cfg = s2pro_args(max_seq_len=seq)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are set by the budgets
    out = {"workload": f"S2-Pro geometry, synthetic weights, LM stage only, {T_PROMPT}-token prompts, sampled "
                       f"(top-k 30, top-p 0.9, temperature 0.8) and greedy requests, {args.load} x slots requests "
                       f"arriving together; fused admission off / on alternated {args.reps} times",
           "card": card(), "engines": []}
    for slots in args.slots:
        model = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        model.max_rows = slots * T_PROMPT
        model.setup_caches(max_batch_size=slots, max_seq_len=seq)
        eng = model.engine
        n = args.load * slots
        g = torch.Generator().manual_seed(17 + slots)
        budgets = torch.randint(args.lo, args.hi + 1, (n,), generator=g).tolist()
        chunks = torch.randint(args.slo, args.shi + 1, (n, 2), generator=g).tolist()
        text = torch.randint(0, 1000, (n, 2, text_rows), generator=g)
        prompts = [p.to(dev) for p in make_prompts(cfg, n, 1000 + slots)]

        timed = {"with_frame": [], "deferred": []}  # CUDA event pairs around each prefill call
        real_prefill = eng.prefill

        def prefill(*a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = real_prefill(*a, **k)
            e1.record()
            timed["deferred" if k.get("defer_first_frame") else "with_frame"].append((e0, e1))
            return r

        eng.prefill = prefill

        def sp(i):
            return dict(temperature=0.8, top_p=0.9, top_k=1 if i % 4 == 0 else 30, seed=7 + i)

        def serve(queue, fused):
            for v in timed.values():
                v.clear()
            b = ContinuousBatcher(model, max_slots=slots, frames_per_poll=8, fused_admission=fused)
            results, made = {}, {}

            def submit(i, c, prompt, budget):
                def on_done(r):
                    results[(i, c)] = r.result.cpu()
                    made[(i, c)] = r.result.shape[1] - prompt.size(1)
                    if queue == "streams" and c == 0:
                        rows = torch.zeros(prompt.size(0), text_rows, dtype=prompt.dtype, device=dev)
                        rows[0] = text[i, 1].to(dev)
                        grown = torch.cat([prompt, r.result[:, prompt.size(1):-1].to(prompt.dtype), rows], dim=1)
                        submit(i, 1, grown, chunks[i][1])

                b.submit(SlotRequest(prompt=prompt, max_new_tokens=budget, reuse_prefix=queue == "streams",
                                     on_done=on_done, **sp(i)))

            for i in range(n):
                submit(i, 0, prompts[i], budgets[i] if queue == "ragged" else chunks[i][0])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b.run()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            b.close()
            frames = sum(made.values())
            kind = "deferred" if fused else "with_frame"
            ms = [e0.elapsed_time(e1) for e0, e1 in timed[kind]]
            return results, {"fused_admission": fused, "wall_s": wall, "frames": frames,
                             "audio_s_per_s": frames * FRAME / SR / wall, "admission_steps": len(ms),
                             "admission_device_ms_total": sum(ms),
                             "admission_device_ms_per_step": sum(ms) / len(ms) if ms else None,
                             "decode_frames": b.frames_run}

        eng_out = {"slots": slots, "queues": []}
        serve("ragged", False)  # warm-up: graph capture and first touch of every buffer, both modes
        serve("ragged", True)
        for queue in ("ragged", "streams"):
            runs, ref, same = [], None, True
            for _ in range(args.reps):
                for fused in (False, True):
                    res, r = serve(queue, fused)
                    if ref is None:
                        ref = res
                    same &= res.keys() == ref.keys() and all(torch.equal(res[k], ref[k]) for k in ref)
                    runs.append(r)
            eng_out["queues"].append({"queue": queue, "requests": n, "identical_tokens": bool(same), "runs": runs})

        # one decode frame with every row live, without and with the splice node (one new request pending)
        eng.prefill = real_prefill
        eng.reset()
        eng.release_kv()
        eng.set_slot_control(True)
        idx = torch.arange(slots, device=dev)
        eng.buffer("slot_limit")[idx] = eng.max_frames
        eng.buffer("slot_temperature")[idx] = bf16_round(0.8)
        eng.buffer("slot_top_p")[idx] = bf16_round(0.9)
        eng.buffer("slot_top_k")[idx] = 30
        eng.buffer("slot_seed")[idx] = idx.to(torch.int64) + 1
        eng.buffer("slot_state")[idx] = 1
        end = T_PROMPT + 2 * args.frames + 8
        eng.prefill(prompts[:slots], list(range(slots)), None, kv_end=[end] * slots)
        eng.set_context_bound_exact(end + 1)
        eng.decode(slots, 2, None)
        plain, fused = [], []
        for i in range(args.frames + 2):
            s = (7 * i) % slots  # this slot's request is replaced by a new one whose first frame is fused
            eng.buffer("n_out")[s] = 0
            eng.buffer("ras_window")[s] = 0
            eng.buffer("slot_state")[s] = 1
            eng.prefill([prompts[s]], [s], None, kv_end=[end], defer_first_frame=True)
            for kind in (fused, plain):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                eng.decode(slots, 1, None)
                e1.record()
                kind.append((e0, e1))
        torch.cuda.synchronize()
        ms = lambda ev: sorted(e0.elapsed_time(e1) for e0, e1 in ev[2:])  # the first two capture graphs
        med = lambda xs: xs[len(xs) // 2]
        eng_out["frame_ms"] = {"plain_median": med(ms(plain)), "with_splice_median": med(ms(fused)),
                               "plain_min": ms(plain)[0], "with_splice_min": ms(fused)[0], "frames": args.frames}
        out["engines"].append(eng_out)
        eng.close()
        del model, eng
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
