"""Streaming serving at 32 and 64 concurrent requests: per-request codec streams against the shared stream pool.

N streaming requests (S2-Pro geometry, synthetic weights, 64-token prompts, seeded ragged lengths of 64..256 frames,
greedy) run through `ContinuousBatcher` (N slots, frames_per_poll 8). Every poll hands each request its finished frames
(`on_frames`); a codec thread decodes them on a CUDA stream of its own while the LM keeps decoding:

  (a) per_request: one `DecodeStream` per request, pushed one request after another (what TTSInferenceEngine does
      without FSB_STREAM_POOL: pushes of different requests serialise on the codec);
  (b) pool: one `DecodeStreamPool` of N slots behind `CodecStreamWorker` (FSB_STREAM_POOL): everything queued is
      decoded in one push.

The two alternate A B A B after one warm-up run each (graph capture). Frames left when a request finishes are pushed
then (the last frame of a request is never part of its audio, as in generate_long). Reported per configuration: audio-s/s (all requests' audio over the wall time until the last sample is ready),
codec stream-elapsed ms per LM poll (the time between CUDA events recorded around every codec push on the codec's
stream: it includes host launch gaps inside a push and time the GPU spends on the concurrently running LM, so it is an
upper bound of the codec's own kernel time), p50 / p95 time to first audio, p95 gap between two segments of a request, device memory of the codec
state; and `identical_audio`: every request's audio equal across (a), (b) and `from_indices` of its codes.

    python tools/serve_stream.py [--streams 32 64] [--reps 2]

Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import queue
import sys
import threading
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def pct(xs, q):
    return float(np.percentile(np.asarray(xs, dtype=np.float64), q)) if xs else None


class _Timed:
    """CUDA events around every call of `fn` on the current stream; total stream-elapsed ms read after a run."""

    def __init__(self, fn):
        self.fn, self.events = fn, []

    def __call__(self, *a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = self.fn(*a, **k)
        e1.record()
        self.events.append((e0, e1))
        return out

    def ms(self):
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.events)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[32, 64])
    ap.add_argument("--reps", type=int, default=2, help="alternated timed runs per configuration")
    args = ap.parse_args()

    from bench import FRAME, SR, T_PROMPT, make_prompts
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.inference_engine import CodecStreamWorker
    from fish_speech_b200.models.dac.inference import load_codec_config
    from fish_speech_b200.models.dac.modded_dac import DAC
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest
    from tools.step_gemm_boundaries import card

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n_max = max(args.streams)
    cfg = s2pro_args(max_seq_len=T_PROMPT + 256)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0  # lengths are set by the per-request budgets
    lm = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
    lm.max_rows = n_max * T_PROMPT
    lm.setup_caches(max_batch_size=n_max, max_seq_len=cfg.max_seq_len)
    del w
    ccfg = load_codec_config("modded_dac_vq")
    dac = DAC(ccfg, synthetic.codec_state_dict(ccfg, dev), device=dev)
    g = torch.Generator().manual_seed(11)
    lens = torch.randint(64, 257, (n_max,), generator=g).tolist()
    prompts = [p.to(dev) for p in make_prompts(cfg, n_max, 42)]
    pools = {n: dac.open_stream_pool(n, k_max=32) for n in args.streams}

    def serve(n, mode):
        """One run of n concurrent streaming requests; returns metrics and each request's audio."""
        b = ContinuousBatcher(lm, max_slots=n, frames_per_poll=8)
        polls = [0]
        step = b.step

        def counted_step():
            polls[0] += 1
            return step()

        b.step = counted_step
        t0 = [0.0]
        seg_t = [[] for _ in range(n)]
        audio = [[] for _ in range(n)]
        delivered = [0] * n
        lock = threading.Lock()

        def got(i, wav):
            with lock:
                seg_t[i].append(time.perf_counter() - t0[0])
                audio[i].append(wav)

        if mode == "pool":
            pool = pools[n]
            timed = _Timed(pool.push)
            pool.push = timed
            worker = CodecStreamWorker(pool, dev)
            slot = [worker.open() for _ in range(n)]
            futs = []

            def feed(i, codes):
                for a in range(0, codes.shape[-1], worker.k_max):
                    f = worker.submit(slot[i], codes[:, a: a + worker.k_max])
                    futs.append(f)
                    f.add_done_callback(lambda f, i=i: got(i, f.result()))
            state_bytes = pool.state_bytes
        else:
            streams = [dac.open_decode_stream(batch=1) for _ in range(n)]
            timed = _Timed(lambda st, c: st.push(c))
            q: queue.Queue = queue.Queue()

            def codec_thread():
                side = torch.cuda.Stream(device=dev)
                with torch.cuda.stream(side):
                    while True:
                        item = q.get()
                        if item is None:
                            return
                        i, codes = item
                        got(i, timed(streams[i], codes[None])[0, 0].float().cpu().numpy())

            th = threading.Thread(target=codec_thread, daemon=True)
            th.start()

            def feed(i, codes):
                q.put((i, codes))
            state_bytes = sum(k.numel() * k.element_size() * 2 for s in streams for k, _ in s.kv)

        def on_frames(req, codes):
            i = req.tag
            delivered[i] += codes.shape[-1]
            feed(i, codes)

        reqs = [b.submit(SlotRequest(prompt=p, max_new_tokens=k, temperature=0.7, top_p=0.7, top_k=1, seed=1,
                                     on_frames=on_frames, tag=i))
                for i, (p, k) in enumerate(zip(prompts[:n], lens[:n]))]
        torch.cuda.synchronize()
        t0[0] = time.perf_counter()
        b.run()
        codes_all = []
        for i, r in enumerate(reqs):
            codes = r.result[1:, T_PROMPT: r.result.shape[1] - 1].cpu()  # the last frame is never kept (scheduler.py)
            codes_all.append(codes)
            if delivered[i] < codes.shape[-1]:  # frames the last poll did not hand out
                feed(i, codes[:, delivered[i]:])
                delivered[i] = codes.shape[-1]
        if mode == "pool":
            for f in list(futs):
                f.result()
            for s in slot:
                worker.release(s)
            worker.close()
            pool.push = timed.fn
        else:
            q.put(None)
            th.join()
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0[0]
        b.close()
        with lock:
            wavs = [np.concatenate(a) if a else np.zeros(0, np.float32) for a in audio]
            ttfa = [t[0] for t in seg_t if t]
            gaps = [y - x for t in seg_t for x, y in zip(t, t[1:])]
        frames = sum(c.shape[-1] for c in codes_all)
        return {
            "audio_s_per_s": frames * FRAME / SR / wall, "wall_s": wall, "lm_polls": polls[0],
            "codec_stream_ms_per_poll": timed.ms() / max(1, polls[0]), "codec_pushes": len(timed.events),
            "ttfa_p50_s": pct(ttfa, 50), "ttfa_p95_s": pct(ttfa, 95), "gap_p95_s": pct(gaps, 95),
            "codec_state_mb": state_bytes / 2 ** 20,
        }, wavs, codes_all

    out = {"workload": "serve_stream: N concurrent streaming requests, 64-token prompts, 64..256 frames each (seeded), "
                       "greedy, frames_per_poll 8, S2-Pro LM + codec geometry, synthetic weights",
           "card": card(), "lengths_mean": sum(lens) / len(lens)}
    identical = True
    for n in args.streams:
        for mode in ("per_request", "pool"):  # warm-up: graph capture, plan caches, first touch
            serve(n, mode)
        runs = {"per_request": [], "pool": []}
        ref = None
        for _ in range(args.reps):
            for mode in ("per_request", "pool"):  # A B A B
                m, wavs, codes = serve(n, mode)
                runs[mode].append(m)
                if ref is None:
                    ref = (wavs, codes)
                    for wv, c in zip(wavs, codes):
                        one = dac.from_indices(c[None].clone().to(dev))[0, 0].cpu().numpy()
                        identical &= np.array_equal(wv, one)
                else:
                    identical &= all(np.array_equal(a, b) for a, b in zip(ref[0], wavs))
                    identical &= all(torch.equal(a, b) for a, b in zip(ref[1], codes))
        out[f"streams_{n}"] = {mode: {k: [r[k] for r in rs] if k not in ("codec_state_mb",) else rs[0][k]
                                      for k in rs[0]} for mode, rs in runs.items()}
        best = {mode: min(r["codec_stream_ms_per_poll"] for r in rs) for mode, rs in runs.items()}
        out[f"streams_{n}"]["codec_stream_ms_per_poll_ratio_pool_over_per_request"] = best["pool"] / best["per_request"]
    out["identical_audio"] = bool(identical)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
