"""ORACLE — TEST / MEASUREMENT INFRASTRUCTURE ONLY (never imported by the product path).

The reference's own CPU implementation of the hot path, timed on the box's host cores for bench.py's
`--impl reference` arm and its `cpu_baseline` object.

What is timed is the oracle restatement of the reference (oracle/lm_oracle.py, oracle/codec_oracle.py; kind
"port"), pinned bit-exact to the reference by oracle/make_golden*.py: `decode_one_token_ar` for the prefill and for
every decode frame (inference.py:96-181, called the way `generate` / `decode_n_tokens` call it, :184-238, :322-352)
and `DAC.from_indices` (modded_dac.py:925-946).

Workload = bench.py's (batch-32 text->codec->wav, 64-token prompts, 256 frames per utterance, S2-Pro 4B +
391 M codec geometry, greedy). The reference is a batch-1 implementation (`max_batch_size=1`, inference.py:285),
so the job is 32 utterances one after another and the throughput of one utterance is the throughput of the job.
One utterance costs  t_prefill + 255 * t_frame + t_codec(256 frames).  A full utterance is ~2.5 minutes of CPU
work, so each measured step is a BOUNDED SAMPLE — `frames_per_step` decode frames at the live context plus a
codec decode of `codec_frames_per_step` frames — and the line reports the explicit extrapolation

    audio-s/s = 256 * 2048 / 44100 / (t_prefill + 255 * mean(t_frame) + mean(t_codec) * 256 / codec_frames_per_step)

with every term in `sample`.  Weights: synthetic at the real sizes; every layer has ITS OWN storage (cloned
values: timing does not depend on the values, and nothing is aliased in memory: 9.1 GB of bf16 LM weights are
streamed per frame exactly as with a real checkpoint).
"""
from __future__ import annotations

import os
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import codec_oracle as CO  # noqa: E402
from oracle import lm_oracle as O  # noqa: E402

SR, FRAME = 44100, 2048
T_PROMPT, N_FRAMES = 64, 256


def usable_cores() -> int:
    """Host cores this process can really use: the affinity mask capped by the cgroup CPU quota (GPU boxes
    expose 100+ hardware threads but a 16-core quota; an oversized OpenMP team thrashes)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = max(1, min(n, int(int(q) / int(p))))
    except Exception:
        pass
    return n


def _lm_weights(cfg: O.LMConfig) -> dict:
    one = O.LMConfig(max_seq_len=cfg.max_seq_len, n_layer=1, n_fast_layer=1)
    w1 = O.make_weights(one, seed=1234, head_gain=4.0)
    w = dict(w1)
    for l in range(1, cfg.n_layer):
        for k, v in w1.items():
            if k.startswith("layers.0."):
                w[k.replace("layers.0.", f"layers.{l}.")] = v.clone()  # own storage: nothing aliased
    for l in range(1, cfg.n_fast_layer):
        for k, v in w1.items():
            if k.startswith("fast_layers.0."):
                w[k.replace("fast_layers.0.", f"fast_layers.{l}.")] = v.clone()
    # fixed-length workload (SURVEY §8(d): "<|im_end|> bias set to -inf"): a zero head row never wins
    w["embeddings.weight"][cfg.im_end_id] = 0
    return w


class CpuHotPath:
    """prefill() / frame() / codec(T): one call = one invocation of the reference's own function."""

    def __init__(self, threads: int | None = None, with_codec: bool = True):
        self.cores = threads or min(usable_cores(), 32)
        torch.set_num_threads(self.cores)
        self.cfg = O.LMConfig(max_seq_len=512)
        w = _lm_weights(self.cfg)
        self.kind = "port"
        self._st = O.setup(self.cfg, w)
        del w
        g = torch.Generator().manual_seed(42)
        self.prompt = torch.zeros(self.cfg.num_codebooks + 1, T_PROMPT, dtype=torch.long)
        self.prompt[0] = torch.randint(0, 151643, (T_PROMPT,), generator=g)
        dt = torch.bfloat16
        self._temp, self._top_p = torch.tensor(0.7, dtype=dt), torch.tensor(0.7, dtype=dt)
        self._bias = O.semantic_logit_bias(self.cfg, dt)
        self._cur = None
        self._pos = T_PROMPT
        self._prev = torch.zeros((self.cfg.num_codebooks + 1, O.RAS_WIN_SIZE), dtype=torch.int)
        self._codec = None
        if with_codec:
            self.ccfg = CO.full_config()
            cw = CO.make_weights(self.ccfg, seed=6)
            self._codec = lambda codes: CO.from_indices(cw, self.ccfg, codes)

    # ---- LM ----
    def _one(self, x, input_pos, prev):
        C1 = self.cfg.num_codebooks + 1
        return O.decode_one_token_ar(self._st, x.view(1, C1, -1), input_pos, self._temp, self._top_p, 1, self._bias,
                                     previous_tokens=prev)

    @torch.inference_mode()
    def prefill(self) -> float:
        """The prefill call of `generate` (inference.py:322-335) on the 64-token prompt; (re)starts the utterance."""
        t0 = time.perf_counter()
        first = self._one(self.prompt, torch.arange(0, T_PROMPT), None)
        dt = time.perf_counter() - t0
        self._cur, self._pos = first, T_PROMPT
        self._prev.zero_()
        return dt

    @torch.inference_mode()
    def frame(self) -> float:
        """One iteration of decode_n_tokens' loop (inference.py:209-236)."""
        from torch.nn.attention import SDPBackend, sdpa_kernel

        if self._pos >= self.cfg.max_seq_len - 1:
            self.prefill()
        t0 = time.perf_counter()
        with sdpa_kernel(SDPBackend.MATH):
            nxt = self._one(self._cur, torch.tensor([self._pos], dtype=torch.long), self._prev).clone()
        dt = time.perf_counter() - t0
        self._pos += 1
        self._cur = nxt
        self._prev = self._prev.roll(-1, dims=1)
        self._prev[:, -1] = nxt.view(self.cfg.num_codebooks + 1, -1)[:, 0]
        return dt

    # ---- codec ----
    @torch.inference_mode()
    def codec(self, T: int) -> float:
        g = torch.Generator().manual_seed(T)
        c = self.ccfg
        codes = torch.stack([torch.randint(0, c.semantic_codebook_size, (1, T), generator=g)] +
                            [torch.randint(0, c.codebook_size, (1, T), generator=g) for _ in range(c.n_codebooks)], dim=1)
        t0 = time.perf_counter()
        wav = self._codec(codes)
        dt = time.perf_counter() - t0
        assert wav.shape[-1] == T * FRAME
        return dt


def measure(steps: int, warmup: int, frames_per_step: int = 2, codec_frames_per_step: int = 16,
            threads: int | None = None) -> dict:
    """`warmup` untimed + `steps` timed sample steps; returns the components and the extrapolated metric."""
    hp = CpuHotPath(threads)
    t_prefill = hp.prefill()  # also the cold start (page-in of 9 GB of weights)
    t_prefill = hp.prefill()
    step_s, frame_s, codec_s = [], [], []
    for i in range(warmup + steps):
        t0 = time.perf_counter()
        f = [hp.frame() for _ in range(frames_per_step)]
        c = hp.codec(codec_frames_per_step)
        dt = time.perf_counter() - t0
        if i >= warmup:
            step_s.append(dt)
            frame_s += f
            codec_s.append(c)
    t_frame = sum(frame_s) / len(frame_s)
    t_codec = sum(codec_s) / len(codec_s)
    utt = t_prefill + (N_FRAMES - 1) * t_frame + t_codec * N_FRAMES / codec_frames_per_step
    value = N_FRAMES * FRAME / SR / utt
    sample = (f"{hp.kind} on {hp.cores} host threads, bf16 LM + fp32 codec, batch-1 (the reference's max_batch_size): "
              f"each step = {frames_per_step} decode frames (decode_one_token_ar, context {T_PROMPT}+) + DAC.from_indices of "
              f"{codec_frames_per_step} frames; 64-token prefill timed once = {t_prefill:.2f} s; mean frame {t_frame:.3f} s; "
              f"mean codec {t_codec:.2f} s per {codec_frames_per_step} frames; utterance of {N_FRAMES} frames extrapolated = "
              f"prefill + 255*frame + codec*{N_FRAMES}/{codec_frames_per_step} = {utt:.1f} s; audio-s/s = "
              f"{N_FRAMES}*2048/44100/utterance (32 utterances run one after another: same throughput)")
    return {"value": value, "unit": "audio-s/s", "cores": hp.cores, "kind": hp.kind, "sample": sample,
            "ms_per_step": 1e3 * sum(step_s) / len(step_s), "t_prefill_s": t_prefill, "t_frame_s": t_frame,
            "t_codec_s": t_codec, "codec_frames_per_step": codec_frames_per_step, "frames_per_step": frames_per_step}


if __name__ == "__main__":
    import json

    print(json.dumps(measure(int(sys.argv[1]) if len(sys.argv) > 1 else 2, 1)))
