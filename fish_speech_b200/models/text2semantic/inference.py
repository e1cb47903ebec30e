"""Drop-in surface of fish_speech/models/text2semantic/inference.py.

Same entry points and semantics (`init_model`, `decode_one_token_ar`, `decode_n_tokens`, `generate`,
`generate_long`, `launch_thread_safe_queue`, `load_codec_model`, `encode_audio`, `decode_to_audio`, the
click `main`), with the per-frame math executed by the CUDA engine.  New on top of the reference:
`generate_batch` — up to 64 independent utterances decoded in lock-step on one GPU (the reference is
batch-1 only: inference.py:87, 284-288).

The CPU-side prompt builder (Conversation / ContentSequence / tokenizer) is the reference's own code
(SURVEY.md §8: ADJACENT, unchanged) and is imported lazily from an installed `fish_speech`.
"""
from __future__ import annotations

import os
import queue
import threading
import time
import traceback
from dataclasses import dataclass
from pathlib import Path
from typing import Callable, Literal, Optional, Sequence, Union

import numpy as np
import torch

from ...engine import KV_PAGE, MAX_DECODE_BATCH
from .llama import IM_END_TOKEN, DualARTransformer

try:  # loguru is what the reference logs with; fall back to stdlib logging if absent
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("fish_speech_b200")

RAS_WIN_SIZE = 10  # inference.py:49-51 (the engine implements the same constants)
RAS_HIGH_TEMP = 1.0
RAS_HIGH_TOP_P = 0.9
_CHECK_EVERY = 8  # frames between host polls of the on-device finished flags


def _as_float(v) -> float:
    return float(v.item()) if isinstance(v, torch.Tensor) else float(v)


def _ensure_engine(model: DualARTransformer, batch: int = 1):
    if model.engine is None or model.max_batch_size < batch:
        model.setup_caches(max_batch_size=max(batch, max(model.max_batch_size, 1)),
                           max_seq_len=model.config.max_seq_len, dtype=model.dtype,
                           prefix_cache=getattr(model, "prefix_cache", False))
        model._cache_setup_done = True
    return model.engine


def decode_one_token_ar(
    model: DualARTransformer,
    x: torch.Tensor,
    input_pos: torch.Tensor,
    temperature,
    top_p,
    top_k: int,
    semantic_logit_bias: Optional[torch.Tensor] = None,
    audio_masks: Optional[torch.Tensor] = None,
    audio_parts: Optional[torch.Tensor] = None,
    previous_tokens: Optional[torch.Tensor] = None,
) -> torch.Tensor:
    """One frame for one sequence (inference.py:96-181): x [1, C+1, S] at positions input_pos [S];
    S > 1 is a prefill. Returns int tensor [C+1, 1].  `semantic_logit_bias` is accepted for signature
    compatibility; the engine applies the same constraint by restricting the LM head to the selectable
    rows (semantic ids + <|im_end|>)."""
    if audio_parts is not None:
        raise NotImplementedError("audio_parts: the reference model has no audio_projector either (llama.py:423-433)")
    eng = _ensure_engine(model, 1)
    seed = int(torch.initial_seed()) & 0x7FFFFFFFFFFFFFFF
    sp = eng.sampling(_as_float(temperature), _as_float(top_p), int(top_k), seed)
    C1 = model.config.num_codebooks + 1
    x = x.view(1, C1, -1)
    S = x.shape[-1]
    if S > 1:
        start = int(input_pos[0].item())
        eng.prefill([x[0]], [0], sp, start_pos=[start], do_sample=True)
    else:
        p0 = int(input_pos.view(-1)[0].item())
        if p0 >= eng.kv_len:
            raise ValueError(f"input_pos {p0} is outside the KV cache ({eng.kv_len} positions)")
        eng.buffer("cur_tok")[0].copy_(x[0, :, 0].to(torch.int32))
        eng.buffer("pos")[0:1].copy_(input_pos.to(torch.int32).view(1))
        eng.reserve(0, p0 + 1, start=p0)
        eng.set_context_bound(p0 + 1)
        win = eng.buffer("ras_window")
        if previous_tokens is not None:
            win[0].copy_(previous_tokens[0].to(torch.int32))
        else:
            win[0].fill_(-1)  # no RAS without a window (inference.py:133)
        eng.decode(1, 1, sp, use_graph=False)
    return eng.buffer("cur_tok")[0].clone().view(C1, 1)


def decode_n_tokens(
    model: DualARTransformer,
    cur_token: torch.Tensor,
    input_pos: torch.Tensor,
    num_new_tokens: int,
    temperature,
    top_p,
    top_k: int,
    semantic_logit_bias: Optional[torch.Tensor] = None,
    audio_masks: Optional[torch.Tensor] = None,
    audio_parts: Optional[torch.Tensor] = None,
    decode_one_token=decode_one_token_ar,
):
    """inference.py:184-238 — up to num_new_tokens frames after `cur_token`, stopping after <|im_end|>.
    The frame loop runs as CUDA-graph replays; the <|im_end|> test stays on the device and is polled
    every few frames instead of synchronising every frame (inference.py:233)."""
    eng = _ensure_engine(model, 1)
    C1 = model.config.num_codebooks + 1
    seed = int(torch.initial_seed()) & 0x7FFFFFFFFFFFFFFF
    sp = eng.sampling(_as_float(temperature), _as_float(top_p), int(top_k), seed)
    eng.buffer("cur_tok")[0].copy_(cur_token.view(C1, -1)[:, -1].to(torch.int32))
    eng.buffer("pos")[0:1].copy_(input_pos.to(torch.int32).view(-1)[:1])
    eng.buffer("n_out").zero_()
    eng.buffer("finished").zero_()
    eng.buffer("ras_window").zero_()
    start = int(input_pos.view(-1)[0].item())
    eng.reserve(0, start + 1, start=start)
    eng.set_context_bound(start + 1)
    num_new_tokens = min(int(num_new_tokens), eng.max_frames, eng.kv_len - start)  # never write past the KV cache
    n = _run_frames(eng, 1, num_new_tokens, sp, first_frame_from_prefill=False)[0]
    return eng.buffer("out_tokens")[0, :, :n].clone()


def _run_frames(eng, batch: int, max_frames: int, sp, first_frame_from_prefill: bool, on_progress=None):
    """Decode until every sequence has emitted <|im_end|> (checked from frame index 1 on, as the
    reference's loop does) or max_frames frames exist. Returns the kept frame count per sequence.
    `on_progress(done)`: called after every poll with the number of frames that exist on the device."""
    im_end = eng.im_end_id
    done = 1 if first_frame_from_prefill else 0
    while done < max_frames:
        step = min(_CHECK_EVERY, max_frames - done)
        eng.decode(batch, step, sp, use_graph=True)
        done += step
        if on_progress is not None:
            on_progress(done)
        if done < max_frames and bool(eng.buffer("finished")[:batch].all().item()):
            # every sequence has produced <|im_end|>; make sure it was at index >= 1
            toks = eng.buffer("out_tokens")[:batch, 0, :done]
            if bool(((toks[:, 1:] == im_end).any(dim=1)).all().item()) or not first_frame_from_prefill:
                break
    toks = eng.buffer("out_tokens")[:batch, 0, :done].cpu()
    counts = []
    for b in range(batch):
        row = toks[b]
        start = 1 if first_frame_from_prefill else 0
        hits = (row[start:] == im_end).nonzero()
        counts.append(int(hits[0].item()) + start + 1 if len(hits) else done)
    return counts


@torch.no_grad()
def generate(
    *,
    model: DualARTransformer,
    prompt: torch.Tensor,
    max_new_tokens: int,
    audio_masks: Optional[torch.Tensor] = None,
    audio_parts: Optional[torch.Tensor] = None,
    decode_one_token=decode_one_token_ar,
    num_samples: int = 1,
    **sampling_kwargs,
):
    """inference.py:243-359 — prompt [C+1, T] -> [C+1, T+n]."""
    return generate_batch(model=model, prompts=[prompt], max_new_tokens=max_new_tokens,
                          audio_masks=audio_masks, audio_parts=audio_parts, **sampling_kwargs)[0]


@torch.no_grad()
def generate_batch(
    *,
    model: DualARTransformer,
    prompts: Sequence[torch.Tensor],
    max_new_tokens: int,
    audio_masks: Optional[torch.Tensor] = None,
    audio_parts: Optional[torch.Tensor] = None,
    **sampling_kwargs,
) -> list[torch.Tensor]:
    """`generate` for up to 64 independent utterances at once (one KV slot each). Every sequence sees
    exactly the computation it would see alone: the kernels are batch-invariant, so the result for a
    prompt does not depend on its batch neighbours. `reuse_prefix=True` (sampling_kwargs) prefills only the
    rows whose K/V is not already in the cache (LmEngine.prefill_reusing): same tokens, less work."""
    if audio_parts is not None:
        raise NotImplementedError("audio_parts is not supported (nor by the reference model, llama.py:423-433)")
    cfg = model.config
    B = len(prompts)
    if B < 1 or B > MAX_DECODE_BATCH:
        raise ValueError(f"generate_batch handles 1..{MAX_DECODE_BATCH} prompts per call")
    T_max = max(int(p.size(1)) for p in prompts)
    for p in prompts:
        if p.size(1) >= cfg.max_seq_len:
            raise ValueError(f"Input sequence length {p.size(1)} exceeds max_seq_len {cfg.max_seq_len}")
    if max_new_tokens:
        if T_max + max_new_tokens > cfg.max_seq_len:
            max_new_tokens = cfg.max_seq_len - T_max
    else:
        max_new_tokens = cfg.max_seq_len - T_max
    eng = _ensure_engine(model, B)
    # the engine's KV cache may be smaller than config.max_seq_len (setup_caches(max_seq_len=...)): never
    # decode past it
    if T_max >= eng.kv_len:
        raise ValueError(f"Input sequence length {T_max} exceeds the KV cache ({eng.kv_len})")
    max_new_tokens = min(max_new_tokens, eng.max_frames, eng.kv_len - T_max)
    seed = int(sampling_kwargs.get("seed", torch.initial_seed())) & 0x7FFFFFFFFFFFFFFF
    sp = eng.sampling(sampling_kwargs.get("temperature", 1.0), sampling_kwargs.get("top_p", 0.9),
                      int(sampling_kwargs.get("top_k", 30)), seed)
    eng.reset()
    if sampling_kwargs.get("reuse_prefix", False):
        # keep the K/V of the rows this prompt shares with what the slot (or another slot) already holds
        eng.prefill_reusing(list(prompts), list(range(B)), sp, do_sample=True)
    else:
        eng.prefill(list(prompts), list(range(B)), sp, do_sample=True)
    out_tokens = eng.buffer("out_tokens")
    frame_callback = sampling_kwargs.get("frame_callback")
    on_progress = None
    if frame_callback is not None:
        # Streaming (SURVEY §8(f).3): hand the codes of finished frames to the caller while decoding goes on. What is
        # emitted over a whole call is exactly what generate_long keeps of it, y[1:, T:-1] (inference.py:708: the last
        # frame -- <|im_end|> or the one at the budget -- is dropped), so the newest frame is always held back.
        emitted = [0] * B
        im_end = eng.im_end_id

        def on_progress(done: int):
            toks = out_tokens[:B, 0, :done].cpu()
            for b in range(B):
                hits = (toks[b, 1:] == im_end).nonzero()
                n = int(hits[0]) + 2 if len(hits) else done  # frames that count, the stopping one included
                if n - 1 > emitted[b]:
                    frame_callback(b, out_tokens[b, 1:, emitted[b]: n - 1].cpu())  # host copy: crosses threads
                    emitted[b] = n - 1

    counts = _run_frames(eng, B, max_new_tokens, sp, first_frame_from_prefill=True, on_progress=on_progress)
    if on_progress is not None:
        on_progress(max(counts))
    outs = []
    for b, p in enumerate(prompts):
        gen = out_tokens[b, :, : counts[b]].to(p.dtype)
        outs.append(torch.cat([p.to(gen.device), gen], dim=1))
    return outs


def init_model(checkpoint_path, device, precision, compile=False):
    """inference.py:362-392. `compile` is accepted and ignored: the frame is already one CUDA graph of
    hand-written kernels, there is nothing for Inductor to do."""
    if precision not in (torch.bfloat16, None):
        logger.warning(f"fish_speech_b200 computes in bf16; requested {precision} is ignored")
    model = DualARTransformer.from_pretrained(checkpoint_path, load_weights=True, device=device)
    logger.info("Restored model from checkpoint")
    logger.info("Using DualARTransformer (fish_speech_b200 CUDA engine)")
    model.fixed_temperature = torch.tensor(0.7, device=device, dtype=torch.float)
    model.fixed_top_p = torch.tensor(0.7, device=device, dtype=torch.float)
    model.fixed_repetition_penalty = torch.tensor(1.5, device=device, dtype=torch.float)
    model._cache_setup_done = False
    return model.eval(), decode_one_token_ar


# ---- codec helpers (inference.py:396-444) -------------------------------------------------------
@torch.inference_mode()
def load_codec_model(codec_checkpoint_path, device, precision=torch.bfloat16):
    from ..dac.inference import load_model

    return load_model("modded_dac_vq", codec_checkpoint_path, device=device)


@torch.inference_mode()
def encode_audio(audio_path, codec, device):
    import torchaudio

    from ...audio import resample

    wav, sr = torchaudio.load(str(audio_path))
    if wav.shape[0] > 1:
        wav = wav.mean(dim=0, keepdim=True)
    wav = resample(wav.to(device), sr, codec.sample_rate)[0]  # on a CUDA device: the codec front end's kernel
    audios = wav[None, None]
    audio_lengths = torch.tensor([len(wav)], device=device, dtype=torch.long)
    indices, feature_lengths = codec.encode(audios, audio_lengths)
    return indices[0, :, : feature_lengths[0]]


@torch.inference_mode()
def decode_to_audio(codes, codec):
    audio = codec.from_indices(codes[None])
    return audio[0, 0]


@dataclass
class GenerateResponse:
    action: Literal["sample", "next", "partial"]  # "partial": streamed codes of a chunk in progress (extension)
    codes: Optional[torch.Tensor] = None
    text: Optional[str] = None


def _reference_frontend():
    """The reference's CPU prompt builder (content_sequence.py / conversation.py) — unchanged code."""
    try:
        from fish_speech.content_sequence import TextPart, VQPart
        from fish_speech.conversation import Conversation, Message
    except Exception as e:  # pragma: no cover
        raise ImportError(
            "generate_long needs the reference's CPU-side prompt builder (fish_speech.conversation / "
            "content_sequence / tokenizer); install fish-speech next to fish_speech_b200") from e
    return TextPart, VQPart, Conversation, Message


def split_text_by_speaker(text: str) -> list[str]:
    """inference.py:454-474."""
    import re

    pattern = r"(<\|speaker:\d+\|>)"
    parts = re.split(pattern, text)
    turns, i = [], 0
    while i < len(parts):
        part = parts[i].strip()
        if re.match(pattern, part):
            if i + 1 < len(parts):
                turn = part + parts[i + 1]
                turns.append(turn.strip())
                i += 2
            else:
                turns.append(part)
                i += 1
        else:
            i += 1
    return turns


def group_turns_into_batches(turns: list[str], max_speakers: int = 3, max_bytes: int = 300) -> list[str]:
    """inference.py:477-520: close the current batch when it already holds `max_speakers` turns or the
    next turn would push it over `max_bytes` UTF-8 bytes."""
    batches: list[str] = []
    held: list[str] = []
    held_bytes = 0
    for turn in turns:
        size = len(turn.encode("utf-8"))
        if len(held) >= max_speakers or (held and held_bytes + size > max_bytes):
            batches.append("\n".join(held))
            held, held_bytes = [], 0
        held.append(turn)
        held_bytes += size
    if held:
        batches.append("\n".join(held))
    return batches


def _generate_long_plan(
    *,
    model,
    device: Union[str, torch.device],
    decode_one_token: Optional[Callable] = None,
    text: str,
    num_samples: int = 1,
    max_new_tokens: int = 0,
    top_p: float = 0.9,
    top_k: int = 30,
    repetition_penalty: float = 1.1,
    temperature: float = 1.0,
    compile: bool = False,
    iterative_prompt: bool = True,
    chunk_length: int = 512,
    prompt_text: Optional[Union[str, list[str]]] = None,
    prompt_tokens: Optional[Union[torch.Tensor, list[torch.Tensor]]] = None,
):
    """inference.py:523-733 as a coroutine: build the conversation and walk the chunk loop, but hand every
    `generate` call to the driver. Yields ("generate", kwargs) and expects the [C+1, T+n] result to be sent
    back; yields ("response", GenerateResponse) for everything the reference's generator yields. One
    request at a time (generate_long) and the slot scheduler (launch_thread_safe_queue) drive the same plan."""
    assert 0 < top_p <= 1, "top_p must be in (0, 1]"
    assert 0 < temperature < 2, "temperature must be in (0, 2)"
    TextPart, VQPart, Conversation, Message = _reference_frontend()

    use_prompt = bool(prompt_text) and bool(prompt_tokens)
    if use_prompt and isinstance(prompt_text, str):
        prompt_text = [prompt_text]
        prompt_tokens = [prompt_tokens]
    if use_prompt:
        assert len(prompt_text) == len(prompt_tokens), "Prompt text and tokens must have the same length"
    if prompt_tokens:
        prompt_tokens = [i.cpu() for i in prompt_tokens]

    tokenizer = model.tokenizer
    max_length = model.config.max_seq_len
    base_conversation = Conversation()
    if use_prompt:
        tagged = []
        for i, t in enumerate(prompt_text):
            import re

            tagged.append(t if re.search(r"<\|speaker:\d+\|>", t) else f"<|speaker:{i}|>{t}")
        system_parts = [TextPart(text="convert the provided text to speech reference to the following:\n\nText:\n",
                                 cal_loss=False)]
        system_parts.append(TextPart(text="\n".join(tagged), cal_loss=False))
        system_parts.append(TextPart(text="\n\nSpeech:\n", cal_loss=False))
        all_codes = torch.cat([c for c in prompt_tokens], dim=1)
        system_parts.append(VQPart(codes=all_codes, cal_loss=False))
    else:
        system_parts = [TextPart(text="convert the provided text to speech", cal_loss=False)]
    base_conversation.append(Message(role="system", parts=system_parts, cal_loss=False, add_im_start=True,
                                     add_im_end=True))

    turns = split_text_by_speaker(text)
    if turns:
        batches = group_turns_into_batches(turns, max_speakers=5, max_bytes=chunk_length)
    else:
        batches = [text]
    logger.info(f"Split into {len(turns)} turns, grouped into {len(batches)} batches")

    for sample_idx in range(num_samples):
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        conversation = __import__("copy").deepcopy(base_conversation)
        for batch_idx, batch_text in enumerate(batches):
            logger.info(f"--- Sample {sample_idx}, Batch {batch_idx} ({len(batch_text.encode('utf-8'))} bytes) ---")
            conversation.append(Message(role="user", parts=[TextPart(text=batch_text, cal_loss=False)],
                                        cal_loss=False, add_im_start=True, add_im_end=True))
            conversation_gen = __import__("copy").deepcopy(conversation)
            conversation_gen.append(Message(role="assistant", parts=[], cal_loss=False, modality="voice",
                                            add_im_start=True, add_im_end=False))
            encoded, audio_masks, audio_parts = conversation_gen.encode_for_inference(
                tokenizer, num_codebooks=model.config.num_codebooks)
            logger.info(f"Encoded prompt shape: {encoded.shape}")
            if encoded.size(1) > max_length - 2048:
                raise ValueError(f"Prompt is too long: {encoded.size(1)} > {max_length - 2048}")
            encoded = encoded.to(device=device)
            prompt_length = encoded.size(1)
            t0 = time.perf_counter()
            # every chunk's prompt extends the previous one (the conversation only grows): reuse its K/V
            y = yield ("generate", dict(prompt=encoded, max_new_tokens=max_new_tokens, audio_masks=audio_masks,
                                        audio_parts=audio_parts, temperature=temperature, top_p=top_p, top_k=top_k,
                                        reuse_prefix=True))
            t_batch = time.perf_counter() - t0
            tokens_generated = y.size(1) - prompt_length
            tokens_sec = tokens_generated / t_batch if t_batch > 0 else 0
            logger.info(f"Batch {batch_idx}: Generated {tokens_generated} tokens in {t_batch:.02f} seconds, "
                        f"{tokens_sec:.02f} tokens/sec")
            codes = y[1:, prompt_length:-1].clone()
            assert (codes >= 0).all(), f"Negative code found: {codes}"
            conversation.append(Message(role="assistant", parts=[VQPart(codes=codes.cpu(), cal_loss=False)],
                                        cal_loss=False, modality="voice", add_im_start=True, add_im_end=True))
            yield ("response", GenerateResponse(action="sample", codes=codes, text=batch_text))
            del y, encoded
        if torch.cuda.is_available():
            logger.info(f"GPU Memory used: {torch.cuda.max_memory_reserved() / 1e9:.02f} GB")
        yield ("response", GenerateResponse(action="next"))


def generate_long(*, model, decode_one_token: Callable = None, on_partial: Optional[Callable] = None, **kwargs):
    """inference.py:523-733: yields GenerateResponse("sample", codes [C, n], text) per chunk, then ("next").
    `on_partial(codes [C, k])` (extension, SURVEY §8(f).3): called from inside the decode loop with the codes of the
    frames finished since the last call; over a chunk the pieces concatenate to that chunk's "sample" codes."""
    plan = _generate_long_plan(model=model, **kwargs)
    reply = None
    while True:
        try:
            kind, payload = plan.send(reply)
        except StopIteration:
            return
        reply = None
        if kind == "generate":
            if on_partial is not None:
                payload = dict(payload, frame_callback=lambda b, codes: on_partial(codes))
            reply = generate(model=model, decode_one_token=decode_one_token or decode_one_token_ar,
                             seed=_next_seed(model), **payload)
            if torch.cuda.is_available():
                torch.cuda.synchronize()
        else:
            yield payload


def _next_seed(model) -> int:
    """Philox key of the next `generate` call: torch's seed (what the CLI's --seed sets) advanced by a per-model
    call counter, so that consecutive chunks / requests do not replay one random stream. Re-seeding torch
    restarts the sequence."""
    base = int(torch.initial_seed())
    last, n = getattr(model, "_seed_state", (None, 0))
    n = n + 1 if last == base else 0
    model._seed_state = (base, n)
    return (base + 0x9E3779B97F4A7C15 * n) & 0x7FFFFFFFFFFFFFFF


@dataclass
class WrappedGenerateResponse:
    status: Literal["success", "error"]
    response: Optional[Union[GenerateResponse, Exception]] = None


@dataclass
class GenerateRequest:
    request: dict
    response_queue: queue.Queue


# Frames per second a listener plays: the codec's sample_rate / frame_length (models/dac/modded_dac.py).
PLAYBACK_FRAMES_PER_S = 44100 / 2048


def serve_requests(model, input_queue: "queue.Queue", max_slots: int, frames_per_poll: int = 8,
                   batcher=None) -> None:
    """Worker loop of the slot scheduler: every queued request's `generate_long` plan advances concurrently,
    their `generate` calls share the decode frames (fish_speech_b200/scheduler.py). Responses of one request
    arrive in the reference's order on its own response queue; `None` shuts the loop down once the running
    requests are finished.

    FSB_SERVE_LIVE=n (n > max_slots) lets up to n requests be live at a time: streaming requests
    (`stream_frames`) are then paced at playback speed, one playback clock per request across its chunks, so
    that the scheduler parks the ones far ahead of their listener and gives their slots to the ones about to run
    dry. FSB_SERVE_KV_GROW=1 (with FSB_SERVE_KV_GB) lets requests take KV pages as they decode instead of reserving
    prompt + budget at admission (ContinuousBatcher kv_growth). FSB_SERVE_COMPACT=1 decodes only the rows up to the
    highest live slot and moves requests below slot 32 whenever they all fit there, so that an engine of more than 32
    slots runs its 32-row frame off-peak (ContinuousBatcher compact_rows). FSB_SERVE_FUSED_ADMIT=1 runs each admitted
    request's first frame inside the next decode frame instead of a frame of its own (ContinuousBatcher
    fused_admission), with the same tokens. A request dict may carry `cancel` (a threading.Event): once it is set the request in flight is taken out
    of the scheduler, the plan ends and nothing more is put on its response queue."""
    from ...scheduler import Cancelled, ContinuousBatcher, SlotRequest, StreamClock

    if batcher is None:
        max_live = max(max_slots, int(os.environ.get("FSB_SERVE_LIVE", "0") or 0))
        grow = serve_kv_grow(os.environ.get("FSB_SERVE_KV_GROW"), os.environ.get("FSB_SERVE_KV_GB"))
        compact = serve_compact(os.environ.get("FSB_SERVE_COMPACT"))
        fused = serve_fused_admit(os.environ.get("FSB_SERVE_FUSED_ADMIT"))
        batcher = ContinuousBatcher(model, max_slots=max_slots, frames_per_poll=frames_per_poll, max_live=max_live,
                                    kv_growth=grow, compact_rows=compact, fused_admission=fused)
    paced = getattr(batcher, "max_live", 0) > getattr(batcher, "max_slots", 0)
    live = 0  # plans not yet exhausted
    waiting_queues: dict = {}  # id(plan) -> response queue of every plan that has a generate call in flight
    streaming: dict = {}  # id(plan) -> playback clock of requests that asked for partial codes (`stream_frames`)
    cancels: dict = {}  # id(plan) -> (cancel event, plan) of requests that carry one
    inflight: dict = {}  # id(plan) -> the SlotRequest of its generate call in flight
    closing = False

    def end(plan):
        nonlocal live
        live -= 1
        streaming.pop(id(plan), None)
        cancels.pop(id(plan), None)
        inflight.pop(id(plan), None)

    def finished(r, plan, response_queue):
        inflight.pop(id(plan), None)
        if r.error is None:
            return advance(plan, response_queue, r.result)
        waiting_queues.pop(id(plan), None)
        plan.close()
        if not isinstance(r.error, Cancelled):
            response_queue.put(WrappedGenerateResponse(status="error", response=r.error))
        end(plan)

    def advance(plan, response_queue, reply):
        """Run a plan until it asks for the next `generate` (submitted to the batcher) or ends."""
        nonlocal live
        waiting_queues.pop(id(plan), None)
        try:
            while True:
                kind, payload = plan.send(reply)
                reply = None
                if kind == "response":
                    response_queue.put(WrappedGenerateResponse(status="success", response=payload))
                    continue
                if payload.get("audio_parts") is not None:
                    raise NotImplementedError("audio_parts is not supported (nor by the reference model)")
                on_frames = None
                if id(plan) in streaming:  # finished frames leave as "partial" responses, ahead of the chunk's "sample"
                    def on_frames(r, codes, q=response_queue):
                        q.put(WrappedGenerateResponse(status="success",
                                                      response=GenerateResponse(action="partial", codes=codes)))
                pace = dict(pace=PLAYBACK_FRAMES_PER_S, stream=streaming[id(plan)]) if paced and on_frames else {}
                inflight[id(plan)] = req = SlotRequest(
                    prompt=payload["prompt"], max_new_tokens=payload["max_new_tokens"],
                    temperature=payload["temperature"], top_p=payload["top_p"], top_k=payload["top_k"],
                    seed=_next_seed(model), reuse_prefix=bool(payload.get("reuse_prefix", False)), on_frames=on_frames,
                    on_done=lambda r, plan=plan, q=response_queue: finished(r, plan, q), **pace)
                batcher.submit(req)
                waiting_queues[id(plan)] = response_queue
                return
        except StopIteration:
            end(plan)
        except Exception as e:
            logger.error(traceback.format_exc())
            response_queue.put(WrappedGenerateResponse(status="error", response=e))
            end(plan)

    try:
        while True:
            # take everything that is waiting; block only when there is nothing to compute
            while not closing:
                try:
                    item = input_queue.get(block=(live == 0 and batcher.idle()))
                except queue.Empty:
                    break
                if item is None:
                    closing = True
                    break
                live += 1
                try:
                    plan = _generate_long_plan(model=model, **{k: v for k, v in item.request.items()
                                                               if k not in ("decode_one_token", "stream_frames", "cancel")})
                except Exception as e:  # pragma: no cover - argument errors surface on first send
                    item.response_queue.put(WrappedGenerateResponse(status="error", response=e))
                    live -= 1
                    continue
                if item.request.get("stream_frames", 0):
                    streaming[id(plan)] = StreamClock()
                if item.request.get("cancel") is not None:
                    cancels[id(plan)] = (item.request["cancel"], plan)
                advance(plan, item.response_queue, None)
            for event, plan in list(cancels.values()):
                if event.is_set() and id(plan) in inflight:
                    batcher.cancel(inflight[id(plan)])  # -> finished(): the plan ends without another response
            if live == 0 and closing:
                return
            try:
                batcher.step()
            except Exception as e:
                # Per-request problems were rejected in submit(); what fails here is the engine itself (e.g. a
                # poisoned CUDA context). Every request in flight hears about it, and so does everything still
                # queued or arriving later: the worker keeps answering (with the error) instead of dying with
                # callers blocked on their response queues.
                logger.error(traceback.format_exc())
                for q_ in waiting_queues.values():
                    q_.put(WrappedGenerateResponse(status="error", response=e))
                waiting_queues.clear()
                while not closing:
                    item = input_queue.get()
                    if item is None:
                        break
                    item.response_queue.put(WrappedGenerateResponse(status="error", response=e))
                return
    finally:
        try:
            batcher.close()
        except Exception:  # a failed engine may not reset cleanly; do not mask the original error
            logger.error(traceback.format_exc())


def slow_kv_bytes_per_position(config) -> int:
    """Bytes of slow-stack K and V cache one sequence slot holds per position (bf16): 147 456 at S2-Pro geometry."""
    return 2 * config.n_layer * config.n_local_heads * config.head_dim * 2


def check_serve_kv_fits(slots: int, kv_len: int, config, free_bytes: int) -> None:
    """Raise a ValueError naming FSB_SERVE_KV_LEN when `slots` slow KV caches of `kv_len` positions do not fit in
    `free_bytes` of device memory (64 slots x 8192 positions need 77 GB at S2-Pro geometry)."""
    need = slots * kv_len * slow_kv_bytes_per_position(config)
    if need > free_bytes:
        fit = free_bytes // max(1, slots * slow_kv_bytes_per_position(config))
        raise ValueError(f"{slots} slots x {kv_len} KV positions need {need / 1e9:.1f} GB of slow KV cache, but only "
                         f"{free_bytes / 1e9:.1f} GB of device memory is free: lower FSB_SERVE_KV_LEN (at most "
                         f"{fit} fits) or FSB_SERVE_SLOTS")


def kv_page_bytes(config) -> int:
    """Bytes of one page of the slow KV cache: 64 positions of every slow layer, K and V (9.44 MB at S2-Pro)."""
    return KV_PAGE * slow_kv_bytes_per_position(config)


def serve_kv_pool_pages(gb: float, config, free_bytes: int) -> int:
    """Pages in a slow KV pool of `gb` GB (FSB_SERVE_KV_GB); a ValueError naming FSB_SERVE_KV_GB when that pool
    does not fit in `free_bytes` of device memory or holds no page."""
    pages = int(float(gb) * 1e9 // kv_page_bytes(config))
    if pages < 1:
        raise ValueError(f"FSB_SERVE_KV_GB={gb} is smaller than one KV page ({kv_page_bytes(config) / 1e9:.3f} GB)")
    need = pages * kv_page_bytes(config)
    if need > free_bytes:
        raise ValueError(f"FSB_SERVE_KV_GB={gb}: a pool of {pages} KV pages needs {need / 1e9:.1f} GB, but only "
                         f"{free_bytes / 1e9:.1f} GB of device memory is free: lower FSB_SERVE_KV_GB")
    return pages


def serve_attn_split(value: Optional[str]) -> int:
    """FSB_ATTN_SPLIT: positions per span of the split decode attention (setup_caches(attn_split=)); unset, empty or
    0 = off. A ValueError naming FSB_ATTN_SPLIT for anything that is not a non-negative multiple of 64."""
    if value is None or value.strip() == "":
        return 0
    try:
        n = int(value)
    except ValueError:
        n = -1
    if n < 0 or n % KV_PAGE != 0:
        raise ValueError(f"FSB_ATTN_SPLIT={value!r} must be 0 (off) or a multiple of {KV_PAGE} positions")
    return n


def serve_kv_grow(value: Optional[str], kv_gb: Optional[str]) -> bool:
    """FSB_SERVE_KV_GROW: 1 = requests take KV pages as they decode (ContinuousBatcher kv_growth); unset, empty or 0
    = prompt + budget reserved at admission. Growth needs the bounded pool of FSB_SERVE_KV_GB: a ValueError naming
    both variables without it, and one naming FSB_SERVE_KV_GROW for any other value."""
    if value is None or value.strip() in ("", "0"):
        return False
    if value.strip() != "1":
        raise ValueError(f"FSB_SERVE_KV_GROW={value!r} must be 0 or 1")
    if not kv_gb:
        raise ValueError("FSB_SERVE_KV_GROW=1 needs FSB_SERVE_KV_GB: growth shares a bounded KV page pool, and without "
                         "FSB_SERVE_KV_GB every slot has its full capacity reserved")
    return True


def serve_compact(value: Optional[str]) -> bool:
    """FSB_SERVE_COMPACT: 1 = decode only the rows up to the highest live slot and move requests below slot 32 when
    they all fit there (ContinuousBatcher compact_rows); unset, empty or 0 = every frame decodes every slot. A
    ValueError naming FSB_SERVE_COMPACT for any other value."""
    if value is None or value.strip() in ("", "0"):
        return False
    if value.strip() != "1":
        raise ValueError(f"FSB_SERVE_COMPACT={value!r} must be 0 or 1")
    return True


def serve_fused_admit(value: Optional[str]) -> bool:
    """FSB_SERVE_FUSED_ADMIT: 1 = an admitted request's first frame runs as a row of the next decode frame, beside the
    running requests, instead of a frame over the new rows alone (ContinuousBatcher fused_admission); unset, empty or
    0 = off. A ValueError naming FSB_SERVE_FUSED_ADMIT for any other value."""
    if value is None or value.strip() in ("", "0"):
        return False
    if value.strip() != "1":
        raise ValueError(f"FSB_SERVE_FUSED_ADMIT={value!r} must be 0 or 1")
    return True


def serve_prefix_cache(value: Optional[str]) -> bool:
    """FSB_SERVE_PREFIX_CACHE: 1 = the prompt pages of a finished request stay in the KV page pool as a prefix later
    requests reuse, until the pool needs them (setup_caches(prefix_cache=)); unset, empty or 0 = off. A ValueError
    naming FSB_SERVE_PREFIX_CACHE for any other value."""
    if value is None or value.strip() in ("", "0"):
        return False
    if value.strip() != "1":
        raise ValueError(f"FSB_SERVE_PREFIX_CACHE={value!r} must be 0 or 1")
    return True


def launch_thread_safe_queue(checkpoint_path, device, precision, compile: bool = False):
    """inference.py:736-799: the model lives in ONE daemon worker thread fed by a queue; `None` shuts
    it down; errors are returned as WrappedGenerateResponse(status="error", response=exc).

    FSB_SERVE_SLOTS=n (2..64) makes the worker a slot scheduler that runs up to n requests concurrently
    (`serve_requests`), each with a KV cache of FSB_SERVE_KV_LEN positions (default 8192; a slot costs
    147 456 B per position at the S2-Pro geometry). Unset / 1: the reference's one-at-a-time loop. If the slots'
    KV caches do not fit in free device memory, this raises a ValueError naming FSB_SERVE_KV_LEN.
    FSB_SERVE_KV_GB=g (with FSB_SERVE_SLOTS > 1) instead gives the slots one shared pool of g GB of KV pages, each
    slot a capacity of FSB_SERVE_KV_LEN (default: the model's max_seq_len) positions, and a request is admitted when
    its pages fit; a pool that does not fit in free device memory raises a ValueError naming FSB_SERVE_KV_GB.
    FSB_ATTN_SPLIT=p (a multiple of 64; 0 or unset = off) makes a decode row whose context is longer than p positions
    split its attention into spans of p positions over several CTAs, so that one long conversation does not slow the
    frames of every slot; requests that stay at or below p keep their bits, longer ones change in the last places.
    FSB_SERVE_KV_GROW=1 (needs FSB_SERVE_KV_GB; else a ValueError naming both) maps a request's prompt and first frames
    at admission and further pages as it decodes; a request that cannot get its next page safely waits parked.
    FSB_SERVE_COMPACT=1 (0 or unset = off; else a ValueError naming it) keeps the live requests in the lowest slots and
    decodes only the rows they occupy: an engine of 33..64 slots runs its faster 32-row frame while load fits in 32.
    FSB_SERVE_FUSED_ADMIT=1 (0 or unset = off; else a ValueError naming it) runs an admitted request's first frame in
    the next decode frame, beside the running requests, instead of a frame that streams the head and fast weights for
    the new rows alone; the tokens are the same.
    FSB_SERVE_PREFIX_CACHE=1 (0 or unset = off; else a ValueError naming it), for the one-at-a-time loop and the slot
    scheduler alike, keeps the prompt pages of a finished request in the KV page pool, so that the next request with
    the same voice prefix prefills only the rows after it; the cache holds only pages no request needs and gives them
    back when a reservation does. The tokens are the same."""
    serve_kv_grow(os.environ.get("FSB_SERVE_KV_GROW"), os.environ.get("FSB_SERVE_KV_GB"))
    serve_compact(os.environ.get("FSB_SERVE_COMPACT"))
    serve_fused_admit(os.environ.get("FSB_SERVE_FUSED_ADMIT"))
    cache = serve_prefix_cache(os.environ.get("FSB_SERVE_PREFIX_CACHE"))
    input_queue = queue.Queue()
    init_event = threading.Event()
    init_error: list = []
    slots = max(1, min(MAX_DECODE_BATCH, int(os.environ.get("FSB_SERVE_SLOTS", "1"))))

    def worker():
        model, decode_one_token = init_model(checkpoint_path, device, precision, compile=compile)
        if slots > 1:
            gb = os.environ.get("FSB_SERVE_KV_GB")
            default_kv = str(model.config.max_seq_len) if gb else "8192"
            kv = min(int(os.environ.get("FSB_SERVE_KV_LEN", default_kv)), model.config.max_seq_len)
            try:
                cuda = torch.device(device).type == "cuda"
                split = serve_attn_split(os.environ.get("FSB_ATTN_SPLIT"))
                if gb:
                    free = torch.cuda.mem_get_info(torch.device(device))[0] if cuda else float("inf")
                    pages = serve_kv_pool_pages(float(gb), model.config, free)
                    model.setup_caches(max_batch_size=slots, max_seq_len=kv, dtype=model.dtype, kv_pages=pages,
                                       attn_split=split, prefix_cache=cache)
                else:
                    if cuda:
                        check_serve_kv_fits(slots, kv, model.config, torch.cuda.mem_get_info(torch.device(device))[0])
                    model.setup_caches(max_batch_size=slots, max_seq_len=kv, dtype=model.dtype, attn_split=split,
                                       prefix_cache=cache)
            except Exception as e:
                init_error.append(e)
                init_event.set()
                return
            init_event.set()
            serve_requests(model, input_queue, slots)
            return
        model.setup_caches(max_batch_size=1, max_seq_len=model.config.max_seq_len, dtype=model.dtype,
                           prefix_cache=cache)
        init_event.set()
        while True:
            item: Optional[GenerateRequest] = input_queue.get()
            if item is None:
                break
            kwargs = dict(item.request)
            response_queue = item.response_queue
            on_partial = None
            kwargs.pop("cancel", None)  # requests are served one at a time here: nothing to give back early
            if kwargs.pop("stream_frames", 0):
                # streaming request (TTSInferenceEngine with req.streaming): codes leave the worker as frames finish
                def on_partial(codes, q=response_queue):
                    q.put(WrappedGenerateResponse(status="success", response=GenerateResponse(action="partial", codes=codes)))
            try:
                for chunk in generate_long(model=model, decode_one_token=decode_one_token, on_partial=on_partial, **kwargs):
                    response_queue.put(WrappedGenerateResponse(status="success", response=chunk))
            except Exception as e:
                logger.error(traceback.format_exc())
                response_queue.put(WrappedGenerateResponse(status="error", response=e))

    threading.Thread(target=worker, daemon=True).start()
    init_event.wait()
    if init_error:
        raise init_error[0]
    return input_queue


def main(argv=None):
    """CLI with the reference's options (inference.py:802-838)."""
    import click

    @click.command()
    @click.option("--text", type=str, default="<|speaker:0|>你说的对, 但是原神是一款由米哈游自主研发的开放世界手游.")
    @click.option("--prompt-text", type=str, default=None, multiple=True)
    @click.option("--prompt-tokens", type=click.Path(path_type=Path, exists=True), default=None, multiple=True)
    @click.option("--prompt-audio", type=click.Path(path_type=Path, exists=True), default=None, multiple=True)
    @click.option("--output", type=click.Path(path_type=Path), default=None)
    @click.option("--num-samples", type=int, default=1)
    @click.option("--max-new-tokens", type=int, default=0)
    @click.option("--top-p", type=float, default=0.9)
    @click.option("--top-k", type=int, default=30)
    @click.option("--temperature", type=float, default=1.0)
    @click.option("--checkpoint-path", type=click.Path(path_type=Path, exists=True), default="checkpoints/s2-pro")
    @click.option("--device", type=str, default="cuda")
    @click.option("--compile/--no-compile", default=False)
    @click.option("--seed", type=int, default=42)
    @click.option("--half/--no-half", default=False)
    @click.option("--iterative-prompt/--no-iterative-prompt", default=True)
    @click.option("--chunk-length", type=int, default=300)
    @click.option("--output-dir", type=Path, default="output")
    def _main(text, prompt_text, prompt_tokens, prompt_audio, output, num_samples, max_new_tokens, top_p, top_k,
              temperature, checkpoint_path, device, compile, seed, half, iterative_prompt, chunk_length, output_dir):
        os_makedirs = __import__("os").makedirs
        os_makedirs(output_dir, exist_ok=True)
        precision = torch.bfloat16
        if prompt_text and not prompt_audio and not prompt_tokens:
            raise ValueError("--prompt-text requires either --prompt-audio or --prompt-tokens")
        if prompt_text and prompt_tokens and len(prompt_text) != len(prompt_tokens):
            raise ValueError("Number of prompt text and prompt tokens should be the same")
        model, decode_one_token = init_model(checkpoint_path, device, precision, compile=compile)
        with torch.cuda.device(device):
            model.setup_caches(max_batch_size=1, max_seq_len=model.config.max_seq_len, dtype=model.dtype)
        codec = None
        codec_path = Path(checkpoint_path) / "codec.pth"
        prompt_tokens_list = None
        if prompt_audio:
            codec = load_codec_model(codec_path, device, precision)
            prompt_tokens_list = [encode_audio(p, codec, device).cpu() for p in prompt_audio]
        elif prompt_tokens:
            prompt_tokens_list = [torch.from_numpy(np.load(p)) for p in prompt_tokens]
        torch.manual_seed(seed)
        if torch.cuda.is_available():
            torch.cuda.manual_seed(seed)
        generator = generate_long(model=model, device=device, decode_one_token=decode_one_token, text=text,
                                  num_samples=num_samples, max_new_tokens=max_new_tokens, top_p=top_p, top_k=top_k,
                                  temperature=temperature, compile=compile, iterative_prompt=iterative_prompt,
                                  chunk_length=chunk_length, prompt_text=list(prompt_text) if prompt_text else None,
                                  prompt_tokens=prompt_tokens_list)
        idx, codes = 0, []
        for response in generator:
            if response.action == "sample":
                codes.append(response.codes)
            elif response.action == "next":
                if codes:
                    merged = torch.cat(codes, dim=1)
                    np.save(Path(output_dir) / f"codes_{idx}.npy", merged.cpu().numpy())
                    if output:
                        if codec is None:
                            codec = load_codec_model(codec_path, device, precision)
                        audio = decode_to_audio(merged.to(device), codec)
                        import soundfile as sf

                        out = Path(output)
                        if num_samples > 1:
                            out = out.with_stem(f"{out.stem}_{idx}")
                        sf.write(str(out), audio.float().cpu().numpy(), codec.sample_rate)
                codes = []
                idx += 1

    return _main(argv, standalone_mode=False) if argv is not None else _main()


if __name__ == "__main__":
    main()
