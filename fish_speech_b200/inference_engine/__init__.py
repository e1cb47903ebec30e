"""TTSInferenceEngine — the surface of fish_speech/inference_engine/__init__.py (`inference` :22-142,
`send_Llama_request` :144-177, `get_audio_segment` :179-192) with the codec stage overlapped with generation.

The reference turns a chunk's codes into audio only after the LM has finished the chunk. Here a streaming request asks
the LM worker for the codes of finished frames while it keeps decoding (`stream_frames`, "partial" responses), and this
thread pushes them through an incremental codec decoder (`DAC.open_decode_stream`) on its own CUDA stream: audio leaves
with a delay of a few frames instead of a whole chunk (SURVEY §8(f).3). With FSB_STREAM_POOL=n the streaming requests
share one n-slot `DAC.open_stream_pool` behind a codec thread (`CodecStreamWorker`) that decodes the pieces of every
stream in one batched push. Non-streaming requests follow the reference:
one `from_indices` per chunk. The result protocol is the reference's: header | segment* | final, or error.
"""
from __future__ import annotations

import os
import queue
import threading
import time
from concurrent.futures import Future
from typing import Generator, Optional

import numpy as np
import torch

from ..models.dac.modded_dac import DAC
from ..models.text2semantic.inference import GenerateRequest, GenerateResponse, WrappedGenerateResponse
from .reference_loader import ReferenceLoader
from .schema import ServeTTSRequest
from .utils import InferenceResult, wav_chunk_header
from .vq_manager import VQManager

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("fish_speech_b200")


def set_seed(seed: int):
    """fish_speech/utils/utils.py:120-134: one seed for every generator the request may touch."""
    import random

    seed = min(abs(int(seed)), 1 << 31)
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed)


class CodecStreamWorker:
    """Owner of a shared DecodeStreamPool (FSB_STREAM_POOL): request threads submit the new codes of their streams and
    wait on a future; one thread takes everything queued, coalesces the queued pieces of each stream in order (up to
    the pool's k_max frames per push) and decodes all streams in one pool push on a CUDA stream of its own. The
    streaming requests of a slot-scheduled LM receive their frames right after the same poll, so their pushes batch.
    An error in a push is delivered to every caller that waits on it; the worker keeps serving."""

    def __init__(self, pool, device: Optional[torch.device] = None):
        self.pool = pool
        self.k_max = int(pool.k_max)
        self._q: queue.Queue = queue.Queue()
        self._lock = threading.Lock()
        self._device = device
        self.pushes = 0  # pool pushes run (tests, measurements)
        self._thread = threading.Thread(target=self._run, name="codec-stream-pool", daemon=True)
        self._thread.start()

    def open(self) -> Optional[int]:
        """A slot of the pool, or None when it is full (the caller decodes on a stream of its own)."""
        with self._lock:
            try:
                return self.pool.open()
            except ValueError:
                return None

    def release(self, slot: int) -> None:
        """Closes a stream's slot of the pool."""
        with self._lock:
            self.pool.close(slot)

    def submit(self, slot: int, codes: torch.Tensor) -> Future:
        """codes [C, k], k <= k_max -> future of the waveform (fp32 numpy [k * frame_length])."""
        if not 1 <= codes.shape[-1] <= self.k_max:
            raise ValueError(f"a piece takes 1 .. {self.k_max} frames, got {codes.shape[-1]}")
        fut: Future = Future()
        self._q.put((slot, codes, fut))
        return fut

    def decode(self, slot: int, codes: torch.Tensor) -> np.ndarray:
        """The next frames of one stream, in pieces of at most k_max frames; blocks until decoded."""
        futs = [self.submit(slot, codes[:, a: a + self.k_max]) for a in range(0, codes.shape[-1], self.k_max)]
        return np.concatenate([f.result() for f in futs]) if len(futs) > 1 else futs[0].result()

    def close(self) -> None:
        """Stops the worker thread once the pieces queued so far are decoded."""
        self._q.put(None)
        self._thread.join()

    def _run(self):
        side = None
        if self._device is not None and self._device.type == "cuda":
            side = torch.cuda.Stream(device=self._device)
        while True:
            items = [self._q.get()]
            while items[-1] is not None:
                try:
                    items.append(self._q.get_nowait())
                except queue.Empty:
                    break
            stop = items[-1] is None
            items = [it for it in items if it is not None]
            try:
                per_slot: dict = {}
                for slot, codes, fut in items:
                    per_slot.setdefault(slot, []).append((codes, fut))
                while per_slot:
                    pieces, waiting = {}, {}
                    for slot in list(per_slot):
                        q = per_slot[slot]
                        take, k = [], 0
                        while q and k + q[0][0].shape[-1] <= self.k_max:
                            take.append(q.pop(0))
                            k += take[-1][0].shape[-1]
                        if not q:
                            del per_slot[slot]
                        waiting[slot] = take
                        pieces[slot] = take[0][0] if len(take) == 1 else torch.cat([c for c, _ in take], dim=-1)
                    self._push(pieces, waiting, side)
            except BaseException as e:  # grouping failed: every caller of this round that is still waiting sees it
                for _, _, fut in items:
                    if not fut.done():
                        fut.set_exception(e)
            if stop:
                return

    def _push(self, pieces: dict, waiting: dict, side):
        try:
            with torch.inference_mode(), (torch.cuda.stream(side) if side is not None else _nullcontext()):
                out = self.pool.push(pieces)
                wavs = {s: w.float().cpu().numpy() for s, w in out.items()}  # synchronises the worker's stream
            self.pushes += 1
        except BaseException as e:  # every caller of this push sees the error; the worker keeps serving
            for take in waiting.values():
                for _, fut in take:
                    fut.set_exception(e)
            return
        for slot, take in waiting.items():
            wav, a = wavs[slot], 0
            n = len(wav) // max(1, pieces[slot].shape[-1])  # samples per frame
            for codes, fut in take:
                k = codes.shape[-1]
                fut.set_result(wav[a * n: (a + k) * n])
                a += k


class _ChunkAudio:
    """Audio of the text chunk being generated: filled piece by piece (streaming) or in one go."""

    def __init__(self, engine: "TTSInferenceEngine"):
        self.engine = engine
        self.stream = None
        self.slot: Optional[int] = None  # slot of the engine's shared stream pool, when it has one free
        self.pieces: list[np.ndarray] = []
        self.frames = 0

    def push_partial(self, codes: torch.Tensor) -> np.ndarray:
        worker = self.engine.codec_worker
        if self.stream is None and self.slot is None:
            self.slot = worker.open() if worker is not None else None
            if self.slot is None:
                self.stream = self.engine.open_decode_stream()
        if self.slot is not None:
            wav = worker.decode(self.slot, codes)
        else:
            wav = self.stream.push(codes[None])[0, 0].float().cpu().numpy()
        self.pieces.append(wav)
        self.frames += codes.shape[-1]
        return wav

    def close(self) -> None:
        """Gives the chunk's pool slot back."""
        if self.slot is not None:
            self.engine.codec_worker.release(self.slot)
            self.slot = None

    def finish(self, codes: torch.Tensor) -> Optional[np.ndarray]:
        """End of the chunk: `codes` are all of its frames. Returns audio that has not been handed out yet."""
        rest = None
        if self.frames == 0:  # nothing was streamed: the reference's one-shot decode
            rest = self.engine.decode_vq_tokens(codes=codes).float().cpu().numpy()
            self.pieces.append(rest)
        elif self.frames < codes.shape[-1]:  # frames the worker did not announce separately
            rest = self.push_partial(codes[:, self.frames:])
        self.close()
        return rest

    def audio(self) -> np.ndarray:
        return np.concatenate(self.pieces, axis=0)


class TTSInferenceEngine(ReferenceLoader, VQManager):
    def __init__(self, llama_queue: queue.Queue, decoder_model: DAC, precision: torch.dtype, compile: bool) -> None:
        super().__init__()
        self.llama_queue = llama_queue
        self.decoder_model = decoder_model
        self.precision = precision
        self.compile = compile
        self.stream_frames = int(os.environ.get("FSB_STREAM_FRAMES", "8"))
        self.last_first_audio_s: Optional[float] = None  # request start -> first audio samples handed out
        # FSB_STREAM_POOL=n: the streaming requests of this engine share one n-slot DecodeStreamPool
        n_pool = int(os.environ.get("FSB_STREAM_POOL", "0") or 0)
        self.codec_worker: Optional[CodecStreamWorker] = None
        if n_pool > 0:
            pool = decoder_model.open_stream_pool(n_pool, k_max=max(32, self.stream_frames))
            self.codec_worker = CodecStreamWorker(pool, decoder_model.device)

    @torch.inference_mode()
    def inference(self, req: ServeTTSRequest) -> Generator[InferenceResult, None, None]:
        t_start = time.perf_counter()
        self.last_first_audio_s = None
        if req.reference_id is not None:
            prompt_tokens, prompt_texts = self.load_by_id(req.reference_id, req.use_memory_cache)
        elif req.references:
            prompt_tokens, prompt_texts = self.load_by_hash(req.references, req.use_memory_cache)
        else:
            prompt_tokens, prompt_texts = [], []
        if req.seed is not None:
            set_seed(req.seed)
            logger.warning(f"set seed: {req.seed}")
        responses = self.send_Llama_request(req, prompt_tokens, prompt_texts)
        rate = self.decoder_model.sample_rate
        if req.streaming:
            yield InferenceResult(code="header", audio=(rate, np.array(wav_chunk_header(sample_rate=rate))), error=None)
        finished: list[np.ndarray] = []
        chunk = _ChunkAudio(self)

        def hand_out(wav):
            if self.last_first_audio_s is None:
                self.last_first_audio_s = time.perf_counter() - t_start
            return InferenceResult(code="segment", audio=(rate, wav), error=None)

        # a CUDA stream of our own: the LM worker thread keeps its stream busy with decode frames meanwhile
        dev = self.decoder_model.device
        side = torch.cuda.Stream(device=dev) if torch.cuda.is_available() and dev.type == "cuda" else None
        try:
            while True:
                wrapped: WrappedGenerateResponse = responses.get()
                if wrapped.status == "error":
                    err = wrapped.response if isinstance(wrapped.response, Exception) else Exception("Unknown error")
                    yield InferenceResult(code="error", audio=None, error=err)
                    return
                result = wrapped.response
                if not isinstance(result, GenerateResponse):
                    raise TypeError(f"Expected GenerateResponse, got {type(result).__name__}")
                if result.action == "next":
                    break
                with (torch.cuda.stream(side) if side is not None else _nullcontext()):
                    if result.action == "partial":
                        wav = chunk.push_partial(result.codes)
                    else:  # "sample": the chunk is complete
                        wav = chunk.finish(result.codes)
                        finished.append(chunk.audio())
                        chunk = _ChunkAudio(self)
                if wav is not None and wav.size and req.streaming:
                    yield hand_out(wav)
        finally:
            chunk.close()  # a request that ends inside a chunk (error, abandoned generator) gives its pool slot back
            cancel = getattr(responses, "cancel", None)
            if cancel is not None:
                cancel.set()  # ... and its LM slot: the slot scheduler takes a request still in flight out
        if not finished:
            yield InferenceResult(code="error", audio=None,
                                  error=RuntimeError("No audio generated, please check the input text."))
            return
        if self.last_first_audio_s is None:
            self.last_first_audio_s = time.perf_counter() - t_start
        yield InferenceResult(code="final", audio=(rate, np.concatenate(finished, axis=0)), error=None)

    def send_Llama_request(self, req: ServeTTSRequest, prompt_tokens: list, prompt_texts: list) -> queue.Queue:
        """Queue one generate_long call on the LM worker (inference.py:736-799); the answer comes on the returned queue."""
        request = dict(
            device=self.decoder_model.device, max_new_tokens=req.max_new_tokens, text=req.text, top_p=req.top_p,
            repetition_penalty=req.repetition_penalty, temperature=req.temperature, compile=self.compile,
            iterative_prompt=req.chunk_length > 0, chunk_length=req.chunk_length, prompt_tokens=prompt_tokens,
            prompt_text=prompt_texts)
        if req.streaming and self.stream_frames > 0:
            request["stream_frames"] = self.stream_frames
        response_queue: queue.Queue = queue.Queue()
        response_queue.cancel = request["cancel"] = threading.Event()  # set when the caller stops listening
        self.llama_queue.put(GenerateRequest(request=request, response_queue=response_queue))
        return response_queue

    def get_audio_segment(self, result: GenerateResponse) -> np.ndarray:
        """One-shot decode of a finished chunk. The codec computes in bf16 with fp32 accumulation whatever `precision`
        says (the reference wraps this call in torch.autocast(bf16), inference_engine/__init__.py:185-189)."""
        return self.decode_vq_tokens(codes=result.codes).float().cpu().numpy()


class _nullcontext:
    def __enter__(self):
        return None

    def __exit__(self, *a):
        return False
