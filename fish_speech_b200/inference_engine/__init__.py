"""TTSInferenceEngine — the surface of fish_speech/inference_engine/__init__.py (`inference` :22-142,
`send_Llama_request` :144-177, `get_audio_segment` :179-192) with the codec stage overlapped with generation.

The reference turns a chunk's codes into audio only after the LM has finished the chunk. Here a streaming request asks
the LM worker for the codes of finished frames while it keeps decoding (`stream_frames`, "partial" responses), and this
thread pushes them through an incremental codec decoder (`DAC.open_decode_stream`) on its own CUDA stream: audio leaves
with a delay of a few frames instead of a whole chunk (SURVEY §8(f).3). With FSB_STREAM_POOL=n the streaming requests
share one n-slot `DAC.open_stream_pool` behind a codec thread (`CodecStreamWorker`) that decodes the pieces of every
stream in one batched push. Non-streaming requests follow the reference:
one `from_indices` per chunk. The result protocol is the reference's: header | segment* | final, or error.

A request may ask for its audio at another `sample_rate` and in another `sample_format` (schema.ServeTTSRequest):
the conversion runs on the device (`audio.convert_out` per chunk, or the decode stream's / pool slot's own
`OutputStream`), and only the converted samples are copied to the host.
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

from .. import audio as _audio
from ..models.dac.modded_dac import DAC
from ..models.text2semantic.inference import GenerateRequest, GenerateResponse, WrappedGenerateResponse
from .reference_loader import ReferenceLoader
from .schema import ServeTTSRequest
from .utils import WAVE_OF_FORMAT, InferenceResult, wav_chunk_header
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
    An error in a push is delivered to every caller that waits on it; the worker keeps serving. A slot opened with a
    sample rate or format gets its converted samples back; they are not a fixed number per frame, so all of a push's
    samples go to the last of the slot's pieces it took, and `finish` flushes the slot on the worker's stream."""

    def __init__(self, pool, device: Optional[torch.device] = None):
        self.pool = pool
        self.k_max = int(pool.k_max)
        self._q: queue.Queue = queue.Queue()
        self._lock = threading.Lock()
        self._device = device
        self.pushes = 0  # pool pushes run (tests, measurements)
        self._converted: set = set()  # slots opened with a sample rate or format
        self._thread = threading.Thread(target=self._run, name="codec-stream-pool", daemon=True)
        self._thread.start()

    def open(self, sample_rate: Optional[int] = None, sample_format: Optional[str] = None) -> Optional[int]:
        """A slot of the pool, or None when it is full (the caller decodes on a stream of its own)."""
        with self._lock:
            try:
                slot = self.pool.open() if sample_rate is None and sample_format is None else \
                    self.pool.open(sample_rate=sample_rate, sample_format=sample_format)
            except ValueError:
                return None
            if sample_rate is None and sample_format is None:
                self._converted.discard(slot)
            else:
                self._converted.add(slot)
            return slot

    def release(self, slot: int) -> None:
        """Closes a stream's slot of the pool."""
        with self._lock:
            self.pool.close(slot)
            self._converted.discard(slot)

    def submit(self, slot: int, codes: Optional[torch.Tensor]) -> Future:
        """codes [C, k], k <= k_max -> future of the waveform (fp32 numpy [k * frame_length], or a converted slot's
        samples); None -> future of the slot's flush (pool.flush)."""
        if codes is not None and not 1 <= codes.shape[-1] <= self.k_max:
            raise ValueError(f"a piece takes 1 .. {self.k_max} frames, got {codes.shape[-1]}")
        fut: Future = Future()
        self._q.put((slot, codes, fut))
        return fut

    def decode(self, slot: int, codes: torch.Tensor) -> np.ndarray:
        """The next frames of one stream, in pieces of at most k_max frames; blocks until decoded."""
        futs = [self.submit(slot, codes[:, a: a + self.k_max]) for a in range(0, codes.shape[-1], self.k_max)]
        return np.concatenate([f.result() for f in futs]) if len(futs) > 1 else futs[0].result()

    def flush(self, slot: int) -> np.ndarray:
        """The samples a converted slot still holds back (after every piece submitted before); blocks until done."""
        return self.submit(slot, None).result()

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
                    pieces, waiting, flushes = {}, {}, []
                    for slot in list(per_slot):
                        q = per_slot[slot]
                        take, k = [], 0
                        while q and q[0][0] is not None and k + q[0][0].shape[-1] <= self.k_max:
                            take.append(q.pop(0))
                            k += take[-1][0].shape[-1]
                        if take:
                            waiting[slot] = take
                            pieces[slot] = take[0][0] if len(take) == 1 else torch.cat([c for c, _ in take], dim=-1)
                        else:  # a flush, after every piece before it
                            flushes.append((slot, q.pop(0)[1]))
                        if not q:
                            del per_slot[slot]
                    if pieces:
                        self._push(pieces, waiting, side)
                    for slot, fut in flushes:
                        self._flush(slot, fut, side)
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
                # synchronises the worker's stream; converted slots keep their dtype
                wavs = {s: (w.cpu() if s in self._converted else w.float().cpu()).numpy() for s, w in out.items()}
            self.pushes += 1
        except BaseException as e:  # every caller of this push sees the error; the worker keeps serving
            for take in waiting.values():
                for _, fut in take:
                    fut.set_exception(e)
            return
        for slot, take in waiting.items():
            wav, a = wavs[slot], 0
            if slot in self._converted:
                for _, fut in take[:-1]:
                    fut.set_result(wav[:0])
                take[-1][1].set_result(wav)
                continue
            n = len(wav) // max(1, pieces[slot].shape[-1])  # samples per frame
            for codes, fut in take:
                k = codes.shape[-1]
                fut.set_result(wav[a * n: (a + k) * n])
                a += k

    def _flush(self, slot: int, fut: Future, side):
        try:
            with torch.inference_mode(), (torch.cuda.stream(side) if side is not None else _nullcontext()):
                rest = self.pool.flush(slot).cpu().numpy()
        except BaseException as e:
            fut.set_exception(e)
            return
        fut.set_result(rest)


class _ChunkAudio:
    """Audio of the text chunk being generated: filled piece by piece (streaming) or in one go. `sample_rate` /
    `sample_format` (None: the codec's fp32 at its own rate) are the request's output conversion."""

    def __init__(self, engine: "TTSInferenceEngine", sample_rate: Optional[int] = None,
                 sample_format: Optional[str] = None):
        self.engine = engine
        self.sample_rate, self.sample_format = sample_rate, sample_format
        self.converted = sample_rate is not None or sample_format is not None
        self.stream = None
        self.slot: Optional[int] = None  # slot of the engine's shared stream pool, when it has one free
        self.pieces: list[np.ndarray] = []
        self.frames = 0

    def push_partial(self, codes: torch.Tensor) -> np.ndarray:
        worker = self.engine.codec_worker
        if self.stream is None and self.slot is None:
            if worker is not None:
                self.slot = worker.open(self.sample_rate, self.sample_format) if self.converted else worker.open()
            if self.slot is None:
                self.stream = self.engine.open_decode_stream(sample_rate=self.sample_rate,
                                                             sample_format=self.sample_format) \
                    if self.converted else self.engine.open_decode_stream()
        if self.slot is not None:
            wav = worker.decode(self.slot, codes)
        else:
            wav = self._host(self.stream.push(codes[None])[0, 0])
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
            wav = self.engine.decode_vq_tokens(codes=codes)
            if self.converted:
                wav = _audio.convert_out(wav, self.sample_rate, self.sample_format,
                                         orig_freq=self.engine.decoder_model.sample_rate)
            rest = self._host(wav)
            self.pieces.append(rest)
        elif self.frames < codes.shape[-1]:  # frames the worker did not announce separately
            rest = self.push_partial(codes[:, self.frames:])
        if self.converted and self.frames > 0:  # the samples the resampler's look-ahead held back
            tail = self.engine.codec_worker.flush(self.slot) if self.slot is not None else \
                self._host(self.stream.flush()[0, 0])
            self.pieces.append(tail)
            rest = tail if rest is None else np.concatenate([rest, tail])
        self.close()
        return rest

    def _host(self, wav: torch.Tensor) -> np.ndarray:
        """Device samples -> numpy: the codec's fp32 (as float) or the converted samples in their own dtype."""
        return (wav.cpu() if self.converted else wav.float().cpu()).numpy()

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
        out_rate, out_format = getattr(req, "sample_rate", None), getattr(req, "sample_format", None)
        if out_rate is not None and int(out_rate) <= 0:
            raise ValueError(f"sample_rate must be positive (got {out_rate})")
        if out_format is not None:
            _audio.output_format(out_format)  # a bad name fails before any work
        responses = self.send_Llama_request(req, prompt_tokens, prompt_texts)
        rate = self.decoder_model.sample_rate if out_rate is None else int(out_rate)
        if req.streaming:
            if out_format is None:
                header = wav_chunk_header(sample_rate=rate)
            else:
                bits, tag = WAVE_OF_FORMAT[out_format]
                header = wav_chunk_header(sample_rate=rate, bit_depth=bits, format_tag=tag)
            yield InferenceResult(code="header", audio=(rate, np.array(header)), error=None)
        finished: list[np.ndarray] = []
        chunk = _ChunkAudio(self, out_rate, out_format)

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
                        chunk = _ChunkAudio(self, out_rate, out_format)
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
