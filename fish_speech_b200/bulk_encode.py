"""Bulk audio -> VQ codes at dataset scale (SURVEY.md 8f.4): the job of tools/vqgan/extract_vq.py:90-240.

Same contract as the reference tool — every audio file under a folder (or in a filelist) gets a `<stem>.npy` with its
codes `[n_codebooks + 1, T]` (int64 in the reference; here too), files that already have one are skipped, rank r of
`world` workers takes `files[r::world]` (SLURM_PROCID / SLURM_NTASKS, or RANK / WORLD_SIZE under torchrun), and
`--num-workers N` re-spawns the script once per GPU — but built around the CUDA codec:

  * one padded-batch `DAC.encode` per batch (the encoder, both downsampling stages, the window-limited transformer and
    the 10 residual VQ stages run as tcgen05 GEMMs / fused kernels; the post-module pass whose result the reference
    throws away is not computed),
  * batches are formed from files of similar duration (sorted by length inside a window of the shard), so a padded
    batch wastes little compute, and capped by total padded seconds as well as by file count,
  * a reader thread reads the next batches while the GPU encodes the current one. With a CUDA codec it only reads
    (the raw frames of a PCM wav, the decoded array of any other file): conversion, down-mix, resampling to the
    codec's rate and padding run on the device (fish_speech_b200.audio.load_batch); a codec on the CPU gets
    converted, resampled waveforms as before.
"""
from __future__ import annotations

import os
import queue
import threading
import time
import wave
from dataclasses import dataclass
from pathlib import Path
from typing import Callable, Iterable, Optional, Sequence

import numpy as np
import torch

from . import audio

try:
    from loguru import logger
except Exception:  # pragma: no cover
    import logging

    logger = logging.getLogger("fish_speech_b200")

AUDIO_EXTENSIONS = {".mp3", ".wav", ".flac", ".ogg", ".m4a", ".wma", ".aac", ".aiff", ".aif", ".aifc"}


def worker_identity() -> tuple[int, int]:
    """(rank, world) of this worker: SLURM variables as in the reference (extract_vq.py:43-44), else torchrun's."""
    if "SLURM_PROCID" in os.environ:
        return int(os.environ["SLURM_PROCID"]), int(os.environ.get("SLURM_NTASKS", 1))
    return int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))


def list_audio_files(folder: Path | str, filelist: Optional[Path] = None) -> list[Path]:
    """Audio files below `folder` (recursive), or the first column of a `|`-separated filelist."""
    if filelist is not None:
        rows = [ln.strip() for ln in Path(filelist).read_text(encoding="utf-8").splitlines() if ln.strip()]
        return [Path(r.split("|")[0]) for r in rows]
    root = Path(folder)
    return sorted(p for p in root.rglob("*") if p.is_file() and p.suffix.lower() in AUDIO_EXTENSIONS)


def pending_files(files: Sequence[Path], rank: int, world: int) -> list[Path]:
    """Files without a `.npy` next to them, then this worker's stride (extract_vq.py:199-203)."""
    todo = [Path(f) for f in files if not Path(f).with_suffix(".npy").exists()]
    return todo[rank::world]


def read_audio(path: Path) -> tuple[torch.Tensor, int]:
    """Mono float32 waveform [N] and its sample rate. soundfile, then torchaudio, then the stdlib PCM-wav reader."""
    try:
        import soundfile as sf

        data, sr = sf.read(str(path), dtype="float32", always_2d=True)
        return torch.from_numpy(data).mean(dim=1), int(sr)
    except Exception:  # not installed, or a format libsndfile cannot decode: the next reader may
        pass
    try:
        import torchaudio

        wav, sr = torchaudio.load(str(path))
        return wav.mean(dim=0).float(), int(sr)
    except Exception:
        if path.suffix.lower() != ".wav":
            raise
    with wave.open(str(path), "rb") as f:
        sr, nch, width, n = f.getframerate(), f.getnchannels(), f.getsampwidth(), f.getnframes()
        raw = f.readframes(n)
    if width == 2:
        x = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif width == 4:
        x = np.frombuffer(raw, dtype="<i4").astype(np.float32) / 2147483648.0
    elif width == 1:
        x = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    else:
        raise ValueError(f"{path}: unsupported PCM width {width}")
    return torch.from_numpy(x.reshape(-1, nch).mean(axis=1).copy()), int(sr)


def resample(wav: torch.Tensor, sr: int, target: int) -> torch.Tensor:
    if sr == target:
        return wav
    import torchaudio

    return torchaudio.functional.resample(wav, sr, target)


@dataclass
class Clip:
    file: Path
    wav: Optional[torch.Tensor]  # [N] float32 at the codec's sample rate (CPU codec)
    pcm: Optional[audio.Pcm] = None  # the file as read, converted on the device (CUDA codec)
    length: int = 0  # samples at the codec's sample rate

    def __post_init__(self):
        if self.wav is not None:
            self.length = int(self.wav.numel())


def _device_front_end(model) -> bool:
    """Whether audio for `model` is converted and resampled on its device: a CUDA codec."""
    return torch.device(model.device).type == "cuda"


def plan_batches(lengths: Sequence[int], batch_size: int, max_padded_samples: int, window: int = 1024) -> list[list[int]]:
    """Indices grouped into batches. Inside consecutive windows of `window` items the clips are sorted by length, so
    a batch holds similar durations; a batch closes at `batch_size` clips or when (clips x longest clip) would exceed
    `max_padded_samples`. Every index appears exactly once; a clip longer than the cap forms a batch of its own."""
    batches: list[list[int]] = []
    for w0 in range(0, len(lengths), window):
        order = sorted(range(w0, min(w0 + window, len(lengths))), key=lambda i: lengths[i])
        cur: list[int] = []
        for i in order:
            longest = max(lengths[i], max((lengths[j] for j in cur), default=0))
            if cur and (len(cur) >= batch_size or (len(cur) + 1) * longest > max_padded_samples):
                batches.append(cur)
                cur = []
            cur.append(i)
        if cur:
            batches.append(cur)
    return batches


@torch.inference_mode()
def encode_batch(clips: Sequence[Clip], model) -> float:
    """One padded `model.encode` call; writes `<file>.npy` = codes[:, :frames] per clip (extract_vq.py:118-140).
    Returns the seconds of audio encoded."""
    if not clips:
        return 0.0
    device = model.device
    lens = [c.length for c in clips]
    if clips[0].pcm is not None:
        audios, audio_lengths = audio.load_batch([c.pcm for c in clips], int(model.sample_rate), device)
    else:
        audios = torch.zeros(len(clips), 1, max(lens), dtype=torch.float32)
        for k, c in enumerate(clips):
            audios[k, 0, : lens[k]] = c.wav
        audios = audios.pin_memory().to(device, non_blocking=True) if torch.device(device).type == "cuda" else audios.to(device)
        audio_lengths = torch.tensor(lens, device=device, dtype=torch.long)
    indices, feature_lengths = model.encode(audios, audio_lengths)
    out = indices.cpu().numpy()
    for c, n, feat in zip(clips, feature_lengths.tolist(), out):
        tmp = c.file.with_suffix(".npy.tmp")
        with open(tmp, "wb") as f:
            np.save(f, feat[:, : int(n)])
        os.replace(tmp, c.file.with_suffix(".npy"))  # a killed worker never leaves a truncated .npy behind
    return sum(lens) / float(model.sample_rate)


def decode_audio_bytes(data: bytes) -> tuple[torch.Tensor, int]:
    """Mono float32 waveform [N] and sample rate of an encoded audio file held in memory (the server receives reference
    audio as bytes): soundfile, then the stdlib PCM-wav reader."""
    import io

    try:
        import soundfile as sf

        x, sr = sf.read(io.BytesIO(data), dtype="float32", always_2d=True)
        return torch.from_numpy(x).mean(dim=1), int(sr)
    except Exception:
        pass
    with wave.open(io.BytesIO(data), "rb") as f:
        sr, nch, width, n = f.getframerate(), f.getnchannels(), f.getsampwidth(), f.getnframes()
        raw = f.readframes(n)
    if width != 2:
        raise ValueError(f"unsupported PCM width {width} in an in-memory wav")
    x = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    return torch.from_numpy(x.reshape(-1, nch).mean(axis=1).copy()), int(sr)


@torch.inference_mode()
def batch_encode(model, audios_list: Sequence) -> list[torch.Tensor]:
    """tools/server/model_utils.py:15-48: several reference audios (encoded bytes, or waveforms [1, N] at the codec's
    sample rate) -> one padded `model.encode` call -> per item its codes [n_codebooks, frames_i] on the host, padding
    frames cut off. (The reference runs this under fp16 autocast; the CUDA codec computes in bf16 / fp32 accumulate.)"""
    sr = int(model.sample_rate)
    if not audios_list:
        return []
    device = model.device
    if _device_front_end(model):
        pcms = [audio.pcm_from_bytes(bytes(a)) if isinstance(a, (bytes, bytearray))
                else audio.pcm_from_array(torch.as_tensor(a, dtype=torch.float32).reshape(-1), sr) for a in audios_list]
        padded, lengths = audio.load_batch(pcms, sr, device)
        features, feature_lengths = model.encode(padded, lengths)
        features, feature_lengths = features.cpu(), feature_lengths.cpu()
        return [f[..., : int(n)] for f, n in zip(features, feature_lengths)]
    audios = []
    for a in audios_list:
        if isinstance(a, (bytes, bytearray)):
            wav, file_sr = decode_audio_bytes(bytes(a))
            audios.append(resample(wav, file_sr, sr)[None])
        else:
            audios.append(torch.as_tensor(a, dtype=torch.float32).reshape(1, -1))
    lens = [int(x.shape[-1]) for x in audios]
    padded = torch.zeros(len(audios), 1, max(lens), dtype=torch.float32)
    for k, x in enumerate(audios):
        padded[k, 0, : lens[k]] = x[0]
    lengths = torch.tensor(lens, device=device, dtype=torch.long)
    features, feature_lengths = model.encode(padded.to(device), lengths)
    features, feature_lengths = features.cpu(), feature_lengths.cpu()
    return [f[..., : int(n)] for f, n in zip(features, feature_lengths)]


@torch.inference_mode()
def batch_vqgan_decode(model, features: Sequence) -> list[np.ndarray]:
    """tools/server/model_utils.py:59-86: codes of several utterances ([1 + n_codebooks, T_i] each, any integer dtype)
    -> per item its waveform, float32 numpy [1, T_i * frame_length], in input order. Instead of padded micro-batches,
    the items share `model.from_indices_list`'s decode pool, each bit-identical to `model.from_indices` of that item
    alone. A malformed item raises ValueError naming it."""
    return [w.cpu().numpy()[None] for w in model.from_indices_list(features)]


def encode_files(files: Sequence[Path], model, batch_size: int = 64, max_batch_seconds: float = 1800.0,
                 reader: Callable[[Path], tuple[torch.Tensor, int]] = read_audio, prefetch: int = 2,
                 progress: Optional[Callable[[int, float], None]] = None) -> tuple[int, float]:
    """Encode `files` with `model` (a DAC): a reader thread loads the clips of the next batches while the current one is
    on the GPU. With a CUDA codec the reader only reads (`audio.read_pcm`, or `reader`'s waveform taken as it is) and
    the device converts, down-mixes and resamples; otherwise the reader thread does that. Unreadable files are logged
    and skipped, like the reference does (extract_vq.py:97-104). Returns (files written, seconds of audio)."""
    files = [Path(f) for f in files]
    sr = int(model.sample_rate)
    on_device = _device_front_end(model)

    def load(p: Path) -> Clip:
        if not on_device:
            wav, file_sr = reader(p)
            return Clip(p, resample(wav.float().flatten(), file_sr, sr).contiguous())
        if reader is read_audio:
            pcm = audio.read_pcm(p)
        else:
            wav, file_sr = reader(p)
            pcm = audio.pcm_from_array(wav.float().flatten(), file_sr)
        return Clip(p, None, pcm, pcm.out_length(sr))

    def probe(p: Path) -> int:
        """Cheap length estimate for batch planning: file size (compressed formats sort roughly by duration too)."""
        try:
            return p.stat().st_size
        except OSError:
            return 0

    sizes = [probe(p) for p in files]
    # the padded-seconds cap is applied on real sample counts after loading; planning uses sizes only to group
    plan = plan_batches(sizes, batch_size, max_padded_samples=max(sizes, default=0) * batch_size + 1)
    q: "queue.Queue[Optional[list[Clip]]]" = queue.Queue(maxsize=max(1, prefetch))

    def produce():
        try:
            for idxs in plan:
                clips: list[Clip] = []
                for i in idxs:
                    try:
                        clips.append(load(files[i]))
                    except Exception as e:  # noqa: BLE001 - a bad file must not stop the shard
                        logger.error(f"Error reading {files[i]}: {e}")
                # split again on true lengths if padding would exceed the cap
                lens = [c.length for c in clips]
                for sub in plan_batches(lens, batch_size, int(max_batch_seconds * sr)):
                    q.put([clips[j] for j in sub])
        finally:
            q.put(None)

    t = threading.Thread(target=produce, daemon=True)
    t.start()
    done, seconds = 0, 0.0
    while True:
        clips = q.get()
        if clips is None:
            break
        seconds += encode_batch(clips, model)
        done += len(clips)
        if progress is not None:
            progress(done, seconds)
    t.join()
    return done, seconds


def run_worker(folder: str, config_name: str, checkpoint_path: str, batch_size: int, filelist: Optional[Path],
               device: str = "cuda") -> tuple[int, float]:
    from .models.dac.inference import load_model

    rank, world = worker_identity()
    files = list_audio_files(folder, filelist)
    logger.info(f"Found {len(files)} files")
    mine = pending_files(files, rank, world)
    logger.info(f"[rank {rank}/{world}] processing {len(mine)} files")
    model = load_model(config_name, checkpoint_path, device=device)
    t0 = time.time()

    def progress(n: int, secs: float):
        if n and (n // batch_size) % 10 == 0:
            eta = (time.time() - t0) / n * (len(mine) - n)
            logger.info(f"Processed {n} files, {secs / 3600:.2f} hours of audio, ETA {eta:.0f}s")

    n, secs = encode_files(mine, model, batch_size=batch_size, progress=progress)
    logger.info(f"Finished processing {n} files, {secs / 3600:.2f} hours of audio")
    return n, secs
