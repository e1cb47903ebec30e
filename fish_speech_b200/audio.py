"""Codec input and output front ends on the device: PCM at any sample rate -> the codec's mono fp32 input, and the
decoder's fp32 44.1 kHz output -> the client's sample rate and sample format.

* `resample(x, orig_freq, new_freq)`: `torchaudio.functional.resample` with its defaults (sinc_interp_hann,
  lowpass_filter_width 6, rolloff 0.99). On a CUDA float32 tensor it runs `fsb_resample` (csrc/audio_kernels.cu); on
  a CPU tensor, or with other filter settings, it is torchaudio itself.
* `Pcm` / `read_pcm` / `pcm_from_bytes` / `pcm_from_array`: what a reader thread produces without converting anything
  (the raw frames of a PCM wav, or a decoded array), and `load_batch`, which turns many of them, at any rates, into the
  zero-padded `[B, 1, N_max]` batch and lengths that `DAC.encode` takes: one upload, one conversion launch, one
  resample launch.
* `StreamResampler`: the same resampler over a signal that arrives in pieces. Each push emits the outputs whose filter
  window is complete and keeps on the device the input history the next outputs read; `flush` emits the tail against
  zero right-padding. The concatenated outputs are bit-identical to `resample` of the whole signal.
* `convert_out` / `OutputStream`: the same resampler run from the decoder's rate to the client's, with the sample
  format (float32, int16 PCM as `inference_engine.utils.pcm16`, or G.711 mu-law) fused into the same launch
  (`fsb_audio_out`), one-shot and streamed with the same bits.

The filter table is built on the host in float64 from torchaudio's formula (`filter_table`) and cast to fp32 once per
rate pair and device. Taps where the Hann window is zero are dropped, so each output is one fixed sequence of fp64
fma over its phase's non-zero taps, in ascending order, rounded to fp32 once: its bits depend only on the samples it
reads.
"""
from __future__ import annotations

import functools
import io
import math
import threading
import wave
from dataclasses import dataclass
from pathlib import Path
from typing import Optional, Sequence, Union

import numpy as np
import torch

from . import _lib

LOWPASS_FILTER_WIDTH = 6
ROLLOFF = 0.99

# fsb_pcm_clip.format (include/fishb200.h FSB_PCM_*), by sample width in bytes for integer PCM
PCM_S16, PCM_S32, PCM_U8, PCM_F32 = 0, 1, 2, 3
_PCM_OF_WIDTH = {2: PCM_S16, 4: PCM_S32, 1: PCM_U8}
_PCM_BYTES = {PCM_S16: 2, PCM_S32: 4, PCM_U8: 1, PCM_F32: 4}


# ---------------------------------------------------------------------------------------------------------------------
# filter table and stream arithmetic (host only)
# ---------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class FilterTable:
    """torchaudio's sinc_interp_hann kernel for orig -> new (both divided by their gcd), non-zero taps only.

    Output j = q * new + p reads input samples q * orig + first[p] + m, m in [0, count[p]), with weights w[p, m]
    (float64; rows padded with zeros to `taps`). `first` and `last` = first + count - 1 never decrease from one
    output to the next, so the outputs whose window lies inside the first M samples form a prefix (`ready`)."""

    orig: int
    new: int
    w: np.ndarray       # float64 [new, taps]
    first: np.ndarray   # int64 [new]
    count: np.ndarray   # int64 [new]

    @property
    def taps(self) -> int:
        return int(self.w.shape[1])

    def total(self, n: int) -> int:
        """Output length of a whole signal of n samples, as torchaudio computes it: ceil(new * n / orig) of the
        quotient rounded to fp32 (torch.as_tensor of a Python float), which for long clips can be one less (or, past
        2^24 outputs, more) than the exact ceiling. Never decreases as n grows."""
        return int(math.ceil(np.float32(self.new * int(n) / self.orig)))

    def ready(self, m: int) -> int:
        """Outputs computable from the first m samples of a signal that goes on: those whose last tap is below m (and
        never more than a signal of exactly m samples has)."""
        last = self.first + self.count - 1
        n = np.maximum(0, -((last - int(m)) // self.orig)).sum()  # per phase: #q >= 0 with q * orig + last < m
        return int(min(n, self.total(m)))

    def first_input(self, j: int) -> int:
        """The first input sample output j reads (may be negative: samples before 0 are zeros)."""
        q, p = divmod(int(j), self.new)
        return q * self.orig + int(self.first[p])


@functools.lru_cache(maxsize=64)
def filter_table(orig_freq: int, new_freq: int) -> FilterTable:
    """The table of torchaudio.functional._get_sinc_resample_kernel (sinc_interp_hann, lowpass_filter_width 6,
    rolloff 0.99) in float64, evaluated in the same order of operations. Taps where |t| reaches the filter width,
    where the Hann window is zero, are dropped."""
    if orig_freq <= 0 or new_freq <= 0:
        raise ValueError(f"sample rates must be positive (got {orig_freq}, {new_freq})")
    g = math.gcd(int(orig_freq), int(new_freq))
    orig, new = int(orig_freq) // g, int(new_freq) // g
    lpw = LOWPASS_FILTER_WIDTH
    base = min(orig, new) * ROLLOFF
    width = math.ceil(lpw * orig / base)
    idx = np.arange(-width, width + orig, dtype=np.float64)[None] / orig
    t = np.arange(0, -new, -1, dtype=np.float64)[:, None] / new + idx
    t *= base
    inside = np.abs(t) < lpw
    t = np.clip(t, -lpw, lpw)
    window = np.cos(t * math.pi / lpw / 2) ** 2
    t *= math.pi
    scale = base / orig
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(t == 0, 1.0, np.sin(t) / t)
    k *= window * scale
    k[~inside] = 0.0
    nz = k != 0
    first_k = nz.argmax(axis=1)
    count = nz.sum(axis=1)
    taps = int(count.max())
    w = np.zeros((new, taps), dtype=np.float64)
    for p in range(new):
        seg = k[p, first_k[p]: first_k[p] + count[p]]
        assert np.all(seg != 0), "non-zero taps of a phase are contiguous"
        w[p, : count[p]] = seg
    first = first_k.astype(np.int64) - width
    last = first + count - 1
    # monotone from one output to the next, across the phase wrap too: `ready` counts a prefix
    assert np.all(np.diff(first) >= 0) and np.all(np.diff(last) >= 0)
    assert first[0] + orig >= first[-1] and last[0] + orig >= last[-1]
    return FilterTable(orig, new, w, first, count.astype(np.int64))


def apply_table(table: FilterTable, x: np.ndarray) -> np.ndarray:
    """The resampler in float64 on the host: what the kernel computes, for checking the table."""
    x = np.asarray(x, dtype=np.float64)
    n = x.shape[-1]
    out_n = table.total(n)
    pad_l = max(0, -int(table.first.min()))
    xp = np.concatenate([np.zeros(pad_l), x, np.zeros(table.orig + table.taps + 1)])
    j = np.arange(out_n)
    q, p = j // table.new, j % table.new
    i0 = q * table.orig + table.first[p] + pad_l
    out = np.zeros(out_n)
    for m in range(table.taps):
        out += table.w[p, m] * xp[i0 + m]  # w is 0 past a phase's count
    return out


class StreamCounts:
    """The host arithmetic of a resampled stream: after each push of `m` samples, which outputs are emitted and from
    which input sample on history must be kept; `flush` emits the rest. `StreamResampler` runs on it."""

    def __init__(self, table: FilterTable):
        self.table = table
        self.received = 0   # input samples pushed
        self.emitted = 0    # outputs emitted
        self.done = False

    def push(self, m: int) -> tuple[int, int, int]:
        """-> (first output, outputs now ready, first input sample still needed)."""
        if self.done:
            raise ValueError("stream was flushed")
        self.received += int(m)
        j0 = self.emitted
        self.emitted = max(j0, self.table.ready(self.received))
        return j0, self.emitted - j0, self.keep_from()

    def flush(self) -> tuple[int, int]:
        """-> (first output, outputs left): everything a whole signal of `received` samples has."""
        if self.done:
            raise ValueError("stream was flushed")
        self.done = True
        j0 = self.emitted
        self.emitted = self.table.total(self.received)
        return j0, self.emitted - j0

    def keep_from(self) -> int:
        return min(max(0, self.table.first_input(self.emitted)), self.received)


# ---------------------------------------------------------------------------------------------------------------------
# device side
# ---------------------------------------------------------------------------------------------------------------------
_dev_tables: dict = {}
_dev_lock = threading.Lock()


def _device_table(orig_freq: int, new_freq: int, device: torch.device) -> tuple:
    """(fp32 weights [taps][new], int32 spans [new][2], orig, new) on `device`, cached per rate pair and device."""
    device = _device(device)
    key = (int(orig_freq), int(new_freq), str(device))
    with _dev_lock:
        hit = _dev_tables.get(key)
        if hit is None:
            t = filter_table(int(orig_freq), int(new_freq))
            w = torch.from_numpy(np.ascontiguousarray(t.w.T).astype(np.float32)).to(device)
            span = torch.from_numpy(np.stack([t.first, t.count], axis=1).astype(np.int32)).to(device)
            hit = (w, span, t.orig, t.new)
            _dev_tables[key] = hit
        return hit


def _device(device) -> torch.device:
    """`device` with its index: "cuda" is the current CUDA device."""
    d = torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if d.type == "cuda" and d.index is None else d


def _stream(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _launch_resample(x: torch.Tensor, rows: list, out: torch.Tensor, max_fill: int) -> None:
    """rows: per clip (x_off, x_start, x_end, j0, out_off, n_out, n_fill, table or None) -> one fsb_resample launch."""
    desc = []
    for x_off, x_start, x_end, j0, out_off, n_out, n_fill, tab in rows:
        if tab is None:
            w_ptr, s_ptr, o, n = 0, 0, 1, 1
        else:
            w_ptr, s_ptr, o, n = tab[0].data_ptr(), tab[1].data_ptr(), tab[2], tab[3]
        desc.append([x_off, x_start, x_end, j0, out_off, n_out, n_fill, w_ptr, s_ptr, o, n])
    d = torch.tensor(desc, dtype=torch.int64).to(x.device)
    _lib.check(_lib.lib().fsb_resample(x.data_ptr(), d.data_ptr(), len(rows), int(max_fill), out.data_ptr(),
                                       _stream(x.device)))


def _default_filter(lowpass_filter_width, rolloff, resampling_method, beta) -> bool:
    return (lowpass_filter_width == LOWPASS_FILTER_WIDTH and rolloff == ROLLOFF
            and resampling_method == "sinc_interp_hann")


def resample(waveform: torch.Tensor, orig_freq: int, new_freq: int, lowpass_filter_width: int = 6,
             rolloff: float = 0.99, resampling_method: str = "sinc_interp_hann",
             beta: Optional[float] = None) -> torch.Tensor:
    """torchaudio.functional.resample(waveform [..., N], orig_freq, new_freq) -> [..., ceil(new * N / orig)].
    A CUDA float32 waveform with the default filter is resampled by the device kernel, every row in one launch;
    orig_freq == new_freq returns the waveform itself. Anything else is torchaudio's own call."""
    if int(orig_freq) == int(new_freq):
        return waveform
    if waveform.device.type != "cuda" or not _default_filter(lowpass_filter_width, rolloff, resampling_method, beta):
        import torchaudio

        return torchaudio.functional.resample(waveform, orig_freq, new_freq, lowpass_filter_width=lowpass_filter_width,
                                              rolloff=rolloff, resampling_method=resampling_method, beta=beta)
    if waveform.dtype != torch.float32:
        raise TypeError(f"resample on CUDA takes float32 waveforms (got {waveform.dtype})")
    shape = waveform.shape
    n = int(shape[-1])
    x = waveform.reshape(-1, n).contiguous()
    rows = x.shape[0]
    with torch.cuda.device(x.device):
        tab = _device_table(orig_freq, new_freq, x.device)
        out_n = filter_table(int(orig_freq), int(new_freq)).total(n)
        out = torch.empty(rows, out_n, dtype=torch.float32, device=x.device)
        if rows and out_n:
            _launch_resample(x, [(r * n, 0, n, 0, r * out_n, out_n, out_n, tab) for r in range(rows)], out, out_n)
    return out.reshape(*shape[:-1], out_n)


@dataclass
class Pcm:
    """One clip as read, not converted: interleaved frames of `channels` samples in `fmt` (PCM_*), as raw little-endian
    bytes (integer PCM) or a float32 array [frames, channels]."""

    data: Union[bytes, np.ndarray]
    sample_rate: int
    channels: int
    fmt: int

    @property
    def frames(self) -> int:
        return len(memoryview(self.data).cast("B")) // (self.channels * _PCM_BYTES[self.fmt])

    def out_length(self, sample_rate: int) -> int:
        """Samples of the clip at `sample_rate`."""
        return filter_table(self.sample_rate, sample_rate).total(self.frames) if self.sample_rate != sample_rate \
            else self.frames


def pcm_from_array(x, sample_rate: int) -> Pcm:
    """A decoded waveform [N] or [N, channels] (numpy or torch, any float dtype) as float32 PCM."""
    a = x.detach().cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)
    a = np.ascontiguousarray(a, dtype=np.float32)
    if a.ndim == 1:
        a = a[:, None]
    if a.ndim != 2:
        raise ValueError(f"a waveform is [N] or [N, channels], got {a.shape}")
    return Pcm(a, int(sample_rate), int(a.shape[1]), PCM_F32)


def _wav_pcm(f) -> Pcm:
    with wave.open(f, "rb") as w:
        sr, nch, width, n = w.getframerate(), w.getnchannels(), w.getsampwidth(), w.getnframes()
        raw = w.readframes(n)
    if width not in _PCM_OF_WIDTH:
        raise ValueError(f"unsupported PCM width {width}")
    return Pcm(raw, int(sr), int(nch), _PCM_OF_WIDTH[width])


def read_pcm(path: Path) -> Pcm:
    """A file as read, for `load_batch`: the raw frames of a PCM wav (stdlib reader), else the array soundfile or
    torchaudio decodes [N, channels]."""
    path = Path(path)
    if path.suffix.lower() == ".wav":
        try:
            return _wav_pcm(str(path))
        except (wave.Error, ValueError, EOFError):
            pass  # not integer PCM (float or extensible wav): a decoder may read it
    try:
        import soundfile as sf

        data, sr = sf.read(str(path), dtype="float32", always_2d=True)
        return pcm_from_array(data, sr)
    except Exception:  # not installed, or a format libsndfile cannot decode: torchaudio may
        pass
    import torchaudio

    wav, sr = torchaudio.load(str(path))
    return pcm_from_array(wav.T, sr)


def pcm_from_bytes(data: bytes) -> Pcm:
    """An encoded audio file held in memory: a PCM wav's raw frames, else soundfile's decoded array."""
    try:
        return _wav_pcm(io.BytesIO(data))
    except (wave.Error, ValueError, EOFError):
        pass
    import soundfile as sf

    x, sr = sf.read(io.BytesIO(data), dtype="float32", always_2d=True)
    return pcm_from_array(x, sr)


def load_batch(clips: Sequence[Pcm], sample_rate: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """Clips at any rates -> (audio fp32 [B, 1, N_max] zero-padded, lengths int64 [B]) on `device` at `sample_rate`:
    one upload of every clip's bytes, one conversion + down-mix launch, one resample launch (clips already at
    `sample_rate` are copied by it)."""
    device = _device(device)
    B = len(clips)
    outs = [c.out_length(sample_rate) for c in clips]
    n_max = max(outs, default=0)
    with torch.cuda.device(device):
        audio = torch.empty(B, 1, n_max, dtype=torch.float32, device=device)
        lengths = torch.tensor(outs, dtype=torch.int64).to(device)
        if B == 0 or n_max == 0:
            return audio.zero_(), lengths
        raws = [np.frombuffer(memoryview(c.data).cast("B"), dtype=np.uint8) for c in clips]
        host = torch.empty(sum(r.size for r in raws), dtype=torch.uint8, pin_memory=True)
        hv = host.numpy()
        pcm_desc, o, mono_off = [], 0, 0
        for c, r in zip(clips, raws):
            hv[o: o + r.size] = r
            pcm_desc.append([o, c.frames, c.channels, c.fmt, mono_off])
            o += r.size
            mono_off += c.frames
        src = host.to(device, non_blocking=True)
        mono = torch.empty(max(1, mono_off), dtype=torch.float32, device=device)
        d = torch.tensor(pcm_desc, dtype=torch.int64).to(device)
        L = _lib.lib()
        _lib.check(L.fsb_pcm_to_mono(src.data_ptr(), d.data_ptr(), B, max(c.frames for c in clips), mono.data_ptr(),
                                     _stream(device)))
        rows = []
        for b, (c, pd) in enumerate(zip(clips, pcm_desc)):
            tab = None if c.sample_rate == sample_rate else _device_table(c.sample_rate, sample_rate, device)
            rows.append((pd[4], 0, c.frames, 0, b * n_max, outs[b], n_max, tab))
        _launch_resample(mono, rows, audio, n_max)
    return audio, lengths


def pcm_to_mono(pcm: torch.Tensor, fmt: int, channels: int = 1) -> torch.Tensor:
    """Interleaved PCM already on a CUDA device (a tensor of its samples, or of its bytes) -> mono fp32 [frames]."""
    raw = pcm.contiguous()
    frames = raw.numel() * raw.element_size() // (channels * _PCM_BYTES[fmt])
    out = torch.empty(frames, dtype=torch.float32, device=raw.device)
    if frames:
        d = torch.tensor([[0, frames, channels, fmt, 0]], dtype=torch.int64).to(raw.device)
        _lib.check(_lib.lib().fsb_pcm_to_mono(raw.data_ptr(), d.data_ptr(), 1, frames, out.data_ptr(),
                                              _stream(raw.device)))
    return out


class StreamResampler:
    """Resample a signal that arrives in pieces, on `device`: `push(x)` -> the outputs now complete, `flush()` -> the
    rest. Concatenated, they are bit-identical to `resample` of the whole signal. Between pushes it keeps the input
    samples the next outputs read (about one filter length) on the device. `orig_freq == new_freq` passes pieces
    through."""

    def __init__(self, orig_freq: int, new_freq: int, device):
        self.orig_freq, self.new_freq = int(orig_freq), int(new_freq)
        self.device = _device(device)
        self.identity = self.orig_freq == self.new_freq
        self.counts = StreamCounts(filter_table(self.orig_freq, self.new_freq))
        self._tab = None if self.identity else _device_table(self.orig_freq, self.new_freq, self.device)
        self._hist = torch.empty(0, dtype=torch.float32, device=self.device)
        self._h0 = 0  # input index of _hist[0]

    def push(self, x: torch.Tensor) -> torch.Tensor:
        return StreamResampler.push_many([(self, x)])[0]

    def flush(self) -> torch.Tensor:
        return StreamResampler.push_many([(self, None)])[0]

    @staticmethod
    def push_many(items: list) -> list:
        """[(resampler, fp32 piece on its device, or None to flush)] -> their outputs, every stream in one launch
        (the resamplers must share a device)."""
        if not items:
            return []
        dev = items[0][0].device
        for rs, _ in items:
            if rs.device != dev:
                raise ValueError("push_many: resamplers on different devices")
        with torch.cuda.device(dev):
            segs, plan, off = [], [], 0
            for rs, x in items:
                if x is not None:
                    x = x.reshape(-1)
                    if x.dtype != torch.float32 or x.device != dev:
                        raise ValueError("a piece must be float32 on the resampler's device")
                if rs.identity:
                    if x is None:
                        rs.counts.flush()
                        plan.append(None)
                    else:
                        rs.counts.push(x.numel())
                        plan.append(x)
                    continue
                seg, h0, n_win, j0, n = rs._take(x)
                segs += seg
                plan.append((rs, off, h0, n_win, j0, n))
                off += n_win
            win = torch.cat(segs) if segs else None
            rows, out_off = [], 0
            for pl in plan:
                if isinstance(pl, tuple):
                    rs, x_off, h0, n_win, j0, n = pl
                    rows.append((x_off, h0, rs.counts.received, j0, out_off, n, n, rs._tab))
                    out_off += n
            out = torch.empty(max(1, out_off), dtype=torch.float32, device=dev)
            live = [r for r in rows if r[5] > 0]
            if live:
                _launch_resample(win, live, out, max(r[5] for r in live))
            res, k = [], 0
            for pl in plan:
                if not isinstance(pl, tuple):
                    res.append(pl if pl is not None else torch.empty(0, dtype=torch.float32, device=dev))
                    continue
                rs, x_off, h0, n_win, j0, n = pl
                res.append(out[rows[k][4]: rows[k][4] + n])
                k += 1
                rs._retain(win, x_off, h0, n_win)
            return res

    def _take(self, x: Optional[torch.Tensor]) -> tuple:
        """Advance the counts by a piece (None: the flush) -> (window pieces [history, piece], input index of the
        window's first sample, window length, first output, outputs now ready)."""
        segs, h0, n_win = [self._hist], self._h0, self._hist.numel()
        if x is None:
            j0, n = self.counts.flush()
        else:
            segs.append(x)
            n_win += x.numel()
            j0, n, _ = self.counts.push(x.numel())
        return segs, h0, n_win, j0, n

    def _retain(self, win: torch.Tensor, x_off: int, h0: int, n_win: int) -> None:
        """Keep, of this stream's window at win[x_off: x_off + n_win], the samples the next outputs read."""
        keep = self.counts.keep_from() if not self.counts.done else self.counts.received
        self._hist = win[x_off + keep - h0: x_off + n_win]
        self._h0 = keep


# ---------------------------------------------------------------------------------------------------------------------
# output front end: the decoder's fp32 waveform -> the client's rate and sample format (fsb_audio_out)
# ---------------------------------------------------------------------------------------------------------------------
CODEC_RATE = 44100  # the decoder's output rate (CodecConfig.sample_rate)
# sample format name -> (fsb_audio_out_row.format, include/fishb200.h FSB_OUT_*; element dtype)
OUTPUT_FORMATS = {"float32": (0, torch.float32), "pcm16": (1, torch.int16), "mulaw": (2, torch.uint8)}


def output_format(sample_format: Optional[str]) -> str:
    """The format name a request's `sample_format` stands for: None is float32."""
    fmt = "float32" if sample_format is None else str(sample_format)
    if fmt not in OUTPUT_FORMATS:
        raise ValueError(f"sample_format must be one of {sorted(OUTPUT_FORMATS)} (got {sample_format!r})")
    return fmt


def _launch_out(x: torch.Tensor, rows: list, out: torch.Tensor) -> None:
    """rows: per output row (x_off, x_start, x_end, j0, out byte offset, n_out, table or None, format code) -> one
    fsb_audio_out launch into the bytes of `out`."""
    desc = []
    for x_off, x_start, x_end, j0, out_off, n_out, tab, code in rows:
        if tab is None:
            w_ptr, s_ptr, o, n = 0, 0, 1, 1
        else:
            w_ptr, s_ptr, o, n = tab[0].data_ptr(), tab[1].data_ptr(), tab[2], tab[3]
        desc.append([x_off, x_start, x_end, j0, out_off, n_out, w_ptr, s_ptr, o, n, code])
    d = torch.tensor(desc, dtype=torch.int64).to(x.device)
    _lib.check(_lib.lib().fsb_audio_out(x.data_ptr(), d.data_ptr(), len(rows), max(r[5] for r in rows),
                                        out.data_ptr(), _stream(x.device)))


def convert_out(wav: torch.Tensor, sample_rate: Optional[int] = None, sample_format: Optional[str] = None,
                orig_freq: int = CODEC_RATE) -> torch.Tensor:
    """A CUDA fp32 waveform [..., N] at `orig_freq` -> [..., M] at `sample_rate` in `sample_format` (float32, pcm16 =
    int16, mulaw = uint8), every row in one fsb_audio_out launch. M is torchaudio's length; the float32 samples are
    the bits of `resample`, pcm16 is utils.pcm16 of them and mulaw G.711 of that. With no rate and no format (or the
    waveform's own rate in float32) the waveform itself is returned."""
    fmt = output_format(sample_format)
    rate = int(orig_freq) if sample_rate is None else int(sample_rate)
    if rate <= 0:
        raise ValueError(f"sample_rate must be positive (got {sample_rate})")
    if wav.device.type != "cuda" or wav.dtype != torch.float32:
        raise TypeError(f"convert_out takes a CUDA float32 waveform (got {wav.dtype} on {wav.device})")
    if rate == int(orig_freq) and fmt == "float32":
        return wav
    code, dtype = OUTPUT_FORMATS[fmt]
    shape = wav.shape
    n = int(shape[-1])
    x = wav.reshape(-1, n).contiguous()
    rows = x.shape[0]
    with torch.cuda.device(x.device):
        identity = rate == int(orig_freq)
        tab = None if identity else _device_table(orig_freq, rate, x.device)
        out_n = n if identity else filter_table(int(orig_freq), rate).total(n)
        out = torch.empty(rows, out_n, dtype=dtype, device=x.device)
        if rows and out_n:
            es = out.element_size()
            _launch_out(x, [(r * n, 0, n, 0, r * out_n * es, out_n, tab, code) for r in range(rows)], out)
    return out.reshape(*shape[:-1], out_n)


class OutputStream(StreamResampler):
    """`convert_out` over a waveform that arrives in pieces: `push(piece)` -> the converted samples now complete,
    `flush()` -> the rest (the filter's look-ahead holds back up to about 6 input samples per output phase). The
    concatenated results are bit-identical to `convert_out` of the whole waveform. History is kept as
    `StreamResampler` keeps it; at the input rate there is none, and float32 there passes pieces through."""

    def __init__(self, sample_rate: Optional[int] = None, sample_format: Optional[str] = None, device="cuda",
                 orig_freq: int = CODEC_RATE):
        rate = int(orig_freq) if sample_rate is None else int(sample_rate)
        if rate <= 0:
            raise ValueError(f"sample_rate must be positive (got {sample_rate})")
        super().__init__(orig_freq, rate, device)
        self.sample_format = output_format(sample_format)
        self._code, self.dtype = OUTPUT_FORMATS[self.sample_format]

    @property
    def sample_rate(self) -> int:
        return self.new_freq

    def push(self, x: torch.Tensor) -> torch.Tensor:
        return OutputStream.push_many([(self, x)])[0]

    def flush(self) -> torch.Tensor:
        return OutputStream.push_many([(self, None)])[0]

    @staticmethod
    def push_many(items: list) -> list:
        """[(stream, fp32 piece on its device, or None to flush)] -> their converted samples, every stream (of any
        rate and format) in one launch (the streams must share a device)."""
        if not items:
            return []
        dev = items[0][0].device
        with torch.cuda.device(dev):
            segs, plan, off = [], [], 0
            for st, x in items:
                if st.device != dev:
                    raise ValueError("push_many: streams on different devices")
                if x is not None:
                    x = x.reshape(-1)
                    if x.dtype != torch.float32 or x.device != dev:
                        raise ValueError("a piece must be float32 on the stream's device")
                if st.identity and st._code == 0:  # float32 at the input rate: the piece itself
                    if x is None:
                        st.counts.flush()
                    else:
                        st.counts.push(x.numel())
                    plan.append(x if x is not None else torch.empty(0, dtype=torch.float32, device=dev))
                    continue
                if st.identity:  # quantise only: output j is input j, no history
                    r0 = st.counts.received
                    seg, h0, n_win, j0 = ([] if x is None else [x]), r0, (0 if x is None else x.numel()), r0
                    if x is None:
                        st.counts.flush()
                    else:
                        st.counts.push(n_win)
                    n = n_win
                else:
                    seg, h0, n_win, j0, n = st._take(x)
                segs += seg
                plan.append((st, off, h0, n_win, j0, n))
                off += n_win
            win = torch.cat(segs) if segs else None
            rows, ob = [], 0
            for pl in plan:
                if isinstance(pl, tuple):
                    st, x_off, h0, n_win, j0, n = pl
                    rows.append((x_off, h0, st.counts.received, j0, ob, n, st._tab, st._code))
                    ob += -(-n * st.dtype.itemsize // 16) * 16  # every row's bytes 16-aligned: a view of any dtype
            out = torch.empty(max(16, ob), dtype=torch.uint8, device=dev)
            live = [r for r in rows if r[5] > 0]
            if live:
                _launch_out(win, live, out)
            res, k = [], 0
            for pl in plan:
                if not isinstance(pl, tuple):
                    res.append(pl)
                    continue
                st, x_off, h0, n_win, j0, n = pl
                b = rows[k][4]
                res.append(out[b: b + n * st.dtype.itemsize].view(st.dtype))
                k += 1
                if not st.identity:
                    st._retain(win, x_off, h0, n_win)
            return res
