"""Codec output front end, host side (no GPU): the stream arithmetic from 44.1 kHz to client rates, the G.711 mu-law
reference the device kernel is checked against, `utils.pcm16` at the edges of its range, and the WAV headers of each
output format."""
import io
import math
import struct
import warnings
import wave

import numpy as np
import pytest

from fish_speech_b200 import audio as A
from fish_speech_b200.inference_engine import utils as U

SR = 44100
OUT_RATES = [8000, 16000, 22050, 24000, 48000]


# ---- references shared with the GPU tests ---------------------------------------------------------------------------
def pcm16_ref(y: float) -> int:
    """utils.pcm16 of one fp32 value without numpy: clip, multiply by 32767 (exact in float64: 24 + 15 bits), round
    once to fp32 (struct rounds to nearest even), truncate toward zero. NaN gives 0."""
    y = struct.unpack("<f", struct.pack("<f", y))[0]
    if math.isnan(y):
        return 0
    y = min(max(y, -1.0), 1.0)
    return math.trunc(struct.unpack("<f", struct.pack("<f", y * 32767.0))[0])


def ulaw_ref(s: int) -> int:
    """G.711 mu-law of a 16-bit sample: the Sun g711.c encoder (linear2ulaw on the sample shifted to 14 bits), which
    audioop.lin2ulaw runs. Magnitude clipped to 8159, bias 132 >> 2, 8 segments, all bits inverted."""
    v = s >> 2
    mask = 0xFF
    if v < 0:
        v, mask = -v, 0x7F
    v = min(v, 8159) + 33
    seg = 0
    while seg < 8 and v > (0x40 << seg) - 1:
        seg += 1
    if seg >= 8:
        return 0x7F ^ mask
    return ((seg << 4) | ((v >> (seg + 1)) & 0xF)) ^ mask


def ulaw_ref_array(s: np.ndarray) -> np.ndarray:
    return np.array([ulaw_ref(int(v)) for v in np.asarray(s, dtype=np.int64)], dtype=np.uint8)


# ---- stream arithmetic ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", OUT_RATES)
def test_output_stream_counts_prefix_and_totals(sr):
    """44.1 kHz -> sr in pieces of one codec frame and of odd sizes: each push emits a prefix of the outputs (never one
    whose last tap has not arrived), and pushes + flush give torchaudio's length."""
    import torch
    import torchaudio

    tab = A.filter_table(SR, sr)
    last = tab.first + tab.count - 1
    for pieces in ([2048] * 9, [1, 2047, 4096, 3, 17, 2048 * 3, 5], [7] * 50):
        c = A.StreamCounts(tab)
        emitted = 0
        for m in pieces:
            j0, n, keep = c.push(m)
            assert j0 == emitted and n >= 0
            emitted += n
            if emitted:  # the last emitted output reads only received samples
                q, p = divmod(emitted - 1, tab.new)
                assert q * tab.orig + last[p] < c.received
            assert keep <= c.received and keep <= max(0, tab.first_input(emitted))
        j0, n = c.flush()
        assert j0 == emitted
        total = sum(pieces)
        want = torchaudio.functional.resample(torch.zeros(total), SR, sr).shape[-1]
        assert emitted + n == want == tab.total(total)


# ---- sample formats ------------------------------------------------------------------------------------------------
def test_ulaw_reference_is_audioop_for_every_int16():
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", DeprecationWarning)
        audioop = pytest.importorskip("audioop")  # removed in Python 3.13: the reference above stands alone there
    s = np.arange(-32768, 32768, dtype=np.int64)
    want = np.frombuffer(audioop.lin2ulaw(s.astype("<i2").tobytes(), 2), dtype=np.uint8)
    assert np.array_equal(ulaw_ref_array(s), want)


def _f32(bits: int) -> float:
    return struct.unpack("<f", struct.pack("<I", bits))[0]


ONE, NEG_ONE = 0x3F800000, 0xBF800000
# (fp32 input bits, utils.pcm16 output)
PCM16_EDGES = [
    (ONE, 32767), (NEG_ONE, -32767),                  # full scale: no wrap to -32768
    (ONE + 1, 32767), (NEG_ONE + 1, -32767),          # just beyond: clipped
    (ONE - 1, 32766), (NEG_ONE - 1, -32766),          # just inside: 0.99999994 * 32767 = 32766.998 in fp32
    (0x3FC00000, 32767), (0xC0000000, -32767),        # 1.5, -2.0 (resampler overshoot)
    (0x7F800000, 32767), (0xFF800000, -32767),        # +-inf
    (0x00000000, 0), (0x80000000, 0), (0x00000001, 0),  # +-0, the smallest subnormal
    (0x380000FF, 0), (0x38000100, 1),                 # fp32 product 1 - 2^-23 and 1.0 (1 - 2^-30 rounded)
    (0x3F000000, 16383), (0xBF000000, -16383),        # 0.5 -> 16383.5, truncated toward zero both ways
]


def _near_integer_cases():
    """Inputs whose fp32 product with 32767 is an integer, and their fp32 neighbours (product just below / above)."""
    out = []
    for k in (1, 2, 3, 100, 1000, 12345, 16384, 32766):
        y = np.float32(k) / np.float32(32767)
        b = int(np.array(y).view(np.uint32))
        for d in (-1, 0, 1):
            out.append(b + d)
            out.append((b + d) | 0x80000000)
    return out


def test_pcm16_at_the_edges():
    xs = np.array([b for b, _ in PCM16_EDGES], dtype=np.uint32).view(np.float32)
    want = np.array([v for _, v in PCM16_EDGES], dtype="<i2")
    got = np.frombuffer(U.pcm16(xs), dtype="<i2")
    assert np.array_equal(got, want), list(zip(got.tolist(), want.tolist()))
    assert [pcm16_ref(float(x)) for x in xs] == want.tolist()
    # products landing either side of an integer: numpy's fp32 multiply and truncation against the exact rounding
    bits = _near_integer_cases()
    ys = np.array(bits, dtype=np.uint32).view(np.float32)
    got = np.frombuffer(U.pcm16(ys), dtype="<i2").tolist()
    assert got == [pcm16_ref(float(y)) for y in ys]
    assert len(set(got)) > 16  # both sides of several integers occur


def test_pcm16_is_not_the_x32768_cast():
    """The reference server's (audio * 32768).astype(int16) wraps a full-scale sample; utils.pcm16 does not."""
    x = np.array([1.0, -1.0], dtype=np.float32)
    assert np.frombuffer(U.pcm16(x), dtype="<i2").tolist() == [32767, -32767]


# ---- WAV headers ---------------------------------------------------------------------------------------------------
def _hand_header(sr, tag, bits):
    block = bits // 8
    return (b"RIFF" + (36).to_bytes(4, "little") + b"WAVE" + b"fmt " + (16).to_bytes(4, "little")
            + tag.to_bytes(2, "little") + (1).to_bytes(2, "little") + sr.to_bytes(4, "little")
            + (sr * block).to_bytes(4, "little") + block.to_bytes(2, "little") + bits.to_bytes(2, "little")
            + b"data" + (0).to_bytes(4, "little"))


def test_wav_headers_for_each_format():
    # the default call is the header it always was: 16-bit PCM at 44.1 kHz
    assert U.wav_chunk_header() == _hand_header(44100, 1, 16)
    assert U.wav_chunk_header(sample_rate=24000) == _hand_header(24000, 1, 16)
    for sr in (8000, 24000, 48000):
        buf = io.BytesIO()
        with wave.open(buf, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(sr)
        bits, tag = U.WAVE_OF_FORMAT["pcm16"]
        assert U.wav_chunk_header(sample_rate=sr, bit_depth=bits, format_tag=tag) == buf.getvalue()
        bits, tag = U.WAVE_OF_FORMAT["float32"]
        assert U.wav_chunk_header(sample_rate=sr, bit_depth=bits, format_tag=tag) == _hand_header(sr, 3, 32)
        bits, tag = U.WAVE_OF_FORMAT["mulaw"]
        assert U.wav_chunk_header(sample_rate=sr, bit_depth=bits, format_tag=tag) == _hand_header(sr, 7, 8)
    assert set(U.WAVE_OF_FORMAT) == set(A.OUTPUT_FORMATS)


def test_output_format_names():
    assert A.output_format(None) == "float32"
    for f in ("float32", "pcm16", "mulaw"):
        assert A.output_format(f) == f
    with pytest.raises(ValueError):
        A.output_format("mp3")


def test_cli_writes_wav_files_of_the_converted_samples(tmp_path):
    from fish_speech_b200.models.dac.inference import write_wav

    s = np.array([0, 1, -1, 32767, -32767, 12345], dtype=np.int16)
    write_wav(tmp_path / "a.wav", s, 24000, "pcm16")
    with wave.open(str(tmp_path / "a.wav"), "rb") as w:
        assert (w.getframerate(), w.getsampwidth(), w.getnchannels()) == (24000, 2, 1)
        assert np.array_equal(np.frombuffer(w.readframes(w.getnframes()), dtype="<i2"), s)
    u = ulaw_ref_array(s)
    write_wav(tmp_path / "u.wav", u, 8000, "mulaw")
    raw = (tmp_path / "u.wav").read_bytes()
    head = bytearray(_hand_header(8000, 7, 8))
    head[4:8] = (36 + u.size).to_bytes(4, "little")
    head[40:44] = u.size.to_bytes(4, "little")
    assert raw == bytes(head) + u.tobytes()
