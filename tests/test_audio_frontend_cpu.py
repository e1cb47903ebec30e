"""Codec input front end (fish_speech_b200/audio.py), host side: the float64 filter table against
torchaudio.functional.resample, and the stream arithmetic (which outputs a push of M samples makes ready, what a flush
adds, how many codec frames follow)."""
import math
import random

import numpy as np
import pytest
import torch

from fish_speech_b200 import audio as A

RATES = [8000, 16000, 22050, 24000, 32000, 48000, 96000]
TARGET = 44100
FL = 2048


def torchaudio_f64(x: np.ndarray, sr: int) -> np.ndarray:
    torchaudio = pytest.importorskip("torchaudio")
    return torchaudio.functional.resample(torch.from_numpy(x), sr, TARGET).numpy()


@pytest.mark.parametrize("sr", RATES)
def test_table_matches_torchaudio_in_float64(sr):
    t = A.filter_table(sr, TARGET)
    g = math.gcd(sr, TARGET)
    assert (t.orig, t.new) == (sr // g, TARGET // g)
    rng = np.random.default_rng(sr)
    n = 3 * t.taps + 2 * t.orig + 5
    for pos in (0, 1, t.orig - 1, n // 2, n - 1):  # impulses, at the edges too
        x = np.zeros(n)
        x[pos] = 1.0
        got, ref = A.apply_table(t, x), torchaudio_f64(x, sr)
        assert got.shape == ref.shape and np.abs(got - ref).max() <= 1e-12
    for n in (1, 7, t.taps - 1, 997, sr // 2):
        x = rng.standard_normal(n)
        got, ref = A.apply_table(t, x), torchaudio_f64(x, sr)
        assert got.shape == ref.shape == (t.total(n),)
        assert np.abs(got - ref).max() <= 1e-12
    assert 12 <= t.count.min() and t.count.max() <= t.taps  # about 13 non-zero taps per output (27 from 96 kHz)


def test_output_length_is_torchaudios():
    """torchaudio rounds new * n / orig to fp32 before its ceiling; a 48 kHz clip of 5 246 004 samples is one sample
    shorter than the exact ceiling."""
    t = A.filter_table(48000, TARGET)
    for n in (1, 159, 160, 161, 5246004, 5246004 + 160, 28_800_000, 40_000_017):
        assert t.total(n) == math.ceil(float(torch.as_tensor(147 * n / 160)))
    assert t.total(5246004) == -(-147 * 5246004 // 160) - 1


def test_same_rate_and_bad_rates():
    t = A.filter_table(TARGET, TARGET)
    assert (t.orig, t.new) == (1, 1)
    with pytest.raises(ValueError):
        A.filter_table(0, TARGET)


def _pieces(rng: random.Random, n: int, taps: int) -> list:
    out, a = [], 0
    while a < n:
        k = rng.choice([1, 2, taps - 1, taps, rng.randint(1, 4000), rng.randint(1, 3 * 48000)])
        k = min(k, n - a)
        out.append(k)
        a += k
    return out


@pytest.mark.parametrize("sr", RATES + [TARGET])
def test_stream_counts_add_up_to_the_one_shot_length(sr):
    t = A.filter_table(sr, TARGET)
    rng = random.Random(sr)
    for trial in range(6):
        n = rng.choice([1, 5, t.taps, rng.randint(1, 5 * sr)])
        sc = A.StreamCounts(t)
        emitted = 0
        for k in _pieces(rng, n, t.taps):
            j0, ready, keep = sc.push(k)
            assert j0 == emitted and ready >= 0
            emitted += ready
            # every emitted output reads only samples already pushed; the next one's first sample is kept
            if emitted:
                assert t.first_input(emitted - 1) + int(t.count[(emitted - 1) % t.new]) - 1 < sc.received
            assert 0 <= keep <= sc.received and keep <= max(0, t.first_input(emitted))
        j0, rest = sc.flush()
        assert j0 == emitted and emitted + rest == t.total(n) == torchaudio_f64(np.zeros(n), sr).shape[-1]
        with pytest.raises(ValueError):
            sc.push(1)


@pytest.mark.parametrize("sr", [16000, 22050, 48000])
def test_stream_outputs_in_float64_equal_the_whole_signal(sr):
    """The stream bookkeeping applied to float64 windows (what StreamResampler hands the kernel) gives the one-shot
    result exactly: the emitted outputs read only kept or new samples."""
    t = A.filter_table(sr, TARGET)
    rng = random.Random(7)
    n = 2 * sr + 13
    x = np.random.default_rng(1).standard_normal(n)
    whole = A.apply_table(t, x)
    sc, out, h0 = A.StreamCounts(t), [], 0
    a = 0

    def window_outputs(j0, m, x_end):
        j = np.arange(j0, j0 + m)
        q, p = j // t.new, j % t.new
        i0 = q * t.orig + t.first[p]
        acc = np.zeros(m)
        for k in range(t.taps):
            i = i0 + k
            ok = (i >= 0) & (i < x_end)
            assert np.all(~ok | (i >= h0)), "an output read a sample that was not kept"
            acc += t.w[p, k] * np.where(ok, x[np.clip(i, 0, n - 1)], 0.0)
        return acc

    for k in _pieces(rng, n, t.taps):
        a += k
        j0, m, keep = sc.push(k)
        out.append(window_outputs(j0, m, a))
        h0 = keep
    j0, m = sc.flush()
    out.append(window_outputs(j0, m, n))
    assert np.array_equal(np.concatenate(out), whole)


@pytest.mark.parametrize("sr", [16000, 22050, 48000, TARGET])
def test_stream_frames_equal_encode_lengths(sr):
    """Frames the encode pool runs for a stream: whole frames of its carry after each push, then the zero-padded rest
    at flush. Their count is encode's indices_lens of the resampled clip, ceil(length / frame_length)."""
    t = A.filter_table(sr, TARGET)
    rng = random.Random(sr + 1)
    for _ in range(4):
        n = rng.randint(1, 4 * sr)
        sc, carry, frames = A.StreamCounts(t), 0, 0
        for k in _pieces(rng, n, t.taps):
            carry += sc.push(k)[1]
            frames += carry // FL
            carry %= FL
        carry += sc.flush()[1]
        frames += -(-carry // FL)
        length = t.total(n)
        assert frames == int(torch.ceil(torch.tensor([length]) / FL).long()[0])
