"""Codec input front end on the device (fish_speech_b200/audio.py, csrc/audio_kernels.cu): resampling against
torchaudio in float64, PCM conversion and down-mix against the numpy reader bit for bit, ragged batches and streams
against the one-shot call bit for bit, and the encode pool's and bulk encode's use of them against `DAC.encode` of the
GPU-resampled clip."""
import random
import wave

import numpy as np
import pytest
import torch

from fish_speech_b200 import audio as A
from oracle import codec_oracle as CO
from tests.test_codec_gpu import VQ_EPS, build, vq_first_mismatches

pytestmark = pytest.mark.gpu
RATES = [8000, 16000, 22050, 24000, 32000, 48000, 96000]
SR = 44100
FL = 2048


def noise(n, seed, ch=None, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    shape = (n,) if ch is None else (n, ch)
    return (scale * torch.randn(*shape, generator=g, dtype=torch.float64)).clamp(-1, 1)


def numpy_mono(raw: np.ndarray, fmt: int, ch: int) -> np.ndarray:
    """bulk_encode.read_audio's stdlib-reader arithmetic (float32 arrays: the same mean)."""
    if fmt == A.PCM_S16:
        x = raw.astype(np.float32) / 32768.0
    elif fmt == A.PCM_S32:
        x = raw.astype(np.float32) / 2147483648.0
    elif fmt == A.PCM_U8:
        x = (raw.astype(np.float32) - 128.0) / 128.0
    else:
        x = raw.astype(np.float32)
    return x.reshape(-1, ch).mean(axis=1)


def rand_pcm(n, fmt, ch, seed, sr=SR):
    rng = np.random.default_rng(seed)
    if fmt == A.PCM_S16:
        raw = rng.integers(-32768, 32768, n * ch).astype("<i2")
    elif fmt == A.PCM_S32:
        raw = rng.integers(-2 ** 31, 2 ** 31, n * ch, dtype=np.int64).astype("<i4")
    elif fmt == A.PCM_U8:
        raw = rng.integers(0, 256, n * ch).astype(np.uint8)
    else:
        raw = rng.standard_normal(n * ch).astype(np.float32)
        raw[::7] = -0.0  # signed zeros in channel sums
    pcm = A.Pcm(raw.tobytes(), sr, ch, fmt) if fmt != A.PCM_F32 else A.pcm_from_array(raw.reshape(n, ch), sr)
    return pcm, raw


# ---- resample ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", RATES)
def test_resample_error_is_within_torchaudio_fp32(sr):
    """Against torchaudio on float64 input: the largest error is no larger than torchaudio's own fp32 result's (at a
    handful of samples both sit at the fp32 rounding of single weights, so 2^-23 is the floor)."""
    import torchaudio

    taps = A.filter_table(sr, SR).taps
    for n in (1, taps - 1, 101, 7919, 3 * sr):
        x = noise(n, n + sr)
        ref = torchaudio.functional.resample(x, sr, SR)
        ta32 = torchaudio.functional.resample(x.float(), sr, SR).double()
        got = A.resample(x.float().cuda(), sr, SR)
        assert got.dtype == torch.float32 and got.shape == ref.shape
        e_got = float((got.cpu().double() - ref).abs().max())
        e_ta = float((ta32 - ref).abs().max())
        print(f"{sr} -> {SR}, n={n}: max error {e_got:.2e} (torchaudio fp32 {e_ta:.2e})")
        assert e_got <= max(e_ta, 2.0 ** -23), f"{sr} Hz, n={n}: {e_got:.3e} > torchaudio fp32 {e_ta:.3e}"


def test_resample_rows_same_rate_and_other_filters():
    import torchaudio

    x = noise(3 * 5000, 1).float().reshape(3, 5000).cuda()
    assert A.resample(x, SR, SR) is x  # no launch, the input itself
    rows = A.resample(x.reshape(3, 1, 5000), 48000, SR)
    assert rows.shape == (3, 1, A.filter_table(48000, SR).total(5000))
    for r in range(3):
        assert torch.equal(rows[r, 0], A.resample(x[r].clone(), 48000, SR))  # each row as if alone
    # a non-default filter is torchaudio's own call, on the device
    k = A.resample(x, 48000, SR, rolloff=0.9)
    assert torch.equal(k, torchaudio.functional.resample(x, 48000, SR, rolloff=0.9))
    with pytest.raises(TypeError):
        A.resample(x.double(), 48000, SR)


# ---- conversion and batching ------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", [A.PCM_S16, A.PCM_S32, A.PCM_U8, A.PCM_F32])
def test_pcm_conversion_is_bitwise_the_numpy_path(fmt):
    clips, want = [], []
    for i, ch in enumerate((1, 2, 6)):
        pcm, raw = rand_pcm(4000 + 37 * i, fmt, ch, seed=10 * fmt + ch)
        clips.append(pcm)
        want.append(numpy_mono(raw, fmt, ch))
    audio, lens = A.load_batch(clips, SR, "cuda")
    assert audio.shape == (3, 1, max(w.size for w in want)) and lens.tolist() == [w.size for w in want]
    for b, w in enumerate(want):
        got = audio[b, 0].cpu().numpy()
        assert np.array_equal(got[: w.size].view(np.uint32), w.view(np.uint32)), f"fmt {fmt}, clip {b}"
        assert not got[w.size:].any()  # zero padding
    # one interleaved piece already on the device
    pcm, raw = rand_pcm(999, fmt, 2, seed=5)
    dev = torch.from_numpy(raw.view(np.uint8).copy()).cuda()
    got = A.pcm_to_mono(dev, fmt, channels=2).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), numpy_mono(raw, fmt, 2).view(np.uint32))


def test_ragged_batch_with_mixed_rates_equals_each_clip_alone():
    specs = [(16000, A.PCM_S16, 2, 16000 * 3 + 7), (48000, A.PCM_S16, 1, 4801), (22050, A.PCM_U8, 6, 1),
             (SR, A.PCM_S32, 2, 30011), (24000, A.PCM_F32, 1, 24000), (96000, A.PCM_S16, 2, 17)]
    clips = [rand_pcm(n, fmt, ch, seed=i, sr=sr)[0] for i, (sr, fmt, ch, n) in enumerate(specs)]
    audio, lens = A.load_batch(clips, SR, "cuda")
    for b, c in enumerate(clips):
        solo, solo_len = A.load_batch([c], SR, "cuda")
        n = int(solo_len[0])
        assert int(lens[b]) == n == c.out_length(SR)
        assert torch.equal(audio[b, 0, :n], solo[0, 0])
        assert not audio[b, 0, n:].any()
        mono, _ = A.load_batch([A.Pcm(c.data, SR, c.channels, c.fmt)], SR, "cuda")
        assert torch.equal(solo[0, 0], A.resample(mono[0, 0], c.sample_rate, SR))  # = convert, then resample


# ---- streams ----------------------------------------------------------------------------------------------------
def piece_sizes(rng, n, taps):
    out, a = [], 0
    while a < n:
        k = min(n - a, rng.choice([1, 2, taps - 1, taps + 1, rng.randint(1, 3000), rng.randint(1, 60000)]))
        out.append(k)
        a += k
    return out


@pytest.mark.parametrize("sr", [16000, 22050, 48000, 96000, SR])
def test_stream_equals_one_shot_bitwise(sr):
    rng = random.Random(sr)
    taps = A.filter_table(sr, SR).taps
    for n in (1, 5, 2 * sr + 333):
        x = noise(n, sr + n).float().cuda()
        whole = A.resample(x, sr, SR)
        rs, outs, a = A.StreamResampler(sr, SR, "cuda"), [], 0
        for k in piece_sizes(rng, n, taps):
            outs.append(rs.push(x[a: a + k]))
            a += k
        outs.append(rs.flush())
        got = torch.cat(outs)
        assert got.shape == whole.shape and torch.equal(got, whole), f"{sr} Hz, n={n}"


def test_streams_pushed_together_equal_each_alone():
    rng = random.Random(3)
    rates = [16000, 22050, 48000, 16000]
    xs = [noise(r + 977 * i, i).float().cuda() for i, r in enumerate(rates)]
    rss = [A.StreamResampler(r, SR, "cuda") for r in rates]
    fed, outs = [0] * len(xs), [[] for _ in xs]
    while any(f < x.numel() for f, x in zip(fed, xs)):
        items = []
        for i, (x, rs) in enumerate(zip(xs, rss)):
            if fed[i] < x.numel() and rng.random() < 0.8:
                k = min(x.numel() - fed[i], rng.randint(1, 9000))
                items.append((rs, x[fed[i]: fed[i] + k]))
                fed[i] += k
        for (rs, _), y in zip(items, A.StreamResampler.push_many(items)):
            outs[rss.index(rs)].append(y)
    for rs, o, y in zip(rss, outs, A.StreamResampler.push_many([(rs, None) for rs in rss])):
        o.append(y)
    for x, r, o in zip(xs, rates, outs):
        assert torch.equal(torch.cat(o), A.resample(x, r, SR))


# ---- encode pool ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tiny():
    cfg = CO.tiny_config()
    w = CO.make_weights(cfg, seed=5)
    return cfg, w, build(cfg, w)


def encode_resampled(dac, x, sr):
    """codes [S, T] of DAC.encode of the whole clip resampled on the GPU."""
    y = A.resample(x.cuda(), sr, SR)
    codes, lens = dac.encode(y.view(1, 1, -1), torch.tensor([y.numel()], device="cuda"))
    return codes[0, :, : int(lens[0])].cpu()


def run_rated(pool, streams, seed, max_piece):
    """streams: {name: (rate or None, clip)}; clips of rated streams are pushed in random pieces (every second piece of
    an int16 clip), a None-rate clip in whole frames of at most k_max; all streams share pushes until each is done,
    rated ones end with flush. Returns {name: codes [S, T]}."""
    rng = random.Random(seed)
    slot = {n: pool.open(sample_rate=r) for n, (r, _) in streams.items()}
    fed = dict.fromkeys(streams, 0)
    codes = {n: [] for n in streams}
    while any(fed[n] < x.numel() for n, (_, x) in streams.items()):
        pieces = {}
        for n, (r, x) in streams.items():
            if fed[n] >= x.numel() or rng.random() < 0.2:
                continue
            if r is None:
                k = rng.randint(1, pool.k_max) * FL
            else:
                k = rng.choice([1, 5, rng.randint(1, max_piece)])
            pieces[slot[n]] = x[fed[n]: fed[n] + k]
            fed[n] += pieces[slot[n]].numel()
        if not pieces:
            continue
        out = pool.push(pieces)
        assert set(out) == set(pieces)
        for n in streams:
            if slot[n] in out:
                c = out[slot[n]]
                assert c.dtype == torch.int64 and c.shape[0] == pool.n_stage
                codes[n].append(c.cpu())
    for n, (r, _) in streams.items():
        codes[n].append(pool.flush(slot[n]).cpu())
        pool.close(slot[n])
    return {n: torch.cat(v, dim=1) for n, v in codes.items()}


def rated_streams(seed, seconds=1.0):
    s16 = (noise(int(16000 * seconds) + 11, seed) * 32767).round().to(torch.int16)
    return {"16k_int16": (16000, s16),
            "22k": (22050, noise(int(22050 * seconds * 1.3) + 5, seed + 1).float()),
            "48k": (48000, noise(int(48000 * seconds * 0.7) + 2047, seed + 2).float()),
            "plain": (None, noise(23 * FL, seed + 3).float())}


def reference_codes(dac, streams):
    out = {}
    for n, (r, x) in streams.items():
        if r is None:
            out[n] = encode_resampled(dac, x, SR)
        elif x.dtype == torch.int16:
            out[n] = encode_resampled(dac, A.pcm_to_mono(x.cuda(), A.PCM_S16), r)
        else:
            out[n] = encode_resampled(dac, x, r)
    return out


def test_pool_streams_at_native_rates_equal_encode_of_the_resampled_clip(tiny):
    cfg, _, dac = tiny
    streams = rated_streams(40)
    ref = reference_codes(dac, streams)
    graphed = dac.open_encode_pool(4, k_max=4)
    eager = dac.open_encode_pool(4, k_max=4, max_graphs=0)
    g = run_rated(graphed, streams, seed=1, max_piece=30000)
    assert graphed._graphs, "no push was replayed from a CUDA graph"
    e = run_rated(eager, streams, seed=1, max_piece=30000)
    for n in streams:
        assert g[n].shape == ref[n].shape, n
        assert torch.equal(g[n], ref[n]), f"{n}: pool codes differ from encode of the resampled clip"
        assert torch.equal(e[n], g[n]), f"{n}: graph replay differs from eager"
    # a piece of many more than k_max frames runs as several frame passes
    pool = dac.open_encode_pool(2, k_max=2)
    s = pool.open(sample_rate=48000)
    x = noise(48000 * 2 - 100, 77).float()
    first = pool.push({s: x})[s]
    assert first.shape[1] > 2 * pool.k_max
    got = torch.cat([first, pool.flush(s)], dim=1)
    assert torch.equal(got.cpu(), encode_resampled(dac, x, 48000))


def test_pool_rated_slot_lifecycle(tiny):
    cfg, _, dac = tiny
    pool = dac.open_encode_pool(2, k_max=4)
    x = noise(22050, 9).float()
    s = pool.open(sample_rate=22050)
    first = pool.push({s: x[:100]})[s]
    assert first.shape == (pool.n_stage, 0)  # no frame complete yet
    pool.push({s: x[100:5000]})
    assert s in pool._rs and s in pool._carry
    pool.close(s)  # mid-stream
    assert s not in pool._rs and s not in pool._carry
    s2 = pool.open(sample_rate=22050)
    got = torch.cat([pool.push({s2: x})[s2], pool.flush(s2)], dim=1)
    assert torch.equal(got.cpu(), encode_resampled(dac, x, 22050))
    with pytest.raises(ValueError):
        pool.push({s2: x[:10]})  # flushed
    with pytest.raises(ValueError):
        pool.flush(s2)
    pool.close(s2)
    s3 = pool.open(sample_rate=16000)
    with pytest.raises(ValueError):
        pool.push({s3: x.double()})
    with pytest.raises(ValueError):
        pool.open(sample_rate=0)
    plain = pool.open()
    assert pool.flush(plain).shape == (pool.n_stage, 0)
    with pytest.raises(ValueError):
        pool.push({plain: x[:100]})  # a slot without a rate keeps the whole-frame contract


def test_pool_full_geometry():
    cfg = CO.full_config()
    dac = build(cfg, CO.make_weights(cfg, seed=6))
    streams = rated_streams(50, seconds=2.0)
    ref = reference_codes(dac, streams)
    got = run_rated(dac.open_encode_pool(4, k_max=8), streams, seed=2, max_piece=40000)
    for n in streams:
        assert torch.equal(got[n], ref[n]), n


# ---- bulk encode ------------------------------------------------------------------------------------------------
def write_wav(path, pcm: np.ndarray, sr, ch):
    with wave.open(str(path), "wb") as f:
        f.setnchannels(ch)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(pcm.astype("<i2").tobytes())


def test_bulk_encode_resamples_on_the_device(tiny, tmp_path):
    from fish_speech_b200 import bulk_encode as BE

    cfg, w, dac = tiny
    rng = np.random.default_rng(4)
    specs = [(48000, 2, 48000 + 555), (22050, 1, 22050 * 2 + 9), (48000, 2, 3000), (22050, 1, 40000)]
    files, mono = [], []
    for i, (sr, ch, n) in enumerate(specs):
        pcm = (np.clip(0.2 * rng.standard_normal(n * ch), -1, 1) * 32767).round().astype(np.int16)
        f = tmp_path / f"c{i}.wav"
        write_wav(f, pcm, sr, ch)
        files.append(f)
        mono.append((torch.from_numpy(numpy_mono(pcm, A.PCM_S16, ch).copy()), sr))
    done, secs = BE.encode_files(files, dac, batch_size=3)
    assert done == len(files)
    for f, (x, sr) in zip(files, mono):
        got = np.load(f.with_suffix(".npy"))
        assert np.array_equal(got, encode_resampled(dac, x, sr).numpy()), f.name
    # against the CPU-torchaudio front end through the same encoder: identical codes except at near-ties of the
    # oracle's fp32 scores for that input. The bound is the codec tests' VQ_EPS (0.03, the largest gap they observed
    # on their five inputs, plus room) raised to 0.04: on c0.wav the encoder picks, on the GPU-resampled clip, a code
    # 0.0311 below the oracle's best (H100, 700 W), a near-tie of the encoder's own bf16 noise that this input shows.
    import torchaudio

    for f, (x, sr) in zip(files[:2], mono[:2]):
        y = torchaudio.functional.resample(x, sr, SR)
        old, lens = dac.encode(y.view(1, 1, -1).cuda(), torch.tensor([y.numel()], device="cuda"))
        new = torch.from_numpy(np.load(f.with_suffix(".npy")))
        assert old.shape[-1] == new.shape[-1] == int(lens[0])
        trace = {}
        CO.encode(w, cfg, y.view(1, 1, -1), torch.tensor([y.numel()]), trace=trace)
        mism = [(s_, abs(g)) for s_, g in vq_first_mismatches(trace["vq_scores"], old.cpu(), new[None])]
        worst = max((g for _, g in mism), default=0.0)
        print(f"{f.name}: {new.shape[-1] - len(mism)}/{new.shape[-1]} frames identical to the CPU front end's, "
              f"worst oracle score gap {worst:.4f}")
        assert worst <= VQ_EPS + 0.01, f"{f.name}: a differing code is not a near-tie ({mism})"


def test_batch_encode_bytes_at_other_rates(tiny, tmp_path):
    from fish_speech_b200 import bulk_encode as BE

    cfg, _, dac = tiny
    pcm = (np.clip(0.2 * np.random.default_rng(8).standard_normal(2 * 30000), -1, 1) * 32767).round().astype(np.int16)
    f = tmp_path / "a.wav"
    write_wav(f, pcm, 24000, 2)
    wav44 = noise(9000, 3).float().reshape(1, -1)
    outs = BE.batch_encode(dac, [f.read_bytes(), wav44])
    x = torch.from_numpy(numpy_mono(pcm, A.PCM_S16, 2).copy())
    assert torch.equal(outs[0], encode_resampled(dac, x, 24000))
    assert torch.equal(outs[1], encode_resampled(dac, wav44[0], SR))
