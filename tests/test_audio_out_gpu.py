"""Codec output front end on the device (fish_speech_b200/audio.py convert_out / OutputStream, csrc/audio_kernels.cu
fsb_audio_out): float32 against `audio.resample` bit for bit and against torchaudio in float64, pcm16 against
`utils.pcm16`, mulaw against the G.711 reference, ragged batches and streams against the one-shot call, and the decode
pool, the decode stream and the TTS engine against the one-shot conversion of `from_indices`."""
import queue
import threading

import numpy as np
import pytest
import torch

from fish_speech_b200 import _lib
from fish_speech_b200 import audio as A
from fish_speech_b200.inference_engine import utils as U
from oracle import codec_oracle as CO
from tests.test_audio_out_cpu import PCM16_EDGES, ulaw_ref_array
from tests.test_codec_gpu import build, rand_codes
from tests.test_codec_stream_pool_gpu import one_shot, ragged_schedule

pytestmark = pytest.mark.gpu
# the finite edge cases of utils.pcm16 (an infinity would turn a resampled window into NaN)
EDGES = [(b, v) for b, v in PCM16_EDGES if (b & 0x7F800000) != 0x7F800000]
SR = 44100
RATES = [8000, 16000, 22050, 24000, 48000, SR]
FORMATS = ["float32", "pcm16", "mulaw"]
ULAW = ulaw_ref_array(np.arange(-32768, 32768))  # G.711 of every int16, indexed by sample + 32768


@pytest.fixture(scope="module")
def tiny():
    cfg = CO.tiny_config()
    return cfg, build(cfg, CO.make_weights(cfg, seed=5))


def noise(n, seed, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    return (scale * torch.randn(n, generator=g, dtype=torch.float64)).clamp(-1, 1)


def loud(n, seed):
    """Noise plus full-scale square bursts and hand-made edge values: resampling rings past +-1 on the bursts, and at
    44.1 kHz the edge values reach the quantiser as they are."""
    x = noise(n, seed, scale=0.5).float()
    x[n // 4: n // 4 + 500] = torch.where(torch.arange(500) % 40 < 20, 1.0, -1.0)
    edges = torch.from_numpy(np.array([b for b, _ in EDGES], dtype=np.uint32).view(np.float32).copy())
    x[n // 2: n // 2 + edges.numel()] = edges
    return x


def expected(y32: torch.Tensor, fmt: str) -> np.ndarray:
    """The host definition of each format applied to the float32 output."""
    y = y32.cpu().numpy()
    if fmt == "float32":
        return y
    p = np.frombuffer(U.pcm16(y), dtype="<i2").reshape(y.shape)
    return p if fmt == "pcm16" else ULAW[p.astype(np.int64) + 32768]


def same(a: torch.Tensor, b) -> bool:
    b = b.cpu().numpy() if isinstance(b, torch.Tensor) else b
    a = a.cpu().numpy()
    return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))


# ---- one-shot -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", RATES)
def test_float32_is_resample_bitwise_and_within_the_input_side_bound(sr):
    import torchaudio

    for n in (1, 13, 2048, 7919, 3 * SR):
        x64 = noise(n, n + sr)
        x = x64.float().cuda()
        got = A.convert_out(x, sr, "float32")
        if sr == SR:
            assert got is x  # no launch
            continue
        assert got.dtype == torch.float32 and got.shape == (A.filter_table(SR, sr).total(n),)
        assert torch.equal(got, A.resample(x, SR, sr))
        ref = torchaudio.functional.resample(x64, SR, sr)
        ta32 = torchaudio.functional.resample(x64.float(), SR, sr).double()
        e_got, e_ta = float((got.cpu().double() - ref).abs().max()), float((ta32 - ref).abs().max())
        assert got.shape == ref.shape
        assert e_got <= max(e_ta, 2.0 ** -23), f"{sr} Hz, n={n}: {e_got:.3e} > torchaudio fp32 {e_ta:.3e}"


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("fmt", ["pcm16", "mulaw"])
def test_pcm16_and_mulaw_are_the_host_definitions_of_the_float_output(sr, fmt):
    x = loud(3 * 2048 + 77, seed=sr).cuda()
    y32 = A.convert_out(x, sr, "float32")
    got = A.convert_out(x, sr, fmt)
    assert got.dtype == A.OUTPUT_FORMATS[fmt][1]
    assert same(got, expected(y32, fmt))
    if sr != SR:
        assert float(y32.abs().max()) > 1.0  # the bursts ring past full scale
    else:  # the edge values reach the quantiser unchanged
        e = x.numel() // 2
        vals = got[e: e + len(EDGES)].cpu().numpy().astype(np.int64)
        want = np.array([v for _, v in EDGES])
        assert np.array_equal(vals, want if fmt == "pcm16" else ULAW[want + 32768])


def test_non_finite_values():
    """+-inf clip to full scale, as utils.pcm16 does; NaN (which the decoder's tanh never makes) gives 0."""
    x = torch.tensor([float("nan"), 0.5, float("inf"), float("-inf")], device="cuda")
    assert A.convert_out(x, SR, "pcm16").tolist() == [0, 16383, 32767, -32767]
    assert A.convert_out(x, SR, "mulaw").tolist() == [int(ULAW[v + 32768]) for v in (0, 16383, 32767, -32767)]


def test_ragged_batch_rows_equal_each_row_alone():
    x = torch.stack([loud(5000, s) for s in range(4)]).cuda()
    for sr in (8000, 24000, SR):
        for fmt in FORMATS:
            rows = A.convert_out(x.reshape(4, 1, 5000), sr, fmt)
            for r in range(4):
                assert same(rows[r, 0], A.convert_out(x[r].clone(), sr, fmt))
    # rows of different rates, formats and lengths in one launch
    specs = [(8000, "mulaw", 1), (24000, "pcm16", 4096), (SR, "pcm16", 333), (48000, "float32", 2048),
             (22050, "float32", 9999), (16000, "pcm16", 7)]
    sts = [A.OutputStream(sr, fmt, "cuda") for sr, fmt, _ in specs]
    xs = [loud(max(n, 1000), i).cuda()[:n].contiguous() for i, (_, _, n) in enumerate(specs)]
    before = _lib.launch_count()
    outs = A.OutputStream.push_many(list(zip(sts, xs)))
    assert _lib.launch_count() - before == 1
    tails = A.OutputStream.push_many([(s, None) for s in sts])
    for (sr, fmt, _), x, o, t in zip(specs, xs, outs, tails):
        assert same(torch.cat([o, t]), A.convert_out(x, sr, fmt)), (sr, fmt)


# ---- streams --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("fmt", FORMATS)
def test_output_stream_equals_one_shot(sr, fmt):
    FL, k_max = 2048, 8
    rng = np.random.default_rng(sr)
    for sizes in ([FL] * 7, [k_max * FL] * 3, [int(v) for v in rng.integers(1, 3 * FL, 12)] + [1, FL, k_max * FL]):
        x = loud(sum(sizes), seed=len(sizes)).cuda()
        st = A.OutputStream(sr, fmt, "cuda")
        got, a = [], 0
        for m in sizes:
            got.append(st.push(x[a: a + m]))
            a += m
        got.append(st.flush())
        assert same(torch.cat(got), A.convert_out(x, sr, fmt))
        with pytest.raises(ValueError):
            st.push(x[:10])


def run_pool(pool, dac, streams, specs, schedule):
    """Like test_codec_stream_pool_gpu.run, with each stream opened at its (rate, format) and flushed after its last
    frame. Returns {name: concatenated audio}."""
    slot_of, fed, out = {}, {n: 0 for n in streams}, {n: [] for n in streams}
    for push in schedule:
        pieces = {}
        for name, k in push.items():
            if name not in slot_of:
                sr, fmt = specs[name]
                slot_of[name] = pool.open() if sr is None and fmt is None else pool.open(sr, fmt)
            pieces[slot_of[name]] = streams[name][:, fed[name]: fed[name] + k].clone()
            fed[name] += k
        res = pool.push(pieces)
        for name in push:
            out[name].append(res[slot_of[name]])
            if specs[name] == (None, None):
                assert res[slot_of[name]].shape == (push[name] * dac.frame_length,)
        for name in push:
            if fed[name] == streams[name].shape[-1]:
                out[name].append(pool.flush(slot_of[name]))
                pool.close(slot_of.pop(name))
    return {n: torch.cat(v) for n, v in out.items()}


POOL_SPECS = {"plain": (None, None), "p24": (24000, "pcm16"), "u8": (8000, "mulaw"), "f48": (48000, "float32"),
              "p44": (None, "pcm16"), "f16": (16000, None), "plain2": (None, None)}


def pool_case(cfg):
    lengths = dict(zip(POOL_SPECS, (37, 5, 60, 1, 23, 44, 18)))
    streams = {n: rand_codes(cfg, 1, T, 700 + i)[0] for i, (n, T) in enumerate(lengths.items())}
    return streams, ragged_schedule(lengths, 8, 4, seed=4, late=("f16", "plain2"))


def test_decode_pool_converted_slots_equal_one_shot(tiny):
    cfg, dac = tiny
    streams, sched = pool_case(cfg)
    assert {1, 8} <= {k for p in sched for k in p.values()}
    assert any(len({POOL_SPECS[n] for n in p}) > 2 for p in sched)  # several formats in one push
    pool = dac.open_stream_pool(4, k_max=8)
    got = run_pool(pool, dac, streams, POOL_SPECS, sched)
    for n, codes in streams.items():
        sr, fmt = POOL_SPECS[n]
        ref = one_shot(dac, codes)
        if (sr, fmt) == (None, None):
            assert torch.equal(got[n], ref), n  # today's bits, in pushes that also convert other slots
        else:
            assert same(got[n], A.convert_out(ref, sr, fmt)), n
    assert pool.n_open() == 0


def test_decode_pool_graph_replay_equals_eager(tiny):
    cfg, dac = tiny
    streams, sched = pool_case(cfg)
    graphed = dac.open_stream_pool(4, k_max=8)
    eager = dac.open_stream_pool(4, k_max=8, max_graphs=0)
    g = run_pool(graphed, dac, streams, POOL_SPECS, sched)
    assert graphed._graphs and len(graphed._graphs) <= 8  # one graph per bucket, whatever the formats
    e = run_pool(eager, dac, streams, POOL_SPECS, sched)
    assert not eager._graphs
    for n in streams:
        assert same(g[n], e[n]), n


def test_decode_pool_slot_lifecycle(tiny):
    cfg, dac = tiny
    pool = dac.open_stream_pool(2, k_max=4)
    with pytest.raises(ValueError):
        pool.open(sample_format="mp3")
    with pytest.raises(ValueError):
        pool.open(sample_rate=0)
    assert pool.n_open() == 0  # a refused open takes no slot
    a, b = pool.open(24000, "pcm16"), pool.open()
    codes = rand_codes(cfg, 1, 3, 9)[0]
    pool.push({a: codes.clone(), b: codes.clone()})
    assert pool.flush(b).numel() == 0  # nothing pending without a format
    pool.flush(a)
    with pytest.raises(ValueError):
        pool.flush(a)
    with pytest.raises(ValueError):
        pool.push({a: codes.clone()})
    pool.close(a)
    c = pool.open()  # the slot comes back without a format
    assert c == a and pool.push({c: codes.clone()})[c].dtype == torch.float32


def test_decode_stream_converted_equals_one_shot(tiny):
    cfg, dac = tiny
    codes = rand_codes(cfg, 2, 40, 11)
    whole = dac.from_indices(codes.clone().cuda())
    for sr, fmt in ((24000, "pcm16"), (8000, "mulaw"), (48000, None), (None, "pcm16")):
        st = dac.open_decode_stream(batch=2, max_frames=64, sample_rate=sr, sample_format=fmt)
        got, a = [], 0
        for k in (1, 8, 3, 16, 12):
            got.append(st.push(codes[:, :, a: a + k].clone()))
            a += k
        got.append(st.flush())
        assert same(torch.cat(got, dim=-1), A.convert_out(whole, sr, fmt))
    plain = dac.open_decode_stream(batch=2, max_frames=64)
    assert plain.flush().shape == (2, 1, 0)


# ---- TTS engine -----------------------------------------------------------------------------------------------------
def _engine_request(dac, cfg, monkeypatch, pool, **fields):
    from fish_speech_b200.inference_engine import TTSInferenceEngine
    from fish_speech_b200.inference_engine.schema import ServeTTSRequest
    from fish_speech_b200.models.text2semantic import inference as inf

    if pool:
        monkeypatch.setenv("FSB_STREAM_POOL", "4")
    else:
        monkeypatch.delenv("FSB_STREAM_POOL", raising=False)
    chunks = [rand_codes(cfg, 1, T, 900 + T)[0] for T in (15, 41, 4)]

    def serve(q):
        item = q.get()
        put = lambda a, c=None: item.response_queue.put(inf.WrappedGenerateResponse(
            status="success", response=inf.GenerateResponse(action=a, codes=c)))
        c1, c2, c3 = chunks
        put("partial", c1[:, :8])
        put("partial", c1[:, 8:13])
        put("sample", c1)
        put("partial", c2[:, :40])  # more than one push of k_max frames
        put("sample", c2)
        put("sample", c3)  # nothing streamed: the one-shot decode
        put("next")

    q = queue.Queue()
    threading.Thread(target=serve, args=(q,), daemon=True).start()
    eng = TTSInferenceEngine(q, dac, torch.bfloat16, compile=False)
    try:
        res = list(eng.inference(ServeTTSRequest(text="hi", streaming=True, **fields)))
    finally:
        if eng.codec_worker is not None:
            eng.codec_worker.close()
    return res, chunks


@pytest.mark.parametrize("pool", [False, True])
def test_engine_streaming_request_at_24k_pcm16(tiny, monkeypatch, pool):
    cfg, dac = tiny
    res, chunks = _engine_request(dac, cfg, monkeypatch, pool, sample_rate=24000, sample_format="pcm16")
    assert [r.code for r in res] == ["header"] + ["segment"] * 6 + ["final"]
    assert bytes(res[0].audio[1]) == U.wav_chunk_header(sample_rate=24000, bit_depth=16, format_tag=1)
    want = np.concatenate([A.convert_out(one_shot(dac, c), 24000, "pcm16").cpu().numpy() for c in chunks])
    segs = [r.audio for r in res[1:-1]]
    assert all(rate == 24000 and a.dtype == np.int16 for rate, a in segs)
    assert np.array_equal(np.concatenate([a for _, a in segs]), want)
    assert res[-1].audio[0] == 24000 and np.array_equal(res[-1].audio[1], want)

    plain, _ = _engine_request(dac, cfg, monkeypatch, pool)  # no fields: today's fp32 segments at 44.1 kHz
    assert bytes(plain[0].audio[1]) == U.wav_chunk_header()
    ref = [one_shot(dac, c).cpu().numpy() for c in chunks]
    segs = [r.audio for r in plain[1:-1]]
    assert all(rate == SR and a.dtype == np.float32 for rate, a in segs)
    assert np.array_equal(np.concatenate([a for _, a in segs]), np.concatenate(ref))
