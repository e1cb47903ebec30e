"""DAC.open_encode_pool (EncodeStreamPool): many independent streams encoded together, each stream's codes bit-identical
to the one-shot `DAC.encode` of its waveform alone; the windowed first conv and strided conv against their zero-history
calls; ring against linear attention at the encoder transformer's window; and `DAC.encode` / `bulk_encode` routed through
the pool when the one-shot pass would not fit in free device memory."""
import ctypes
import random

import numpy as np
import pytest
import torch

from oracle import codec_oracle as CO
from tests.test_codec_gpu import GOLD, build
from tests.test_codec_stream_pool_gpu import ragged_schedule

pytestmark = pytest.mark.gpu
FL = 2048


@pytest.fixture(scope="module")
def tiny():
    cfg = CO.tiny_config()  # encoder transformer window 32, pre_module window 16
    return cfg, build(cfg, CO.make_weights(cfg, seed=5))


def rand_wav(n, seed):
    g = torch.Generator().manual_seed(seed)
    return 0.1 * torch.randn(n, generator=g)


def one_shot(dac, wav, n_quantizers=None):
    """codes [S, T] of the one-shot pass over one clip (whatever the free-memory probe says)."""
    codes, _ = dac._encode_one_shot(wav.view(1, 1, -1).cuda(), None, n_quantizers)
    return codes[0]


def run(pool, streams, schedule):
    """streams: {name: waveform [n] (any n)}; schedule: list of pushes {name: frames}; a name is opened at its first
    push and closed after its last frame, its last piece zero-padded to a whole frame. Returns {name: codes [S, T]}."""
    slot_of, fed, codes = {}, {n: 0 for n in streams}, {n: [] for n in streams}
    frames = {n: -(-w.numel() // FL) for n, w in streams.items()}
    for push in schedule:
        pieces = {}
        for name, k in push.items():
            if name not in slot_of:
                slot_of[name] = pool.open()
            a = fed[name]
            piece = streams[name][a * FL: (a + k) * FL]
            pieces[slot_of[name]] = torch.nn.functional.pad(piece, (0, k * FL - piece.numel()))
            fed[name] += k
        out = pool.push(pieces)
        for name, k in push.items():
            assert out[slot_of[name]].shape == (pool.n_stage, k) and out[slot_of[name]].dtype == torch.int64
            codes[name].append(out[slot_of[name]].cpu())
        for name in push:
            if fed[name] == frames[name]:
                pool.close(slot_of.pop(name))
    assert all(fed[n] == frames[n] for n in streams)
    return {n: torch.cat(v, dim=1) for n, v in codes.items()}


def check(dac, got, streams, n_quantizers=None):
    for n, w in streams.items():
        assert torch.equal(got[n], one_shot(dac, w, n_quantizers).cpu()), f"stream {n} differs from its one-shot encode"


def test_ragged_streams_equal_one_shot(tiny):
    cfg, dac = tiny
    k_max = 8
    pool = dac.open_encode_pool(4, k_max=k_max)
    lengths = {f"s{i}": T for i, T in enumerate((37, 5, 60, 1, 23, 44, 18))}
    # lengths that are not a multiple of 2048: the caller zero-pads the last piece, encode pads the clip
    streams = {n: rand_wav(T * FL - (0 if i % 2 else 700 + 97 * i), 300 + i) for i, (n, T) in enumerate(lengths.items())}
    sched = ragged_schedule(lengths, k_max, 4, seed=1, late=("s4", "s5", "s6"))
    ks = {k for p in sched for k in p.values()}
    assert 1 in ks and k_max in ks and len({len(p) for p in sched}) > 1
    got = run(pool, streams, sched)
    check(dac, got, streams)
    assert pool.n_open() == 0
    # slots are reused by the late streams
    assert len(lengths) > pool.slots


def test_idle_slot_state_is_untouched(tiny):
    cfg, dac = tiny
    pool = dac.open_encode_pool(3, k_max=8)
    streams = {"a": rand_wav(30 * FL, 41), "b": rand_wav(60 * FL, 42)}
    sched = [{"a": 8, "b": 3}, {"a": 5}] + [{"b": 8}] * 7 + [{"b": 1, "a": 8}, {"a": 8}, {"a": 1}]
    check(dac, run(pool, streams, sched), streams)


def test_n_quantizers(tiny):
    cfg, dac = tiny
    pool = dac.open_encode_pool(2, k_max=8, n_quantizers=1)
    assert pool.n_stage == 2
    streams = {"a": rand_wav(21 * FL + 5, 51), "b": rand_wav(13 * FL, 52)}
    sched = ragged_schedule({"a": 22, "b": 13}, 8, 2, seed=4)
    check(dac, run(pool, streams, sched), streams, n_quantizers=1)


def test_rings_wrap_and_streams_past_4096_frames(tiny):
    cfg, dac = tiny
    pool = dac.open_encode_pool(2, k_max=32)
    T = 4096 + 70
    wav = rand_wav(T * FL - 1234, 7)
    pieces = [32] * (T // 32) + [T % 32]
    assert T * 4 > 20 * pool.rings[0] and T > 20 * pool.rings[-1]  # both windows crossed and both rings wrapped often
    check(dac, run(pool, {"x": wav}, [{"x": k} for k in pieces]), {"x": wav})


def test_graph_replay_equals_eager(tiny):
    """Buckets are captured into CUDA graphs the second time they are seen; replays give the eager bits. The schedule
    also puts padding rows (and the scratch sequence) in the same attention tiles as valid rows in many pushes."""
    cfg, dac = tiny
    lengths = {f"g{i}": T for i, T in enumerate((40, 33, 25, 48))}
    streams = {n: rand_wav(T * FL, 500 + i) for i, (n, T) in enumerate(lengths.items())}
    sched = ragged_schedule(lengths, 8, 4, seed=3)
    graphed = dac.open_encode_pool(4, k_max=8)
    eager = dac.open_encode_pool(4, k_max=8, max_graphs=0)
    g = run(graphed, streams, sched)
    assert graphed._graphs, "no push was replayed from a CUDA graph"
    e = run(eager, streams, sched)
    assert not eager._graphs
    for n in streams:
        assert torch.equal(g[n], e[n])
    check(dac, g, streams)


def test_argument_errors(tiny):
    cfg, dac = tiny
    pool = dac.open_encode_pool(2, k_max=4)
    s0, s1 = pool.open(), pool.open()
    with pytest.raises(ValueError):
        pool.open()  # full
    w = rand_wav(5 * FL, 9)
    with pytest.raises(ValueError):
        pool.push({s0: w})  # 5 > k_max
    with pytest.raises(ValueError):
        pool.push({s0: w[: FL + 3]})  # not whole frames
    with pytest.raises(ValueError):
        pool.push({s0: w[:0]})  # no frames
    with pytest.raises(ValueError):
        pool.push({s0: w[: 2 * FL].double()})  # not fp32
    pool.close(s1)
    with pytest.raises(ValueError):
        pool.push({s1: w[: 2 * FL]})  # closed
    with pytest.raises(ValueError):
        pool.push({7: w[: 2 * FL]})  # unknown
    with pytest.raises(ValueError):
        pool.close(s1)
    before = w.clone()
    out = pool.push({s0: w[: 3 * FL]})
    assert torch.equal(w, before)
    assert torch.equal(out[s0].cpu(), one_shot(dac, w[: 3 * FL]).cpu())


def test_failed_push_leaves_its_slots_unusable_until_closed(tiny, monkeypatch):
    cfg, dac = tiny
    pool = dac.open_encode_pool(2, k_max=4)
    a, b = pool.open(), pool.open()
    w = rand_wav(4 * FL, 21)

    def boom(*args, **kw):
        raise RuntimeError("device work failed")

    monkeypatch.setattr(pool, "_body", boom)
    with pytest.raises(RuntimeError):
        pool.push({a: w[: 2 * FL]})
    monkeypatch.undo()
    with pytest.raises(ValueError, match="close the slot"):
        pool.push({a: w[2 * FL:]})
    assert torch.equal(pool.push({b: w[: 2 * FL]})[b].cpu(), one_shot(dac, w[: 2 * FL]).cpu())  # others unaffected
    pool.close(a)
    a2 = pool.open()
    assert torch.equal(pool.push({a2: w})[a2].cpu(), one_shot(dac, w).cpu())


def test_full_geometry_streams_equal_one_shot():
    cfg = CO.full_config()
    dac = build(cfg, CO.make_weights(cfg, seed=6))
    pool = dac.open_encode_pool(4, k_max=32)
    streams = {"long": rand_wav(310 * FL - 999, 61), "short": rand_wav(45 * FL, 62)}
    # mixed piece sizes, 1 and k_max among them, the short stream alongside in the first pushes
    long_k = [1, 32, 7, 32, 3, 16, 1, 32, 32, 5, 32, 32, 32, 32, 21]
    short_k = [8, 1, 32, 4]
    assert sum(long_k) == 310 and sum(short_k) == 45
    sched = [dict([("long", a)] + ([("short", b)] if i < len(short_k) else []))
             for i, (a, b) in enumerate(zip(long_k, short_k + [0] * len(long_k)))]
    check(dac, run(pool, streams, sched), streams)
    # the committed 1 s input, whose one-shot codes the codec tests hold against the reference's
    z = np.load(GOLD / "codec_full_1s.npz")
    dac = build(cfg, CO.make_weights(cfg, seed=int(z["weight_seed"])))
    audio = torch.from_numpy(z["audio"]).reshape(-1)
    pool = dac.open_encode_pool(1, k_max=8)
    n = -(-audio.numel() // FL)
    got = run(pool, {"g": audio}, [{"g": k} for k in [3, 8, 1] + [8] * ((n - 12) // 8) + [(n - 12) % 8] if k])
    check(dac, got, {"g": audio})


# ---- kernels ----------------------------------------------------------------------------------------------------
def _lib():
    from fish_speech_b200 import _lib as lib_mod

    return lib_mod, lib_mod.lib()


@pytest.mark.parametrize("C,n", [(64, 2048 * 3), (16, 1000)])
def test_first_conv_window_equals_the_zero_history_call(C, n):
    lib_mod, L = _lib()
    g = torch.Generator().manual_seed(C)
    B, K, H = 3, 7, 8
    x = torch.randn(B, n, generator=g).cuda()
    w, b = torch.randn(C, K, generator=g).cuda(), torch.randn(C, generator=g).cuda()
    alpha = (1 + 0.3 * torch.randn(C, generator=g)).abs().cuda()
    inv = (alpha + 1e-9).reciprocal()
    st = torch.cuda.current_stream().cuda_stream
    win = torch.zeros(B, H + n, device="cuda")
    win[:, H:] = x
    outs = []
    for call in range(2):
        raw = torch.empty(B, n, C, dtype=torch.bfloat16, device="cuda")
        act = torch.empty_like(raw)
        if call == 0:
            lib_mod.check(L.fsb_first_conv(x.data_ptr(), w.data_ptr(), b.data_ptr(), alpha.data_ptr(), inv.data_ptr(), B,
                                           n, C, K, raw.data_ptr(), act.data_ptr(), st))
        else:
            lib_mod.check(L.fsb_first_conv_window(win.data_ptr(), w.data_ptr(), b.data_ptr(), alpha.data_ptr(),
                                                  inv.data_ptr(), B, H + n, H, n, C, K, raw.data_ptr(), act.data_ptr(), st))
        outs.append((raw, act))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    # with real history: the window's samples H.. are the plain call's last n samples over [history | x]
    hist = torch.randn(B, H, generator=g).cuda()
    win[:, :H] = hist
    full = torch.cat([hist, x], 1).contiguous()
    raw2 = torch.empty(B, H + n, C, dtype=torch.bfloat16, device="cuda")
    lib_mod.check(L.fsb_first_conv(full.data_ptr(), w.data_ptr(), b.data_ptr(), alpha.data_ptr(), inv.data_ptr(), B,
                                   H + n, C, K, raw2.data_ptr(), None, st))
    raw = torch.empty(B, n, C, dtype=torch.bfloat16, device="cuda")
    lib_mod.check(L.fsb_first_conv_window(win.data_ptr(), w.data_ptr(), b.data_ptr(), None, None, B, H + n, H, n, C, K,
                                          raw.data_ptr(), None, st))
    assert torch.equal(raw2[:, H:], raw)
    with pytest.raises(lib_mod.FsbError):
        lib_mod.check(L.fsb_first_conv_window(win.data_ptr(), w.data_ptr(), b.data_ptr(), None, None, B, H + n, H + 1, n,
                                              C, K, raw.data_ptr(), None, st))


@pytest.mark.parametrize("c,s,n", [(64, 2, 700), (512, 8, 33), (16, 4, 64)])
def test_strided_conv_over_a_window_equals_the_zero_history_call(c, s, n):
    """The encoder's down convs (k = 2 * stride) read the activation as [T / s][s * c] rows with 2 taps: one history row
    of that view before the new rows gives the bits of the plain causal call."""
    lib_mod, L = _lib()
    g = torch.Generator().manual_seed(c + s)
    B, co, taps, H = 2, 2 * c, 2, 1
    Ci = s * c
    kpad = (Ci + 63) // 64 * 64
    x = torch.randn(B, n * s, c, generator=g).to(torch.bfloat16).cuda()  # [T][c] = [T / s][s * c]
    w = torch.zeros(co, taps, kpad)
    w[:, :, :Ci] = torch.randn(co, taps, Ci, generator=g) / (taps * Ci) ** 0.5
    w = w.reshape(co, taps * kpad).to(torch.bfloat16).cuda()
    bias = torch.randn(co, generator=g).cuda()
    win = torch.zeros(B, H + n, Ci, dtype=torch.bfloat16, device="cuda")
    win[:, H:] = x.view(B, n, Ci)
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for src, T_in, sh in ((x, n, [-1, 0]), (win, H + n, [0, 1])):
        o = torch.empty(B, n, co, dtype=torch.bfloat16, device="cuda")
        lib_mod.check(L.fsb_conv_gemm(src.data_ptr(), B, T_in, Ci, Ci, T_in * Ci, w.data_ptr(), co, taps, kpad,
                                      (ctypes.c_int * taps)(*sh), n, bias.data_ptr(), None, None, 0, o.data_ptr(), None,
                                      None, None, 0, st))
        outs.append(o)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("per_row", [False, True])
def test_ring_kv_attention_equals_linear_cache_at_the_encoder_window(per_row):
    """The encoder transformer's attention (window 512, head_dim 64, 4 rows per frame): ring of
    round_up(512 + 4 * k_max + 63, 64) positions against a linear cache holding every position, for pieces of 1 frame
    (4 rows) up to k_max frames per sequence, three sequences."""
    lib_mod, L = _lib()
    H, Dh, W, k_max, P = 4, 64, 512, 32, 2600
    R = (W + 4 * k_max + 63 + 63) // 64 * 64
    g = torch.Generator().manual_seed(8)
    freqs = torch.randn(P, Dh // 2, 2, generator=g).to(torch.bfloat16).cuda()
    nseq = 3
    lin = [torch.zeros(nseq * H * P * Dh, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    ring = [torch.zeros(nseq * H * (R + 64) * Dh, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    rnd = random.Random(6)
    done = [0] * nseq
    st = torch.cuda.current_stream().cuda_stream
    L.fsb_op_attn_per_row(int(per_row))
    try:
        while min(done) < P:
            seq, pos = [], []
            for b in range(nseq):
                k = min(P - done[b], 4 * rnd.choice([1, 1, 2, 5, 8, 16, k_max]))
                seq += [b] * k
                pos += list(range(done[b], done[b] + k))
                done[b] += k
            rows = len(seq)
            qkv = torch.randn(rows, 3 * H * Dh, generator=g).cuda()
            dseq = torch.tensor(seq, dtype=torch.int32, device="cuda")
            dpos = torch.tensor(pos, dtype=torch.int32, device="cuda")
            outs = []
            for caches, S, is_ring in ((lin, P, 0), (ring, R, 1)):
                q = torch.empty(rows * H * Dh, dtype=torch.bfloat16, device="cuda")
                out = torch.empty_like(q)
                lib_mod.check(L.fsb_qkv_rope_ring(qkv.data_ptr(), rows, H, H, Dh, freqs.data_ptr(), dseq.data_ptr(),
                                                  dpos.data_ptr(), q.data_ptr(), caches[0].data_ptr(),
                                                  caches[1].data_ptr(), S, is_ring, st))
                lib_mod.check(L.fsb_window_attn_ring(q.data_ptr(), caches[0].data_ptr(), caches[1].data_ptr(),
                                                     dseq.data_ptr(), dpos.data_ptr(), rows, H, H, Dh, S, W, is_ring,
                                                     out.data_ptr(), st))
                outs.append(out)
            assert torch.equal(outs[0], outs[1]), f"ring != linear at positions up to {done}"
    finally:
        L.fsb_op_attn_per_row(0)


# ---- bounded memory and routing -----------------------------------------------------------------------------------
def test_streaming_8x_longer_grows_memory_by_the_rope_table_only(tiny):
    cfg, dac = tiny
    pool = dac.open_encode_pool(1, k_max=32)

    def stream(frames, seed):
        s = pool.open()
        wav = rand_wav(frames * FL, seed)
        for f0 in range(0, frames, 32):
            pool.push({s: wav[f0 * FL: (f0 + 32) * FL]})[s].cpu()
        pool.close(s)
        torch.cuda.synchronize()

    def rope_bytes():
        return sum(v.numel() * v.element_size() for v in dac._rope.values())

    stream(512, 1)  # sizes every workspace
    torch.cuda.reset_peak_memory_stats()
    r0 = rope_bytes()
    stream(512, 2)
    peak1 = torch.cuda.max_memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    stream(8 * 512, 3)
    peak8 = torch.cuda.max_memory_allocated()
    r8 = rope_bytes()
    growth = r8 if r8 != r0 else 0  # a grown table is allocated while the old one still exists
    print(f"peak allocated: {peak1} B streaming 512 frames, {peak8} B streaming 4096 frames; RoPE tables {r0} -> {r8} B")
    assert peak8 - peak1 <= growth


def _patched_low(monkeypatch, dac):
    calls = []
    real = dac._encode_streamed

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(dac, "_free_device_bytes", lambda: 0)
    monkeypatch.setattr(dac, "_encode_streamed", spy)
    return calls


def test_encode_routes_to_the_pool_when_the_one_shot_does_not_fit(tiny, monkeypatch):
    cfg, dac = tiny
    g = torch.Generator().manual_seed(4)
    lens = torch.tensor([2048 * 150 + 77, 2048 * 20, 2048 * 131 + 2047, 999, 2048 * 60 + 1])
    audio = 0.1 * torch.randn(len(lens), 1, int(lens.max()), generator=g)
    for b, n in enumerate(lens.tolist()):
        audio[b, :, n:] = 0
    cases = [(audio, lens, None), (audio[:1, 0], None, None), (audio[2:4], lens[2:4], 2)]
    ref = [dac._encode_one_shot(a.cuda(), None if l is None else l.cuda(), q) for a, l, q in cases]
    calls = _patched_low(monkeypatch, dac)
    for (a, l, q), (rc, rl) in zip(cases, ref):
        codes, out_lens = dac.encode(a.cuda(), None if l is None else l.cuda(), n_quantizers=q)
        assert codes.dtype == rc.dtype and codes.shape == rc.shape and torch.equal(codes, rc)
        assert torch.equal(out_lens, rl)
    assert len(calls) == len(cases)


def test_bulk_encode_writes_the_same_files_either_way(tiny, tmp_path, monkeypatch):
    import wave

    from fish_speech_b200 import bulk_encode as BE

    cfg, dac = tiny
    g = torch.Generator().manual_seed(5)
    files = []
    for i, n in enumerate([2048 * 300 + 17, 2048 * 9, 2048 * 41 + 1000]):
        pcm = ((0.1 * torch.randn(n, generator=g)).clamp(-1, 1) * 32767).round().to(torch.int16)
        f = tmp_path / f"clip{i}.wav"
        with wave.open(str(f), "wb") as wf:
            wf.setnchannels(1)
            wf.setsampwidth(2)
            wf.setframerate(cfg.sample_rate)
            wf.writeframes(pcm.numpy().tobytes())
        files.append(f)
    BE.encode_files(files, dac, batch_size=2)
    first = [f.with_suffix(".npy").read_bytes() for f in files]
    for f in files:
        f.with_suffix(".npy").unlink()
    calls = _patched_low(monkeypatch, dac)
    BE.encode_files(files, dac, batch_size=2)
    assert calls
    assert [f.with_suffix(".npy").read_bytes() for f in files] == first
