"""DAC.open_stream_pool (DecodeStreamPool): many independent streams decoded together, each stream's audio bit-identical
to `from_indices` of its codes alone; and the ring K/V cache of its post-transformer against the linear cache, for both
attention kernels."""
import random

import pytest
import torch

from oracle import codec_oracle as CO
from tests.test_codec_gpu import build, rand_codes

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    cfg = CO.tiny_config()
    return cfg, build(cfg, CO.make_weights(cfg, seed=5))


def one_shot(dac, codes):
    return dac.from_indices(codes[None].clone().cuda())[0, 0]


def run(pool, dac, streams, schedule):
    """streams: {name: codes [C, T]}; schedule: list of pushes, each {name: k}; a name is opened at its first push and
    closed after its last frame. Returns {name: concatenated audio}."""
    slot_of, fed, audio = {}, {n: 0 for n in streams}, {n: [] for n in streams}
    for push in schedule:
        pieces = {}
        for name, k in push.items():
            if name not in slot_of:
                slot_of[name] = pool.open()
            a = fed[name]
            pieces[slot_of[name]] = streams[name][:, a: a + k].clone()
            fed[name] += k
        out = pool.push(pieces)
        for name in push:
            audio[name].append(out[slot_of[name]])
            assert out[slot_of[name]].shape == (push[name] * dac.frame_length,)
        for name in push:
            if fed[name] == streams[name].shape[-1]:
                pool.close(slot_of.pop(name))
    assert all(fed[n] == streams[n].shape[-1] for n in streams)
    return {n: torch.cat(v) for n, v in audio.items()}


def ragged_schedule(lengths, k_max, max_live, seed, late=()):
    """Random pushes: at most max_live streams at a time, streams in `late` join only after others pushed, each push
    takes 1..k_max frames of a random subset of the live streams."""
    rnd = random.Random(seed)
    left = dict(lengths)
    waiting = [n for n in lengths if n not in late] + list(late)
    live, sched = [], []
    while left:
        while waiting and len(live) < max_live and (waiting[0] not in late or sched):
            live.append(waiting.pop(0))
        push = {}
        for n in live:
            if rnd.random() < 0.75 or len(live) == 1:
                push[n] = min(left[n], rnd.randint(1, k_max))
        if not push:
            push[live[0]] = min(left[live[0]], k_max)
        for n, k in push.items():
            left[n] -= k
            if left[n] == 0:
                del left[n]
                live.remove(n)
        sched.append(push)
    return sched


def test_ragged_streams_equal_one_shot(tiny):
    cfg, dac = tiny
    k_max = 8
    pool = dac.open_stream_pool(4, k_max=k_max)
    lengths = {f"s{i}": T for i, T in enumerate((37, 5, 60, 1, 23, 44, 18))}
    streams = {n: rand_codes(cfg, 1, T, 300 + i)[0] for i, (n, T) in enumerate(lengths.items())}
    sched = ragged_schedule(lengths, k_max, 4, seed=1, late=("s4", "s5", "s6"))
    ks = {k for p in sched for k in p.values()}
    assert 1 in ks and k_max in ks and len({len(p) for p in sched}) > 1
    got = run(pool, dac, streams, sched)
    for n, codes in streams.items():
        assert torch.equal(got[n], one_shot(dac, codes)), f"stream {n} differs from its one-shot decode"
    assert pool.n_open() == 0


def test_idle_slot_state_is_untouched(tiny):
    cfg, dac = tiny
    pool = dac.open_stream_pool(3, k_max=8)
    a, b = rand_codes(cfg, 1, 30, 41)[0], rand_codes(cfg, 1, 60, 42)[0]
    sched = [{"a": 8, "b": 3}, {"a": 5}] + [{"b": 8}] * 7 + [{"b": 1, "a": 8}, {"a": 8}, {"a": 1}]
    got = run(pool, dac, {"a": a, "b": b}, sched)
    assert torch.equal(got["a"], one_shot(dac, a)) and torch.equal(got["b"], one_shot(dac, b))


def test_ring_wraps_and_streams_past_4096_frames(tiny):
    cfg, dac = tiny
    pool = dac.open_stream_pool(2, k_max=32)
    T = 4096 + 70
    codes = rand_codes(cfg, 1, T, 7)[0]
    pieces = [32] * (T // 32) + [T % 32]
    assert T > 20 * pool.ring
    got = run(pool, dac, {"x": codes}, [{"x": k} for k in pieces])
    assert torch.equal(got["x"], one_shot(dac, codes))


def test_graph_replay_equals_eager(tiny):
    cfg, dac = tiny
    lengths = {f"g{i}": T for i, T in enumerate((40, 33, 25, 48))}
    streams = {n: rand_codes(cfg, 1, T, 500 + i)[0] for i, (n, T) in enumerate(lengths.items())}
    sched = ragged_schedule(lengths, 8, 4, seed=3)
    graphed = dac.open_stream_pool(4, k_max=8)
    eager = dac.open_stream_pool(4, k_max=8, max_graphs=0)
    g = run(graphed, dac, streams, sched)
    assert graphed._graphs, "no push was replayed from a CUDA graph"
    e = run(eager, dac, streams, sched)
    assert not eager._graphs
    for n in streams:
        assert torch.equal(g[n], e[n])
        assert torch.equal(g[n], one_shot(dac, streams[n]))


def test_argument_errors(tiny):
    cfg, dac = tiny
    pool = dac.open_stream_pool(2, k_max=4)
    s0, s1 = pool.open(), pool.open()
    with pytest.raises(ValueError):
        pool.open()  # full
    c = rand_codes(cfg, 1, 5, 9)[0]
    with pytest.raises(ValueError):
        pool.push({s0: c})  # 5 > k_max
    with pytest.raises(ValueError):
        pool.push({s0: c[:, :0]})  # no frames
    with pytest.raises(ValueError):
        pool.push({s0: c[1:, :2]})  # wrong number of codebooks
    pool.close(s1)
    with pytest.raises(ValueError):
        pool.push({s1: c[:, :2]})  # closed
    with pytest.raises(ValueError):
        pool.push({7: c[:, :2]})  # unknown
    with pytest.raises(ValueError):
        pool.close(s1)
    before = c.clone()
    c[0, 0] = cfg.semantic_codebook_size + 9  # clamped on the pool's copy, the caller's tensor stays as it is
    out = pool.push({s0: c[:, :3]})
    assert c[0, 0].item() == cfg.semantic_codebook_size + 9 and torch.equal(c[1:], before[1:])
    c[0, 0] = cfg.semantic_codebook_size - 1
    assert torch.equal(out[s0], one_shot(dac, c[:, :3]))


def test_full_geometry_streams_equal_one_shot():
    cfg = CO.full_config()
    dac = build(cfg, CO.make_weights(cfg, seed=6))
    pool = dac.open_stream_pool(8, k_max=32)
    lengths = {f"f{i}": T for i, T in enumerate((40, 37, 44, 41))}
    streams = {n: rand_codes(cfg, 1, T, 900 + i)[0] for i, (n, T) in enumerate(lengths.items())}
    sched = ragged_schedule(lengths, 8, 4, seed=11)
    got = run(pool, dac, streams, sched)
    for n, codes in streams.items():
        assert torch.equal(got[n], one_shot(dac, codes)), f"stream {n} differs from its one-shot decode"


@pytest.mark.parametrize("per_row", [False, True])
def test_ring_kv_attention_equals_linear_cache(per_row):
    """fsb_qkv_rope_ring + fsb_window_attn_ring over a ring of 128 positions give the bits of fsb_qkv_rope +
    fsb_window_attn over a linear cache holding all 600 positions, chunk after chunk, for two sequences."""
    from fish_speech_b200 import _lib

    L = _lib.lib()
    H, Dh, W, R, P = 4, 64, 48, 128, 600
    g = torch.Generator().manual_seed(3)
    freqs = torch.randn(P, Dh // 2, 2, generator=g).to(torch.bfloat16).cuda()
    lin = [torch.zeros(2 * H * P * Dh, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    ring = [torch.zeros(2 * H * (R + 64) * Dh, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    rnd = random.Random(5)
    done = [0, 0]
    st = torch.cuda.current_stream().cuda_stream
    L.fsb_op_attn_per_row(int(per_row))
    try:
        while min(done) < P:
            seq, pos = [], []
            for b in range(2):
                k = min(P - done[b], rnd.randint(0, R - W - 32))  # the ring needs R >= W + k - 1
                seq += [b] * k
                pos += list(range(done[b], done[b] + k))
                done[b] += k
            rows = len(seq)
            if rows == 0:
                continue
            qkv = torch.randn(rows, 3 * H * Dh, generator=g).cuda()
            dseq = torch.tensor(seq, dtype=torch.int32, device="cuda")
            dpos = torch.tensor(pos, dtype=torch.int32, device="cuda")
            outs = []
            for caches, S, is_ring in ((lin, P, 0), (ring, R, 1)):
                q = torch.empty(rows * H * Dh, dtype=torch.bfloat16, device="cuda")
                out = torch.empty_like(q)
                _lib.check(L.fsb_qkv_rope_ring(qkv.data_ptr(), rows, H, H, Dh, freqs.data_ptr(), dseq.data_ptr(),
                                               dpos.data_ptr(), q.data_ptr(), caches[0].data_ptr(),
                                               caches[1].data_ptr(), S, is_ring, st))
                _lib.check(L.fsb_window_attn_ring(q.data_ptr(), caches[0].data_ptr(), caches[1].data_ptr(),
                                                  dseq.data_ptr(), dpos.data_ptr(), rows, H, H, Dh, S, W, is_ring,
                                                  out.data_ptr(), st))
                outs.append(out)
            assert torch.equal(outs[0], outs[1]), f"ring != linear at positions up to {done}"
    finally:
        L.fsb_op_attn_per_row(0)


def test_failed_push_leaves_its_slots_unusable_until_closed(tiny, monkeypatch):
    cfg, dac = tiny
    pool = dac.open_stream_pool(2, k_max=4)
    a, b = pool.open(), pool.open()
    c = rand_codes(cfg, 1, 4, 21)[0]

    def boom(*args, **kw):
        raise RuntimeError("device work failed")

    monkeypatch.setattr(pool, "_body", boom)
    with pytest.raises(RuntimeError):
        pool.push({a: c[:, :2]})
    monkeypatch.undo()
    with pytest.raises(ValueError, match="close the slot"):
        pool.push({a: c[:, 2:]})
    assert torch.equal(pool.push({b: c[:, :2]})[b], one_shot(dac, c[:, :2]))  # other slots are unaffected
    pool.close(a)
    a2 = pool.open()
    assert torch.equal(pool.push({a2: c})[a2], one_shot(dac, c))


def _lib():
    from fish_speech_b200 import _lib as lib_mod

    return lib_mod, lib_mod.lib()


@pytest.mark.parametrize("C,H,n,taps,dil", [(64, 6, 40, 7, 1), (128, 54, 300, 7, 9), (96, 1, 17, 2, 1)])
def test_conv_gemm_over_a_window_equals_the_zero_history_call(C, H, n, taps, dil):
    """The pool's conv layers: taps shifted by H over [B][H + n][C] with zero history rows give the bits of the plain
    causal call on the n rows."""
    import ctypes

    lib_mod, L = _lib()
    g = torch.Generator().manual_seed(C + H)
    B, co, kpad = 3, 2 * C, (C + 63) // 64 * 64
    x = torch.randn(B, n, C, generator=g).to(torch.bfloat16).cuda()
    w = torch.zeros(co, taps, kpad)
    w[:, :, :C] = torch.randn(co, taps, C, generator=g) / (taps * C) ** 0.5
    w = w.reshape(co, taps * kpad).to(torch.bfloat16).cuda()
    bias = torch.randn(co, generator=g).cuda()
    shifts = [-(taps - 1 - j) * dil for j in range(taps)]
    win = torch.zeros(B, H + n, C, dtype=torch.bfloat16, device="cuda")
    win[:, H:] = x
    st = torch.cuda.current_stream().cuda_stream
    outs = []
    for src, T_in, sh in ((x, n, shifts), (win, H + n, [s + H for s in shifts])):
        o = torch.empty(B, n, co, dtype=torch.bfloat16, device="cuda")
        lib_mod.check(L.fsb_conv_gemm(src.data_ptr(), B, T_in, C, C, T_in * C, w.data_ptr(), co, taps, kpad,
                                      (ctypes.c_int * taps)(*sh), n, bias.data_ptr(), None, None, 0, o.data_ptr(), None,
                                      None, None, 0, st))
        outs.append(o)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("C,n", [(256, 33), (1024, 64)])
def test_dwconv_ln_window_equals_the_zero_history_call(C, n):
    lib_mod, L = _lib()
    g = torch.Generator().manual_seed(C)
    B, K, H = 2, 7, 6
    x = torch.randn(B, n, C, generator=g).to(torch.bfloat16).cuda()
    w, b = torch.randn(C, K, generator=g).cuda(), torch.randn(C, generator=g).cuda()
    lw, lb = torch.randn(C, generator=g).cuda(), torch.randn(C, generator=g).cuda()
    win = torch.zeros(B, H + n, C, dtype=torch.bfloat16, device="cuda")
    win[:, H:] = x
    st = torch.cuda.current_stream().cuda_stream
    y0 = torch.empty(B, n, C, dtype=torch.bfloat16, device="cuda")
    y1 = torch.empty_like(y0)
    lib_mod.check(L.fsb_dwconv_ln(x.data_ptr(), w.data_ptr(), b.data_ptr(), lw.data_ptr(), lb.data_ptr(), B, n, C, K,
                                  1e-6, y0.data_ptr(), st))
    lib_mod.check(L.fsb_dwconv_ln_window(win.data_ptr(), w.data_ptr(), b.data_ptr(), lw.data_ptr(), lb.data_ptr(), B,
                                         H + n, H, n, C, K, 1e-6, y1.data_ptr(), st))
    assert torch.equal(y0, y1)
    # with real history: the window's rows H.. are the plain call's last n rows over [history | x]
    hist = torch.randn(B, H, C, generator=g).to(torch.bfloat16).cuda()
    win[:, :H] = hist
    full = torch.cat([hist, x], 1).contiguous()
    y2 = torch.empty(B, H + n, C, dtype=torch.bfloat16, device="cuda")
    lib_mod.check(L.fsb_dwconv_ln(full.data_ptr(), w.data_ptr(), b.data_ptr(), lw.data_ptr(), lb.data_ptr(), B, H + n,
                                  C, K, 1e-6, y2.data_ptr(), st))
    lib_mod.check(L.fsb_dwconv_ln_window(win.data_ptr(), w.data_ptr(), b.data_ptr(), lw.data_ptr(), lb.data_ptr(), B,
                                         H + n, H, n, C, K, 1e-6, y1.data_ptr(), st))
    assert torch.equal(y2[:, H:], y1)


def test_window_fill_and_roll_against_a_reference():
    lib_mod, L = _lib()
    g = torch.Generator().manual_seed(1)
    slots, nb, H, n, C = 5, 4, 6, 16, 24
    state = torch.randn(slots, H, C, generator=g).to(torch.bfloat16).cuda()
    dense = torch.randn(nb, n, C, generator=g).to(torch.bfloat16).cuda()
    win = torch.full((nb, H + n, C), 7.0, dtype=torch.bfloat16, device="cuda")
    slot = torch.tensor([3, 0, -1, 4], dtype=torch.int32, device="cuda")
    valid = torch.tensor([16, 2, 0, 9], dtype=torch.int32, device="cuda")
    ref_win, ref_state = win.clone(), state.clone()
    for i, (s, v) in enumerate(zip(slot.tolist(), valid.tolist())):
        if s < 0:
            continue
        ref_win[i, :H] = state[s]
        ref_win[i, H: H + v] = dense[i, :v]
        ref_state[s] = ref_win[i, v: v + H]
    st = torch.cuda.current_stream().cuda_stream
    lib_mod.check(L.fsb_window_fill(state.data_ptr(), dense.data_ptr(), win.data_ptr(), slot.data_ptr(),
                                    valid.data_ptr(), nb, H, n, C * 2, st))
    lib_mod.check(L.fsb_window_roll(win.data_ptr(), state.data_ptr(), slot.data_ptr(), valid.data_ptr(), nb, H, n,
                                    C * 2, st))
    assert torch.equal(win, ref_win) and torch.equal(state, ref_state)
