"""Host side of DAC.from_indices' routing and of the ragged batch decode (no GPU), with a stand-in codec: the one-shot
pass runs when its workspaces fit in free device memory and its post-transformer rows fit one launch, the streamed path
otherwise, and a shape with a captured graph never probes memory; the one-shot workspace estimate; the pool driver's
pieces, slot reuse and output placement; and the argument checks of `from_indices_list` / `batch_vqgan_decode`."""
import contextlib
import threading

import numpy as np
import pytest
import torch

from fish_speech_b200 import bulk_encode as BE
from fish_speech_b200.models.dac import modded_dac as M

FL = 2048


def bare_codec(monkeypatch):
    dac = M.DAC.__new__(M.DAC)
    dac.cfg = M.CodecConfig()
    dac.frame_length, dac.n_stage = FL, 1 + dac.cfg.n_codebooks
    dac.post_tfm = {"cfg": dac.cfg.quant_tfm}
    dac._device = torch.device("cpu")
    dac._lock = threading.RLock()
    dac._bufs, dac._graphs, dac._graph_seen = {}, {}, {}
    dac._dec_pool = None
    monkeypatch.setattr(M.torch.cuda, "device", lambda d: contextlib.nullcontext())
    return dac


def fake_codec(monkeypatch, free: int, need: int):
    """A DAC with no device: the probe, the estimate and both paths replaced by recorders."""
    dac = bare_codec(monkeypatch)
    calls = []
    monkeypatch.setattr(dac, "_free_device_bytes", lambda: free)
    monkeypatch.setattr(dac, "_decode_one_shot_bytes", lambda B, T: need)
    monkeypatch.setattr(dac, "_from_indices_body",
                        lambda idx, B, S, T: calls.append("one_shot") or torch.zeros(B, T * FL))
    monkeypatch.setattr(dac, "_from_indices_streamed",
                        lambda idx: calls.append("streamed") or torch.ones(idx.shape[0], 1, idx.shape[2] * FL))
    return dac, calls


def codes(B, T, seed=0, hi=4096):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, hi, (B, 10, T), generator=g)


@pytest.mark.parametrize("need,free,path", [
    (1 << 30, 80 << 30, "one_shot"),
    (1 << 30, (1 << 30) + (512 << 20) + (1 << 30) // 20, "one_shot"),  # exactly need + margin
    (1 << 30, (1 << 30) + (512 << 20) + (1 << 30) // 20 - 1, "streamed"),
    (61 << 30, 79 << 30, "one_shot"),
    (122 << 30, 79 << 30, "streamed"),
    (0, 0, "streamed"),
])
def test_routing_rule(monkeypatch, need, free, path):
    dac, calls = fake_codec(monkeypatch, free, need)
    wav = dac.from_indices(codes(1, 7))
    assert wav.shape == (1, 1, 7 * FL) and calls == [path]


@pytest.mark.parametrize("B,T,path", [(1, 65535, "one_shot"), (1, 65536, "streamed"),
                                      (3, 21845, "one_shot"), (3, 21846, "streamed")])
def test_routing_rule_post_transformer_rows(monkeypatch, B, T, path):
    """The one-shot pass launches B x T post-transformer rows, at most 65 535."""
    dac, calls = fake_codec(monkeypatch, 1 << 50, 1 << 30)
    dac.from_indices(torch.zeros(B, 10, T, dtype=torch.int64))
    assert calls == [path]


def test_captured_shape_replays_without_probing_memory(monkeypatch):
    dac, calls = fake_codec(monkeypatch, 0, 1 << 30)
    monkeypatch.setattr(dac, "_free_device_bytes", lambda: pytest.fail("probed free memory"))
    monkeypatch.setattr(dac, "_decode_one_shot_bytes", lambda B, T: pytest.fail("estimated workspaces"))
    replays = []
    g_idx, g_wav = torch.zeros(2 * 10 * 5, dtype=torch.int32), torch.full((2, 5 * FL), 3.0)
    dac._graphs[(2, 10, 5)] = (type("G", (), {"replay": lambda self: replays.append(1)})(), g_idx, g_wav)
    c = codes(2, 5, 1)
    wav = dac.from_indices(c)
    assert replays == [1] and calls == [] and torch.equal(g_idx, c.reshape(-1).int())
    assert wav.shape == (2, 1, 5 * FL) and torch.equal(wav, g_wav.view(2, 1, -1))


@pytest.mark.parametrize("path", ["one_shot", "streamed"])
def test_codes_are_clamped_in_place_on_both_routes(monkeypatch, path):
    dac, calls = fake_codec(monkeypatch, 1 << 50 if path == "one_shot" else 0, 1 << 30)
    c = codes(2, 6, 3, hi=1024)
    c[0, 0, 1], c[1, 0, 5], c[1, 3, 2], c[0, 9, 0] = 4096 + 9, 10 ** 6, 1024, 5000
    want = c.clone()
    want[:, 0].clamp_(max=4095)
    want[:, 1:].clamp_(max=1023)
    dac.from_indices(c)
    assert calls == [path] and torch.equal(c, want)


def test_one_shot_estimate_grows_and_counts_only_workspaces_that_grow(monkeypatch):
    dac = bare_codec(monkeypatch)
    cfg = dac.cfg
    one = dac._decode_one_shot_bytes(1, 10_000)
    assert dac._decode_one_shot_bytes(1, 20_000) > one and dac._decode_one_shot_bytes(4, 10_000) > one
    # 393 KB per frame in each of the decoder's three bf16 buffers (96 channels x 2048 samples), and the waveform
    act = 3 * 10_000 * 96 * 2048 * 2
    assert dac._decoder_numel(1, 4 * 10_000) == 10_000 * 96 * 2048
    assert act + 10_000 * FL * 4 <= one <= act * 1.4
    dac._bufs = {f"dec_{k}": torch.empty(1, dtype=torch.bfloat16).expand(10_000 * 96 * 2048) for k in range(3)}
    assert dac._decode_one_shot_bytes(1, 10_000) == one - act
    # a larger transformer workspace than needed counts 0 as well
    rows, HD = 10_000, cfg.quant_tfm.n_head * cfg.quant_tfm.head_dim
    ws = rows * max(3 * HD, 2 * cfg.quant_tfm.intermediate_size, cfg.quant_tfm.dim)
    dac._bufs["tf_ws"] = torch.empty(1, dtype=torch.float32).expand(ws + 1)
    assert dac._decode_one_shot_bytes(1, 10_000) == one - act - 4 * ws


class _FakePool:
    """A push returns, per frame of a piece, its semantic code repeated over the frame's samples; records every push."""

    def __init__(self, slots, k_max):
        self.slots, self.k_max = slots, k_max
        self.live, self.pushes = [False] * slots, []

    def open(self):
        s = self.live.index(False)
        self.live[s] = True
        return s

    def close(self, s):
        assert self.live[s]
        self.live[s] = False

    def push(self, pieces):
        self.pushes.append({s: c.shape[1] for s, c in pieces.items()})
        out = {}
        for s, c in pieces.items():
            assert self.live[s] and c.dtype == torch.int32 and c.shape[0] == 10 and 1 <= c.shape[1] <= self.k_max
            out[s] = c[0].float().repeat_interleave(FL)
        return out


def pooled_codec(monkeypatch):
    dac = bare_codec(monkeypatch)
    pools = []
    monkeypatch.setattr(dac, "open_stream_pool", lambda slots, k_max: pools.append(_FakePool(slots, k_max)) or pools[-1])
    return dac, pools


def test_streamed_from_indices_pieces_and_output(monkeypatch):
    dac, pools = pooled_codec(monkeypatch)
    K, N = M.DAC.DECODE_STREAM_FRAMES, M.DAC.DECODE_STREAM_SLOTS
    B, T = N + 2, 3 * K + 5
    c = codes(B, T, 4)
    wav = dac._from_indices_streamed(c)
    assert wav.shape == (B, 1, T * FL) and wav.dtype == torch.float32
    assert torch.equal(wav[:, 0], c[:, 0].float().repeat_interleave(FL, dim=1))
    (pool,) = pools
    assert pool.slots == N and pool.k_max == K and not any(pool.live)
    # N rows side by side in pieces of K frames and a remainder, then the last rows
    assert pool.pushes == [{s: K for s in range(N)}] * 3 + [{s: 5 for s in range(N)}] + [{0: K, 1: K}] * 3 + [{0: 5, 1: 5}]
    dac._from_indices_streamed(codes(1, 2, 5))
    assert len(pools) == 1, "the pool is kept for later calls"


def test_ragged_items_take_slots_as_earlier_ones_finish(monkeypatch):
    dac, pools = pooled_codec(monkeypatch)
    K, N = M.DAC.DECODE_STREAM_FRAMES, M.DAC.DECODE_STREAM_SLOTS
    lengths = [1, 37, 2 * K, 500, 3000, K - 1, K + 1, 7]
    items = [codes(1, T, 10 + i)[0] for i, T in enumerate(lengths)]
    before = [c.clone() for c in items]
    outs = BE.batch_vqgan_decode(dac, items)
    assert [o.shape for o in outs] == [(1, T * FL) for T in lengths] and all(o.dtype == np.float32 for o in outs)
    for o, c in zip(outs, items):
        assert np.array_equal(o[0], c[0].float().repeat_interleave(FL).numpy())
    assert all(torch.equal(a, b) for a, b in zip(items, before)), "the caller's codes were modified"
    (pool,) = pools
    assert not any(pool.live)
    # every push is full while items wait; an item is never split into more pieces than its length needs
    assert [len(p) for p in pool.pushes[:2]] == [N, N]
    assert sum(sum(p.values()) for p in pool.pushes) == sum(lengths)
    assert len(pool.pushes) == -(-3000 // K) + 1  # the longest item joins at the second push


def test_ragged_items_are_clamped_on_a_copy(monkeypatch):
    dac, _ = pooled_codec(monkeypatch)
    got = []
    monkeypatch.setattr(dac, "_decode_streamed", lambda items, outs: got.extend(items))
    a = np.full((10, 3), 7, dtype=np.int64)
    a[0, 0], a[0, 1], a[2, 2], a[5, 0] = 4096, -3, 1024, 1 << 40
    dac.from_indices_list([a, torch.tensor([[1]] * 10, dtype=torch.int16)])
    assert got[0].dtype == torch.int32 and got[0].tolist()[0] == [4095, 0, 7] and got[0][2, 2] == 1023
    assert got[0][5, 0] == 1023 and a[0, 0] == 4096 and got[1].tolist() == [[1]] * 10


@pytest.mark.parametrize("bad,msg", [
    (torch.zeros(9, 4, dtype=torch.int64), r"item 1: codes must be \[10, frames\], got \(9, 4\)"),
    (torch.zeros(10, 4, 1, dtype=torch.int64), r"item 1: codes must be \[10, frames\]"),
    (torch.zeros(10, dtype=torch.int64), r"item 1: codes must be \[10, frames\]"),
    (torch.zeros(10, 0, dtype=torch.int64), "item 1: no frames"),
    (torch.zeros(10, 4), "item 1: codes must be integers, got torch.float32"),
    (np.zeros((10, 4), dtype=np.float16), "item 1: codes must be integers"),
    (torch.zeros(10, 4, dtype=torch.bool), "item 1: codes must be integers"),
])
def test_ragged_decode_rejects_malformed_items(monkeypatch, bad, msg):
    dac, pools = pooled_codec(monkeypatch)
    with pytest.raises(ValueError, match=msg):
        BE.batch_vqgan_decode(dac, [torch.zeros(10, 3, dtype=torch.int64), bad, torch.zeros(10, 2, dtype=torch.int64)])
    assert pools == [], "nothing was decoded"


def test_ragged_decode_of_nothing(monkeypatch):
    dac, _ = pooled_codec(monkeypatch)
    assert BE.batch_vqgan_decode(dac, []) == []


def test_a_failed_push_leaves_the_pool_usable(monkeypatch):
    dac, pools = pooled_codec(monkeypatch)
    dac.from_indices_list([torch.zeros(10, 3, dtype=torch.int64)])
    (pool,) = pools
    real = pool.push
    pool.push = lambda pieces: (_ for _ in ()).throw(RuntimeError("device error"))
    with pytest.raises(RuntimeError, match="device error"):
        dac.from_indices_list([torch.zeros(10, 300, dtype=torch.int64)] * 6)
    assert not any(pool.live)
    pool.push = real
    (w,) = dac.from_indices_list([torch.ones(10, 2, dtype=torch.int64)])
    assert torch.equal(w, torch.ones(2 * FL))
