"""Host side of DAC.encode's routing and of EncodeStreamPool (no GPU), with a stand-in codec: the one-shot pass runs when
its workspaces fit in free device memory and the streamed path when they do not; the streamed path's pieces, tail padding,
code assembly and lengths; the one-shot workspace estimate; and the pool's validation of its arguments."""
import contextlib
import math
import threading

import pytest
import torch

from fish_speech_b200.models.dac import modded_dac as M

FL = 2048


def fake_codec(monkeypatch, free: int, need: int):
    """A DAC with no device: the probe, the estimate and both paths replaced by recorders."""
    dac = M.DAC.__new__(M.DAC)
    dac.cfg = M.CodecConfig()
    dac.frame_length, dac.hop_length, dac.encoder_rates = FL, 512, [2, 4, 8, 8]
    dac.enc_blocks = [{"tfm": None}] * 3 + [{"tfm": {"cfg": dac.cfg.enc_tfm(1024, 4)}}]
    dac.pre_tfm = {"cfg": dac.cfg.quant_tfm}
    dac._device = torch.device("cpu")
    dac._lock = threading.RLock()
    dac._bufs = {}
    calls = []
    monkeypatch.setattr(M.torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(dac, "_free_device_bytes", lambda: free)
    monkeypatch.setattr(dac, "_encode_one_shot_bytes", lambda B, N: need)
    monkeypatch.setattr(dac, "_encode_one_shot", lambda *a: calls.append("one_shot") or "one_shot")
    monkeypatch.setattr(dac, "_encode_streamed", lambda *a: calls.append("streamed") or "streamed")
    return dac, calls


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
    assert dac.encode(torch.zeros(1, 1, 5000)) == path and calls == [path]


@pytest.mark.parametrize("B,N,path", [(1, 2048 * 16383, "one_shot"), (1, 2048 * 16383 + 1, "streamed"),
                                      (64, 2048 * 255, "one_shot"), (64, 2048 * 256, "streamed")])
def test_routing_rule_transformer_rows(monkeypatch, B, N, path):
    """The one-shot pass launches at most 65 535 encoder transformer rows (B x padded N / 512, 4 per frame)."""
    dac, calls = fake_codec(monkeypatch, 80 << 30, 1 << 30)
    assert dac.encode(torch.zeros(B, 1, N)) == path and calls == [path]


def test_routing_rule_counts_the_rows_of_every_transformer(monkeypatch):
    """A transformer after an earlier encoder block runs more rows than one after the last: the rule takes the most."""
    dac, calls = fake_codec(monkeypatch, 80 << 30, 1 << 30)
    N = 2048 * 2048  # 16 384 rows after the last block, 262 144 after the second
    assert dac.encode(torch.zeros(1, 1, N)) == "one_shot"
    dac.enc_blocks = [{"tfm": None}, {"tfm": {"cfg": dac.cfg.enc_tfm(256, 1)}}] + [{"tfm": None}] * 2
    assert dac.encode(torch.zeros(1, 1, N)) == "streamed" and calls == ["one_shot", "streamed"]


def test_pool_refuses_more_rows_than_one_launch_takes():
    cfg = M.CodecConfig()
    dac = type("D", (), {})()
    dac.cfg, dac.frame_length, dac.n_stage, dac.device = cfg, FL, 10, torch.device("cpu")
    dac.enc_blocks = [{"stride": s, "tfm": None} for s in cfg.encoder_rates[:3]] + [
        {"stride": cfg.encoder_rates[3], "tfm": {"cfg": cfg.enc_tfm(1024, 4), "layers": [None] * 4}}]
    dac.pre_tfm = {"cfg": cfg.quant_tfm, "layers": [None] * 8}
    with pytest.raises(ValueError, match="exceeds the 65535 rows"):
        M.EncodeStreamPool(dac, 1024, 32, None, 8)  # 1024 x 32 x 4 encoder transformer rows


class _FakePool:
    """Codes of a piece: stage s of frame j = 1000 * s + (slot's absolute frame index); records every piece."""

    def __init__(self, slots, k_max, n_stage):
        self.slots, self.k_max, self.n_stage = slots, k_max, n_stage
        self.live, self.pos, self.pieces = [False] * slots, [0] * slots, []

    def open(self):
        s = self.live.index(False)
        self.live[s], self.pos[s] = True, 0
        return s

    def close(self, s):
        assert self.live[s]
        self.live[s] = False

    def push(self, pieces):
        out = {}
        for s, w in pieces.items():
            assert self.live[s] and w.dtype == torch.float32 and w.ndim == 1 and w.numel() % FL == 0
            k = w.numel() // FL
            assert 1 <= k <= self.k_max
            self.pieces.append((s, w.clone()))
            f = torch.arange(self.pos[s], self.pos[s] + k)
            out[s] = torch.stack([1000 * st + f for st in range(self.n_stage)])
            self.pos[s] += k
        return out


@pytest.mark.parametrize("B,n,lens,nq", [(1, FL * 300 + 17, None, None), (3, FL * 9 + 1, [FL * 9 + 1, 5, FL * 4], 2),
                                         (6, FL * 2, [FL * 2] * 6, None), (2, 100, torch.tensor([100, 1]), None)])
def test_streamed_path_pieces_padding_and_lengths(monkeypatch, B, n, lens, nq):
    dac = M.DAC.__new__(M.DAC)
    dac.frame_length, dac._device, dac.n_stage = FL, torch.device("cpu"), 10
    pools = []

    def open_pool(slots, k_max, n_quantizers):
        pools.append(_FakePool(slots, k_max, dac.n_stage if n_quantizers is None else 1 + n_quantizers))
        return pools[-1]

    monkeypatch.setattr(dac, "open_encode_pool", open_pool)
    g = torch.Generator().manual_seed(B)
    audio = torch.randn(B, 1, n, generator=g)
    lens_t = None if lens is None else torch.as_tensor(lens)
    codes, out_lens = dac._encode_streamed(audio, lens_t, nq)
    T = math.ceil(n / FL)
    S = 10 if nq is None else 1 + nq
    (pool,) = pools
    assert pool.slots == min(B, M.DAC.ENCODE_STREAM_SLOTS) and pool.k_max == M.DAC.ENCODE_STREAM_FRAMES
    assert codes.shape == (B, S, T) and codes.dtype == torch.int64
    assert torch.equal(codes, torch.stack([1000 * s + torch.arange(T) for s in range(S)]).expand(B, S, T))
    assert not any(pool.live)
    # each stream's pieces, in order, are its row of the batch zero-padded to T whole frames
    per_slot_round = {}
    for s, w in pool.pieces:
        per_slot_round.setdefault(s, []).append(w)
    padded = torch.nn.functional.pad(audio[:, 0], (0, T * FL - n))
    got_rows = []
    rows_per_round = pool.slots
    chunks = {s: torch.cat(v) for s, v in per_slot_round.items()}
    for b in range(B):
        # row b ran in slot b % slots, in round b // slots; each round streams T frames per slot
        s, rnd = b % rows_per_round, b // rows_per_round
        got_rows.append(chunks[s][rnd * T * FL: (rnd + 1) * T * FL])
    assert torch.equal(torch.stack(got_rows), padded)
    want = torch.ceil(torch.as_tensor([T * FL] if lens is None else lens) / FL).long()
    assert torch.equal(out_lens, want)


def test_one_shot_estimate_counts_only_workspaces_that_grow():
    cfg = M.CodecConfig()
    dac = M.DAC.__new__(M.DAC)
    dac.cfg, dac.hop_length, dac.encoder_rates, dac.n_stage = cfg, cfg.hop_length, list(cfg.encoder_rates), 10
    tf = lambda t: {"cfg": t}
    dac.enc_blocks = [{"tfm": tf(cfg.enc_tfm(1024, 4)) if n else None} for n in cfg.encoder_transformer_layers]
    dac.pre_tfm = tf(cfg.quant_tfm)
    dac._bufs = {}
    hour = 3600 * 44100 // FL * FL
    need = dac._encode_one_shot_bytes(1, hour)
    act = 3 * hour * cfg.encoder_dim * 2
    # 384 B per sample of encoder activations (about 61 GB for one hour), plus the encoder transformer's workspaces
    assert act <= need <= act * 1.4 and act > 60e9
    dac._bufs = {f"enc_{k}": torch.empty(1, dtype=torch.bfloat16).expand(hour * cfg.encoder_dim) for k in range(3)}
    assert dac._encode_one_shot_bytes(1, hour) == need - act


def _bare_pool(slots=2, k_max=4):
    """EncodeStreamPool's host-side checks run before any device work: a pool without device state."""
    pool = M.EncodeStreamPool.__new__(M.EncodeStreamPool)
    pool.dac = type("D", (), {"frame_length": FL, "_lock": threading.RLock()})()
    pool.slots, pool.k_max = slots, k_max
    pool.live, pool.broken, pool.pos = [True] * slots, [False] * slots, [0] * slots
    return pool


def test_pool_validation():
    pool = _bare_pool()
    w = torch.zeros(5 * FL)
    bad = [
        ({0: w}, "push takes 1 .. 4"),
        ({0: w[: FL + 1]}, "whole number"),
        ({0: w[:0]}, "push takes 1 .. 4"),
        ({0: w[:FL].double()}, "float32"),
        ({0: w[:FL].view(1, -1)}, "1-D"),
        ({0: [0.0] * FL}, "1-D"),
        ({2: w[:FL]}, "not an open stream"),
        ({"0": w[:FL]}, "not an open stream"),
    ]
    for pieces, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pool.push(pieces)
    pool.close(1)
    with pytest.raises(ValueError, match="not an open stream"):
        pool.push({1: w[:FL]})
    with pytest.raises(ValueError, match="not an open stream"):
        pool.close(1)
    pool.broken[0] = True
    with pytest.raises(ValueError, match="close the slot"):
        pool.push({0: w[:FL]})
    assert pool.push({}) == {}
