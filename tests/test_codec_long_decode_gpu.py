"""DAC.from_indices of any length: the streamed route (a DecodeStreamPool of DECODE_STREAM_SLOTS rows in pieces of
DECODE_STREAM_FRAMES frames) is byte-identical to the one-shot pass wherever both run, is taken by itself past the one-shot
pass's post-transformer rows, and holds memory that grows with length only by its output; codes are clamped in the
caller's tensor on both routes; and the ragged batch decode (`from_indices_list`, `bulk_encode.batch_vqgan_decode`)
gives every item the samples of `from_indices` of that item alone."""
import numpy as np
import pytest
import torch

from fish_speech_b200 import bulk_encode as BE
from fish_speech_b200.models.dac.modded_dac import DAC
from oracle import codec_oracle as CO
from tests.test_codec_gpu import build, rand_codes

pytestmark = pytest.mark.gpu
K = DAC.DECODE_STREAM_FRAMES


@pytest.fixture(scope="module")
def tiny():
    cfg = CO.tiny_config()  # post-transformer window 16
    return cfg, build(cfg, CO.make_weights(cfg, seed=5))


@pytest.fixture(scope="module")
def full():
    cfg = CO.full_config()  # post-transformer window 128
    return cfg, build(cfg, CO.make_weights(cfg, seed=6))


def spy_streamed(monkeypatch, dac):
    calls = []
    real = dac._from_indices_streamed
    monkeypatch.setattr(dac, "_from_indices_streamed", lambda idx: calls.append(tuple(idx.shape)) or real(idx))
    return calls


def forced_stream(monkeypatch, dac, codes):
    """from_indices with a free-memory probe that reports 0: the streamed route."""
    calls = spy_streamed(monkeypatch, dac)
    monkeypatch.setattr(dac, "_free_device_bytes", lambda: 0)
    try:
        return dac.from_indices(codes)
    finally:
        monkeypatch.undo()
        assert calls == [tuple(codes.shape)], "the streamed route did not run"


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("T", [1, K - 1, K, K + 1, 3 * K + 17])
def test_streamed_route_equals_one_shot_tiny(tiny, monkeypatch, B, T):
    cfg, dac = tiny
    codes = rand_codes(cfg, B, T, 1000 * B + T).cuda()
    ref = dac.from_indices(codes.clone())
    got = forced_stream(monkeypatch, dac, codes.clone())
    assert got.shape == ref.shape == (B, 1, T * dac.frame_length) and got.dtype == torch.float32
    assert torch.equal(got, ref)


@pytest.mark.parametrize("B,T", [(1, 1), (3, K - 1), (1, K + 1), (3, 300), (1, 2 * K)])
def test_streamed_route_equals_one_shot_full(full, monkeypatch, B, T):
    """The S2-Pro geometry, across the post-transformer's 128-frame window."""
    cfg, dac = full
    codes = rand_codes(cfg, B, T, 2000 * B + T).cuda()
    ref = dac.from_indices(codes.clone())
    got = forced_stream(monkeypatch, dac, codes.clone())
    assert torch.equal(got, ref)


@pytest.mark.parametrize("stream", [False, True])
def test_codes_are_clamped_in_the_callers_tensor(tiny, monkeypatch, stream):
    cfg, dac = tiny
    T = 41 if stream else 40  # a shape with a captured graph replays it whatever the memory probe says
    codes = rand_codes(cfg, 2, T, 77).cuda()
    codes[0, 0, 3] = cfg.semantic_codebook_size + 50
    codes[1, 2, T - 1] = cfg.codebook_size + 7
    clamped = codes.clone()
    clamped[:, 0].clamp_(max=cfg.semantic_codebook_size - 1)
    clamped[:, 1:].clamp_(max=cfg.codebook_size - 1)
    ref = dac.from_indices(clamped.clone())
    got = forced_stream(monkeypatch, dac, codes) if stream else dac.from_indices(codes)
    assert torch.equal(codes, clamped) and torch.equal(got, ref)


def test_past_the_one_shot_rows_the_route_is_taken_by_itself(tiny, monkeypatch):
    """B x T above ONE_SHOT_MAX_ROWS: decoded through the pool with no probe patched. Causality gives the reference (the
    first n frames' samples are those of the one-shot decode of the first n frames), and peak memory above the resident
    state grows with T only by the output's 8 KB per frame (and the 80 B per frame of the in-place clamp's temporaries)."""
    cfg, dac = tiny
    FL = dac.frame_length
    T1 = DAC.ONE_SHOT_MAX_ROWS + 465  # 66 000 frames
    T2 = T1 + 40 * K  # the same last piece
    codes = rand_codes(cfg, 1, T2, 5).cuda()
    calls = spy_streamed(monkeypatch, dac)

    def decode(T):
        c = codes[..., :T].clone()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        wav = dac.from_indices(c)
        torch.cuda.synchronize()
        return wav, torch.cuda.max_memory_allocated() - base

    decode(T1)  # the pool, its workspaces and graphs
    wav1, peak1 = decode(T1)
    wav2, peak2 = decode(T2)
    assert calls == [(1, cfg.n_codebooks + 1, T1)] * 2 + [(1, cfg.n_codebooks + 1, T2)]
    print(f"peak above resident: {peak1} B at {T1} frames, {peak2} B at {T2} frames")
    assert 0 <= peak2 - peak1 <= (T2 - T1) * (FL * 4 + 80) + (256 << 10)
    assert torch.equal(wav1, wav2[..., : T1 * FL])
    n = 3000
    assert torch.equal(wav2[..., : n * FL], dac.from_indices(codes[..., :n].clone()))
    assert torch.isfinite(wav2).all()


LENGTHS = [1, 37, 128, 500, 3000, 129, 7, 64, 250]  # more items than the pool has slots


@pytest.mark.parametrize("geometry,lengths", [("tiny", LENGTHS), ("full", [1, 37, 128, 500, 129, 300])])
def test_batch_vqgan_decode_items_equal_from_indices_alone(request, geometry, lengths):
    cfg, dac = request.getfixturevalue(geometry)
    assert len(lengths) > DAC.DECODE_STREAM_SLOTS
    items = [rand_codes(cfg, 1, T, 3000 + i)[0] for i, T in enumerate(lengths)]
    items[2] = items[2].numpy().astype(np.int32)  # any integer array
    before = [torch.as_tensor(c).clone() for c in items]
    outs = BE.batch_vqgan_decode(dac, items)
    assert len(outs) == len(lengths)
    for i, (o, c, T) in enumerate(zip(outs, items, lengths)):
        assert isinstance(o, np.ndarray) and o.dtype == np.float32 and o.shape == (1, T * dac.frame_length)
        alone = dac.from_indices(torch.as_tensor(c)[None].long().cuda())[0].cpu().numpy()
        assert o.tobytes() == alone.tobytes(), f"item {i} ({T} frames) differs from its from_indices"
    assert all(torch.equal(torch.as_tensor(c), b) for c, b in zip(items, before))
    assert dac._dec_pool.n_open() == 0


def test_batch_vqgan_decode_refuses_malformed_items(tiny):
    cfg, dac = tiny
    good = rand_codes(cfg, 1, 5, 1)[0]
    for bad, msg in [(good[:-1], r"item 1: codes must be \[4, frames\]"), (good[:, :0], "item 1: no frames"),
                     (good.float(), "item 1: codes must be integers")]:
        with pytest.raises(ValueError, match=msg):
            BE.batch_vqgan_decode(dac, [good, bad])
    (w,) = BE.batch_vqgan_decode(dac, [good])
    assert w.tobytes() == dac.from_indices(good[None].clone().cuda())[0].cpu().numpy().tobytes()
