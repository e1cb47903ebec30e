"""The 64-row decode step: engines of 33..64 slots (csrc/lm_gemm.cu step_gemm_kernel<NORM, 64>, the RT = 64 finalize,
attention and sampler consumers, the RT-sized decode state of csrc/lm_engine.cu).

A request's tokens must not depend on its slot, its neighbours or the engine it runs in. The 64-row kernel issues, per
32-row half of its operand tile, the wgmma the 32-row kernel issues, so every output element must be bit-identical to
the 32-row result on the same rows; these tests check that bitwise, from one GEMM up to whole S2-Pro frames, and check
the 64-row GEMM against float64 with the bound of tests/test_step_gemm_gpu.py.
"""
from __future__ import annotations

import ctypes
import math

import pytest
import torch

from oracle import lm_oracle as O
from tests.kernel_ref import acc_bound, fp64_gemm, norm_operand, tile_ssq
from tests.lm_util import (SHAPES, STAGES, _bits, _ctas, _gen, _lib, _randn, _sms, build_model, layer_configs,
                           make_prompt)

pytestmark = pytest.mark.gpu

ROWS64 = (1, 33, 47, 64)


def step_gemm_tile(w, x, row_tile, rows, num_ctas, stages, norm_w=None, ssq=None, eps=1e-6):
    """fsb_op_step_gemm_tile: w bf16 [n_out, K], x bf16 [row_tile, K] -> (fp32 [rows, n_out], plan info)."""
    L = _lib()
    n_out, K = w.shape
    assert x.shape == (row_tile, K) and x.is_contiguous() and w.is_contiguous()
    out = torch.full((max(rows, 1), n_out), float("nan"), device="cuda")
    info = (ctypes.c_int * 5)()
    L.check(L.lib().fsb_op_step_gemm_tile(
        w.data_ptr(), n_out, K, x.data_ptr(), row_tile, rows, norm_w.data_ptr() if norm_w is not None else None,
        ssq.data_ptr() if ssq is not None else None, eps, num_ctas, stages, out.data_ptr(), info,
        torch.cuda.current_stream().cuda_stream))
    return out[:rows], dict(ctas=info[0], stages=info[1], parts=info[2], units=info[3], items=info[4])


# ---------------------------------------------------------------------------------------------------------------------
# one GEMM at RT = 64 against float64, over the shapes and schedules of test_step_gemm_matches_fp64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_out,K", SHAPES)
def test_step_gemm64_matches_fp64(n_out, K):
    w = _randn((n_out, K), seed=n_out * 7 + K)
    x = _randn((64, K), seed=n_out * 7 + K + 3)
    ref, absprod = fp64_gemm(x, w)
    tiles, kblocks = math.ceil(n_out / 128), math.ceil(K / 64)
    infos = []
    for ci, ctas in enumerate(_ctas()):
        for si, stages in enumerate(STAGES):
            rows = ROWS64[(ci + si) % len(ROWS64)]
            out, info = step_gemm_tile(w, x, 64, rows, ctas, stages)
            infos.append((ctas, stages, info))
            bound = acc_bound(absprod[:rows], K, info["parts"])
            err = (out.double() - ref[:rows]).abs()
            bad = ~(err <= bound)
            assert not bad.any(), (
                f"ctas={ctas} stages={stages} rows={rows} {info}: {int(bad.sum())} elements off, first at "
                f"{bad.nonzero()[0].tolist()}, max err/bound {float((err / bound).nan_to_num(float('inf')).max()):.3g}")
    for ctas, stages, info in infos:
        assert 1 <= info["ctas"] <= min(ctas, tiles * kblocks)
        assert 2 <= info["stages"] <= stages
    assert any(i["units"] > i["stages"] for _, _, i in infos), "no CTA wrapped its ring"
    if kblocks >= 3:
        assert any(i["parts"] >= 3 for _, _, i in infos), "no tile was split into 3 or more partial slots"


def test_step_gemm64_keeps_two_ctas_per_sm_at_the_engine_schedule():
    """Same stream-K split as the 32-row kernel: the engine's request (2 CTAs per SM, 4 stages) is granted as it is,
    with normalise-on-load at K = 4096 too."""
    for n_out, K, norm in ((19456, 2560, True), (2560, 9728, False), (6144, 4096, True)):
        w = _randn((n_out, K), seed=K + 1, scale=0.02)
        nw = torch.ones(K, device="cuda").bfloat16() if norm else None
        infos = []
        for rt in (32, 64):
            x = _randn((rt, K), seed=K)
            ssq = torch.zeros(rt, 32, device="cuda") if norm else None
            if norm:
                ssq[:, : math.ceil(K / 128)] = tile_ssq(x).float()
            infos.append(step_gemm_tile(w, x, rt, rt, 2 * _sms(), 4, nw, ssq)[1])
        assert infos[0] == infos[1], infos
        assert infos[1]["ctas"] == 2 * _sms() and infos[1]["stages"] == 4, infos[1]


# ---------------------------------------------------------------------------------------------------------------------
# bits: the 64-row tile against the 32-row tile, and rows against their neighbours
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_out,K,norm", [(2560, 9728, False), (19456, 2560, True), (6144, 2560, True),
                                          (97, 256, True), (200, 528, False)])
def test_step_gemm64_halves_equal_the_32_row_tile_bitwise(n_out, K, norm):
    eps = 1e-6
    sched = (2 * _sms(), 4)
    w = _randn((n_out, K), seed=K + 5, scale=0.02)
    scale = torch.tensor([2.0 ** (j % 7 - 3) for j in range(64)], device="cuda")[:, None]
    x = (_randn((64, K), seed=K + 6) * scale).bfloat16()
    nw = (1 + 0.1 * torch.randn(K, generator=_gen(K + 7), device="cuda")).bfloat16() if norm else None
    nt = math.ceil(K / 128)
    ssq = torch.full((64, 32), float("nan"), device="cuda")
    if norm:
        ssq[:, :nt] = tile_ssq(x).float()
    s = ssq if norm else None
    full, _ = step_gemm_tile(w, x, 64, 64, *sched, nw, s, eps)
    assert torch.isfinite(full).all()
    for h in (0, 1):
        half, _ = step_gemm_tile(w, x[32 * h: 32 * h + 32].contiguous(), 32, 32, *sched, nw,
                                 s[32 * h: 32 * h + 32].contiguous() if norm else None, eps)
        assert torch.equal(_bits(full[32 * h: 32 * h + 32]), _bits(half)), f"rows {32 * h}..{32 * h + 31} differ"
    # a row keeps its bits whatever the other 63 rows hold and whatever `rows` is
    for j in (0, 31, 32, 47, 63):
        for junk in (float("nan"), 1e30, -1e30):
            xj = torch.full((64, K), junk, device="cuda").bfloat16()
            xj[j] = x[j]
            sj = torch.full((64, 32), float("nan") if junk != junk else 1e38, device="cuda")
            sj[j] = ssq[j]
            for rows in sorted({j + 1, 33 if j < 33 else 64, 64}):
                out, _ = step_gemm_tile(w, xj, 64, rows, *sched, nw, sj if norm else None, eps)
                assert torch.equal(_bits(out[j]), _bits(full[j])), f"row {j} changed with rows={rows}, others = {junk}"


def test_step_gemm64_normalise_on_load_identity():
    """Identity weights expose X' element by element: every one of the 64 rows is normalised with its own sums of
    squares (inside the rsqrtf bracket), bit-identically to the 32-row tile on each half."""
    K, eps = 2560, 1e-6
    nt = math.ceil(K / 128)
    scale = torch.tensor([2.0 ** (j % 9 - 4) for j in range(64)], device="cuda")[:, None]
    x = (_randn((64, K), seed=K + 11) * scale).bfloat16()
    nw = (1 + 0.1 * torch.randn(K, generator=_gen(K + 12), device="cuda")).bfloat16()
    ssq = torch.full((64, 32), float("nan"), device="cuda")
    ssq[:, :nt] = tile_ssq(x).float()
    eye = torch.eye(K, device="cuda").bfloat16()
    for ctas, stages in ((7, 3), (2 * _sms(), 4)):
        out, info = step_gemm_tile(eye, x, 64, 64, ctas, stages, nw, ssq, eps)
        _, lo, hi = norm_operand(x, ssq, nw, eps, K)
        inside = (out >= lo) & (out <= hi)
        assert inside.all(), f"ctas={ctas} {info}: X' off at {(~inside).nonzero()[0].tolist()}"
        for h in (0, 1):
            half, _ = step_gemm_tile(eye, x[32 * h: 32 * h + 32].contiguous(), 32, 32, ctas, stages, nw,
                                     ssq[32 * h: 32 * h + 32].contiguous(), eps)
            assert torch.equal(_bits(out[32 * h: 32 * h + 32]), _bits(half)), f"ctas={ctas}: half {h} differs"


# ---------------------------------------------------------------------------------------------------------------------
# one decode layer: a 64-slot engine against a 32-slot engine on the two halves
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def layer_models():
    built = {}

    def get(name):
        if name not in built:
            for m in built.values():
                for e in m[1:]:
                    e.engine.close()
            built.clear()
            cfg = layer_configs()[name]
            w = O.make_weights(cfg, seed=97)
            built[name] = (cfg, build_model(cfg, w, max_batch=64, debug=False, max_rows=128),
                           build_model(cfg, w, max_batch=32, debug=False, max_rows=128))
        return built[name]

    yield get
    for m in built.values():
        for e in m[1:]:
            e.engine.close()


@pytest.mark.parametrize("name", ["tiny", "s2pro"])
@pytest.mark.parametrize("fast", [0, 1])
def test_decode_layer64_equals_two_32_row_halves(layer_models, name, fast):
    L = _lib()
    cfg, m64, m32 = layer_models(name)
    assert m64.engine.row_tile == 64 and m32.engine.row_tile == 32
    D = cfg.fast_dim if fast else cfg.dim
    I = cfg.fast_intermediate_size if fast else cfg.intermediate_size
    HD = (cfg.fast_n_head * cfg.fast_head_dim) if fast else (cfg.n_head * cfg.head_dim)
    nt = math.ceil(D / 128)
    nl = cfg.n_fast_layer if fast else cfg.n_layer
    stream = torch.cuda.current_stream().cuda_stream

    def run(model, x, attn, rows, upto, layer):
        eng = model.engine
        rt = eng.row_tile
        xb, sb = eng.buffer("x_fast" if fast else "x_slow"), eng.buffer("ssq_fast" if fast else "ssq_slow")
        ab, hb = eng.buffer("attn")[: rt * HD].view(rt, HD), eng.buffer("ffn_h")
        xb.zero_()
        xb[: x.shape[0]].copy_(x)
        sb.fill_(float("nan"))
        ab.fill_(float("nan"))
        ab[: attn.shape[0]].copy_(attn)
        hb.zero_()
        torch.cuda.synchronize()
        L.check(L.lib().fsb_lm_test_layer_gemms(eng.h, fast, layer, rows, upto, stream))
        torch.cuda.synchronize()
        return xb[:rows].clone(), sb[:rows, :nt].clone(), hb[: rows * I].clone()

    for layer in sorted({0, nl - 1}):
        for rows in (33, 47, 64):
            x = _randn((rows, D), seed=rows + 7 * layer + 100 * fast)
            attn = _randn((rows, HD), seed=rows + 7 * layer + 100 * fast + 1)
            for upto in (1, 2, 3):
                what = f"{name} {'fast' if fast else 'slow'} layer {layer} rows={rows} upto={upto}"
                x64, s64, h64 = run(m64, x, attn, rows, upto, layer)
                parts = [run(m32, x[:32], attn[:32], 32, upto, layer),
                         run(m32, x[32:], attn[32:], rows - 32, upto, layer)]
                x32 = torch.cat([p[0] for p in parts])
                s32 = torch.cat([p[1] for p in parts])
                h32 = torch.cat([p[2] for p in parts])
                assert torch.equal(x64.view(torch.int16), x32.view(torch.int16)), f"{what}: x differs"
                assert torch.equal(_bits(s64), _bits(s32)), f"{what}: sums of squares differ"
                if upto >= 2:
                    assert torch.equal(h64.view(torch.int16), h32.view(torch.int16)), f"{what}: ffn_h differs"


# ---------------------------------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------------------------------
def _gen_alone(model, prompt, n, **kw):
    from fish_speech_b200.models.text2semantic.inference import generate

    return generate(model=model, prompt=prompt.cuda(), max_new_tokens=n, **kw).cpu()


def test_generate_batch_of_64_equals_each_solo_run():
    from fish_speech_b200.models.text2semantic.inference import generate_batch

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=33, head_gain=8.0)
    prompts = [make_prompt(cfg, 400 + i, 5 + (7 * i) % 29) for i in range(64)]
    n = 8
    model = build_model(cfg, w, max_batch=64, debug=False)
    assert model.engine.row_tile == 64
    outs = generate_batch(model=model, prompts=[p.cuda() for p in prompts], max_new_tokens=n, temperature=0.7,
                          top_p=0.7, top_k=1)
    solo = build_model(cfg, w, max_batch=1, debug=False)
    for i, p in enumerate(prompts):
        one = _gen_alone(solo, p, n, temperature=0.7, top_p=0.7, top_k=1)
        assert torch.equal(outs[i].cpu().to(torch.int32), one.to(torch.int32)), f"seq {i}: batch of 64 != solo"


def test_64_sampled_requests_with_their_own_seeds_equal_each_solo_run():
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=34, head_gain=2.5)
    specs = [dict(prompt=make_prompt(cfg, 500 + i, 4 + (5 * i) % 23), max_new_tokens=6 + i % 5, temperature=0.8,
                  top_p=0.9, top_k=30, seed=7000 + 13 * i) for i in range(64)]
    model = build_model(cfg, w, max_batch=64, debug=False)
    b = ContinuousBatcher(model, max_slots=64, frames_per_poll=4)
    reqs = [b.submit(SlotRequest(**{**s, "prompt": s["prompt"].cuda()})) for s in specs]
    b.run()
    b.close()
    assert sorted(r.slot for r in reqs) == list(range(64))
    solo = build_model(cfg, w, max_batch=1, debug=False)
    for i, (s, r) in enumerate(zip(specs, reqs)):
        one = _gen_alone(solo, s["prompt"], s["max_new_tokens"], temperature=s["temperature"], top_p=s["top_p"],
                         top_k=s["top_k"], seed=s["seed"])
        assert torch.equal(r.result.cpu(), one), f"request {i} (slot {r.slot}) != its solo run"


def test_sampled_probe_in_slot_63_equals_the_probe_alone():
    """test_slot_position_in_the_batch_does_not_change_a_sampled_request at 64 slots."""
    from fish_speech_b200.scheduler import ContinuousBatcher, SlotRequest

    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=71, head_gain=2.5)
    model = build_model(cfg, w, max_batch=64, debug=False)
    probe = dict(prompt=make_prompt(cfg, 7, 11).cuda(), max_new_tokens=12, temperature=0.8, top_p=0.9, top_k=30, seed=99)
    b = ContinuousBatcher(model, max_slots=64, frames_per_poll=6)
    r_alone = b.submit(SlotRequest(**probe))
    b.run()
    others = [b.submit(SlotRequest(prompt=make_prompt(cfg, 200 + i, 6 + i % 9).cuda(), max_new_tokens=13 + i % 13,
                                   temperature=0.8, top_p=0.9, top_k=30, seed=i)) for i in range(63)]
    r_last = b.submit(SlotRequest(**probe))
    b.run()
    b.close()
    assert r_last.slot == 63 and r_alone.slot == 0
    assert all(o.done.is_set() for o in others)
    assert torch.equal(r_alone.result, r_last.result)
    # the 32-slot engine gives the probe the same tokens too
    m32 = build_model(cfg, w, max_batch=32, debug=False)
    b32 = ContinuousBatcher(m32, max_slots=32, frames_per_poll=6)
    r32 = b32.submit(SlotRequest(**probe))
    b32.run()
    b32.close()
    assert torch.equal(r32.result, r_alone.result)


def test_s2pro_frames_of_64_equal_a_32_slot_engine_on_the_two_halves():
    """Full S2-Pro geometry (36 slow + 4 fast layers, real vocabulary, synthetic weights): 64 greedy sequences for a few
    frames equal a 32-slot engine run on rows 0..31 and 32..63, tokens and debug logits bitwise."""
    from fish_speech_b200 import synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID, s2pro_args
    from fish_speech_b200.models.text2semantic.inference import generate_batch
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    dev = torch.device("cuda", 0)
    cfg = s2pro_args(max_seq_len=64)
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    g = torch.Generator().manual_seed(5)
    prompts = []
    for i in range(64):
        p = torch.zeros(cfg.num_codebooks + 1, 8 + i % 13, dtype=torch.int32)
        p[0] = torch.randint(0, 151643, (p.shape[1],), generator=g, dtype=torch.int32)
        prompts.append(p.to(dev))
    n = 4
    results = {}
    for slots in (64, 32):
        model = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
        model.debug = True
        model.max_rows = 64 * 24
        model.setup_caches(max_batch_size=slots, max_seq_len=cfg.max_seq_len)
        eng = model.engine
        assert eng.row_tile == slots
        toks, slow, fast = [], [], []
        for lo in range(0, 64, slots):
            out = generate_batch(model=model, prompts=prompts[lo: lo + slots], max_new_tokens=n, temperature=0.7,
                                 top_p=0.7, top_k=1, seed=1)
            torch.cuda.synchronize()
            toks += [o.cpu() for o in out]
            slow.append(eng.buffer("slow_logits")[:slots].cpu())
            fast.append(eng.buffer("fast_logits")[:, :slots].cpu())
        results[slots] = (toks, torch.cat(slow), torch.cat(fast, dim=1))
        eng.close()
        del model
    del w
    t64, s64, f64 = results[64]
    t32, s32, f32 = results[32]
    for i in range(64):
        assert torch.equal(t64[i], t32[i]), f"sequence {i}: tokens differ"
    assert torch.equal(_bits(s64), _bits(s32)), "slow logits differ"
    assert torch.equal(_bits(f64), _bits(f32)), "fast logits differ"


# ---------------------------------------------------------------------------------------------------------------------
# limits
# ---------------------------------------------------------------------------------------------------------------------
def test_limits_of_the_64_row_path():
    from fish_speech_b200.scheduler import ContinuousBatcher

    L = _lib()
    cfg = O.tiny_config()
    w = O.make_weights(cfg, seed=3)
    with pytest.raises(L.FsbError, match="max_batch"):
        build_model(cfg, w, max_batch=65, debug=False)
    model = build_model(cfg, w, max_batch=33, debug=False)
    assert model.engine.row_tile == 64 and tuple(model.engine.buffer("pos").shape) == (64,)
    with pytest.raises(ValueError, match="max_slots"):
        ContinuousBatcher(model, max_slots=65)
    wt, x = _randn((128, 64), seed=1), _randn((64, 64), seed=2)
    with pytest.raises(L.FsbError, match="rows"):
        step_gemm_tile(wt, x, 64, 65, 4, 4)
    with pytest.raises(L.FsbError, match="rows"):
        step_gemm_tile(wt, x, 64, 0, 4, 4)
    for rt in (16, 48, 128):
        xx = _randn((rt, 64), seed=rt)
        with pytest.raises(L.FsbError, match="row_tile"):
            step_gemm_tile(wt, xx, rt, 1, 4, 4)
    with pytest.raises(L.FsbError, match="rows"):  # the 32-row hook keeps its contract
        step_gemm_tile(wt, _randn((32, 64), seed=3), 32, 33, 4, 4)
