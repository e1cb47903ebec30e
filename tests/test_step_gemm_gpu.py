"""The decode step GEMM (csrc/lm_gemm.cu: step_gemm_kernel, the stream-K schedule of step_plan_init, the slot-ordered
partial sums of step_partial_sum(s)) and its finalize kernels (residual add, SwiGLU), against float64 references built
from the same bf16 operands.

Two hooks drive the kernels directly: fsb_op_step_gemm runs one GEMM with any schedule request, and
fsb_lm_test_layer_gemms runs one decode layer's wo -> residual -> w1|w3 -> SwiGLU -> w2 -> residual chain with the
engine's own plans. The whole-model tests only compare sampled tokens; these compare every element.

Accumulation bound. The step GEMM adds bf16 products in fp32: one wgmma step per 16-deep slice of a 64-wide k-block
(the products are exact, the running sum is rounded once per step), then the consumer adds the P partial slots of a
tile in fp32. Each of these n <= K/16 + P roundings is off by at most one fp32 ulp (2^-23 relative, whether the
hardware truncates or rounds to nearest) of a value no larger than sum_k |W_ik X_jk|, so
    |out_ij - ref_ij| <= (K/16 + P + 1) * 2^-23 * (|W| |X|^T)_ij                                      (ACC)
holds for every schedule. The finalize checks need most of the kernel's bf16 roundings to be decided, which a
worst-case bound that grows with K cannot do. There the result of a GEMM may round either way only where its float64
value lies within C_AMB * (|W| |X|^T)_ij of a bf16 rounding boundary; everywhere else the kernel's bf16 output must be
bit-identical to the reference's, and fewer than 1 % of the elements may differ at all. C_AMB = 2^-19 is 7x the
largest error measured at the engine's schedules (2 CTAs per SM, 4 stages): 2^-21.9 * (|W| |X|^T)_ij, for w1|w3 at 24
units per CTA, on an H100 SXM (132 SMs). test_step_gemm_error_at_engine_schedules keeps that margin at least 4x.
"""
from __future__ import annotations

import ctypes
import math

import pytest
import torch

from tests.kernel_ref import (C_AMB, acc_bound, bracket_bf16, check_bracket, check_ssq, fp64_gemm, norm_operand,
                              normed_gemm, rbf, swiglu_from, tile_ssq)
from tests.lm_util import SHAPES, STAGES, _ctas, _gen, _lib, _randn, _sms, build_model, layer_configs

pytestmark = pytest.mark.gpu

ROWS = (1, 5, 31, 32)


def step_gemm(w, x, rows, num_ctas, stages, norm_w=None, ssq=None, eps=1e-6):
    """fsb_op_step_gemm: w bf16 [n_out, K], x bf16 [32, K] (cuda) -> (fp32 [rows, n_out], plan info)."""
    L = _lib()
    n_out, K = w.shape
    assert x.shape == (32, K) and x.is_contiguous() and w.is_contiguous()
    out = torch.full((max(rows, 1), n_out), float("nan"), device="cuda")  # a valid pointer even for rows = 0
    info = (ctypes.c_int * 5)()
    L.check(L.lib().fsb_op_step_gemm(
        w.data_ptr(), n_out, K, x.data_ptr(), rows, norm_w.data_ptr() if norm_w is not None else None,
        ssq.data_ptr() if ssq is not None else None, eps, num_ctas, stages, out.data_ptr(), info,
        torch.cuda.current_stream().cuda_stream))
    return out[:rows], dict(ctas=info[0], stages=info[1], parts=info[2], units=info[3], items=info[4])


# ---------------------------------------------------------------------------------------------------------------------
# 3a: one GEMM against float64 over the engine's shapes and the whole range of schedules
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_out,K", SHAPES)
def test_step_gemm_matches_fp64(n_out, K):
    w = _randn((n_out, K), seed=n_out * 7 + K)
    x = _randn((32, K), seed=n_out * 7 + K + 1)
    ref, absprod = fp64_gemm(x, w)
    tiles, kblocks = math.ceil(n_out / 128), math.ceil(K / 64)
    infos = []
    full = None
    for ci, ctas in enumerate(_ctas()):
        for si, stages in enumerate(STAGES):
            rows = ROWS[(ci + si) % len(ROWS)]
            out, info = step_gemm(w, x, rows, ctas, stages)
            infos.append((ctas, stages, info))
            bound = acc_bound(absprod[:rows], K, info["parts"])
            err = (out.double() - ref[:rows]).abs()
            bad = ~(err <= bound)  # NaN (unwritten slot, or the two partial-sum helpers disagree) fails too
            assert not bad.any(), (
                f"ctas={ctas} stages={stages} rows={rows} {info}: {int(bad.sum())} elements off, first at "
                f"{bad.nonzero()[0].tolist()}, max err/bound {float((err / bound).nan_to_num(float('inf')).max()):.3g}")
            if rows == 32 and full is None:
                full = (out.double(), info)
    # the bound has teeth: one 64-wide k-block dropped from (or counted twice in) the reference is out of it
    out, info = full
    bound = acc_bound(absprod, K, info["parts"])
    blk = x[:, :64].double() @ w[:, :64].double().T
    for sign, what in ((-1, "dropped"), (1, "doubled")):
        assert ((out - (ref + sign * blk)).abs() > bound).any(), f"a {what} k-block stays inside the bound"
    # the sweep reached what it is for
    for ctas, stages, info in infos:
        assert 1 <= info["ctas"] <= min(ctas, tiles * kblocks)
        assert 2 <= info["stages"] <= stages
        assert info["units"] >= math.ceil(tiles * kblocks / info["ctas"])
    assert any(i["units"] > i["stages"] for _, _, i in infos), "no CTA wrapped its ring"
    assert any(i["stages"] < s for _, s, i in infos), "no stages request was shrunk"
    assert any(i["ctas"] < c for c, _, i in infos), "no CTA request was clamped"
    if tiles >= 2:
        assert any(i["items"] >= 2 for _, _, i in infos), "no CTA range crossed a tile boundary"
    if kblocks >= 3:
        assert any(i["parts"] >= 3 for _, _, i in infos), "no tile was split into 3 or more partial slots"


def test_step_gemm_error_at_engine_schedules():
    """C_AMB (module docstring) stays at least 4x the error at the schedules the engine runs: 2 CTAs per SM, 4 stages."""
    for n_out, K in ((6144, 2560), (2560, 4096), (19456, 2560), (2560, 9728), (384, 256)):
        w = _randn((n_out, K), seed=K, scale=0.02)
        x = _randn((32, K), seed=K + 1)
        ref, absprod = fp64_gemm(x, w)
        out, info = step_gemm(w, x, 32, 2 * _sms(), 4)
        ratio = float(((out.double() - ref).abs() / absprod).max())
        assert ratio <= C_AMB / 4, f"{n_out}x{K} {info}: max error 2^{math.log2(ratio):.2f} * sum|w x|"


def test_step_gemm_rejects_bad_arguments():
    L = _lib()
    w, x = _randn((128, 64), seed=1), _randn((32, 64), seed=2)
    for rows in (0, 33):
        with pytest.raises(L.FsbError, match="rows"):
            step_gemm(w, x, rows, 4, 4)
    with pytest.raises(L.FsbError):
        step_gemm(w, x, 1, 0, 4)
    with pytest.raises(L.FsbError):
        step_gemm(_randn((128, 68), seed=3), _randn((32, 68), seed=4), 1, 4, 4)  # K % 8 != 0


# ---------------------------------------------------------------------------------------------------------------------
# 3b: normalise-on-load
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [2560, 1000])  # 20 tiles; 8 tiles, the last one partial, and a partial last k-block
def test_step_gemm_normalise_on_load(K):
    eps = 1e-6
    nt = math.ceil(K / 128)
    # rows of different scales, so that every row has its own rsqrt
    scale = torch.tensor([2.0 ** (j % 7 - 3) for j in range(32)], device="cuda")[:, None]
    x = (_randn((32, K), seed=K) * scale).bfloat16()
    norm_w = (1 + 0.1 * torch.randn(K, generator=_gen(K + 1), device="cuda")).bfloat16()
    ssq_live = tile_ssq(x).float()
    schedules = [(1, 2), (7, 3), (2 * _sms(), 4), (10 ** 6, 8)]
    # identity weights: out = X' itself, so every element of the normalised operand is checked, not only their sums
    eye = torch.eye(K, device="cuda").bfloat16()
    w = _randn((640, K), seed=K + 2)
    for i, (ctas, stages) in enumerate(schedules):
        rows = ROWS[i]
        # sums of squares only in the live rows and the tiles of K: NaN anywhere else must not reach the result
        ssq = torch.full((32, 32), float("nan"), device="cuda")
        ssq[:rows, :nt] = ssq_live[:rows]
        mid, lo, hi = norm_operand(x[:rows], ssq[:rows], norm_w, eps, K)
        amb = lo != hi
        assert amb.double().mean() < 0.01

        out, info = step_gemm(eye, x, rows, ctas, stages, norm_w, ssq, eps)
        inside = (out >= lo) & (out <= hi)
        assert inside.all(), (f"ctas={ctas} stages={stages} rows={rows} {info}: X' off at "
                              f"{(~inside).nonzero()[0].tolist()} ({int((~inside).sum())} elements)")

        out, info = step_gemm(w, x, rows, ctas, stages, norm_w, ssq, eps)
        ref, absprod = fp64_gemm(mid, w)
        slack = (hi - lo).double() @ w.double().abs().T  # zero wherever the rounding of X' is unambiguous
        bound = acc_bound(fp64_gemm(torch.maximum(lo.abs(), hi.abs()), w)[1], K, info["parts"]) + slack
        bad = ~((out.double() - ref).abs() <= bound)
        assert not bad.any(), f"ctas={ctas} stages={stages} rows={rows} {info}: {int(bad.sum())} elements off"


# ---------------------------------------------------------------------------------------------------------------------
# 3c: bits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_out,K,norm", [(2560, 9728, False), (19456, 2560, True), (97, 256, True)])
def test_step_gemm_bits_reproducible_and_row_independent(n_out, K, norm):
    eps = 1e-6
    w = _randn((n_out, K), seed=K + 5, scale=0.02)
    x = _randn((32, K), seed=K + 6)
    nw = (1 + 0.1 * torch.randn(K, generator=_gen(K + 7), device="cuda")).bfloat16() if norm else None
    nt = math.ceil(K / 128)
    ssq = torch.full((32, 32), float("nan"), device="cuda")
    if norm:
        ssq[:, :nt] = tile_ssq(x).float()
    sched = (2 * _sms(), 4)
    base, _ = step_gemm(w, x, 32, *sched, nw, ssq if norm else None, eps)
    again, _ = step_gemm(w, x, 32, *sched, nw, ssq if norm else None, eps)
    assert torch.equal(base.view(torch.int32), again.view(torch.int32)), "two runs of one plan differ"
    assert torch.isfinite(base).all()
    for j in (0, 12, 31):
        for junk in (float("nan"), 1e30, -1e30, None):
            if junk is None:
                xj = _randn((32, K), seed=K + j, scale=100.0)
            else:
                xj = torch.full((32, K), junk, device="cuda").bfloat16()
            xj[j] = x[j]
            sj = torch.full((32, 32), float("nan") if junk is None or junk != junk else 1e38, device="cuda")
            sj[j] = ssq[j]
            for rows in sorted({j + 1, 17 if j < 17 else 32, 32}):
                out, _ = step_gemm(w, xj, rows, *sched, nw, sj if norm else None, eps)
                assert torch.equal(out[j].view(torch.int32), base[j].view(torch.int32)), (
                    f"row {j} changed with rows={rows} and the other rows of X = {junk}")


# ---------------------------------------------------------------------------------------------------------------------
# 3d: one decode layer through the engine's own plans
# ---------------------------------------------------------------------------------------------------------------------
_MODELS: dict = {}


def _model(name):
    if name not in _MODELS:
        from oracle import lm_oracle as O

        for _, _, m in _MODELS.values():  # one at a time on the device
            m.engine.close()
        _MODELS.clear()
        cfg = layer_configs()[name]
        w = O.make_weights(cfg, seed=97)
        _MODELS[name] = (cfg, w, build_model(cfg, w, max_batch=32, debug=False, max_rows=128))
    return _MODELS[name]


@pytest.fixture(scope="module", autouse=True)
def _free_models():
    yield
    for _, _, m in _MODELS.values():
        m.engine.close()
    _MODELS.clear()


def _check_resid(x_new, x_old, y, b, absprod, what):
    """x_new = rbf(x_old + rbf(y + b)) with y the float64 GEMM; the rounding of y + b may go either way within
    C_AMB * absprod of a bf16 rounding boundary."""
    v = y + (b.double()[None, :] if b is not None else 0.0)
    y_lo, y_hi = bracket_bf16(v, C_AMB * absprod)
    x_old = x_old.float()
    check_bracket(x_new.float(), rbf(x_old + y_lo), rbf(x_old + y_hi), f"{what}: x", rbf(x_old + rbf(v)))


def _check_swiglu(h, x, ssq, w, prefix, eps, what):
    """h = rbf(rbf(silu(g)) * u), g = rbf(w1 X'), u = rbf(w3 X') from the SEPARATE w1 / w3 (not the interleaved
    matrix), X' = ffn_norm(x) normalised on load with the sums of squares the residual-add finalize left. Ambiguity
    sources: the accumulation (C_AMB), the rounding of X' (rsqrtf) and expf."""
    nw = w[f"{prefix}.ffn_norm.weight"].cuda()
    g, u = (normed_gemm(x, ssq, nw, eps, w[f"{prefix}.feed_forward.{name}.weight"].cuda()) for name in ("w1", "w3"))
    # h is monotone in u, and in g wherever a bracket of g holds more than two bf16 values (|g| small, silu rising):
    # the extremes over the corners bracket it
    lo, hi, mid = swiglu_from(*bracket_bf16(*g), rbf(g[0]), *bracket_bf16(*u), rbf(u[0]))
    check_bracket(h.float(), lo, hi, f"{what}: h", mid)


LAYER_CASES = [pytest.param(name, fast, last, id=f"{name}-{'fast' if fast else 'slow'}-{'last' if last else 'first'}")
               for name in ("tiny", "s2pro") for fast in (0, 1) for last in (False, True)]


@pytest.mark.parametrize("name,fast,last", LAYER_CASES)
def test_decode_layer_gemms(name, fast, last):
    """wo + residual add, w1|w3 (normalised on load) + SwiGLU, w2 + residual add, each stage against float64 from the
    kernel's own output of the stage before."""
    L = _lib()
    cfg, w, model = _model(name)
    eng = model.engine
    nl = cfg.n_fast_layer if fast else cfg.n_layer
    layer = nl - 1 if last else 0
    prefix = f"{'fast_layers' if fast else 'layers'}.{layer}"
    D = cfg.fast_dim if fast else cfg.dim
    I = cfg.fast_intermediate_size if fast else cfg.intermediate_size
    HD = (cfg.fast_n_head * cfg.fast_head_dim) if fast else (cfg.n_head * cfg.head_dim)
    nt = math.ceil(D / 128)
    xb = eng.buffer("x_fast" if fast else "x_slow")
    sb = eng.buffer("ssq_fast" if fast else "ssq_slow")
    ab = eng.buffer("attn")[: 32 * HD].view(32, HD)
    hb = eng.buffer("ffn_h")
    wo = w[f"{prefix}.attention.wo.weight"].cuda()
    bo = w.get(f"{prefix}.attention.wo.bias")
    bo = bo.cuda() if bo is not None else None
    w2 = w[f"{prefix}.feed_forward.w2.weight"].cuda()
    stream = torch.cuda.current_stream().cuda_stream
    sentinel = torch.tensor([-12345.0], device="cuda").bfloat16()

    for rows in (1, 13, 32):
        what = f"{name} {'fast' if fast else 'slow'} layer {layer} rows={rows}"
        x0 = _randn((32, D), seed=rows + 11 * layer + 100 * fast)
        x0[rows:] = sentinel
        attn = _randn((32, HD), seed=rows + 11 * layer + 100 * fast + 1)
        attn[rows:] = float("nan")  # dead rows of the wo operand must not reach live rows

        def run(upto):
            xb.copy_(x0)
            sb.fill_(float("nan"))
            ab.copy_(attn)
            hb.fill_(sentinel.item())
            torch.cuda.synchronize()
            L.check(L.lib().fsb_lm_test_layer_gemms(eng.h, fast, layer, rows, upto, stream))
            torch.cuda.synchronize()
            return xb.clone(), sb.clone(), hb.clone()

        def dead_regions_untouched(x, ssq, h, h_written):
            assert torch.equal(x[rows:].view(torch.int16), x0[rows:].view(torch.int16)), f"{what}: dead x rows written"
            assert torch.isnan(ssq[rows:]).all() and torch.isnan(ssq[:, nt:]).all(), f"{what}: dead ssq written"
            tail = h[rows * I:] if h_written else h
            assert (tail.view(torch.int16) == sentinel.view(torch.int16)).all(), f"{what}: ffn_h written past rows*I"

        # upto = 1: x1 = rbf(x0 + rbf(wo attn + bo)) and its sums of squares
        x1, s1, h1 = run(1)
        y, absprod = fp64_gemm(attn[:rows], wo)
        _check_resid(x1[:rows], x0[:rows], y, bo, absprod, f"{what} wo")
        check_ssq(s1[:rows], x1[:rows], f"{what} wo")
        dead_regions_untouched(x1, s1, h1, False)

        # upto = 2: the same x, then h = SwiGLU of the w1|w3 GEMM normalised on load with those sums of squares
        x2, s2, h2 = run(2)
        assert torch.equal(x2.view(torch.int16), x1.view(torch.int16)), f"{what}: x differs between runs"
        assert torch.equal(s2.view(torch.int32), s1.view(torch.int32)), f"{what}: sums of squares differ between runs"
        hl = h2[: rows * I].view(rows, I)
        _check_swiglu(hl, x1[:rows], s1[:rows], w, prefix, cfg.norm_eps, f"{what} w13")
        dead_regions_untouched(x2, s2, h2, True)

        # upto = 3: x3 = rbf(x1 + rbf(w2 h)) (w2 has no bias) and its sums of squares, finished by the next consumer
        x3, s3, h3 = run(3)
        assert torch.equal(h3.view(torch.int16), h2.view(torch.int16)), f"{what}: h differs between runs"
        y, absprod = fp64_gemm(hl, w2)
        _check_resid(x3[:rows], x1[:rows], y, None, absprod, f"{what} w2")
        check_ssq(s3[:rows], x3[:rows], f"{what} w2")
        dead_regions_untouched(x3, s3, h3, True)
