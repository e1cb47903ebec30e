"""Micro-benchmark: one decoder ResidualUnit at the codec's real sizes (B = 32 utterances x 256 frames), as two conv
GEMM launches (conv7, conv1) and as the fused kernel (csrc/codec_resunit.cu).  python tools/bench_res_unit.py"""
import ctypes as Ct
import sys
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import torch  # noqa: E402

from fish_speech_b200 import _lib  # noqa: E402

L = _lib.lib()
st = lambda: torch.cuda.current_stream().cuda_stream
B = 32
dev = "cuda"


def timed(fn, n=5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


print("| C | T/utt | dilation | conv7 ms | conv1 ms | two launches ms | fused ms | fused TFLOP/s | fused GB/s (3 N C x 2 B) |")
print("|---|---|---|---|---|---|---|---|---|")
for C, T in ((384, 65536), (192, 262144), (96, 524288)):
    cp = (C + 63) // 64 * 64
    g = torch.Generator(device=dev).manual_seed(C)
    x = torch.randn(B, T, C, device=dev, generator=g, dtype=torch.float32).bfloat16()
    a = torch.randn(B, T, C, device=dev, generator=g, dtype=torch.float32).bfloat16()
    w7 = (torch.randn(C, 7 * cp, device=dev, generator=g) * (7 * C) ** -0.5).bfloat16()
    w1 = (torch.randn(C, cp, device=dev, generator=g) * C ** -0.5).bfloat16()
    vec = lambda: torch.rand(C, device=dev, generator=g) + 0.5
    b7, b1, a1, i1, an, inn = vec(), vec(), vec(), vec(), vec(), vec()
    h = torch.empty_like(a)
    y1 = torch.empty_like(a)
    for dil in (1, 9):
        sh7 = (Ct.c_int * 7)(*[-(6 - j) * dil for j in range(7)])
        sh1 = (Ct.c_int * 1)(0)
        c7 = lambda: _lib.check(L.fsb_conv_gemm(a.data_ptr(), B, T, C, C, T * C, w7.data_ptr(), C, 7, cp, sh7, T, b7.data_ptr(),
                                                 None, None, 0, None, h.data_ptr(), a1.data_ptr(), i1.data_ptr(), 0, st()))
        c1 = lambda: _lib.check(L.fsb_conv_gemm(h.data_ptr(), B, T, C, C, T * C, w1.data_ptr(), C, 1, cp, sh1, T, b1.data_ptr(),
                                                 None, x.data_ptr(), 0, x.data_ptr(), y1.data_ptr(), an.data_ptr(),
                                                 inn.data_ptr(), 0, st()))
        fu = lambda: _lib.check(L.fsb_res_unit(a.data_ptr(), x.data_ptr(), B, T, C, dil, w7.data_ptr(), b7.data_ptr(),
                                               a1.data_ptr(), i1.data_ptr(), w1.data_ptr(), b1.data_ptr(), x.data_ptr(),
                                               y1.data_ptr(), an.data_ptr(), inn.data_ptr(), st()))
        t7, t1, tf = timed(c7), timed(c1), timed(fu)
        flops = 2.0 * B * T * C * C * 8
        print(f"| {C} | {T} | {dil} | {t7:.2f} | {t1:.2f} | {t7 + t1:.2f} | {tf:.2f} | {flops / tf / 1e9:.0f} | "
              f"{4 * B * T * C * 2 / tf / 1e6:.0f} |")
    del x, a, h, y1
    torch.cuda.empty_cache()
