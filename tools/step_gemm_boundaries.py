"""Where the decode step GEMMs lose time against a plain weight stream: the cost of a GEMM boundary.

Replays the 36 slow layers' step GEMMs of ONE kind (qkv, wo, w1|w3 or w2) back to back through the decode path's own
plans (fsb_lm_bench_step_kind), with and without the finalize kernels between them, and fits per-launch time against
per-launch weight bytes over the four kinds:

    t = t0 + bytes / BW

t0 is the fixed cost of a boundary, BW the streaming rate inside a GEMM. For reference it also times the frame's whole
step GEMM chain (the replay line of bench.py) and decode frames.

    python tools/step_gemm_boundaries.py [--min-s 0.5] [--batch 32]

Prints one JSON object, with the card's name, power limit and maximum SM clock. Needs a GPU; S2-Pro geometry with
synthetic weights, batch 32 by default (an engine of --batch slots: above 32 it runs the 64-row step GEMM).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import numpy as np  # noqa: E402
import torch  # noqa: E402

KINDS = ("qkv", "wo", "w13", "w2")
T_PROMPT = 64


def card() -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), (v.strip() for v in out.split(","))))
    except Exception as e:  # pragma: no cover
        return {"name": torch.cuda.get_device_name(0), "error": repr(e)}


def timed(fn, min_s: float) -> tuple[float, int]:
    """(ms per call, calls): fn() repeated until the timed window is at least min_s seconds."""
    fn()
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    fn()
    ev1.record()
    torch.cuda.synchronize()
    n = max(1, math.ceil(min_s * 1e3 / max(ev0.elapsed_time(ev1), 1e-3)))
    ev0.record()
    for _ in range(n):
        fn()
    ev1.record()
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1) / n, n


def fit(points) -> dict:
    """Least squares t_us = t0_us + bytes / BW over (bytes, t_us) points."""
    x = np.array([p[0] for p in points], dtype=np.float64)
    y = np.array([p[1] for p in points], dtype=np.float64)
    slope, t0 = np.polyfit(x, y, 1)
    resid = y - (t0 + slope * x)
    return {"t0_us": float(t0), "bw_gbs": float(1e-3 / slope), "max_resid_us": float(np.abs(resid).max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-s", type=float, default=0.5, help="least length of each timed window")
    ap.add_argument("--frames", type=int, default=64, help="decode frames timed")
    ap.add_argument("--batch", type=int, default=32, help="engine slots = rows of every step (1..64)")
    args = ap.parse_args()
    B = args.batch

    from bench import make_prompts, s2pro_cfg
    from fish_speech_b200 import _lib, synthetic
    from fish_speech_b200.configs import S2PRO_IM_END_ID
    from fish_speech_b200.models.text2semantic.llama import DualARTransformer

    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    cfg = s2pro_cfg()
    w = synthetic.lm_state_dict(cfg, dev)
    w["embeddings.weight"][S2PRO_IM_END_ID] = 0
    model = DualARTransformer(cfg, w, device=dev, im_end_id=S2PRO_IM_END_ID)
    model.max_rows = B * T_PROMPT
    model.setup_caches(max_batch_size=B, max_seq_len=cfg.max_seq_len)
    del w
    eng = model.engine
    L = _lib.lib()
    stream = torch.cuda.current_stream().cuda_stream

    result = {"card": card(), "sms": torch.cuda.get_device_properties(0).multi_processor_count,
              "layers": cfg.n_layer, "batch": B, "kinds": {}}
    wb, nl = C.c_double(), C.c_int()
    for fin in (1, 0):
        sfx = "" if fin else "_no_finalize"
        pts = []
        for k, name in enumerate(KINDS):
            ms, _ = timed(lambda: _lib.check(L.fsb_lm_bench_step_kind(eng.h, k, 1, fin, C.byref(wb), C.byref(nl),
                                                                       stream)), args.min_s)
            us = ms * 1e3 / nl.value
            per = wb.value / nl.value
            pts.append((per, us))
            entry = result["kinds"].setdefault(name, {"mb_per_launch": per / 1e6})
            entry["us_per_launch" + sfx] = us
            entry["gbs" + sfx] = per / us / 1e3
        result["fit" + sfx] = fit(pts)
    ms, _ = timed(lambda: _lib.check(L.fsb_lm_bench_gemms(eng.h, 1, C.byref(wb), C.byref(nl), stream)), args.min_s)
    result["frame_chain"] = {"launches": nl.value, "gbs": wb.value / (ms / 1e3) / 1e9, "us_per_launch": ms * 1e3 / nl.value}
    sp = eng.sampling(0.7, 0.7, 1, 42)
    eng.reset()
    eng.prefill([p.to(dev) for p in make_prompts(cfg, B, 42)], list(range(B)), sp, do_sample=True)
    eng.decode(B, 2, sp, use_graph=True)  # captures the frame graph
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    eng.decode(B, args.frames, sp, use_graph=True)
    ev1.record()
    torch.cuda.synchronize()
    result["ms_per_decode_frame"] = ev0.elapsed_time(ev1) / args.frames
    print(json.dumps(result))


if __name__ == "__main__":
    main()
