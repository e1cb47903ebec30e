"""Record the oracle's sampling traces of the stochastic goldens (lm_tiny_topk / lm_tiny_ras) for the GPU suite.

    python -m oracle.make_golden_traces

The GPU test that replays the reference's RNG compares the CUDA path against the recorded reference tokens and, at a
first differing frame, needs the reference's decision margins (scores, top-p cumulative sums, top-k logits): the
oracle's trace of the same run.  The oracle runs its bf16 matmuls on the CPU, whose kernels depend on the host's
instruction set, and a high-temperature draw can turn on the last bit of a score; so the trace is recorded here, where
the oracle reproduces the reference's tokens exactly (asserted), and stored as trace_<golden>.npz.
"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import lm_oracle as O  # noqa: E402
from tests.lm_util import load_golden  # noqa: E402

GOLD = ROOT / "tests" / "golden"


def record(name: str) -> Path:
    cfg, w, z = load_golden(GOLD / name)
    traces = []
    torch.manual_seed(int(z["rng_seed"]))
    out = O.generate(O.setup(cfg, w), torch.from_numpy(z["prompt"]), int(z["new_frames"]),
                     temperature=float(z["temperature"]), top_p=float(z["top_p"]), top_k=int(z["top_k"]), traces=traces)
    assert torch.equal(out.to(torch.int32), torch.from_numpy(z["ref_tokens"])), "the oracle does not reproduce the reference run here"
    arrays = {"ras_changed": np.array([bool(t.get("ras_changed")) for t in traces])}
    for f, t in enumerate(traces):
        for r, (s_, cum, tp, topl) in enumerate(t["scores"]):
            arrays[f"s_{f}_{r}"] = s_.numpy().astype(np.float32)
            arrays[f"cum_{f}_{r}"] = cum.numpy().astype(np.float32)
            arrays[f"tp_{f}_{r}"] = np.float64(tp)
            arrays[f"topl_{f}_{r}"] = topl.numpy().astype(np.float32)
    path = GOLD / ("trace_" + name)
    np.savez_compressed(path, **arrays)
    return path


if __name__ == "__main__":
    for n in ("lm_tiny_topk.npz", "lm_tiny_ras.npz"):
        print(record(n))
