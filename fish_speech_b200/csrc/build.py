"""Build libfishb200.so in-tree with nvcc for sm_90a (H100; no other architecture, no JIT cache)."""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
LIB = HERE.parent / "libfishb200.so"
SOURCES = ["error.cu", "gemm_tc.cu", "lm_gemm.cu", "lm_kernels.cu", "attn_tile.cu", "lm_engine.cu", "codec_kernels.cu", "codec_resunit.cu", "audio_kernels.cu", "api.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-diag-suppress", "550",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (Path(cand).exists() or cand == "nvcc"):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not LIB.exists():
        return True
    t = LIB.stat().st_mtime
    deps = list(HERE.glob("*.cu")) + list(HERE.glob("*.cuh")) + [HERE.parent.parent / "include" / "fishb200.h"]
    return any(p.stat().st_mtime > t for p in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not needs_build():
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    build_dir = HERE / "build"
    build_dir.mkdir(exist_ok=True)
    for src in SOURCES:
        if not (HERE / src).exists():
            continue
        obj = build_dir / (src + ".o")
        objs.append(str(obj))
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(HERE / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src} ---\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    cmd = [nvcc, "-shared", "-o", str(LIB), *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
