"""Build libtiny_llm_b200.so (sm_90a only) in-tree with nvcc.

The reference drives CMake through mlx.extension.CMakeBuild
(src/extensions_ref/build.py:11-24, CMakeLists.txt:32-84) to
produce a metallib plus a nanobind module; here one nvcc invocation per
translation unit produces objects that are linked into a C-ABI shared library
loaded with ctypes.  nvcc cross-compiles without a GPU.
"""

from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

CSRC = Path(__file__).resolve().parent
ROOT = CSRC.parent.parent
OUT_DIR = CSRC.parent / "extensions_b200" / "tiny_llm_ext_b200"
# Experiment builds: TL_DEFINES="-DS5_DEPTH_SMALL=3 ..." TL_LIB_SUFFIX=_d3 python build.py
# -> libtiny_llm_b200_d3.so next to the product library (tools/kbench.py --lib selects it).
SUFFIX = os.environ.get("TL_LIB_SUFFIX", "")
LIB = OUT_DIR / f"libtiny_llm_b200{SUFFIX}.so"
BUILD = CSRC / f"build{SUFFIX}"

SOURCES = [
    "c_abi.cu",
    "elementwise.cu",
    "w4a16_matvec.cu",
    "w4a16_skinny.cu",
    "attention_decode.cu",
    "attention_prefill.cu",
    "attention_prefill_tc.cu",
    "decode_attention_fused.cu",
    "sampling.cu",
    "spec_sample.cu",
    "ngram.cu",
    "beam.cu",
    "logprobs.cu",
    "constrained.cu",
    "json.cu",
    "json_schema.cu",
    "moe.cu",
    "moe_router.cu",
    "lora.cu",
    "embed.cu",
    "tma.cu",
]

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", str(ROOT / "include"),
    *os.environ.get("TL_DEFINES", "").split(),
]


def _digest(path: Path) -> str:
    h = hashlib.sha256()
    for dep in sorted(list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [ROOT / "include" / "tiny_llm_b200.h", path]):
        h.update(dep.read_bytes())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src: str, verbose: bool) -> Path:
    path = CSRC / src
    obj = BUILD / (path.stem + ".o")
    stamp = BUILD / (path.stem + ".sha")
    want = _digest(path)
    if obj.exists() and stamp.exists() and stamp.read_text() == want:
        return obj
    cmd = [NVCC, *FLAGS, "-c", str(path), "-o", str(obj)]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    proc = subprocess.run(cmd, capture_output=True, text=True)
    if proc.returncode != 0:
        sys.stderr.write(proc.stdout + proc.stderr)
        raise RuntimeError(f"nvcc failed on {src}")
    if verbose:
        sys.stderr.write(proc.stderr)
    stamp.write_text(want)
    return obj


def build(verbose: bool = False) -> Path:
    BUILD.mkdir(exist_ok=True)
    OUT_DIR.mkdir(parents=True, exist_ok=True)
    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as pool:
        objs = list(pool.map(lambda s: _compile(s, verbose), SOURCES))
    newest = max(o.stat().st_mtime for o in objs)
    if not LIB.exists() or LIB.stat().st_mtime < newest:
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
               "-o", str(LIB), *map(str, objs), "-lcuda"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            sys.stderr.write(proc.stdout + proc.stderr)
            raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv))
