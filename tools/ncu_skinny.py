"""One skinny-GEMM shape for an `ncu --set full --import-source on` capture:

  ncu --set full --clock-control none --import-source on -k regex:w4a16_skinny_kernel -s 3 -c 1 -o tools_out/skinny \
      python tools/ncu_skinny.py [M N K]          # default: the tied head at 64 rows (2560 -> 151936)
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

M, N, K = (int(v) for v in sys.argv[1:4]) if len(sys.argv) >= 4 else (64, 2560, 151936)
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
w = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
s = (torch.randn(K, N // 128, device=dev, generator=g) * 0.01).to(torch.bfloat16)
b = (-7.5 * s.float()).to(torch.bfloat16)
a = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
for _ in range(4):
    ext.quantized_matmul(s, b, 128, 4, a, w, True)
    torch.cuda.synchronize()
print("done", ext.launch_count())
