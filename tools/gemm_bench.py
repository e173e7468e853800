"""Per-shape timing of the prefill GEMM (Qwen3-4B projections at M rows, default 4096):
  python tools/gemm_bench.py [M]
CUDA events around 20 back-to-back launches after 5 warm-up calls; weights of the next launch differ (4 copies > L2)."""
import json
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]
from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

M = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
dev = torch.device("cuda:0")
g = torch.Generator(device=dev).manual_seed(0)
out = {"M": M, "env": {k: v for k, v in os.environ.items() if k.startswith("TL_")}, "shapes": {}}
for name, N, K in [("qkv", 2560, 6144), ("o", 4096, 2560), ("gate_up", 2560, 19456), ("down", 9728, 2560)]:
    copies = []
    for _ in range(4):
        w = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
        s = (torch.randn(K, N // 128, device=dev, generator=g) * 0.01).to(torch.bfloat16)
        copies.append((w, s, (-7.5 * s.float()).to(torch.bfloat16)))
    a = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
    for i in range(5):
        w, s, b = copies[i % 4]
        ext.quantized_matmul(s, b, 128, 4, a, w, True)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    start.record()
    for i in range(reps):
        w, s, b = copies[i % 4]
        ext.quantized_matmul(s, b, 128, 4, a, w, True)
    end.record()
    torch.cuda.synchronize()
    us = start.elapsed_time(end) * 1e3 / reps
    tf = 2.0 * M * N * K / us / 1e6
    out["shapes"][name] = {"N": N, "K": K, "us": round(us, 1), "tflops": round(tf, 1)}
    print(f"{name:8s} M={M} {N}->{K}: {us:8.1f} us  {tf:7.1f} TF/s", flush=True)
print(json.dumps(out))
