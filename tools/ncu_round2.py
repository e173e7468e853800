"""Driver for `ncu --set full` captures of the hot-path kernels (one launch of each kernel is captured):

  ncu --set full --clock-control none --import-source on \
      -k regex:"paged_prefill_tc|w4a16_skinny_kernel|w4a16_stream5" -s 21 -c 7 -o tools_out/kernels python tools/ncu_round2.py

Order of launches after the warm-up (3 of each): wgmma flash prefill (L = S = 4096), the same kernel as split-KV
decode attention (B = 64, S = 8192), swap-AB GEMM M = 64 at the gate|up and tied-head shapes, streaming matvec M = 1 at
the gate|up and tied-head shapes, the swap-AB GEMM on 128-token tiles at 4096 rows (gate|up)."""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

dev = torch.device("cuda:0")
BF = torch.bfloat16
g = torch.Generator(device=dev).manual_seed(0)


def packed(K, N):
    w = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
    s = (torch.randn(K, N // 128, device=dev, generator=g) * 0.01).to(BF)
    return w, s, (-7.5 * s.float()).to(BF)


def attention_inputs(B, L, S, page=128, Hq=32, Hkv=8, D=128):
    pages = (S + page - 1) // page
    kp = torch.randn(B * pages, Hkv, page, D, device=dev, generator=g).to(BF)
    vp = torch.randn(B * pages, Hkv, page, D, device=dev, generator=g).to(BF)
    q = torch.randn(B * Hq, L, D, device=dev, generator=g).to(BF)
    bt = torch.arange(B * pages, dtype=torch.int32, device=dev).reshape(B, pages)
    cl = torch.full((B,), S, dtype=torch.int32, device=dev)
    return lambda: ext.paged_attention(q, kp, vp, bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)


def matmul(M, N, K):
    w, s, b = packed(K, N)
    a = torch.randn(M, N, device=dev, generator=g).to(BF)
    return lambda: ext.quantized_matmul(s, b, 128, 4, a, w, True)


calls = [attention_inputs(1, 4096, 4096), attention_inputs(64, 1, 8192), matmul(64, 2560, 19456), matmul(64, 2560, 151936),
         matmul(1, 2560, 19456), matmul(1, 2560, 151936), matmul(4096, 2560, 19456)]
for rep in range(4):  # three warm-up rounds, the fourth is the one to capture
    for c in calls:
        c()
    torch.cuda.synchronize()
print("done", ext.launch_count())
