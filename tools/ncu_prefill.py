"""Driver for `ncu` captures of the two prefill kernels (the GEMM on 128-token tiles, the flash attention):

  ncu --set full --clock-control none --import-source on -k regex:"w4a16_skinny_kernel|paged_prefill_tc" -s 4 -c 2 \
      -o tools_out/prefill python tools/ncu_prefill.py
"""
from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(0)
    M, N, K = 4096, 2560, 19456  # gate|up of Qwen3-4B
    w = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
    s = (torch.randn(K, N // 128, device=dev, generator=g) * 0.01).to(torch.bfloat16)
    b = (-7.5 * s.float()).to(torch.bfloat16)
    x = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
    Hq, Hkv, D, page, L = 32, 8, 128, 128, 4096
    pages = L // page
    kp = torch.randn(pages, Hkv, page, D, device=dev, generator=g).to(torch.bfloat16)
    vp = torch.randn(pages, Hkv, page, D, device=dev, generator=g).to(torch.bfloat16)
    q = torch.randn(Hq, L, D, device=dev, generator=g).to(torch.bfloat16)
    bt = torch.arange(pages, dtype=torch.int32, device=dev).reshape(1, pages)
    cl = torch.tensor([L], dtype=torch.int32, device=dev)
    for _ in range(3):  # launches 0..5: warm-up (skipped by -s 4), 4 and 5 are captured
        ext.quantized_matmul(s, b, 128, 4, x, w, True)
        ext.paged_attention(q, kp, vp, bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
