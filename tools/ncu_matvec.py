"""Small driver for `ncu` captures of the W4A16 streaming kernel:

  ncu --set full --clock-control none --import-source on -k regex:w4a16_stream -s 4 -c 2 \
      -o tools_out/matvec python tools/ncu_matvec.py [lm_head|gate_up|down|q|o]
"""

from __future__ import annotations

import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

SHAPES = {"q": (2560, 4096), "kv": (2560, 1024), "o": (4096, 2560), "gate_up": (2560, 19456), "down": (9728, 2560), "lm_head": (2560, 151936)}


def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "lm_head"
    M = int(sys.argv[2]) if len(sys.argv) > 2 else 1
    N, K = SHAPES[name]
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(1)
    copies = max(2, min(8, int(300e6 // (K * N // 2)) + 1))
    ws = [torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=dev, generator=g).to(torch.int32) for _ in range(copies)]
    sc = [(torch.randn(K, N // 128, device=dev, generator=g) * 0.01).to(torch.bfloat16) for _ in range(copies)]
    bi = [(-7.5 * s.float()).to(torch.bfloat16) for s in sc]
    a = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
    for rep in range(3):
        for i in range(copies):
            ext.quantized_matmul(sc[i], bi[i], 128, 4, a, ws[i], True)
    torch.cuda.synchronize()


if __name__ == "__main__":
    main()
