"""In-kernel timeline of the swap-AB GEMM (debug build with -DTL_TRACE=1, CTA 0):
  TL_LIB=.../libtiny_llm_b200_trace.so python tools/skinny_timeline.py
Tags: 30 entry, 31 set-up done (barriers), 34 accumulators complete, 36 exit."""
import ctypes
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]
from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

dev = torch.device("cuda:0")
lib = ctypes.CDLL(str(ext.current_library_path()))
g = torch.Generator(device=dev).manual_seed(0)
for M, N, K in [(64, 2560, 6144), (64, 4096, 2560), (64, 2560, 19456), (64, 9728, 2560), (128, 2560, 19456), (16, 2560, 1024)]:
    w = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=dev, generator=g).to(torch.int32)
    s = (torch.randn(K, N // 128, device=dev, generator=g) * 0.01).to(torch.bfloat16)
    b = (-7.5 * s.float()).to(torch.bfloat16)
    a = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
    for _ in range(3):
        ext.quantized_matmul(s, b, 128, 4, a, w, True)
    torch.cuda.synchronize()
    cap = 4096
    events = torch.zeros(2 * cap, dtype=torch.int64, device=dev)
    count = torch.zeros(1, dtype=torch.int32, device=dev)
    lib.tl_debug_trace(ctypes.c_void_p(events.data_ptr()), ctypes.c_void_p(count.data_ptr()), ctypes.c_uint(cap))
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    ext.quantized_matmul(s, b, 128, 4, a, w, True)
    end.record()
    torch.cuda.synchronize()
    lib.tl_debug_trace(None, None, ctypes.c_uint(0))
    n = int(count[0])
    ev = sorted(events[: 2 * n].cpu().reshape(-1, 2).tolist(), key=lambda e: e[1])
    t0 = ev[0][1] if ev else 0
    print(f"M={M} N={N} K={K}: event-timed {start.elapsed_time(end) * 1e3:.1f} us;", " ".join(f"{tag}@{(t - t0) / 1e3:.2f}" for tag, t in ev), flush=True)
