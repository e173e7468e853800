"""Prefill-side kernels on one H100 (config 3 shapes): the wgmma W4A16 GEMM at M = 4096 for the
Qwen3-4B layer shapes, paged causal prefill attention at L = S = 4096, and the whole-model chunked
prefill of a 4096-token prompt through the public API.

  python tools/prefill_bench.py [--out tools_out/prefill_bench.json]
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

DEV = torch.device("cuda:0")
BF16 = torch.bfloat16


def peaks():
    path = ROOT / "MEASURED_PEAKS.json"
    d = json.loads(path.read_text()) if path.exists() else {}
    return float(d.get("bf16_tflops", d.get("bf16_tflops_burst", 1682.0))), float(d.get("hbm_gbs", 6650.0))


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "tools_out" / "prefill_bench.json"))
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--skip-model", action="store_true")
    ap.add_argument("--profile", action="store_true", help="torch.profiler kernel table of one whole-model prefill")
    args = ap.parse_args()
    tf_peak, _ = peaks()
    M = args.tokens
    report = {"bf16_peak_tflops": tf_peak, "gemm": [], "attention": [], "model": None}
    g = torch.Generator(device=DEV).manual_seed(0)
    for name, N, K in [("qkv", 2560, 6144), ("o", 4096, 2560), ("gate_up", 2560, 19456), ("down", 9728, 2560)]:
        w = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=DEV, generator=g).to(torch.int32)
        s = (torch.randn(K, N // 128, device=DEV, generator=g) * 0.01).to(BF16)
        b = (-7.5 * s.float()).to(BF16)
        x = torch.randn(M, N, device=DEV, generator=g).to(BF16)
        ms = timed(lambda: ext.quantized_matmul(s, b, 128, 4, x, w, True))
        tf = 2.0 * M * N * K / (ms * 1e-3) / 1e12
        report["gemm"].append(dict(name=name, M=M, N=N, K=K, ms=round(ms, 3), tflops=round(tf, 1), frac=round(tf / tf_peak, 3)))
        print(f"gemm {name:8s} M={M} {N}->{K}: {ms:7.3f} ms  {tf:7.1f} TF/s  {tf / tf_peak:5.1%}", flush=True)
    Hq, Hkv, D, page = 32, 8, 128, 128
    for L in (512, M):
        pages = (L + page - 1) // page
        kp = torch.randn(pages, Hkv, page, D, device=DEV, generator=g).to(BF16)
        vp = torch.randn(pages, Hkv, page, D, device=DEV, generator=g).to(BF16)
        q = torch.randn(Hq, L, D, device=DEV, generator=g).to(BF16)
        bt = torch.arange(pages, dtype=torch.int32, device=DEV).reshape(1, pages)
        cl = torch.tensor([L], dtype=torch.int32, device=DEV)
        ms = timed(lambda: ext.paged_attention(q, kp, vp, bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq), reps=3)
        flops = 4.0 * Hq * D * (L * (L + 1) / 2)  # causal: QK^T and PV over the lower triangle
        tf = flops / (ms * 1e-3) / 1e12
        report["attention"].append(dict(L=L, ms=round(ms, 3), tflops=round(tf, 2), frac=round(tf / tf_peak, 4)))
        print(f"paged causal prefill attention L=S={L}: {ms:8.3f} ms  {tf:7.2f} TF/s  {tf / tf_peak:6.2%}", flush=True)
    if not args.skip_model:
        from tiny_llm_b200 import Qwen3ModelWeek3
        from tiny_llm_b200.synthetic import synthetic_qwen3

        ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV)
        model = Qwen3ModelWeek3(ns, page_size=128)
        prompt = torch.randint(0, 150000, (1, M), dtype=torch.int32, device=DEV, generator=g)
        for rep in range(2):
            cache = model.create_kv_cache()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model(prompt, 0, cache, logits_to_keep=1)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            for c in cache:
                c.release()
        report["model"] = dict(tokens=M, seconds=round(dt, 4), tok_per_s=round(M / dt, 1))
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            cache = model.create_kv_cache()
            with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
                model(prompt, 0, cache, logits_to_keep=1)
                torch.cuda.synchronize()
            print(prof.key_averages().table(sort_by="cuda_time_total", row_limit=18, max_name_column_width=60))
        print(f"Qwen3-4B prefill of {M} tokens through model(): {dt * 1e3:.1f} ms -> {M / dt:.0f} tok/s", flush=True)
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
