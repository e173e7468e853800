"""Per-kernel micro-benchmark on one H100: CUDA-event timing of CUDA-graph
replays (so host launch overhead is out of the picture), rotating over enough
distinct buffers that every launch misses L2 (50 MB on H100), reported against the
HBM peak of MEASURED_PEAKS.json (else the H100 SXM data sheet).

  python tools/kbench.py [--out tools_out/kbench.json] [--quick]
"""

from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

DEV = torch.device("cuda:0")
BF16 = torch.bfloat16


def peak_gbs() -> float:
    path = ROOT / "MEASURED_PEAKS.json"
    if path.exists():
        return float(json.loads(path.read_text())["hbm_gbs"])
    return 3350.0  # NVIDIA H100 SXM data sheet


def time_graph(fn_list, reps=5, inner=1):
    """fn_list: callables launched back to back inside one captured graph.
    Returns mean microseconds per callable."""
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for f in fn_list[: min(3, len(fn_list))]:
            f()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(inner):
                for f in fn_list:
                    f()
        graph.replay()
        torch.cuda.synchronize()
        best = float("inf")
        for _ in range(reps):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            graph.replay()
            end.record()
            end.synchronize()
            best = min(best, start.elapsed_time(end))
    return best * 1e3 / (len(fn_list) * inner)


def matvec_case(M, N, K, copies):
    g = torch.Generator(device=DEV).manual_seed(N + K)
    ws = [torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, device=DEV, generator=g).to(torch.int32) for _ in range(copies)]
    sc = [(torch.randn(K, N // 128, device=DEV, generator=g) * 0.01).to(BF16) for _ in range(copies)]
    bi = [(-7.5 * s.float()).to(BF16) for s in sc]
    a = torch.randn(M, N, device=DEV, generator=g).to(BF16)
    fns = [(lambda i=i: ext.quantized_matmul(sc[i], bi[i], 128, 4, a, ws[i], True)) for i in range(copies)]
    us = time_graph(fns)
    nbytes = K * N * 17 // 32 + 2 * M * N + 2 * M * K
    return us, nbytes


def attention_case(B, S, page=128, Hq=32, Hkv=8, D=128):
    pages_per = (S + page - 1) // page
    P = B * pages_per
    copies = max(1, min(8, int(300e6 // (2 * P * Hkv * page * D * 2)) + 1))
    g = torch.Generator(device=DEV).manual_seed(S + B)
    sets = []
    for _ in range(copies):
        kp = torch.randn(P, Hkv, page, D, device=DEV, generator=g, dtype=torch.float32).to(BF16)
        vp = torch.randn(P, Hkv, page, D, device=DEV, generator=g, dtype=torch.float32).to(BF16)
        sets.append((kp, vp))
    bt = torch.arange(P, dtype=torch.int32, device=DEV).reshape(B, pages_per)
    cl = torch.full((B,), S, dtype=torch.int32, device=DEV)
    q = torch.randn(B * Hq, 1, D, device=DEV, generator=g).to(BF16)
    fns = [(lambda kv=kv: ext.paged_attention(q, kv[0], kv[1], bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)) for kv in sets]
    us = time_graph(fns, inner=max(1, 8 // copies))
    nbytes = B * (2 * Hkv * S * D * 2 + 2 * Hq * D * 2)
    return us, nbytes


def small_ops():
    out = {}
    x = torch.randn(1, 2560, device=DEV).to(BF16)
    w = torch.ones(2560, device=DEV, dtype=BF16)
    out["rms_norm_1x2560"] = time_graph([lambda: ext.rms_norm(x, w, 1e-6)], inner=20)
    h = torch.randn(1, 1, 40, 128, device=DEV).to(BF16)
    w128 = torch.ones(128, device=DEV, dtype=BF16)
    out["rms_norm_40x128"] = time_graph([lambda: ext.rms_norm(h, w128, 1e-6)], inner=20)
    off = torch.tensor([777], dtype=torch.int32, device=DEV)
    out["rope_1x1x32x128"] = time_graph([lambda: ext.rope(h[:, :, :32].contiguous(), off, 128, 1e6)], inner=20)
    gte = torch.randn(1, 9728, device=DEV).to(BF16)
    out["swiglu_9728"] = time_graph([lambda: ext.swiglu(gte, gte)], inner=20)
    out["add_2560"] = time_graph([lambda: ext.add(x, x)], inner=20)
    logits = torch.randn(1, 151936, device=DEV).to(BF16)
    out["argmax_151936"] = time_graph([lambda: ext.argmax(logits)], inner=20)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=str(ROOT / "tools_out" / "kbench.json"))
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--lib", default=None, help="alternative libtiny_llm_b200*.so (experiment builds)")
    ap.add_argument("--only", default=None, help="comma-separated matvec shape names; skips attention and small ops")
    ap.add_argument("--attention-only", action="store_true")
    ap.add_argument("--batches", default=None, help="comma-separated activation row counts for the projection sweep")
    args = ap.parse_args()
    import os

    if args.lib:
        ext.load_library(args.lib)
    if os.environ.get("TL_PDL", "0") == "1":
        ext.set_pdl(True)
    peak = peak_gbs()
    report = {"hbm_peak_gbs": peak, "gpu": torch.cuda.get_device_name(0), "matvec": [], "attention": [], "small_ops_us": {}}
    shapes = [("q", 2560, 4096), ("kv", 2560, 1024), ("o", 4096, 2560), ("gate_up", 2560, 9728), ("down", 9728, 2560), ("lm_head", 2560, 151936)]
    batches = [1, 8] if args.quick else [1, 2, 4, 8, 16, 32]
    if args.batches:
        batches = [int(b) for b in args.batches.split(",")]
    if args.only:
        shapes = [s for s in shapes if s[0] in args.only.split(",")]
    if args.attention_only:
        shapes = []
    for name, N, K in shapes:
        copies = max(2, min(48, int(300e6 // (K * N // 2)) + 1))
        for M in batches:
            us, nbytes = matvec_case(M, N, K, copies)
            gbs = nbytes / us / 1e3
            report["matvec"].append(dict(name=name, M=M, N=N, K=K, us=round(us, 2), gbs=round(gbs, 1), frac=round(gbs / peak, 3)))
            print(f"matvec {name:8s} M={M:2d} {N}->{K}: {us:8.2f} us  {gbs:7.1f} GB/s  {gbs / peak:5.1%}", flush=True)
    for B, S in [] if args.only else ([(1, 1024), (1, 8192)] if args.quick else [(1, 128), (1, 1024), (1, 4096), (1, 8192), (8, 4096), (32, 2048), (64, 1024), (64, 8192)]):
        try:
            us, nbytes = attention_case(B, S)
        except torch.OutOfMemoryError:
            print(f"attention B={B} S={S}: OOM", flush=True)
            continue
        gbs = nbytes / us / 1e3
        report["attention"].append(dict(B=B, S=S, us=round(us, 2), gbs=round(gbs, 1), frac=round(gbs / peak, 3)))
        print(f"paged decode attention B={B:2d} S={S:5d}: {us:9.2f} us  {gbs:7.1f} GB/s  {gbs / peak:5.1%}", flush=True)
    report["small_ops_us"] = {} if args.only else {k: round(v, 2) for k, v in small_ops().items()}
    print("small ops (us):", report["small_ops_us"], flush=True)
    Path(args.out).parent.mkdir(parents=True, exist_ok=True)
    Path(args.out).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
