"""Qwen3-30B-A3B-shaped synthetic weights, saved and loaded through load_checkpoint, on one GPU:
  python tools/moe_bench.py [--rounds R] [--layers L] [--save-dir DIR]

  load     seconds to save and to load the checkpoint (48 layers: about 16 GB), and the peak device memory once the
           model is built (the weights plus the interleaved gate|up copy the grouped GEMM reads)
  kernels  per sparse layer at T = 1, 64 and 4096 rows: each launch of the MoE block (router in both layouts - 4-bit
           group 128 and mlx_lm's 8-bit group 64 - top-k, group, gather, gate|up, down, combine) timed alone, repeated
           in one CUDA graph, with CUDA events, with its algorithmic bytes and FLOPs and the share of the bound min time (3.35 TB/s HBM, 989 TFLOP/s
           dense bf16; the H100 SXM data sheet at 700 W)
  decode   device-resident greedy decode tok/s through DecodeEngine at B = 1, 8, 32 and 64 (128-token prompts, 32 steps)
  prefill  one 4096-token prompt through the public call, tok/s

The checkpoint's routers are 8-bit group 64 (what current mlx_lm writes).  Every measurement is repeated for --rounds
rounds, the configurations of one measurement alternating within a round; the JSON gives the median and the
[min, max] spread, beside the card name and its power limit."""

import argparse
import json
import shutil
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]
from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

from bench import _prefill_request, cuda_time_ms, synthetic_prompt  # noqa: E402

HBM_BPS, BF16_FLOPS = 3.35e12, 989e12


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:  # the numbers stay; the card line says why it is missing
        return f"unknown ({exc})"


def fill_random(node, gen):
    """Fill an ``empty=True`` synthetic model in place on its device, with the value ranges of synthetic._random_layer
    (codes uniform, weights ~ N(0, 1 / in_dim)); norms near 1."""
    from types import SimpleNamespace

    if isinstance(node, list):
        for item in node:
            fill_random(item, gen)
        return
    if not isinstance(node, SimpleNamespace):
        return
    if hasattr(node, "scales"):
        w = node.weight.view(torch.int32)
        w.copy_(torch.randint(-(2**31), 2**31 - 1, w.shape, generator=gen, device=w.device, dtype=torch.int64).to(torch.int32))
        in_dim = node.scales.shape[-1] * node.group_size
        sigma = 1.0 / (4.717 * in_dim**0.5)
        centre, step = (7.5, 1.0) if node.bits == 4 else (127.5, 15.0 / 255.0)
        s = torch.randn(node.scales.shape, generator=gen, device=w.device) * (sigma * step)
        node.scales.copy_(s.to(torch.bfloat16))
        node.biases.copy_((-centre * node.scales.float() + torch.randn(s.shape, generator=gen, device=w.device) * sigma).to(torch.bfloat16))
        return
    if set(vars(node)) == {"weight"}:
        node.weight.copy_((1 + 0.1 * torch.randn(node.weight.shape, generator=gen, device=node.weight.device)).to(torch.bfloat16))
        return
    for value in vars(node).values():
        fill_random(value, gen)


def spread(xs):
    return {"median": round(statistics.median(xs), 4), "min": round(min(xs), 4), "max": round(max(xs), 4)}


def timed(fn, reps):
    """Device time of one call: `reps` calls captured in one CUDA graph, the replay timed with CUDA events (so the
    host's per-call cost, about 20 us through the shim, does not count)."""
    fn()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        fn()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(reps):
                fn()
        graph.replay()
        ms = cuda_time_ms(graph.replay, stream) / reps
    stream.synchronize()
    return ms


def layer_steps(moe, T, device, gen):
    """The launches of one sparse layer at T rows as (name, fn, bytes, flops), on random rows of layer 0's block."""
    from tiny_llm_b200 import moe as moe_mod

    E, H, inter, k = moe.num_experts, moe.hidden_size, moe.intermediate_size, moe.num_experts_per_tok
    R = T * k
    h = torch.randn(T, H, generator=gen, device=device).to(torch.bfloat16)
    w4 = torch.randint(-(2**31), 2**31 - 1, (E, H // 8), generator=gen, device=device, dtype=torch.int64).to(torch.int32)
    s4 = (torch.randn(E, H // 128, generator=gen, device=device) * 0.01).to(torch.bfloat16)
    g64 = moe.w_router
    logits = ext.moe_router(h, g64.weight, g64.scales, g64.biases)
    _, ids, scores = ext.moe_topk(logits, k, moe.norm_topk_prob)
    nt = max(ext.moe_grouped_matmul_route(T, k, E, H, 2 * inter, ext.EPI_SWIGLU_PAIRS, h.dtype, h, moe.w_gate_up.weight)[1],
             ext.moe_grouped_matmul_route(T, k, E, inter, H, ext.EPI_NONE, h.dtype, h, moe.w_down.weight)[1])
    flat = ids.reshape(-1).contiguous()
    offsets, perm, tiles = moe_mod._group(flat, E, nt)
    xs = ext.moe_gather(h, perm, k)
    act = moe_mod._grouped(xs, moe.w_gate_up, offsets, tiles, k, None, ext.EPI_SWIGLU_PAIRS)
    y = moe_mod._grouped(act, moe.w_down, offsets, tiles, k, perm, ext.EPI_NONE)
    used = int(torch.unique(flat).numel())  # experts whose weights a projection streams
    return [
        ("router_g128_w4", lambda: ext.quantized_matmul(s4, s4, 128, 4, h, w4, True), E * H // 2 + E * H // 128 * 4 + 2 * T * (H + E), 2 * T * E * H),
        ("router_g64_w8", lambda: ext.moe_router(h, g64.weight, g64.scales, g64.biases), E * H + E * H // 64 * 4 + 2 * T * (H + E), 2 * T * E * H),
        ("topk", lambda: ext.moe_topk(logits, k, moe.norm_topk_prob), 4 * T * E + 6 * R, 0),
        ("group", lambda: ext.moe_group(flat, E, nt), 8 * R + 4 * (E + 1), 0),
        ("gather", lambda: ext.moe_gather(h, perm, k), 4 * R * H + 4 * R, 0),
        ("gate_up", lambda: moe_mod._grouped(xs, moe.w_gate_up, offsets, tiles, k, None, ext.EPI_SWIGLU_PAIRS),
         used * 2 * inter * H * 17 // 32 + 2 * R * (H + inter), 2 * R * 2 * inter * H),
        ("down", lambda: moe_mod._grouped(act, moe.w_down, offsets, tiles, k, perm, ext.EPI_NONE),
         used * H * inter * 17 // 32 + 2 * R * (inter + H), 2 * R * H * inter),
        ("combine", lambda: ext.moe_combine(y, scores, h), 2 * R * H + 6 * T * H + 2 * R, 2 * R * H),
    ], used


def decode_ms(model, device, B, vocab):
    from tiny_llm_b200.batch import greedy_tokens
    from tiny_llm_b200.kv_cache import BatchingKvCache

    S, steps = 128, 32
    engine = model.decode_engine(B)
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=512) for _ in range(model.num_hidden_layers)]
    tokens = []
    for b in range(B):
        cache, logits = _prefill_request(model, device, synthetic_prompt(100 + b, S, vocab))
        tokens.append(int(greedy_tokens(logits[:, -1, :])[0]))
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, b)
    engine.decode_on_device(tokens, [S] * B, tables, 4)
    torch.cuda.synchronize()
    tokens = engine.next_tokens.tolist()
    ms = cuda_time_ms(lambda: engine.decode_on_device(tokens, [S + 4] * B, tables, steps)) / steps
    for table in tables:
        for b in range(B):
            table.remove_request(b)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=48, help="decoder layers of the Qwen3-30B-A3B shape (48 = the published model)")
    ap.add_argument("--save-dir", default=None, help="where the checkpoint is written (a temporary directory, removed afterwards, if not given)")
    opts = ap.parse_args()
    from tiny_llm_b200 import Qwen3ModelWeek3
    from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
    from tiny_llm_b200.synthetic import synthetic_qwen3

    if not torch.cuda.is_available():
        raise SystemExit("moe_bench.py measures on a CUDA device; none is visible")
    device = torch.device("cuda:0")
    out = {"card": card(), "layers": opts.layers, "rounds": opts.rounds, "router": "8-bit group 64"}
    gen = torch.Generator(device=device).manual_seed(0)
    ns = synthetic_qwen3("qwen3-30b-a3b", empty=True, device=device, num_hidden_layers=opts.layers, max_position_embeddings=4096,
                         router_bits=8, router_group_size=64)
    fill_random(ns, gen)
    path = Path(opts.save_dir) if opts.save_dir else Path(tempfile.mkdtemp(prefix="moe_bench_"))
    try:
        t0 = time.perf_counter()
        save_checkpoint(ns, path)
        out["checkpoint_gb"] = round(sum(f.stat().st_size for f in path.iterdir()) / 1e9, 2)
        del ns
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(device)
        t1 = time.perf_counter()
        loaded = load_checkpoint(path, device=device)
        model = Qwen3ModelWeek3(loaded, page_size=128)
        model.decode_graph_max_seq_len = 512  # the decode window: KV pages for 64 slots fit beside the weights
        torch.cuda.synchronize()
        t2 = time.perf_counter()
    finally:
        if opts.save_dir is None:
            shutil.rmtree(path, ignore_errors=True)
    out["load"] = {"save_s": round(t1 - t0, 1), "load_s": round(t2 - t1, 1), "peak_device_gb_after_load": round(torch.cuda.max_memory_allocated(device) / 1e9, 2),
                   "allocated_gb_after_load": round(torch.cuda.memory_allocated(device) / 1e9, 2)}

    # per-kernel table of one sparse layer
    moe = model.layers_inner[0].mlp
    out["kernels"] = {}
    for T in (1, 64, 4096):
        steps, used = layer_steps(moe, T, device, torch.Generator(device=device).manual_seed(T))
        reps = 200 if T <= 64 else 20
        times = {name: [] for name, *_ in steps}
        for _ in range(opts.rounds):
            for name, fn, _, _ in steps:
                times[name].append(timed(fn, reps) * 1e3)  # us
        rows = {}
        for name, _, nbytes, flops in steps:
            us = statistics.median(times[name])
            bound_us = max(nbytes / HBM_BPS, flops / BF16_FLOPS) * 1e6
            rows[name] = {"us": spread(times[name]), "bytes": nbytes, "flops": flops, "bound": "flops" if flops / BF16_FLOPS > nbytes / HBM_BPS else "bytes",
                          "share_of_bound": round(bound_us / us, 3)}
        rows["layer_us_g64"] = round(sum(statistics.median(times[n]) for n in times if n != "router_g128_w4"), 2)
        out["kernels"][f"T{T}"] = {"experts_used": used, **rows}

    vocab = loaded.args.vocab_size
    out["decode"] = {}
    t = {B: [] for B in (1, 8, 32, 64)}
    for _ in range(opts.rounds):
        for B in t:
            t[B].append(B * 1e3 / decode_ms(model, device, B, vocab))
    for B, xs in t.items():
        out["decode"][f"B{B}_tok_s"] = spread(xs)

    prompt = synthetic_prompt(7, 4096, vocab)
    rates = []
    for _ in range(opts.rounds):
        cache = None

        def run():
            nonlocal cache
            cache, _ = _prefill_request(model, device, prompt, chunk=4096)

        run()
        for c in cache:
            c.release()
        rates.append(4096 * 1e3 / cuda_time_ms(run))
        for c in cache:
            c.release()
    out["prefill_4096_tok_s"] = spread(rates)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
