"""Prefix caching on one GPU, at the Qwen3-4B shape (36 layers, 8 KV heads, 128-slot pages, head_dim 128, bf16):

* the copy-on-write kernel ``tl_paged_cache_copy_prefix``: one page's first ``r`` in {1, 64, 127} slots, K and V, across
  the 36 layers in one launch, against the 72 torch slice copies it replaces.  CUDA events over 200 calls; successive
  calls cycle through 16 page pairs per layer (600 MB of slab), so the source is not served from L2;
* serving: 64 slots, 256 requests of one 1,024-token shared system prompt plus U[32, 256] unique tokens, outputs
  U[32, 128], ``prefill_step`` 128, Qwen3-4B-shaped synthetic weights, greedy.  The cache off and on alternate, twice
  each, on two models over the same weights (the index is cleared before every run with it on).  Time to first token is
  taken from the scheduler iteration that pops the request to the end of the one that produced its first token.

  python tools/prefix_cache_bench.py [--out tools_out/prefix_cache_bench.json]
"""
from __future__ import annotations

import argparse
import json
import random
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3  # noqa: E402
from tiny_llm_b200.batch import ContinuousBatcher  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
LAYERS, HKV, PAGE, D = 36, 8, 128, 128
HBM_TBS = 3.35  # H100 SXM data sheet


def card() -> str:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                          timeout=30).stdout.strip()


def events_ms(fn, calls: int, host_us_per_call: float) -> float:
    """Device time per call: the stream first runs a spin kernel longer than the host needs to enqueue every call, so
    the calls execute back to back and the events time the device, not the host."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(3e9 * 2 * calls * host_us_per_call * 1e-6) + 1000)  # ~2x the enqueue time at up to 3 GHz
    start.record()
    for i in range(calls):
        fn(i)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / calls


def host_us(fn, calls: int) -> float:
    """Host time per call to enqueue (no synchronise inside the window): what the scheduler pays."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(calls):
        fn(i)
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    return (t1 - t0) / calls * 1e6


def cow_bench(calls: int = 200) -> list[dict]:
    pairs = 16
    ks = [torch.randn(2 * pairs, HKV, PAGE, D, device=DEV).to(torch.bfloat16) for _ in range(LAYERS)]
    vs = [torch.randn(2 * pairs, HKV, PAGE, D, device=DEV).to(torch.bfloat16) for _ in range(LAYERS)]
    rows = []
    for r in (1, 64, 127):
        lists = [[(layer, p, pairs + p, r) for layer in range(LAYERS)] for p in range(pairs)]

        def kernel(i):
            ext.paged_cache_copy_prefix(ks, vs, lists[i % pairs])

        def slices(i):
            p = i % pairs
            for k, v in zip(ks, vs):
                k[pairs + p, :, :r].copy_(k[p, :, :r])
                v[pairs + p, :, :r].copy_(v[p, :, :r])

        for fn in (kernel, slices):
            for i in range(20):
                fn(i)
        want = [k.clone() for k in ks[:2]]
        kernel_host = host_us(kernel, calls)
        slices_host = host_us(slices, calls)
        kernel_ms = min(events_ms(kernel, calls, kernel_host) for _ in range(3))
        slices_ms = min(events_ms(slices, calls, slices_host) for _ in range(3))
        assert all(torch.equal(a, b) for a, b in zip(ks[:2], want))  # both paths wrote the same bytes
        moved = 2 * 2 * LAYERS * HKV * r * D * 2  # K and V, read and written
        rows.append({
            "slots": r, "bytes_moved": moved,
            "kernel_us": round(kernel_ms * 1e3, 2), "kernel_gbs": round(moved / (kernel_ms / 1e3) / 1e9, 1),
            "kernel_share_of_3.35_tbs": round(moved / (kernel_ms / 1e3) / (HBM_TBS * 1e12), 3),
            "kernel_host_us_per_call": round(kernel_host, 1),
            "torch_72_slices_us": round(slices_ms * 1e3, 2), "torch_72_slices_host_us_per_call": round(slices_host, 1),
            "timing": "device time per call with the calls queued behind a spin kernel; host time to enqueue one call",
        })
    return rows


def build_requests(seed: int, vocab: int):
    rng = random.Random(seed)
    system = [rng.randint(256, vocab - 1) for _ in range(1024)]
    reqs = []
    for _ in range(256):
        n_in, n_out = rng.randint(32, 256), rng.randint(32, 128)
        reqs.append((system + [rng.randint(256, vocab - 1) for _ in range(n_in)], n_out))
    return reqs


def serve(model, reqs, prefix_cache: bool) -> tuple[dict, dict]:
    slots, max_seq = 64, 1024 + 256 + 128 + PAGE
    if model.prefix_cache is not None:
        model.prefix_cache.clear()
    b = ContinuousBatcher(model, None, [p for p, _ in reqs], max_seq_len=max_seq, batch_size=slots, prefill_step=128, verbose=False,
                          device=DEV, max_new_tokens=[n for _, n in reqs], prefix_cache=prefix_cache)
    b.record_timing = True
    popped, first = {}, {}
    before = dict(model.prefix_cache.stats()) if prefix_cache else {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        while not b.idle():
            nxt = b.next_request_idx
            t = time.perf_counter()
            b.step()
            if b.next_request_idx > nxt:
                popped[nxt] = t
            now = time.perf_counter()
            for idx in b.generated:
                first.setdefault(idx, now)
    finally:
        b.release_all()
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    ttft = sorted((first[i] - popped[i]) * 1e3 for i in first)
    pct = lambda q: round(ttft[min(len(ttft) - 1, int(q * len(ttft)))], 1)
    decode_ms = sum(b.gpu_phase_ms()["decode"])
    stats = {k: v - before[k] for k, v in model.prefix_cache.stats().items()} if prefix_cache else {}
    prompt_tokens = sum(len(p) for p, _ in reqs)
    row = {
        "prefix_cache": prefix_cache, "prompt_tokens": prompt_tokens, "prompt_tokens_prefilled": b.prefill_tokens,
        "hit_rate": round(stats.get("hits", 0) / len(reqs), 3), "reused_tokens": b.reused_total,
        "cow_copies": stats.get("cow_copies", 0), "evictions": stats.get("evictions", 0), "wall_s": round(wall, 2),
        "ttft_ms_p50": pct(0.5), "ttft_ms_p99": pct(0.99), "decode_tok_s": round(b.decode_tokens / (decode_ms / 1e3), 1),
        "generated_tokens": sum(b.generated.values()), "output_tok_s": round(sum(b.generated.values()) / wall, 1),
    }
    return row, dict(b.results)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-serving", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "prefix_cache_bench measures on a GPU"
    result = {"card": card(), "cow": cow_bench()}
    print(json.dumps({"card": result["card"], "cow": result["cow"]}), flush=True)
    if not args.skip_serving:
        ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV)
        models = {False: Qwen3ModelWeek3(ns, page_size=PAGE), True: Qwen3ModelWeek3(ns, page_size=PAGE)}
        reqs = build_requests(0, ns.args.vocab_size)
        warm = [(p[:300], 4) for p, _ in reqs[:66]]
        for on, model in models.items():
            model.decode_graph_max_seq_len = 1024 + 256 + 128 + PAGE
            model.prefill_graph_len = 128
            serve(model, warm, on)  # captures the 64-slot decode graph and the 128-row prefill graph, sizes the pools
        runs, outputs = [], {}
        for on in (False, True, False, True):
            row, out = serve(models[on], reqs, on)
            runs.append(row)
            print(json.dumps(row), flush=True)
            outputs.setdefault(on, []).append(out)
        result["serving"] = runs
        result["tokens_identical_on_off"] = all(o == outputs[False][0] for o in outputs[False] + outputs[True])
        result["card_after"] = card()
    print(json.dumps({"tokens_identical_on_off": result.get("tokens_identical_on_off")}), flush=True)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
