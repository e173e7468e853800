"""Multi-LoRA serving on the GPU (DESIGN.md section 12), CUDA events over graph replays, variants alternated in one process:

* ``tl_lora_apply`` alone per site at Qwen3-4B shapes, ranks 8 / 16 / 64, rows 1 / 8 / 64 / 1024: microseconds per launch
  and achieved bytes/s against the algorithmic bytes (x, A and B of the one adapter read once, y read and written once);
* ``decode_on_device`` at B = 1, 8, 64 on Qwen3-4B-shaped synthetic weights: a model without adapters, a LoRA engine with
  every slot at -1, with every slot on one rank-16 adapter, and with four adapters mixed;
* a 4,096-token prefill in 512-token chunk graphs, without adapters, on a LoRA engine at -1 and under an adapter.

It prints the card, its power limit and its clocks as it finds them and changes nothing.

    python tools/lora_bench.py [--shape qwen3-4b] [--skip-model]
"""

from __future__ import annotations

import argparse
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
for extra in (ROOT, ROOT / "tiny-llm_b200"):
    if str(extra) not in sys.path:
        sys.path.insert(0, str(extra))

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3  # noqa: E402
from tiny_llm_b200.kv_cache import BatchingKvCache  # noqa: E402
from tiny_llm_b200.lora import LoraAdapter, projection_shapes  # noqa: E402
from tiny_llm_b200.synthetic import make_args, synthetic_qwen3  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError as exc:
        return f"nvidia-smi unavailable: {exc}"


def timed(fn, reps: int) -> float:
    """Milliseconds per call of ``fn`` over ``reps`` calls between two CUDA events."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps


def site_bytes(M: int, N: int, Ks, rank: int) -> int:
    ktot = sum(Ks)
    return 2 * (M * N + 2 * M * ktot + len(Ks) * rank * N + ktot * rank)


def kernel_table(args, dev) -> None:
    shapes = projection_shapes(args)
    sites = {"q|k|v": ("q", "k", "v"), "o": ("o",), "gate|up": ("gate", "up"), "down": ("down",)}
    gen = torch.Generator().manual_seed(0)
    print("\n| site | rank | rows | us / launch | GB/s (algorithmic bytes) |\n|---|---|---|---|---|")
    for name, projs in sites.items():
        N, Ks = shapes[projs[0]][1], [shapes[p][0] for p in projs]
        for rank in (8, 16, 64):
            A = (torch.randn(1, len(Ks) * rank, N, generator=gen) * N**-0.5).to(torch.bfloat16).to(dev)
            Bs = [(torch.randn(1, K, rank, generator=gen) * 0.02).to(torch.bfloat16).to(dev) for K in Ks]
            site = ext.LoraSite(A, Bs, torch.full((1,), 1e-3, device=dev), torch.tensor([rank], dtype=torch.int32, device=dev),
                                torch.tensor([(1 << len(Ks)) - 1], dtype=torch.int32, device=dev))
            for M in (1, 8, 64, 1024):
                x = torch.randn(M, N, generator=gen).to(torch.bfloat16).to(dev)
                y = torch.zeros(M, sum(Ks), dtype=torch.bfloat16, device=dev)
                ids = torch.zeros(M, dtype=torch.int32, device=dev)
                stream = torch.cuda.Stream()
                inner = 20
                with torch.cuda.stream(stream):
                    ext.lora_apply(x, y, ids, site)
                    stream.synchronize()
                    graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(graph, stream=stream):
                        for _ in range(inner):
                            ext.lora_apply(x, y, ids, site)
                    graph.replay()
                    us = timed(graph.replay, 10) / inner * 1e3
                    stream.synchronize()
                print(f"| {name} | {rank} | {M} | {us:.2f} | {site_bytes(M, N, Ks, rank) / us / 1e3:.0f} |")


def slots(model, B: int, dev, prompt_len: int, max_seq_len: int, adapter_ids):
    """``B`` requests prefilled with ``prompt_len`` random tokens each, in a slot table: (table, tokens, offsets)."""
    gen = torch.Generator().manual_seed(B)
    table = [BatchingKvCache(max_active_requests=B, max_seq_len=max_seq_len) for _ in range(model.num_hidden_layers)]
    tokens = []
    for b in range(B):
        cache = model.create_kv_cache()
        prompt = torch.randint(1, 1000, (1, prompt_len), generator=gen).to(torch.int32).to(dev)
        kw = {} if model.adapters is None else {"adapter_ids": [adapter_ids[b]]}
        logits = model(prompt, 0, cache, logits_to_keep=1, **kw)
        tokens.append(int(torch.argmax(logits[0, -1].float())))
        for layer_cache, t in zip(cache, table):
            t.add_request(layer_cache, b)
    return table, tokens, [prompt_len] * B


def decode_table(ns, dev, steps: int = 32, rounds: int = 3) -> None:
    adapters = [LoraAdapter.synthetic(ns.args, 16, seed=i, name=f"a{i}") for i in range(4)]
    plain = Qwen3ModelWeek3(ns, page_size=128)
    lora = Qwen3ModelWeek3(ns, page_size=128)
    lora.load_adapters(adapters)
    print("\n| B | mode | launches / step | ms / step | tok/s |\n|---|---|---|---|---|")
    for B in (1, 8, 64):
        modes = {"no adapters loaded": (plain, None), "LoRA engine, every slot -1": (lora, [-1] * B),
                 "LoRA engine, every slot on one rank-16 adapter": (lora, [0] * B),
                 "LoRA engine, four rank-16 adapters mixed": (lora, [b % 4 for b in range(B)])}
        state = {}
        for name, (model, ids) in modes.items():
            engine = model.decode_engine(B, 1024)
            table, tokens, offsets = slots(model, B, dev, 128, 1024, ids or [-1] * B)
            state[name] = [engine, table, tokens, offsets, ids, []]
        for _ in range(rounds + 1):  # the first round warms up: captures, lazy attributes
            for name, (engine, table, tokens, offsets, ids, times) in state.items():
                kw = {} if ids is None else {"adapter_ids": ids}
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                out = engine.decode_on_device(tokens, offsets, table, steps, **kw)
                end.record()
                end.synchronize()
                times.append(start.elapsed_time(end) / steps)
                state[name][2] = out[-1].tolist()
                state[name][3] = [o + steps for o in offsets]
        for name, (engine, table, _, _, _, times) in state.items():
            ms = sorted(times[1:])[len(times[1:]) // 2]
            print(f"| {B} | {name} | {engine.kernels_per_step} | {ms:.3f} | {B / ms * 1e3:.0f} |")
            for t in table:
                for b in range(B):
                    cache = t.kv_caches[b]
                    t.remove_request(b)
                    cache.release()


def prefill_table(ns, dev, tokens: int = 4096, chunk: int = 512, rounds: int = 2) -> None:
    gen = torch.Generator().manual_seed(1)
    prompt = torch.randint(1, 1000, (1, tokens), generator=gen).to(torch.int32).to(dev)
    plain = Qwen3ModelWeek3(ns, page_size=128)
    lora = Qwen3ModelWeek3(ns, page_size=128)
    lora.load_adapters([LoraAdapter.synthetic(ns.args, 16, seed=0, name="a0")])
    for model in (plain, lora):
        model.prefill_graph_len = chunk
        model.decode_engine(1, 8192)  # reserves the page slabs the chunk graph runs over
    modes = {"no adapters loaded": (plain, None), "LoRA engine, id -1": (lora, [-1]), "LoRA engine, rank-16 adapter": (lora, [0])}
    times = {name: [] for name in modes}
    for _ in range(rounds + 1):
        for name, (model, ids) in modes.items():
            kw = {} if ids is None else {"adapter_ids": ids}
            cache = model.create_kv_cache()
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for off in range(0, tokens, chunk):
                model(prompt[:, off:off + chunk], off, cache, logits_to_keep=1, **kw)
            end.record()
            end.synchronize()
            times[name].append(start.elapsed_time(end))
            for c in cache:
                c.release()
    print(f"\n| {tokens}-token prefill, {chunk}-token chunk graphs | launches / chunk | ms | tok/s |\n|---|---|---|---|")
    for name, (model, _) in modes.items():
        ms = min(times[name][1:])
        print(f"| {name} | {model.prefill_engine(chunk).kernels_per_chunk} | {ms:.1f} | {tokens / ms * 1e3:.0f} |")


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="qwen3-4b")
    ap.add_argument("--skip-model", action="store_true", help="only the kernel table")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_bench needs a CUDA device: there is no CPU timing")
    dev = torch.device("cuda:0")
    print(f"card: {card()}")
    kernel_table(make_args(args.shape), dev)
    if not args.skip_model:
        ns = synthetic_qwen3(args.shape, seed=0, device=dev, max_position_embeddings=8192)
        decode_table(ns, dev)
        prefill_table(ns, dev)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
