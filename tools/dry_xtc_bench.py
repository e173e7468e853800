"""DRY and XTC on one GPU (DESIGN.md section 24):

* ``tl_dry_penalty`` us per call at histories of 1K, 8K and 32K tokens for 1, 8 and 64 rows, on repetitive (a
  period-7 cycle: every end matches up to the cap) and random histories, V = 151,936: 50 calls captured in one CUDA
  graph and replayed 20 times between CUDA events (each call writes the same history entry again, so replays are
  identical);
* ``tl_sample_penalized`` with and without XTC (q = 1, theta = 0.05, so every row takes the exclusion passes) at
  V = 151,936 bf16 for 1, 8 and 64 rows, timed the same way;
* ``decode_on_device`` tok/s on Qwen3-4B-shaped synthetic weights at B = 1 and 64, context 128: sampled against
  sampled with DRY + XTC on every slot, the two modes alternated over 4 rounds after a capture round.

  python tools/dry_xtc_bench.py [--out tools_out/dry_xtc_bench.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams  # noqa: E402
from tiny_llm_b200.dry import DryRows  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
from tiny_llm_b200.sampler import penalty_tensors, sampling_tensors, xtc_tensors  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
V = 151936


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return f"unknown ({exc})"


def graph_timed(fn, launches=50, reps=20) -> float:
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(launches):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / (reps * launches) * 1e3


def dry_table() -> dict:
    out = {}
    g = torch.Generator().manual_seed(0)
    p = SamplingParams(0.7, dry_multiplier=0.8)
    for n in (1024, 8192, 32768):
        for kind in ("repetitive", "random"):
            for rows in (1, 8, 64):
                tab = DryRows(rows, n, DEV)
                h = ([int(t) for t in torch.randint(0, V, (7,), generator=g)] * (n // 7 + 1))[:n] if kind == "repetitive" else \
                    torch.randint(0, V, (n,), generator=g).tolist()
                for r in range(rows):
                    tab.set_row(r, p, h)
                x = torch.randn(rows, V, device=DEV)
                pos = torch.full((rows,), n, dtype=torch.int32, device=DEV)
                tok = torch.full((rows,), h[-1], dtype=torch.int32, device=DEV)
                us = graph_timed(lambda: ext.dry_penalty(x, tab.table, pos, tok, tab.history, tab.scratch))
                out[f"{kind} n={n} rows={rows}"] = us
                print(f"tl_dry_penalty {kind} history {n} rows {rows}: {us:.2f} us", flush=True)
    return out


def xtc_table() -> dict:
    out = {}
    g = torch.Generator(device=DEV).manual_seed(1)
    for rows in (1, 8, 64):
        logits = (torch.randn(rows, V, generator=g, device=DEV) * 3).to(torch.bfloat16)
        pos = torch.full((rows,), 7, dtype=torch.int32, device=DEV)
        state = torch.zeros((rows, V), dtype=torch.int32, device=DEV)
        for mode in ("penalized", "penalized+xtc"):
            params = [SamplingParams(0.8, top_k=50, top_p=0.9, seed=r, presence_penalty=0.5,
                                     **(dict(xtc_probability=1.0, xtc_threshold=0.05) if mode != "penalized" else {})) for r in range(rows)]
            base, pen = sampling_tensors(params, DEV), penalty_tensors(params, DEV)
            kw = {}
            if mode != "penalized":
                kw = dict(zip(("xtc_threshold", "xtc_probability"), xtc_tensors(params, DEV)))
            us = graph_timed(lambda: ext.sample_penalized(logits, *base, pos, *pen, state, **kw))
            out[f"{mode} rows={rows}"] = us
            print(f"tl_sample_penalized {mode} rows {rows}: {us:.2f} us", flush=True)
    return out


def decode_rates(model, B, ctx=128, steps=64, rounds=4) -> dict:
    modes = ("sampled", "sampled+dry+xtc")
    msl = ctx + len(modes) * (rounds + 2) * steps + 64
    engine = DecodeEngine(model, B, msl, DEV)
    engine.reserve_pools()
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b in range(B):
        cache = model.create_kv_cache()
        for c, t in zip(cache, tables):
            c.append_slots(ctx)
            t.add_request(c, b)
    plain = [SamplingParams(0.7, top_k=50, top_p=0.9, seed=b) for b in range(B)]
    both = [SamplingParams(0.7, top_k=50, top_p=0.9, seed=b, dry_multiplier=0.8, xtc_probability=0.5) for b in range(B)]
    offsets, tokens = [ctx] * B, [1] * B
    times = {m: [] for m in modes}
    hist = [list(range(ctx)) for _ in range(B)]
    for r in range(rounds + 1):
        for mode in modes:
            kw = {"sampling": plain}
            if mode != "sampled":
                kw = {"sampling": both, "history": [(hist[b][:-1], [hist[b][-1]]) for b in range(B)]}
            tokens = [hist[b][-1] for b in range(B)]
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = engine.decode_on_device(tokens, offsets, tables, steps, **kw)
            e.record()
            e.synchronize()
            for b in range(B):
                hist[b].extend(out[:, b].tolist())
            offsets = [o + steps for o in offsets]
            if r:  # round 0 captures the graphs
                times[mode].append(a.elapsed_time(e))
    res = {m: B * steps * len(v) / (sum(v) / 1e3) for m, v in times.items()}
    res["kernels_per_step"] = {"sampled": engine.kernels_per_sampled_step, "sampled+dry+xtc": engine.kernels_per_controlled_step}
    for t in tables:
        for c in t.kv_caches:
            if c is not None:
                c.release()
        t.kv_caches = [None] * t.max_active_requests
    print(f"B {B}: " + ", ".join(f"{m} {res[m]:.1f} tok/s" for m in modes), flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print(card(), flush=True)
    result = {"gpu": card(), "dry_us": dry_table(), "sample_us": xtc_table()}
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV, max_position_embeddings=8192)
    result["decode"] = {B: decode_rates(Qwen3ModelWeek3(ns, page_size=64), B) for B in (1, 64)}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
