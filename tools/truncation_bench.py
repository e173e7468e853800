"""Top-n-sigma, locally typical sampling and Mirostat 2.0 on one GPU (DESIGN.md section 25):

* ``tl_sample_penalized`` (presence penalty 0.5, top-k 50, top-p 0.9) us per call at V = 151,936 bf16 for 1, 8 and
  64 rows, without a truncation sampler and with each of typical (p = 0.9), top-n-sigma (n = 1.5) and Mirostat
  (tau = 5, eta = 0.1, no top-k or top-p: Mirostat replaces them): 50 calls captured in one CUDA graph and replayed 20
  times between CUDA events;
* ``decode_on_device`` tok/s on Qwen3-4B-shaped synthetic weights at B = 1 and 64, context 128: penalised sampling
  against penalised sampling with typical + top-n-sigma on every slot and with Mirostat on every slot, the modes
  alternated over 4 rounds after a capture round.

  python tools/truncation_bench.py [--out tools_out/truncation_bench.json]
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
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
from tiny_llm_b200.sampler import mirostat_start, penalty_tensors, sampling_tensors, truncation_tensors  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
V = 151936
NAMES = ("typical_p", "top_n_sigma", "mirostat_tau", "mirostat_eta")


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


MODES = {
    "penalized": lambda r: SamplingParams(0.8, top_k=50, top_p=0.9, seed=r, presence_penalty=0.5),
    "+typical": lambda r: SamplingParams(0.8, top_k=50, top_p=0.9, seed=r, presence_penalty=0.5, typical_p=0.9),
    "+top_n_sigma": lambda r: SamplingParams(0.8, top_k=50, top_p=0.9, seed=r, presence_penalty=0.5, top_n_sigma=1.5),
    "mirostat": lambda r: SamplingParams(0.8, seed=r, presence_penalty=0.5, mirostat=2, mirostat_tau=5.0, mirostat_eta=0.1),
}


def sample_table() -> dict:
    out = {}
    g = torch.Generator(device=DEV).manual_seed(1)
    for rows in (1, 8, 64):
        logits = (torch.randn(rows, V, generator=g, device=DEV) * 3).to(torch.bfloat16)
        pos = torch.full((rows,), 0, dtype=torch.int32, device=DEV)  # position 0: replays leave the counts and mu alone
        state = torch.zeros((rows, V), dtype=torch.int32, device=DEV)
        for mode, make in MODES.items():
            params = [make(r) for r in range(rows)]
            base, pen = sampling_tensors(params, DEV), penalty_tensors(params, DEV)
            kw = {}
            if mode != "penalized":
                kw = dict(zip(NAMES, truncation_tensors(params, DEV)))
                kw["mirostat_mu"] = torch.tensor([mirostat_start(p) if p.mirostat else 0.0 for p in params], device=DEV)
            us = graph_timed(lambda: ext.sample_penalized(logits, *base, pos, *pen, state, **kw))
            out[f"{mode} rows={rows}"] = us
            print(f"tl_sample_penalized {mode} rows {rows}: {us:.2f} us", flush=True)
    return out


def decode_rates(model, B, ctx=128, steps=64, rounds=4) -> dict:
    modes = {"penalized": MODES["penalized"],
             "typical+top_n_sigma": lambda b: SamplingParams(0.8, top_k=50, top_p=0.9, seed=b, presence_penalty=0.5, typical_p=0.9,
                                                             top_n_sigma=1.5),
             "mirostat": MODES["mirostat"]}
    msl = ctx + len(modes) * (rounds + 2) * steps + 64
    engine = DecodeEngine(model, B, msl, DEV)
    engine.reserve_pools()
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b in range(B):
        cache = model.create_kv_cache()
        for c, t in zip(cache, tables):
            c.append_slots(ctx)
            t.add_request(c, b)
    offsets = [ctx] * B
    times = {m: [] for m in modes}
    hist = [list(range(ctx)) for _ in range(B)]
    for r in range(rounds + 1):
        for mode, make in modes.items():
            params = [make(b) for b in range(B)]
            tokens = [hist[b][-1] for b in range(B)]
            a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = engine.decode_on_device(tokens, offsets, tables, steps, sampling=params,
                                          history=[(hist[b][:-1], [hist[b][-1]]) for b in range(B)])
            e.record()
            e.synchronize()
            for b in range(B):
                hist[b].extend(out[:, b].tolist())
            offsets = [o + steps for o in offsets]
            if r:  # round 0 captures the graphs
                times[mode].append(a.elapsed_time(e))
    res = {m: B * steps * len(v) / (sum(v) / 1e3) for m, v in times.items()}
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
    result = {"gpu": card(), "sample_us": sample_table()}
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV, max_position_embeddings=8192)
    result["decode"] = {B: decode_rates(Qwen3ModelWeek3(ns, page_size=64), B) for B in (1, 64)}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
