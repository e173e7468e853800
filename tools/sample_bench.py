"""Seeded sampling on one GPU (V = 151,936, bf16 logits):

* ``tl_argmax`` against ``tl_sample`` with temperature only, top-k 50, top-p 0.9 and both, and ``make_sampler`` (torch
  ops: sort + cumsum + multinomial) on the same rows, at 1, 8 and 64 rows (CUDA events over 200 launches);
* ``tl_sample_penalized`` (repetition 1.1, presence 0.5, frequency 0.3, with and without min-p 0.05; temperature 0.7,
  top-p 0.9, top-k 50) against ``tl_sample`` with the same top-k / top-p, same rows, random token states;
* ``decode_on_device`` tok/s, greedy against sampled (temperature 0.7, top-p 0.9, top-k 50) and sampled with those
  penalties, at B = 1 and B = 64 on Qwen3-4B-shaped synthetic weights, context 128 + steps, alternated in one process.

  python tools/sample_bench.py [--out tools_out/sample_bench.json] [--kernels-only]
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
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, make_sampler  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
from tiny_llm_b200.sampler import penalty_tensors, sampling_tensors  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
V = 151936
CONFIGS = {"temperature": dict(), "top_k 50": dict(top_k=50), "top_p 0.9": dict(top_p=0.9), "both": dict(top_k=50, top_p=0.9)}
PENALTIES = dict(repetition_penalty=1.1, presence_penalty=0.5, frequency_penalty=0.3)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return f"unknown ({exc})"


def timed(fn, reps=200, warmup=10) -> float:
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e3  # us


def kernel_table() -> dict:
    out = {}
    g = torch.Generator(device=DEV).manual_seed(0)
    for rows in (1, 8, 64):
        logits = (torch.randn(rows, V, generator=g, device=DEV) * 3).to(torch.bfloat16)
        res = {"argmax": timed(lambda: ext.argmax(logits))}
        pos = torch.arange(rows, dtype=torch.int32, device=DEV) + 128
        for name, kw in CONFIGS.items():
            t, k, p, s = sampling_tensors([SamplingParams(0.7, seed=i, **kw) for i in range(rows)], DEV)
            res[f"sample {name}"] = timed(lambda: ext.sample(logits, t, k, p, s, pos))
            sampler = make_sampler(0.7, top_p=kw.get("top_p"), top_k=kw.get("top_k"), generator=torch.Generator(device=DEV).manual_seed(0))
            lp = torch.log_softmax(logits.float(), dim=-1)
            res[f"make_sampler {name}"] = timed(lambda: sampler(lp), reps=50)
        # the penalised kernel on the same rows; positions 0 keep the states as they are across the repetitions
        state = torch.randint(0, 3, (rows, V), generator=g, device=DEV, dtype=torch.int32)
        zero = torch.zeros(rows, dtype=torch.int32, device=DEV)
        for name, kw in (("penalties", PENALTIES), ("penalties + min_p 0.05", dict(PENALTIES, min_p=0.05))):
            params = [SamplingParams(0.7, top_k=50, top_p=0.9, seed=i, **kw) for i in range(rows)]
            t, k, p, s = sampling_tensors(params, DEV)
            pen = penalty_tensors(params, DEV)
            res[f"sample_penalized {name}"] = timed(lambda: ext.sample_penalized(logits, t, k, p, s, zero, *pen, state))
        out[rows] = res
        print(f"rows {rows}: " + ", ".join(f"{k} {v:.1f} us" for k, v in res.items()), flush=True)
    return out


def decode_rates(model, B, ctx=128, steps=64, rounds=3) -> dict:
    msl = ctx + 3 * (rounds + 1) * steps + 64
    engine = DecodeEngine(model, B, msl, DEV)
    engine.reserve_pools()
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b in range(B):
        cache = model.create_kv_cache()
        for c, t in zip(cache, tables):
            c.append_slots(ctx)
            t.add_request(c, b)
    modes = {"greedy": None, "sampled": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1),
             "penalized": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1, **PENALTIES)}
    offsets, tokens = [ctx] * B, [1] * B
    times = {m: [] for m in modes}
    for r in range(rounds + 1):
        for mode, sampling in modes.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            log = engine.decode_on_device(tokens, offsets, tables, steps, sampling=sampling)
            b.record()
            b.synchronize()
            tokens = log[-1].tolist()
            offsets = [o + steps for o in offsets]
            if r:  # round 0 captures the graphs
                times[mode].append(a.elapsed_time(b))
    res = {m: B * steps * len(v) / (sum(v) / 1e3) for m, v in times.items()}
    res["step_ms"] = {m: sum(v) / len(v) / steps for m, v in times.items()}
    res["kernels_per_step"] = {"greedy": engine.kernels_per_step, "sampled": engine.kernels_per_sampled_step,
                               "penalized": engine.kernels_per_penalized_step}
    print(f"B {B}: greedy {res['greedy']:.1f} tok/s, sampled {res['sampled']:.1f} tok/s "
          f"({(res['sampled'] / res['greedy'] - 1) * 100:+.2f} %), penalized {res['penalized']:.1f} tok/s "
          f"({(res['penalized'] / res['sampled'] - 1) * 100:+.2f} % against sampled)", flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--kernels-only", action="store_true", help="the per-call kernel table alone, no decode run")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sample_bench needs a CUDA device")
    result = {"card": card()}
    print(f"card: {result['card']}", flush=True)
    result["kernels_us"] = kernel_table()
    if args.kernels_only:
        print(json.dumps(result))
        return
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV)
    model = Qwen3ModelWeek3(ns, page_size=64)
    result["decode"] = {B: decode_rates(model, B) for B in (1, 64)}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
