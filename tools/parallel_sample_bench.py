"""Parallel sampling on one GPU (DESIGN.md section 16), on the Qwen3-4B-shaped synthetic model (``--layers``, default
36), for n = 1 / 2 / 4 / 8 / 16 samples of prompts of 256 / 1,024 / 4,096 / 8,192 tokens:

* attention alone, one layer: ``tl_shared_prefix_attention`` over one group of n slots (prefix pass, suffix pass and
  merge together) against ``tl_paged_attention`` on the same n full tables, CUDA events over 50 launches captured in
  one graph, with block tables as wide as the context ("tight") and as wide as the engine's graph window ("window",
  what the decode step passes); the algorithmic K/V bytes each way and the achieved bandwidth;
* the same launches per kernel (prefix pass, suffix pass, merge; the plain kernels they replace), from
  ``torch.profiler`` over 20 eager calls after the timed loops, at the window width, with programmatic dependent
  launch off so that the durations do not overlap;
* the decode step: ``decode_on_device`` over n forks of the prompt, grouped (the rule forced on) and ungrouped,
  alternated three times each in one process, CUDA events around ``--steps`` steps (min and max of the three);
* the same step for 4 prompts of n samples each (B = 4n, four groups);
* end to end: ``parallel_sample_ids`` (its own rule) against n sequential ``greedy_generate_ids(sampling=...)``
  calls, ``--tokens`` new tokens each with no EOS, host clock around each call (both end in a device read).

The card's name and power limit are read in the same run.

  python tools/parallel_sample_bench.py [--layers 36] [--steps 32] [--tokens 32] [--out tools_out/parallel_sample_bench.json]
"""

from __future__ import annotations

import argparse
import gc
import json
import sys
import time
from dataclasses import replace
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200"), str(ROOT / "tools")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from spec_bench import card, graphed  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, greedy_generate_ids, parallel_sample_ids  # noqa: E402
from tiny_llm_b200 import engine as eng  # noqa: E402
from tiny_llm_b200 import generate as gen  # noqa: E402
from tiny_llm_b200 import paged_kv_cache as pkv  # noqa: E402
from tiny_llm_b200.kv_cache import BatchingKvCache  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
SAMPLES = (1, 2, 4, 8, 16)
PROMPTS = (256, 1024, 4096, 8192)
HQ, HKV, D = 32, 8, 128
KV_BYTES_PER_TOKEN = HKV * D * 2 * 2  # K and V, bf16, one layer


def _events(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def kernel_us(fn, reps: int = 20) -> dict:
    """Device microseconds per call of each kernel ``fn`` launches, from ``torch.profiler`` over ``reps`` eager calls.
    Programmatic dependent launch is off meanwhile: with it, a dependent kernel starts early and its duration includes
    the wait for its predecessor, so the durations would overlap."""
    ext.set_pdl(False)
    try:
        fn()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                fn()
            torch.cuda.synchronize()
    finally:
        ext.set_pdl(True)
    out = {}
    for evt in prof.key_averages():
        t = getattr(evt, "device_time_total", None)
        if t is None:
            t = evt.cuda_time_total
        if t > 0 and "Memset" not in evt.key and "Memcpy" not in evt.key:
            out[evt.key[:60]] = round(t / reps, 2)
    return out


def attention_case(n: int, prompt: int, page: int, window: int, private: int = 16, reps: int = 50) -> dict:
    """One layer's decode attention for n forks of a prompt of ``prompt`` tokens, ``private`` tokens past it each, with
    tables as wide as the context and as wide as ``window`` tokens."""
    row = {}
    for width, max_pages in (("tight", -(-(prompt + private + 64) // page)), ("window", -(-window // page))):
        row.update({f"{k}_{width}": v for k, v in _attention(n, prompt, page, max_pages, private, reps, width == "window").items()})
    return row


def _attention(n, prompt, page, max_pages, private, reps, per_kernel):
    shared = prompt // page
    ctx = prompt + private
    own = -(-ctx // page) - shared
    P = shared + n * own + 1
    tables = torch.full((n, max_pages), -1, dtype=torch.int32)
    for b in range(n):
        tables[b, :shared] = torch.arange(shared)
        tables[b, shared : shared + own] = torch.arange(shared + b * own, shared + (b + 1) * own)
    tables, lens = tables.to(DEV), torch.full((n,), ctx, dtype=torch.int32, device=DEV)
    q = torch.randn(n * HQ, 1, D, device=DEV).to(torch.bfloat16)
    kp = torch.randn(P, HKV, page, D, device=DEV).to(torch.bfloat16)
    vp = torch.randn(P, HKV, page, D, device=DEV).to(torch.bfloat16)
    groups_host = torch.tensor([[0, n, shared]], dtype=torch.int32)
    groups = groups_host.to(DEV)
    ws = torch.empty(ext.shared_prefix_attention_workspace(n, HQ, HKV, page, max_pages), dtype=torch.uint8, device=DEV)
    scale = D ** -0.5
    plain = graphed(lambda: ext.paged_attention(q, kp, vp, tables, lens, scale, is_causal=True, num_kv_heads=HKV, num_heads=HQ), reps)
    grouped = graphed(lambda: ext.shared_prefix_attention(q, kp, vp, tables, lens, groups, groups_host, scale, HKV, HQ, workspace=ws), reps)
    times = {"plain": [], "grouped": []}
    for _ in range(3):  # alternated
        times["plain"].append(_events(plain) * 1e3 / reps)
        times["grouped"].append(_events(grouped) * 1e3 / reps)
    t_plain, t_grp = min(times["plain"]), min(times["grouped"])
    bytes_plain = n * ctx * KV_BYTES_PER_TOKEN
    bytes_grp = (shared * page + n * (ctx - shared * page)) * KV_BYTES_PER_TOKEN
    out = {"attention_us_plain": round(t_plain, 2), "attention_us_grouped": round(t_grp, 2),
           "kv_bytes_plain": bytes_plain, "kv_bytes_grouped": bytes_grp,
           "gbps_plain": round(bytes_plain / t_plain / 1e3, 1), "gbps_grouped": round(bytes_grp / t_grp / 1e3, 1)}
    if per_kernel:
        out["kernels_plain"] = kernel_us(lambda: ext.paged_attention(q, kp, vp, tables, lens, scale, is_causal=True, num_kv_heads=HKV, num_heads=HQ))
        out["kernels_grouped"] = kernel_us(lambda: ext.shared_prefix_attention(q, kp, vp, tables, lens, groups, groups_host, scale, HKV, HQ,
                                                                               workspace=ws))
    return out


def step_case(model, n: int, prompt_ids: list, steps: int, prompts: int = 1) -> dict:
    """ms per decode step over n forks of each of ``prompts`` copies of the prompt, grouped (rule forced on) and
    ungrouped, alternated three times each: (min, max)."""
    B = prompts * n
    engine = model.decode_engine(B, model.decode_graph_max_seq_len)
    sampling = [SamplingParams(1.0, seed=j) for j in range(B)]
    out = {}
    saved = (eng.SHARED_PREFIX_MIN_COUNT, eng.SHARED_PREFIX_MIN_TOKENS)
    eng.SHARED_PREFIX_MIN_COUNT, eng.SHARED_PREFIX_MIN_TOKENS = 1, 1
    try:
        for grouped in (False, True) * 3:
            caches = []
            for _ in range(prompts):
                cache = model.create_kv_cache()
                model(torch.as_tensor(prompt_ids, dtype=torch.int32, device=DEV)[None], 0, cache, logits_to_keep=1)
                caches += [cache] + (pkv.fork([(cache, n - 1)])[0] if n > 1 else [])
            slots = [BatchingKvCache(B) for _ in range(len(caches[0]))]
            for layer, s in enumerate(slots):
                s.kv_caches = [c[layer] for c in caches]
            groups = [(i * n, n) for i in range(prompts)] if grouped else None
            offsets = [len(prompt_ids)] * B
            engine.decode_on_device([1] * B, offsets, slots, 2, sampling=sampling, groups=groups)  # warm / capture
            offsets = [o + 2 for o in offsets]
            ms = _events(lambda: engine.decode_on_device([1] * B, offsets, slots, steps, sampling=sampling, groups=groups)) / steps
            out.setdefault("grouped" if grouped else "plain", []).append(ms)
            for c in caches:
                gen._release_kv_cache(c)
    finally:
        eng.SHARED_PREFIX_MIN_COUNT, eng.SHARED_PREFIX_MIN_TOKENS = saved
    return {"step_ms_plain": [round(min(out["plain"]), 3), round(max(out["plain"]), 3)],
            "step_ms_grouped": [round(min(out["grouped"]), 3), round(max(out["grouped"]), 3)]}


def end_to_end(model, n: int, prompt_ids: list, tokens: int) -> dict:
    s = SamplingParams(1.0, seed=3)
    parallel_sample_ids(model, [prompt_ids], n, s, 2, device=DEV)  # warm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = parallel_sample_ids(model, [prompt_ids], n, s, tokens, device=DEV)
    t_par = time.perf_counter() - t0
    t0 = time.perf_counter()
    for j in range(n):
        greedy_generate_ids(model, prompt_ids, tokens, sampling=replace(s, seed=gen.sample_seed(3, j)), device=DEV)
    torch.cuda.synchronize()
    t_seq = time.perf_counter() - t0
    made = sum(len(x.ids) for x in got[0])
    return {"tok_s_parallel": round(made / t_par, 1), "tok_s_sequential": round(n * tokens / t_seq, 1)}


def main(argv=None) -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--steps", type=int, default=32)
    ap.add_argument("--tokens", type=int, default=32)
    ap.add_argument("--samples", default=",".join(map(str, SAMPLES)))
    ap.add_argument("--prompts", default=",".join(map(str, PROMPTS)))
    ap.add_argument("--out", default=None)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("parallel_sample_bench needs a CUDA device")
    ns = synthetic_qwen3("qwen3-4b", device=DEV, seed=1, num_hidden_layers=args.layers)
    model = Qwen3ModelWeek3(ns)
    model.set_max_context(max(int(p) for p in args.prompts.split(",")) + args.steps + args.tokens + 256)
    rows = []
    result = {"card": card(), "layers": args.layers, "page_size": model.page_size, "rows": rows}
    for prompt in (int(p) for p in args.prompts.split(",")):
        ids = torch.randint(0, 4096, (prompt,), generator=torch.Generator().manual_seed(prompt)).tolist()
        for n in (int(x) for x in args.samples.split(",")):
            row = {"n": n, "prompt": prompt, **attention_case(n, prompt, model.page_size, model.decode_graph_max_seq_len)}
            row.update(step_case(model, n, ids, args.steps))
            row.update(end_to_end(model, n, ids, args.tokens))
            row["rule"] = eng.shared_prefix_attention_applies(n, prompt // model.page_size * model.page_size, model)
            rows.append(row)
            print(json.dumps(row), flush=True)
    multi = []
    result["four_prompts"] = multi
    del model  # the four-prompt engines (B up to 64) need the memory of the first model's page slabs
    gc.collect()
    torch.cuda.empty_cache()
    model = Qwen3ModelWeek3(ns)
    model.set_max_context(4096 + args.steps + 256, batch_size=64)
    for prompt, n in ((1024, 2), (4096, 8), (4096, 16)):
        ids = torch.randint(0, 4096, (prompt,), generator=torch.Generator().manual_seed(prompt)).tolist()
        row = {"prompts": 4, "n": n, "prompt": prompt, **step_case(model, n, ids, args.steps, prompts=4)}
        multi.append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": result["card"], "layers": args.layers, "page_size": model.page_size}))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
