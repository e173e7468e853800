"""Embedding throughput: packed ``embed_ids`` passes against one prompt at a time through the chunked-prefill graph.

Workloads: Qwen3-0.6B- and Qwen3-4B-shaped synthetic models, prompts with lengths drawn (seeded) from U[16, 128]
(queries) and U[128, 1024] (passages).  Compared:
  * ``embed_ids`` at ``max_tokens`` 2048 and 8192 over all ``--prompts`` prompts;
  * the nearest path that existed before it: each prompt alone through the B = 1 ``PrefillEngine`` at chunk 128
    (``prefill_chunk`` per 128 tokens, which also runs the LM head on the last row), over the first
    ``--baseline-prompts`` prompts (a rate: tokens/s does not depend on how many prompts are timed).
Tokens/s counts prompt tokens (not padding) over CUDA-event time.  A separate profiled pass gives the time of the
segment-causal attention and ``tl_embed_pool`` kernels per pass.  The card's name and power limit are read in the
same run.  Writes one JSON line per row to stdout and to ``--out``.

    python tools/embed_bench.py [--models qwen3-0.6b,qwen3-4b] [--prompts 4096] [--baseline-prompts 256] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200"), str(ROOT / "tools")]

from spec_bench import card  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3, embed_ids  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
RANGES = {"short": (16, 128), "long": (128, 1024)}


def prompts_of(model, lo, hi, n, seed):
    g = np.random.default_rng(seed)
    lengths = g.integers(lo, hi + 1, size=n)
    return [g.integers(0, model.vocab_size, size=int(L)).tolist() for L in lengths]


def events_time(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def packed(model, prompts, max_tokens) -> float:
    embed_ids(model, prompts[:64], max_tokens=max_tokens)  # warm-up: slabs, modules, tensor maps
    return events_time(lambda: embed_ids(model, prompts, max_tokens=max_tokens))


def one_at_a_time(model, prompts, chunk=128) -> float:
    longest = max(len(p) for p in prompts)
    engine = model.prefill_engine(chunk, max_seq_len=-(-longest // chunk) * chunk)
    engine.reserve_pools(engine.max_pages + 1)

    def run(batch):
        for p in batch:
            cache = model.create_kv_cache()
            for a in range(0, len(p), chunk):
                engine.prefill_chunk(p[a:a + chunk], a, cache)
            for c in cache:
                c.release()

    run(prompts[:8])
    return events_time(lambda: run(prompts))


def kernel_times(model, prompts, max_tokens) -> dict:
    """Mean device time per pass of the segment attention (summed over layers) and of the pooling kernel."""
    from torch.profiler import ProfilerActivity, profile

    sel = prompts[:256]
    embed_ids(model, sel, max_tokens=max_tokens)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        embed_ids(model, sel, max_tokens=max_tokens)
        torch.cuda.synchronize()
    attn = pool = 0.0
    n_attn = n_pool = 0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        name = e.name
        if "paged_prefill_tc_kernel<3" in name or ("paged_prefill_tc_kernel" in name and "Li3E" in name):
            attn += e.device_time
            n_attn += 1
        elif "embed_pool_kernel" in name:
            pool += e.device_time
            n_pool += 1
    passes = max(n_pool, 1)
    return {"passes": n_pool, "attention_ms_per_pass": attn / passes / 1e3, "attention_launches": n_attn,
            "pool_ms_per_pass": pool / passes / 1e3}


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="qwen3-0.6b,qwen3-4b")
    ap.add_argument("--prompts", type=int, default=4096)
    ap.add_argument("--baseline-prompts", type=int, default=256)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("embed_bench needs a CUDA device")
    out = Path(args.out) if args.out else None
    if out is not None:
        out.parent.mkdir(parents=True, exist_ok=True)
        out.write_text("")

    def emit(row):
        row["gpu"] = gpu
        print(json.dumps(row), flush=True)
        if out is not None:
            with out.open("a") as f:
                f.write(json.dumps(row) + "\n")

    gpu = card()
    for name in args.models.split(","):
        model = Qwen3ModelWeek3(synthetic_qwen3(name, seed=0, device=DEV), page_size=128)
        for label, (lo, hi) in RANGES.items():
            prompts = prompts_of(model, lo, hi, args.prompts, args.seed)
            tokens = sum(len(p) for p in prompts)
            for max_tokens in (2048, 8192):
                t = packed(model, prompts, max_tokens)
                emit({"model": name, "lengths": f"U[{lo},{hi}]", "path": f"embed_ids max_tokens={max_tokens}", "prompts": len(prompts),
                      "tokens": tokens, "seconds": round(t, 4), "tokens_per_s": round(tokens / t)})
                emit({"model": name, "lengths": f"U[{lo},{hi}]", "path": f"kernels max_tokens={max_tokens}",
                      **{k: round(v, 4) if isinstance(v, float) else v for k, v in kernel_times(model, prompts, max_tokens).items()}})
            base = prompts[:args.baseline_prompts]
            btok = sum(len(p) for p in base)
            t = one_at_a_time(model, base)
            emit({"model": name, "lengths": f"U[{lo},{hi}]", "path": "PrefillEngine chunk=128, one prompt at a time", "prompts": len(base),
                  "tokens": btok, "seconds": round(t, 4), "tokens_per_s": round(btok / t)})
        del model
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
