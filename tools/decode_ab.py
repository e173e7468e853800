"""A/B timing of the device-resident decode loop (Qwen3-4B shapes, synthetic weights).

  [TL_S5_HALF=0] [TL_S5_GRID=...] python tools/decode_ab.py [--batch 1] [--context 128] [--steps 128] [--tag name]

Launch-geometry switches of the streaming kernel are read once per process, so every variant is
its own process; the script appends one JSON line to tools_out/decode_ab.jsonl.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from tiny_llm_b200 import Qwen3ModelWeek3  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--context", type=int, default=128)
    ap.add_argument("--steps", type=int, default=128)
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--tag", default="")
    ap.add_argument("--max-seq", type=int, default=0, help="engine max_seq_len (default: context + 2 * steps + 80 rounded up to pages)")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=dev, num_hidden_layers=args.layers)
    model = Qwen3ModelWeek3(ns, page_size=128)
    B = args.batch
    engine = DecodeEngine(model, B, args.max_seq or (args.context + 2 * args.steps + 80), dev)
    engine.reserve_pools()
    if B == 1:
        caches = model.create_kv_cache()
        for c in caches:
            for _ in range(args.context):
                c.append_token_slot()
    else:
        from tiny_llm_b200.kv_cache import BatchingKvCache
        from tiny_llm_b200.paged_kv_cache import TinyKvPagedCache

        caches = []
        for pool in model.page_pools:
            bc = BatchingKvCache(B, max_seq_len=engine.max_seq_len)
            for b in range(B):
                rc = TinyKvPagedCache(pool)
                for _ in range(args.context):
                    rc.append_token_slot()
                bc.add_request(rc, b)
            caches.append(bc)
    toks, offs = [1000 + b for b in range(B)], [args.context] * B
    engine.decode_on_device(toks, offs, caches, 16)
    torch.cuda.synchronize()
    best = float("inf")
    offs = [args.context + 16] * B
    for rep in range(2):
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        engine.decode_on_device(toks, offs, caches, args.steps)
        end.record()
        end.synchronize()
        best = min(best, start.elapsed_time(end) / args.steps)
        offs = [o + args.steps for o in offs]
    rec = dict(tag=args.tag, batch=B, context=args.context, steps=args.steps, ms_per_step=round(best, 4),
               tok_s=round(B * 1e3 / best, 1), kernels_per_step=engine.kernels_per_step,
               env={k: v for k, v in os.environ.items() if k.startswith("TL_")})
    print(json.dumps(rec), flush=True)
    out = ROOT / "tools_out"
    out.mkdir(exist_ok=True)
    with open(out / "decode_ab.jsonl", "a") as f:
        f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
