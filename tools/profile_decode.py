"""Run a few eager (non-graph) decode steps of the fused path inside an NVTX
range so that ncu can be pointed at exactly the decode kernels:

  ncu --nvtx --nvtx-include "decode/" --metrics gpu__time_duration.sum --clock-control none \
      --csv --log-file tools_out/launches.csv python tools/profile_decode.py --layers 36 --steps 2
"""

from __future__ import annotations

import argparse
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--context", type=int, default=128)
    ap.add_argument("--unfused", action="store_true")
    ap.add_argument("--pdl", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    if args.pdl:
        ext.set_pdl(True)
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=dev, num_hidden_layers=args.layers)
    model = Qwen3ModelWeek3(ns, page_size=128)
    engine = DecodeEngine(model, args.batch, args.context + 256, dev, fused=not args.unfused)
    engine.reserve_pools()
    # pretend `context` tokens are already cached: bookkeeping only (K/V bytes are whatever the slab holds)
    caches = [model.create_kv_cache() for _ in range(args.batch)]
    for cache in caches:
        for layer_cache in cache:
            for _ in range(args.context):
                layer_cache.append_token_slot()
    from tiny_llm_b200 import BatchingKvCache

    if args.batch == 1:
        tables = caches[0]
    else:
        tables = [BatchingKvCache(args.batch, max_seq_len=args.context + 256) for _ in range(model.num_hidden_layers)]
        for slot, cache in enumerate(caches):
            for layer_cache, table in zip(cache, tables):
                table.add_request(layer_cache, slot)
    forward = engine._forward_unfused if args.unfused else engine._forward_fused
    ctx = engine._advance_host(tables, 1)
    B = args.batch
    engine.meta_np[0:B] = 1000
    engine.meta_np[B : 2 * B] = args.context
    engine.meta_np[2 * B : 3 * B] = ctx
    engine._upload()
    for _ in range(2):
        forward()
    torch.cuda.synchronize()
    torch.cuda.nvtx.range_push("decode")
    for _ in range(args.steps):
        forward()
    torch.cuda.synchronize()
    torch.cuda.nvtx.range_pop()
    print("profiled", args.steps, "eager decode steps;", ext.launch_count(), "launches total")


if __name__ == "__main__":
    main()
