"""Workloads for an ncu launch list (per-kernel gpu__time_duration of ONE step, captured graph included):

  ncu --metrics gpu__time_duration.sum --clock-control none --profile-from-start off --csv \
      --log-file tools_out/launches.csv python tools/launch_list.py --mode decode --batch 64 --context 1024
  ... --mode chunk --chunk 128 --context 512      # one chunked-prefill step of the serving loop

The profiler range covers exactly one decode step / one prefill chunk after warm-up.  Times under ncu are serialised
and cold-cache: use the SHARES, not the absolute step time.
"""
from __future__ import annotations

import argparse
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from tiny_llm_b200 import Qwen3ModelWeek3  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine, PrefillEngine  # noqa: E402
from tiny_llm_b200.kv_cache import BatchingKvCache  # noqa: E402
from tiny_llm_b200.paged_kv_cache import TinyKvPagedCache  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=["decode", "chunk"], default="decode")
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--context", type=int, default=1024)
    ap.add_argument("--chunk", type=int, default=128)
    ap.add_argument("--layers", type=int, default=36)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=dev, num_hidden_layers=args.layers)
    model = Qwen3ModelWeek3(ns, page_size=128)
    if args.mode == "decode":
        B = args.batch
        engine = DecodeEngine(model, B, args.context + 256, dev)
        engine.reserve_pools()
        caches = []
        for pool in model.page_pools:
            bc = BatchingKvCache(B, max_seq_len=engine.max_seq_len)
            for b in range(B):
                rc = TinyKvPagedCache(pool)
                for _ in range(args.context):
                    rc.append_token_slot()
                bc.add_request(rc, b)
            caches.append(bc if B > 1 else bc.kv_caches[0])
        toks, offs = [1000 + b for b in range(B)], [args.context] * B
        engine.decode_on_device(toks, offs, caches, 8)
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        engine.decode_on_device(toks, [o + 8 for o in offs], caches, 1)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        print("kernels per step", engine.kernels_per_step)
    else:
        engine = PrefillEngine(model, args.chunk, args.context + 4 * args.chunk, dev)
        engine.reserve_pools(64)
        cache = [TinyKvPagedCache(pool) for pool in model.page_pools]
        ids = list(range(10, 10 + args.chunk))
        offset = 0
        while offset < args.context:  # warm-up chunks build the context
            engine.prefill_chunk(ids, offset, cache)
            offset += args.chunk
        torch.cuda.synchronize()
        torch.cuda.profiler.start()
        engine.prefill_chunk(ids, offset, cache)
        torch.cuda.synchronize()
        torch.cuda.profiler.stop()
        print("kernels per chunk", engine.kernels_per_chunk)


if __name__ == "__main__":
    main()
