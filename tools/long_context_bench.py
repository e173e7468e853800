"""Long context on one GPU (DESIGN.md "Long context"), Qwen3-4B-shaped synthetic W4A16 weights with the YaRN
configuration of Qwen3's 131,072-token window:

* decode attention per layer alone (32 query heads, 8 KV heads, head dim 128, 128-token pages, bf16) at 8K / 32K / 64K /
  128K, on the path the decode engine picks for that window (fused up to 16,384 slot-tokens, q/k norm + RoPE + append
  and the paged attention kernel beyond), CUDA events over 200 graph-captured calls, beside the reference's published
  M4 Pro figures.  The calls re-read the same pages: the 8K row's 33.5 MB fit the 50 MB L2, so it is a warm-cache figure;
  from 32K on the pages exceed L2;
* the whole model (``--layers``, default 36) at 32K and 128K: the prompt prefilled in one call (the model runs prompts
  past 32,768 tokens as 8,192-token pieces), then the B = 1 decode step as graph replays (CUDA events around 15 steps);
* the same prompt at 32K as 128-token chunks through the chunk graph, with the split of the prefix's key range on and
  forced off (the script drops the engine's split workspace before the first capture).

The card's name and power limit are read in the same run.

  python tools/long_context_bench.py [--layers 36] [--out tools_out/long_context_bench.json]
"""

from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200"), str(ROOT / "tools")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from spec_bench import card, graphed, timed  # noqa: E402
from tiny_llm_b200.engine import FUSED_ATTENTION_MAX_SLOT_TOKENS  # noqa: E402
from tiny_llm_b200.rope_scaling import parse_rope_scaling, rope_inv_freq  # noqa: E402

DEV = torch.device("cuda:0")
HQ, HKV, D, PAGE = 32, 8, 128, 128
YARN = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}
REFERENCE_MS = {2048: 0.142, 8192: 0.287, 32768: 0.917, 65536: 1.728, 131072: 3.651}  # benches/bench_long_context_attention.py, M4 Pro
REPS = 200


def attention_ms(ctx: int, table: torch.Tensor) -> dict:
    pages = -(-ctx // PAGE)
    need = 2 * pages * HKV * PAGE * D * 2
    if need > 0.5 * torch.cuda.mem_get_info(DEV)[0]:
        return {"context": ctx, "skipped": f"{need} bytes of pages do not fit"}
    g = torch.Generator(device=DEV).manual_seed(ctx)
    kp = torch.randn(pages, HKV, PAGE, D, device=DEV, generator=g).to(torch.bfloat16)
    vp = torch.randn(pages, HKV, PAGE, D, device=DEV, generator=g).to(torch.bfloat16)
    qkv = torch.randn(1, (HQ + 2 * HKV) * D, device=DEV, generator=g).to(torch.bfloat16)
    qw = torch.ones(D, dtype=torch.bfloat16, device=DEV)
    table_row = torch.arange(pages, dtype=torch.int32, device=DEV).view(1, pages)
    off = torch.tensor([ctx - 1], dtype=torch.int32, device=DEV)
    cl = torch.tensor([ctx], dtype=torch.int32, device=DEV)
    scale = D**-0.5 * parse_rope_scaling(YARN, 40960).mscale ** 2
    fused = ctx <= FUSED_ATTENTION_MAX_SLOT_TOKENS
    if fused:
        ws = torch.empty(ext.decode_attention_fused_workspace(1, HQ, HKV), dtype=torch.float32, device=DEV)
        out = torch.empty(1, HQ * D, dtype=torch.bfloat16, device=DEV)

        def call():
            ext.decode_attention_fused(qkv, qw, qw, off, table_row, cl, table, kp, vp, HQ, HKV, 1e-6, scale, ctx, out=out, workspace=ws)
    else:
        def call():
            q = ext.decode_qk_norm_rope_append(qkv, qw, qw, off, table_row, cl, kp, vp, HQ, HKV, 1e6, 1e-6, inv_freq=table)
            ext.paged_attention(q.view(HQ, 1, D), kp, vp, table_row, cl, scale, is_causal=True, num_kv_heads=HKV, num_heads=HQ)

    replay = graphed(call, REPS)
    ms = timed(replay, reps=5, warmup=2) / REPS
    row = {"context": ctx, "path": "fused" if fused else "qk_norm_rope_append + paged_attention", "ms_per_layer": round(ms, 4)}
    if ctx in REFERENCE_MS:
        row["reference_m4_pro_ms"] = REFERENCE_MS[ctx]
    del kp, vp
    torch.cuda.empty_cache()
    return row


def _model(layers: int, window: int):
    from tiny_llm_b200 import Qwen3ModelWeek3
    from tiny_llm_b200.synthetic import synthetic_qwen3

    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV, num_hidden_layers=layers, rope_scaling=YARN)
    return Qwen3ModelWeek3(ns, page_size=PAGE, max_context=window)


def _ids(n: int) -> torch.Tensor:
    return torch.randint(1, 151936, (1, n), generator=torch.Generator().manual_seed(n)).to(torch.int32).to(DEV)


def _ms(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def model_rows(layers: int) -> list:
    rows = []
    for ctx in (32768, 131072):
        model = _model(layers, ctx)
        try:
            model.decode_engine(1)  # reserves the window's pages (refused here if they do not fit)
        except MemoryError as exc:
            rows.append({"context": ctx, "layers": layers, "skipped": str(exc)})
            continue
        ids = _ids(ctx - 21)
        cache = model.create_kv_cache()
        out = {}
        prefill_ms = _ms(lambda: out.setdefault("logits", model(ids, 0, cache, logits_to_keep=1)))
        tok = torch.tensor([[int(out["logits"][0, -1].argmax())]], dtype=torch.int32, device=DEV)
        off = ctx - 21
        for _ in range(3):  # warm: capture and first replays
            model(tok, off, cache)
            off += 1
        steps = 15

        def decode():
            nonlocal off
            for _ in range(steps):
                model(tok, off, cache)
                off += 1

        step_ms = _ms(decode) / steps
        rows.append({"context": ctx, "layers": layers, "prefill_one_call_ms": round(prefill_ms, 1), "prompt_tokens": ctx - 21,
                     "decode_step_ms": round(step_ms, 3)})
        for c in cache:
            c.release()
        del model, cache
        torch.cuda.empty_cache()
    return rows


def chunked_rows(layers: int, ctx: int = 32768) -> list:
    rows = []
    for split in (True, False):
        model = _model(layers, ctx)
        model.decode_engine(1)
        model.prefill_graph_len = 128
        engine = model.prefill_engine(128)
        if not split:
            engine._attn_ws = None  # before the first capture: the unsplit chunk attention
        ids = _ids(ctx - 128)
        cache = model.create_kv_cache()

        def run():
            for s0 in range(0, ids.shape[1], 128):
                model(ids[:, s0:s0 + 128], s0, cache, logits_to_keep=1)

        ms = _ms(run)
        rows.append({"context": ctx, "layers": layers, "chunk": 128, "split": split and engine._attn_ws is not None,
                     "prefill_chunked_ms": round(ms, 1), "chunk_graph_replays": engine.replays})
        for c in cache:
            c.release()
        del model, cache, engine
        torch.cuda.empty_cache()
    return rows


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--contexts", default="8192,32768,65536,131072")
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("long_context_bench needs a GPU")
    table = rope_inv_freq(D, 1e6, parse_rope_scaling(YARN, 40960), DEV)
    result = {"card": card(), "attention_per_layer": [attention_ms(int(c), table) for c in args.contexts.split(",")]}
    result["model"] = model_rows(args.layers)
    result["chunked_prefill"] = chunked_rows(args.layers)
    print(json.dumps(result, indent=1))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
