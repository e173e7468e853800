"""Reranking throughput: ``rerank_ids`` with shared query prefixes against the same pairs with the prefix repeated per
document, and against one pair at a time through the chunked-prefill graph.

Workloads: Qwen3-0.6B- and Qwen3-4B-shaped synthetic models; Q queries x n documents with n in {8, 64}, a shared
prefix of P in {64, 512} tokens and document lengths drawn (seeded) from U[64, 512]; Q is chosen so that every
workload holds ``--docs`` documents.  Compared, (a) and (b) alternating in one process over ``--rounds`` rounds:
  (a) ``rerank_ids`` with one group per query: the prefix is laid out once per pass that takes its documents;
  (b) the same pairs with every document as its own one-document group: the prefix is repeated per document;
  (c) the nearest path that existed before: each whole prompt (prefix + document) alone through the B = 1
      ``PrefillEngine`` at chunk 128, reading the last row's logits, over the first ``--baseline-docs`` pairs.
Documents/s is over CUDA-event time; rows report the median round.  The prompt tokens sharing saves, (n - 1) * P per
query before alignment, are counted on the host.

A separate ``torch.profiler`` run gives, per pass of (a), the device time of the prefixed-segment attention (summed
over layers) and of ``tl_select_logits``.  A kernel-level probe then times one attention launch over an 8,192-row
pass holding a 512-token prefix and as many documents of 288 tokens (the mean of U[64, 512]) as fit, with only the
first or only the last document live (every other row padding): with the tile skip both cost the same; without it the
last document would walk all its siblings' tiles.  The card's name and power limit are read in the same run.  Writes
one JSON line per row to stdout and to ``--out``.

    python tools/rerank_bench.py [--models qwen3-0.6b,qwen3-4b] [--docs 512] [--baseline-docs 64] [--rounds 3] [--out FILE]
"""

from __future__ import annotations

import argparse
import json
import statistics
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200"), str(ROOT / "tools")]

from spec_bench import card  # noqa: E402
from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3, rerank_ids  # noqa: E402
from tiny_llm_b200.rerank import group_layout  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
TRUE_ID, FALSE_ID = 9454, 2152  # any two ids: the synthetic weights are random
MAX_TOKENS = 8192


def workload(model, n_queries, n_docs, prefix_len, seed):
    g = np.random.default_rng(seed)
    out = []
    for _ in range(n_queries):
        prefix = g.integers(0, model.vocab_size, size=prefix_len).tolist()
        docs = [g.integers(0, model.vocab_size, size=int(L)).tolist() for L in g.integers(64, 513, size=n_docs)]
        out.append((prefix, docs))
    return out


def events_time(fn) -> float:
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3


def split(queries):
    return [(p, [d]) for p, docs in queries for d in docs]


def one_at_a_time(model, queries, count, chunk=128) -> tuple[float, int]:
    pairs = [p + d for p, docs in queries for d in docs][:count]
    longest = max(len(x) for x in pairs)
    engine = model.prefill_engine(chunk, max_seq_len=-(-longest // chunk) * chunk)
    engine.reserve_pools(engine.max_pages + 1)

    def run(batch):
        for ids in batch:
            cache = model.create_kv_cache()
            for a in range(0, len(ids), chunk):
                logits, _ = engine.prefill_chunk(ids[a:a + chunk], a, cache)
            logits[0, -1, [FALSE_ID, TRUE_ID]].float().softmax(-1)
            for c in cache:
                c.release()

    run(pairs[:4])
    return events_time(lambda: run(pairs)), len(pairs)


def kernel_times(model, queries) -> dict:
    """Mean device time per pass of the prefixed attention (summed over layers) and of tl_select_logits."""
    from torch.profiler import ProfilerActivity, profile

    rerank_ids(model, queries, TRUE_ID, FALSE_ID, max_tokens=MAX_TOKENS)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rerank_ids(model, queries, TRUE_ID, FALSE_ID, max_tokens=MAX_TOKENS)
        torch.cuda.synchronize()
    attn = head = 0.0
    n_attn = n_head = 0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        if "paged_prefill_tc_kernel" in e.name and ("Li4E" in e.name or "<4" in e.name):
            attn += e.device_time
            n_attn += 1
        elif "select_logits_kernel" in e.name:
            head += e.device_time
            n_head += 1
    passes = max(n_head, 1)
    return {"passes": n_head, "attention_ms_per_pass": attn / passes / 1e3, "attention_launches": n_attn,
            "select_logits_ms_per_pass": head / passes / 1e3}


def skip_probe(model, reps=200) -> dict:
    """One attention launch over an 8,192-row pass (512-token prefix, 288-token documents) with only the first or only
    the last document live, in ms per launch."""
    at = model.layers_inner[0].self_attn
    Hq, Hkv, D = at.num_heads, at.num_kv_heads, at.head_dim
    P, doc = 512, 288
    n = (MAX_TOKENS - 512) // 320
    entries = [(0, -1)] + [(0, d) for d in range(n)]
    _, _, seg, pst, pen, _, starts = group_layout(entries, [P], [[doc] * n], MAX_TOKENS)
    gen = torch.Generator().manual_seed(0)
    q = torch.randn((Hq, MAX_TOKENS, D), generator=gen).to(torch.bfloat16).to(DEV)
    page = 128
    kp = torch.randn((MAX_TOKENS // page, Hkv, page, D), generator=gen).to(torch.bfloat16).to(DEV)
    vp = torch.randn((MAX_TOKENS // page, Hkv, page, D), generator=gen).to(torch.bfloat16).to(DEV)
    table = torch.arange(MAX_TOKENS // page, dtype=torch.int32, device=DEV)
    out = {"documents_in_pass": n}
    for label, d in (("first", 1), ("last", n)):
        s = seg.copy()
        a, b = starts[d], starts[d] + doc
        keep = np.zeros(MAX_TOKENS, dtype=bool)
        keep[a:b] = True
        s[~keep] = MAX_TOKENS
        ps, pe = np.where(keep, pst, 0).astype(np.int32), np.where(keep, pen, 0).astype(np.int32)
        args = [torch.from_numpy(x).to(DEV) for x in (s, ps, pe)]
        for _ in range(10):
            ext.paged_attention_prefixed_segments(q, kp, vp, table, *args, at.scale, Hkv, Hq)
        t = events_time(lambda: [ext.paged_attention_prefixed_segments(q, kp, vp, table, *args, at.scale, Hkv, Hq) for _ in range(reps)])
        out[f"{label}_document_ms"] = t / reps * 1e3
        out[f"{label}_document_rows"] = [a, b]
    return out


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="qwen3-0.6b,qwen3-4b")
    ap.add_argument("--docs", type=int, default=512, help="documents per workload (Q = docs / n queries)")
    ap.add_argument("--baseline-docs", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rerank_bench needs a CUDA device")
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
        emit({"model": name, "path": "tile-skip probe, one attention launch", **skip_probe(model)})
        for n in (8, 64):
            for P in (64, 512):
                queries = workload(model, max(args.docs // n, 1), n, P, args.seed)
                docs = sum(len(d) for _, d in queries)
                alone = split(queries)
                tag = {"model": name, "n": n, "P": P, "queries": len(queries), "documents": docs,
                       "doc_tokens": sum(len(x) for _, ds in queries for x in ds),
                       "prefix_tokens_saved": len(queries) * (n - 1) * P}
                rerank_ids(model, queries[:1], TRUE_ID, FALSE_ID, max_tokens=MAX_TOKENS)  # warm-up: slabs, modules, tensor maps
                ta, tb = [], []
                for _ in range(args.rounds):
                    ta.append(events_time(lambda: rerank_ids(model, queries, TRUE_ID, FALSE_ID, max_tokens=MAX_TOKENS)))
                    tb.append(events_time(lambda: rerank_ids(model, alone, TRUE_ID, FALSE_ID, max_tokens=MAX_TOKENS)))
                a, b = statistics.median(ta), statistics.median(tb)
                same = all(torch.equal(x, y) for x, y in zip(torch.cat(rerank_ids(model, queries, TRUE_ID, FALSE_ID)).split(1),
                                                            torch.cat(rerank_ids(model, alone, TRUE_ID, FALSE_ID)).split(1)))
                emit({**tag, "path": "(a) shared prefix", "seconds": [round(t, 4) for t in ta], "docs_per_s": round(docs / a, 1)})
                emit({**tag, "path": "(b) prefix repeated per document", "seconds": [round(t, 4) for t in tb], "docs_per_s": round(docs / b, 1),
                      "a_over_b": round(b / a, 3), "a_and_b_bit_identical": same})
                t, count = one_at_a_time(model, queries, args.baseline_docs)
                emit({**tag, "path": "(c) PrefillEngine chunk=128, one pair at a time", "documents": count, "seconds": round(t, 4),
                      "docs_per_s": round(count / t, 1)})
                if n == 64:
                    emit({**tag, "path": "(a) kernels", **{k: round(v, 4) if isinstance(v, float) else v
                                                           for k, v in kernel_times(model, queries[:2]).items()}})
        del model
        torch.cuda.empty_cache()
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
