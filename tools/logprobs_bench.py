"""Token log-probabilities on one GPU (DESIGN.md section 8a):

* ``tl_logprobs`` us per call at 1, 8 and 64 rows and max_n 0 / 5 / 20 (V = 151,936, bf16 logits, a target per row),
  against torch ``log_softmax`` + ``gather`` + ``topk`` on the same rows: device time per call, 50 calls captured in one
  CUDA graph and replayed 20 times between CUDA events (outputs preallocated, no host enqueue in the figure);
* ``decode_on_device`` tok/s on Qwen3-4B-shaped synthetic weights, B = 1 and B = 64, context 128: greedy against
  greedy with ``logprobs=5``, sampled against sampled with ``logprobs=5``, the four modes alternated 3 times;
* ``score_ids`` tokens/s on a 4096-token prompt at chunk 512, against the same chunked forward without scoring.

  python tools/logprobs_bench.py [--out tools_out/logprobs_bench.json]
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
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, score_ids  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
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
    """us per call of ``fn`` on the device: ``launches`` calls captured in one CUDA graph, replayed ``reps`` times
    between two events, so the host's enqueue cost per call does not enter the figure."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):  # lazy attribute setup and library warm-up outside the capture
            fn()
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            for _ in range(launches):
                fn()
    torch.cuda.current_stream().wait_stream(s)
    graph.replay()  # warm replay
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        graph.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / (reps * launches) * 1e3


def kernel_table() -> dict:
    out = {}
    g = torch.Generator(device=DEV).manual_seed(0)
    for rows in (1, 8, 64):
        logits = (torch.randn(rows, V, generator=g, device=DEV) * 3).to(torch.bfloat16)
        targets = torch.randint(0, V, (rows,), generator=g, device=DEV, dtype=torch.int32)
        index = torch.zeros(1, dtype=torch.int32, device=DEV)
        res = {}
        for n in (0, 5, 20):
            logs = (torch.empty(1, rows, device=DEV), torch.empty(1, rows, device=DEV), torch.empty(1, rows, dtype=torch.int32, device=DEV),
                    torch.empty(1, rows, n, dtype=torch.int32, device=DEV), torch.empty(1, rows, n, device=DEV))
            res[f"tl_logprobs max_n {n}"] = graph_timed(lambda: ext.logprobs(logits, targets, None, n, out=logs, out_index=index))

            def torch_path():
                lp = torch.log_softmax(logits.float(), dim=-1)
                picked = lp.gather(1, targets.long()[:, None])
                return picked, (torch.topk(lp, n, dim=-1) if n else None)

            res[f"torch max_n {n}"] = graph_timed(torch_path)
        out[rows] = res
        print(f"rows {rows}: " + ", ".join(f"{k} {v:.1f} us" for k, v in res.items()), flush=True)
    return out


def decode_rates(model, B, ctx=128, steps=64, rounds=3) -> dict:
    modes = ("greedy", "greedy+logprobs", "sampled", "sampled+logprobs")
    msl = ctx + len(modes) * (rounds + 1) * steps + 64
    engine = DecodeEngine(model, B, msl, DEV)
    engine.reserve_pools()
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b in range(B):
        cache = model.create_kv_cache()
        for c, t in zip(cache, tables):
            c.append_slots(ctx)
            t.add_request(c, b)
    sampling = SamplingParams(0.7, top_k=50, top_p=0.9, seed=1)
    offsets, tokens = [ctx] * B, [1] * B
    times = {m: [] for m in modes}
    for r in range(rounds + 1):
        for mode in modes:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = engine.decode_on_device(tokens, offsets, tables, steps, sampling=sampling if mode.startswith("sampled") else None,
                                          logprobs=5 if mode.endswith("logprobs") else None)
            b.record()
            b.synchronize()
            log = out[0] if isinstance(out, tuple) else out
            tokens = log[-1].tolist()
            offsets = [o + steps for o in offsets]
            if r:  # round 0 captures the graphs
                times[mode].append(a.elapsed_time(b))
    res = {m: B * steps * len(v) / (sum(v) / 1e3) for m, v in times.items()}
    res["step_ms"] = {m: sum(v) / len(v) / steps for m, v in times.items()}
    res["kernels_per_step"] = {"greedy": engine.kernels_per_step, "sampled": engine.kernels_per_sampled_step,
                               "sampled+logprobs (last captured)": engine.kernels_per_logprobs_step}
    print(f"B {B}: " + ", ".join(f"{m} {res[m]:.1f} tok/s" for m in modes)
          + f" (logprobs cost: greedy {(res['greedy+logprobs'] / res['greedy'] - 1) * 100:+.2f} %,"
          f" sampled {(res['sampled+logprobs'] / res['sampled'] - 1) * 100:+.2f} %)", flush=True)
    return res


def scoring_rate(model, L=4096, chunk=512, rounds=3) -> dict:
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(1, 150000, (L,), generator=g).tolist()

    def forward_only():
        cache = model.create_kv_cache()
        try:
            for start in range(0, L, chunk):
                piece = torch.tensor([ids[start : start + chunk]], dtype=torch.int32, device=DEV)
                model(piece, start, cache, logits_to_keep=None)
        finally:
            for c in cache:
                c.release()

    times = {"forward": [], "score_ids": []}
    for r in range(rounds + 1):
        for mode, fn in (("forward", forward_only), ("score_ids", lambda: score_ids(model, ids, chunk=chunk, top_n=5))):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            if r:
                times[mode].append(a.elapsed_time(b))
    res = {m: L * len(v) / (sum(v) / 1e3) for m, v in times.items()}
    print(f"scoring {L} tokens at chunk {chunk}: forward {res['forward']:.0f} tok/s, score_ids {res['score_ids']:.0f} tok/s "
          f"({(res['score_ids'] / res['forward'] - 1) * 100:+.2f} %)", flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("logprobs_bench needs a CUDA device")
    result = {"card": card()}
    print(f"card: {result['card']}", flush=True)
    result["kernels_us"] = kernel_table()
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV, max_position_embeddings=8192)
    model = Qwen3ModelWeek3(ns, page_size=64)
    result["decode"] = {B: decode_rates(model, B) for B in (1, 64)}
    result["scoring"] = scoring_rate(model)
    result["card_after"] = card()
    print(json.dumps(result))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
