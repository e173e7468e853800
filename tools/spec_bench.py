"""Speculative decoding on one GPU with a Qwen3-4B-shaped synthetic target:

* B = 1 decode step vs verify step (T = 2, 4, 6, 8) at contexts 128 and 4096 (CUDA events over graph replays);
* draft step time of Qwen3-0.6B- and Qwen3-1.7B-shaped drafts (``decode_on_device``);
* end-to-end speculative vs greedy tok/s, alternated in one process, ids compared token for token, for the target's
  own weights as draft (every proposal accepted: the round overhead) and a random 0.6B draft (acceptance ~ 0);
* per-kernel breakdown of the verify cost: the layer's four projections at M = 1 vs M = 8 and the fused attention at
  R = 1 vs R = 8 (36 repetitions captured in one CUDA graph, CUDA events over replays);
* tok/s PROJECTED from those times for acceptance rates 0.5-0.9 (random weights say nothing about real acceptance).

  python tools/spec_bench.py [--out tools_out/spec_bench.json]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids, speculative_generate_ids  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        return f"unknown ({exc})"


def timed(fn, reps=50, warmup=5) -> float:
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def prefilled(model, n):
    cache = model.create_kv_cache()
    ids = torch.randint(0, 1000, (n,), dtype=torch.int32, device=DEV)
    model(ids[None], 0, cache, logits_to_keep=1)
    return cache


def release(cache):
    for layer in cache:
        layer.release()


def step_times(target, ctx):
    dec = target.decode_engine(1)
    out = {}
    cache = prefilled(target, ctx)
    dec.step([1], [ctx], cache)  # metadata of a real step; replays re-run it in place
    out["decode"] = timed(dec._graph.replay)
    release(cache)
    for T in range(2, 9):
        cache = prefilled(target, ctx)
        ver = target.verify_engine(T)
        ver.verify(1, [2] * (T - 1), ctx, cache)
        out[f"verify{T}"] = timed(ver._graph.replay)
        release(cache)
    return out


def graphed(fn, n):
    """``n`` calls of ``fn`` captured into one CUDA graph (the launches chain as in the engine's step graph, with no
    host dispatch between them); returns its replay."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(n):
            fn()
    return graph.replay


def kernel_breakdown(target, ctx, T=8):
    """ms per step of the 36 layers' projections (qkv, o, gate|up, down) at M = 1 and M = T, and of the fused attention
    at R = 1 and R = T rows (layer 0's weights and shapes, 36 repetitions in one graph)."""
    pk, blk = target.packed_layers()[0], target.layers_inner[0]
    at, ln1, wd = blk.self_attn, blk.input_layernorm, blk.mlp.w_down
    Hq, Hkv, D = at.num_heads, at.num_kv_heads, at.head_dim
    H = pk.qkv.weight.shape[1] * 8  # packed W4: 8 input features per int32
    inter = wd.weight.shape[1] * 8
    out = {}
    for M in (1, T):
        x = torch.randn(M, H, device=DEV).to(torch.bfloat16)
        y = torch.randn(M, Hq * D, device=DEV).to(torch.bfloat16)
        act = torch.randn(M, inter, device=DEV).to(torch.bfloat16)
        lw = ln1._weight_as(x.dtype, x.device)

        def projections():
            ext.quantized_matmul_fused(pk.qkv.scales, pk.qkv.biases, pk.qkv.weight, x, lw, prologue=ext.PRO_RMSNORM, eps=ln1.eps)
            ext.quantized_matmul_fused(at.wo.scales, at.wo.biases, at.wo.weight, y, residual=x, epilogue=ext.EPI_RESIDUAL)
            ext.quantized_matmul_fused(pk.gate_up.scales, pk.gate_up.biases, pk.gate_up.weight, x, lw, prologue=ext.PRO_RMSNORM,
                                       eps=ln1.eps, epilogue=ext.EPI_SWIGLU_PAIRS)
            ext.quantized_matmul_fused(wd.scales, wd.biases, wd.weight, act, residual=x, epilogue=ext.EPI_RESIDUAL)

        out[f"projections_M{M}"] = timed(graphed(projections, target.num_hidden_layers))
    page, maxc = 128, 8192
    mp = maxc // page
    kp = torch.randn(mp + 1, Hkv, page, D, device=DEV).to(torch.bfloat16)
    vp = torch.randn_like(kp)
    table = torch.arange(mp, dtype=torch.int32, device=DEV)[None]
    freq = ext.rope_inv_freq_table(D, 1e6, DEV)
    qn = torch.ones(D, device=DEV).to(torch.bfloat16)
    ws = torch.empty(ext.decode_attention_fused_workspace(1, Hq, Hkv, rows_per_request=T), dtype=torch.float32, device=DEV)
    for R in (1, T):
        qkv = torch.randn(R, (Hq + 2 * Hkv) * D, device=DEV).to(torch.bfloat16)
        pos = torch.arange(ctx, ctx + R, dtype=torch.int32, device=DEV)
        ctxs = pos + 1
        out[f"attention_R{R}"] = timed(graphed(lambda: ext.decode_attention_fused(qkv, qn, qn, pos, table, ctxs, freq, kp, vp, Hq, Hkv, 1e-6,
                                                                                  D ** -0.5, maxc, workspace=ws, rows_per_request=R),
                                               target.num_hidden_layers))
    return out


def draft_time(draft, k=4):
    cache = prefilled(draft, 128)
    eng = draft.decode_engine(1)
    offset = 128

    def run():
        nonlocal offset
        eng.decode_on_device([1], [offset], cache, k)
        offset += k
        for layer in cache:
            layer.rewind(k)
        offset -= k

    ms = timed(run, reps=20) / k
    release(cache)
    return ms


def e2e(target, draft, k, n, prompt):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    want = greedy_generate_ids(target, prompt, n, device=DEV)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    got, stats = speculative_generate_ids(draft, target, prompt, n, proposal_length=k, device=DEV)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    proposed, accepted = sum(p for p, _ in stats), sum(a for _, a in stats)
    return dict(k=k, greedy_tok_s=len(want) / (t1 - t0), spec_tok_s=len(got) / (t2 - t1), identical=got == want, rounds=len(stats),
                acceptance=accepted / max(proposed, 1), round_ms=(t2 - t1) * 1e3 / max(len(stats), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="tools_out/spec_bench.json")
    ap.add_argument("--tokens", type=int, default=256)
    args = ap.parse_args()
    res = {"card": card()}
    print("card (name, power limit):", res["card"], flush=True)
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV)
    target = Qwen3ModelWeek3(ns, page_size=128)
    target.prefill_graph_len = 0  # greedy and speculative prefill the prompt through the same path
    res["steps_ms"] = {ctx: step_times(target, ctx) for ctx in (128, 4096)}
    for ctx, row in res["steps_ms"].items():
        print(f"ctx {ctx}: " + "  ".join(f"{k} {v:.3f} ms" for k, v in row.items()), flush=True)
    res["breakdown_ms"] = {ctx: kernel_breakdown(target, ctx) for ctx in (128, 4096)}
    for ctx, row in res["breakdown_ms"].items():
        print(f"breakdown ctx {ctx} (36 layers in one graph): " + "  ".join(f"{k} {v:.3f} ms" for k, v in row.items()), flush=True)
    drafts = {}
    for name in ("qwen3-0.6b", "qwen3-1.7b"):
        drafts[name] = Qwen3ModelWeek3(synthetic_qwen3(name, seed=3, device=DEV), page_size=128)
        drafts[name].prefill_graph_len = 0
    res["draft_step_ms"] = {name: draft_time(m) for name, m in drafts.items()}
    print("draft step ms:", {k: round(v, 3) for k, v in res["draft_step_ms"].items()}, flush=True)
    prompt = list(range(5, 69))
    self_draft = Qwen3ModelWeek3(ns, page_size=128)
    self_draft.prefill_graph_len = 0
    res["e2e"] = []
    for label, draft in (("target weights", self_draft), ("random 0.6b", drafts["qwen3-0.6b"])):
        for k in (2, 4, 7):
            r = dict(draft=label, **e2e(target, draft, k, args.tokens, prompt))
            res["e2e"].append(r)
            print(json.dumps(r), flush=True)
    # projection: a round costs k draft steps, one verify of k + 1 rows, the draft's catch-up step when all k were
    # accepted, and the host time of a round (round_ms of the full-acceptance k = 4 run with the target as its own
    # draft, minus its 4 draft steps, its verify of 5 rows and its catch-up step - each about one decode step)
    dec = res["steps_ms"][128]["decode"]
    d06 = res["draft_step_ms"]["qwen3-0.6b"]
    r4 = next(r for r in res["e2e"] if r["draft"] == "target weights" and r["k"] == 4)
    overhead = max(0.0, r4["round_ms"] - 5 * dec - res["steps_ms"][128]["verify5"])
    res["round_overhead_ms"] = overhead
    greedy_e2e = sum(r["greedy_tok_s"] for r in res["e2e"]) / len(res["e2e"])
    proj = []
    for k in range(1, 8):
        ver = res["steps_ms"][128][f"verify{k + 1}"]
        for a in (0.5, 0.6, 0.7, 0.8, 0.9):
            tokens = (1 - a ** (k + 1)) / (1 - a)  # expected tokens per round at per-proposal acceptance a
            ms = k * d06 + ver + a ** k * d06 + overhead
            proj.append(dict(k=k, acceptance=a, projected_tok_s=tokens / ms * 1e3))
    res["projection_0.6b_draft_ctx128"] = proj
    res["greedy_e2e_tok_s"] = greedy_e2e
    print(f"PROJECTION (not measured): 0.6B-shaped draft, context 128, host time per round {overhead:.3f} ms; "
          f"compare with greedy end to end {greedy_e2e:.0f} tok/s (same basis: device + host)")
    for k in range(1, 8):
        row = [p for p in proj if p["k"] == k]
        print(f"  k={k}: " + "  ".join(f"a={p['acceptance']:.1f} {p['projected_tok_s']:.0f}" for p in row))
    out = Path(args.out)
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
