"""W8A16 against W4A16 on Qwen3-4B-shaped synthetic weights, in one process, the two widths alternating:
  python tools/w8a16_bench.py [--rounds R]

  chain    the 145 projection launches of one decode token at M = 1 (bench.py's matvec_roofline body: per layer
           rms_norm+q|k|v, o+residual, rms_norm+gate|up+swiglu, down+residual, then rms_norm+head) captured in one graph;
           GB/s over the algorithmic bytes (weight_stream_bytes at the width + activations), and the share of HBM
  decode   device-resident greedy decode tok/s at B = 1, 16 and 64 (128-token prompts, 32 timed steps)
  prefill  the four projection GEMMs of one layer at 4096 tokens (tiles kernel), TFLOP/s

Prints one JSON object with the card name and power limit beside the numbers.  Each measurement alternates
W4, W8, W4, W8 ... for --rounds rounds and reports the median of each width."""

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]
from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402

from bench import _prefill_request, cuda_time_ms, measured_peaks, synthetic_prompt  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as exc:  # the numbers stay; the card line says why it is missing
        return f"unknown ({exc})"


def chain_body(model, engine, device):
    H = model.hidden_size
    bf = torch.bfloat16
    x = torch.randn(1, H, device=device).to(bf)
    y = torch.randn(1, engine.Hq * engine.D, device=device).to(bf)
    res = torch.randn(1, H, device=device).to(bf)
    norm_w = torch.ones(H, device=device, dtype=bf)
    inter = model.layers_inner[0].mlp.hidden_dim
    act = torch.randn(1, inter, device=device).to(bf)
    head = model.w_lm_head if model.w_lm_head is not None else model.embedding.weight

    def body():
        for block, pk in zip(model.layers_inner, engine._packed):
            wo, wd = block.self_attn.wo, block.mlp.w_down
            ext.quantized_matmul_fused(pk.qkv.scales, pk.qkv.biases, pk.qkv.weight, x, norm_w, prologue=ext.PRO_RMSNORM, eps=1e-6)
            ext.quantized_matmul_fused(wo.scales, wo.biases, wo.weight, y, residual=res, epilogue=ext.EPI_RESIDUAL)
            ext.quantized_matmul_fused(pk.gate_up.scales, pk.gate_up.biases, pk.gate_up.weight, x, norm_w, prologue=ext.PRO_RMSNORM,
                                       eps=1e-6, epilogue=ext.EPI_SWIGLU_PAIRS)
            ext.quantized_matmul_fused(wd.scales, wd.biases, wd.weight, act, residual=res, epilogue=ext.EPI_RESIDUAL)
        ext.quantized_matmul_fused(head.scales, head.biases, head.weight, x, norm_w, prologue=ext.PRO_RMSNORM, eps=1e-6)

    io = 2 * len(model.layers_inner) * (H + (engine.Hq + 2 * engine.Hkv) * engine.D + engine.Hq * engine.D + 2 * H + H + inter + inter + 2 * H)
    return body, io + 2 * (H + model.mlx_model.args.vocab_size)


def capture(body, device):
    stream = torch.cuda.Stream(device=device)
    with torch.cuda.stream(stream):
        body()
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            body()
        for _ in range(3):
            graph.replay()
        stream.synchronize()
    return graph, stream


def decode_ms(model, device, B, margs):
    from tiny_llm_b200.batch import greedy_tokens
    from tiny_llm_b200.kv_cache import BatchingKvCache

    S, steps = 128, 32
    engine = model.decode_engine(B)
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=512) for _ in range(model.num_hidden_layers)]
    tokens = []
    for b in range(B):
        cache, logits = _prefill_request(model, device, synthetic_prompt(100 + b, S, margs.vocab_size))
        tokens.append(int(greedy_tokens(logits[:, -1, :])[0]))
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, b)
    engine.decode_on_device(tokens, [S] * B, tables, 4)
    torch.cuda.synchronize()
    tokens = engine.next_tokens.tolist()
    ms = cuda_time_ms(lambda: engine.decode_on_device(tokens, [S + 4] * B, tables, steps)) / steps
    for table in tables:
        for b in range(B):
            table.remove_request(b)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--layers", type=int, default=36, help="decoder layers of the Qwen3-4B shape (36 = the published model)")
    opts = ap.parse_args()
    from tiny_llm_b200 import Qwen3ModelWeek3
    from tiny_llm_b200.synthetic import synthetic_qwen3, weight_stream_bytes

    device = torch.device("cuda:0")
    peak = measured_peaks()
    models, chains = {}, {}
    for bits in (4, 8):
        ns = synthetic_qwen3("qwen3-4b", seed=0, device=device, bits=bits, num_hidden_layers=opts.layers, max_position_embeddings=4096)
        model = Qwen3ModelWeek3(ns, page_size=128)
        model.decode_graph_max_seq_len = 512
        engine = model.decode_engine(1)
        body, io = chain_body(model, engine, device)
        graph, stream = capture(body, device)
        models[bits] = model
        chains[bits] = (graph, stream, weight_stream_bytes(ns.args, bits=bits) + io)
    out = {"card": card(), "layers": opts.layers, "peak_hbm_gbs": peak["hbm_gbs"], "peak_source": peak["source"]}

    # decode projection chain, alternating widths
    times = {4: [], 8: []}
    for _ in range(opts.rounds):
        for bits in (4, 8):
            graph, stream, _ = chains[bits]
            with torch.cuda.stream(stream):  # the replay goes to the current stream: the events must be on it
                times[bits].append(statistics.median(cuda_time_ms(graph.replay, stream) for _ in range(10)))
    out["chain"] = {}
    for bits in (4, 8):
        ms = statistics.median(times[bits])
        gbs = chains[bits][2] / (ms / 1e3) / 1e9
        out["chain"][f"w{bits}"] = {"ms": round(ms, 4), "bytes": chains[bits][2], "gbs": round(gbs, 1), "hbm_frac": round(gbs / peak["hbm_gbs"], 4)}
    out["chain"]["w8_over_w4_gbs"] = round(out["chain"]["w8"]["gbs"] / out["chain"]["w4"]["gbs"], 3)
    del chains

    # device-resident decode
    out["decode"] = {}
    for B in (1, 16, 64):
        t = {4: [], 8: []}
        for _ in range(max(1, opts.rounds // 2)):
            for bits in (4, 8):
                t[bits].append(decode_ms(models[bits], device, B, models[bits].mlx_model.args))
        out["decode"][f"B{B}"] = {f"w{bits}_tok_s": round(B * 1e3 / statistics.median(t[bits]), 1) for bits in (4, 8)}

    # prefill projection GEMMs at 4096 tokens (layer 0's weights of each model: q|k|v, o, gate|up, down)
    M = 4096
    a_by_n = {}
    t = {4: [], 8: []}
    flops = 0
    for _ in range(opts.rounds):
        for bits in (4, 8):
            model = models[bits]
            pk, block = model.decode_engine(1)._packed[0], model.layers_inner[0]
            ws = [pk.qkv, block.self_attn.wo, pk.gate_up, block.mlp.w_down]
            shapes = [(w.scales.shape[1] * 128, w.weight.shape[0]) for w in ws]
            for N, _ in shapes:
                if N not in a_by_n:
                    a_by_n[N] = torch.randn(M, N, device=device).to(torch.bfloat16)
            flops = sum(2.0 * M * N * K for N, K in shapes)

            def run():
                for w, (N, _) in zip(ws, shapes):
                    ext.quantized_matmul(w.scales, w.biases, 128, bits, a_by_n[N], w.weight, True)

            run()
            t[bits].append(cuda_time_ms(run))
    out["prefill"] = {f"w{bits}_tflops": round(flops / (statistics.median(t[bits]) / 1e3) / 1e12, 1) for bits in (4, 8)}
    out["prefill"]["w8_over_w4"] = round(out["prefill"]["w8_tflops"] / out["prefill"]["w4_tflops"], 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
