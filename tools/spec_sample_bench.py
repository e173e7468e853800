"""Speculative sampling on one GPU (DESIGN.md section 8d), Qwen3-4B-shaped synthetic target:
* us per tl_speculative_sample call at T = 2, 4, 8 on V = 151,936 bf16 rows, temperature only and top-k 50 + top-p 0.9,
  beside tl_sample and tl_argmax on the same T rows (CUDA events over 200 graph-captured launches per replay);
* the greedy against the sampled verify graph at contexts 128 and 4096;
* the draft step with and without the logits log (0.6B-shaped draft, decode_on_device);
* end-to-end tok/s of sampled speculation against sampled generate, alternated in one process, for the target's own
  weights as draft (acceptance 1: the upper bound) and a random 0.6B-shaped draft (acceptance ~ 0: the lower bound).
The card's name and power limit are read in the same run.

  python tools/spec_sample_bench.py [--out tools_out/spec_sample_bench.json]
"""

from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200"), str(ROOT / "tools")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from spec_bench import card, graphed, prefilled, release, timed  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids, speculative_generate_ids  # noqa: E402
from tiny_llm_b200.sampler import SamplingParams, sampling_tensors  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
V = 151936
REPS = 200


def kernel_us(T, params):
    g = torch.Generator(device=DEV).manual_seed(T)
    x = (torch.randn(T, V, device=DEV, generator=g) * 3).to(torch.bfloat16)
    y = (x[: T - 1].float() + torch.randn(T - 1, V, device=DEV, generator=g)).to(torch.bfloat16)
    per = sampling_tensors([params] * T, DEV)
    pos = torch.arange(100, 100 + T, dtype=torch.int32, device=DEV)
    d = ext.sample(y, *[t[: T - 1] for t in per], pos[: T - 1])
    out = torch.empty(T, dtype=torch.int32, device=DEV)
    calls = {
        "speculative_sample": lambda: ext.speculative_sample(x, y, d, *per, pos, out=out),
        "sample": lambda: ext.sample(x, *per, pos),
        "argmax": lambda: ext.argmax(x),
    }
    return {name: timed(graphed(fn, REPS), reps=20) * 1e3 / REPS for name, fn in calls.items()}


def verify_ms(target, ctx, k, params):
    """Greedy and sampled verify graph replays of T = k + 1 rows at context ``ctx``."""
    ver = target.verify_engine(k + 1)
    draft_rows = torch.randn(k, V, device=DEV).to(torch.bfloat16)
    cache = prefilled(target, ctx)
    ver.verify(1, [2] * k, ctx, cache)
    greedy = timed(ver._graph.replay)
    release(cache)
    cache = prefilled(target, ctx)
    ver.verify(1, [2] * k, ctx, cache, sampling=params, draft_logits=draft_rows)
    sampled = timed(ver._graph_spec[(draft_rows.data_ptr(), draft_rows.dtype)].replay)
    release(cache)
    return dict(greedy=greedy, sampled=sampled)


def draft_ms(draft, params, k=4):
    """ms per draft step of ``decode_on_device(sampling=...)`` with and without ``keep_logits`` (alternated)."""
    eng = draft.decode_engine(1)
    res = {"sampled": [], "sampled_keep_logits": []}
    for _ in range(3):
        for keep, name in ((False, "sampled"), (True, "sampled_keep_logits")):
            cache = prefilled(draft, 128)

            def run():
                eng.decode_on_device([1], [128], cache, k, sampling=params, keep_logits=keep)
                for layer in cache:
                    layer.rewind(k)

            res[name].append(timed(run, reps=20) / k)
            release(cache)
    return {name: min(v) for name, v in res.items()}


def e2e(target, draft, k, n, prompt, params):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    want = greedy_generate_ids(target, prompt, n, device=DEV, sampling=params)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    got, stats = speculative_generate_ids(draft, target, prompt, n, proposal_length=k, device=DEV, sampling=params)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    proposed, accepted = sum(p for p, _ in stats), sum(a for _, a in stats)
    return dict(k=k, sampled_generate_tok_s=len(want) / (t1 - t0), spec_tok_s=len(got) / (t2 - t1), identical=got == want,
                rounds=len(stats), acceptance=accepted / max(proposed, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="tools_out/spec_sample_bench.json")
    ap.add_argument("--tokens", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("spec_sample_bench measures on a CUDA device; none is available")
    res = {"card": card()}
    print("card (name, power limit):", res["card"], flush=True)
    configs = {"temperature 1.0": SamplingParams(1.0, seed=1), "top-k 50 + top-p 0.9": SamplingParams(1.0, top_k=50, top_p=0.9, seed=1)}
    res["kernel_us"] = {}
    for label, params in configs.items():
        for T in (2, 4, 8):
            r = kernel_us(T, params)
            res["kernel_us"][f"{label} T={T}"] = r
            print(f"{label} T={T}: " + "  ".join(f"{k} {v:.2f} us" for k, v in r.items()), flush=True)
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV)
    target = Qwen3ModelWeek3(ns, page_size=128)
    target.prefill_graph_len = 0
    params = configs["top-k 50 + top-p 0.9"]
    res["verify_ms"] = {}
    for ctx in (128, 4096):
        for k in (1, 4, 7):
            r = verify_ms(target, ctx, k, params)
            res["verify_ms"][f"ctx {ctx} T={k + 1}"] = r
            print(f"verify ctx {ctx} T={k + 1}: greedy {r['greedy']:.3f} ms  sampled {r['sampled']:.3f} ms", flush=True)
    draft = Qwen3ModelWeek3(synthetic_qwen3("qwen3-0.6b", seed=3, device=DEV), page_size=128)
    draft.prefill_graph_len = 0
    res["draft_step_ms"] = draft_ms(draft, params)
    print("draft step ms (0.6B-shaped):", {k: round(v, 4) for k, v in res["draft_step_ms"].items()}, flush=True)
    self_draft = Qwen3ModelWeek3(ns, page_size=128)
    self_draft.prefill_graph_len = 0
    prompt = list(range(5, 69))
    res["e2e"] = []
    for label, d in (("target weights", self_draft), ("random 0.6b", draft)):
        for k in (2, 4, 7):
            r = dict(draft=label, **e2e(target, d, k, args.tokens, prompt, params))
            res["e2e"].append(r)
            print(json.dumps(r), flush=True)
    out = Path(args.out)
    out.parent.mkdir(parents=True, exist_ok=True)
    out.write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
