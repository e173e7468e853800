"""Prompt-lookup speculative decoding on one GPU (DESIGN.md section 14):

* the proposer kernel ``tl_ngram_propose``: microseconds per call at L = 1K / 8K / 32K / 131,072, k = 4 and 7, with and
  without the one-hot rows (V = 151,936, bf16).  "device" is CUDA events over 200 calls captured in one graph (the
  kernel alone); "call+read" is the host clock around 200 eager calls each followed by the small device->host read of
  the match length and proposals, as a generation round issues them;
* end to end on the Qwen3-4B-shaped synthetic model (``--layers``, default 36): tokens/s of ``greedy_generate_ids``
  against ``prompt_lookup_generate_ids``, alternated in one process (greedy, lookup, greedy, lookup), on (a) a prompt
  of a repeated passage, the case that copies text, (b) a random prompt, the overhead case, and (c) a 32K-token
  repeated prompt at ``--max-context 65536``; and, as a control, draft-model speculation with the target's own weights
  on (a), which runs the same verify graph with every proposal accepted.  Random weights say nothing about acceptance on real text: the
  acceptance here is that of this synthetic model on these prompts.

The card's name and power limit are read in the same run.

  python tools/prompt_lookup_bench.py [--layers 36] [--tokens 128] [--out tools_out/prompt_lookup_bench.json]
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
from spec_bench import card, graphed  # noqa: E402
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids, prompt_lookup_generate_ids, speculative_generate_ids  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
V = 151936
REPS = 200


def kernel_rows() -> list[dict]:
    rows = []
    g = torch.Generator().manual_seed(0)
    for L in (1024, 8192, 32768, 131072):
        passage = torch.randint(0, V, (512,), generator=g)
        hist = passage.repeat(L // 512 + 1)[: L + 8].to(torch.int32).to(DEV)
        for k in (4, 7):
            for onehot in (False, True):
                rows_buf = torch.full((k, V), float("-inf"), dtype=torch.bfloat16, device=DEV) if onehot else None
                state = torch.zeros(ext.NGRAM_STATE_WORDS, dtype=torch.int32, device=DEV)
                out = torch.empty(2 + k, dtype=torch.int32, device=DEV)

                tok = [int(hist[L - 1])]  # the pending token travels by argument, as in a generation round

                def call():
                    ext.ngram_propose(hist, L - 1, tok, k, 2, 3, out, state, rows_buf)

                replay = graphed(call, REPS)
                replay()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                replay()
                b.record()
                b.synchronize()
                device_us = a.elapsed_time(b) * 1e3 / REPS
                for _ in range(10):
                    call()
                    out.tolist()
                t0 = time.perf_counter()
                for _ in range(REPS):
                    call()
                    out.tolist()
                read_us = (time.perf_counter() - t0) * 1e6 / REPS
                rows.append(dict(L=L, k=k, onehot=onehot, device_us=round(device_us, 2), call_and_read_us=round(read_us, 2),
                                 match=out.tolist()[:2]))
                print(rows[-1], flush=True)
    return rows


def e2e(model, prompt, tokens, k, ngram) -> dict:
    res = {"greedy": [], "lookup": []}
    ids = {}
    for rep in range(2):
        for mode in ("greedy", "lookup"):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if mode == "greedy":
                out = greedy_generate_ids(model, prompt, tokens, device=DEV)
                st = None
            else:
                out, st = prompt_lookup_generate_ids(model, prompt, tokens, proposal_length=k, ngram=ngram, device=DEV)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            res[mode].append(dt)
            ids[mode] = out
            if st is not None:
                res["stats"] = st
    st = res.pop("stats")
    proposed, accepted = sum(p for p, _ in st), sum(a for _, a in st)
    matched = sum(1 for p, _ in st if p)
    best = {m: min(v) for m, v in res.items()}
    return dict(prompt_tokens=len(prompt), new_tokens=tokens, k=k, ngram=list(ngram), same_ids=ids["greedy"] == ids["lookup"],
                first_difference=next((i for i, (a, b) in enumerate(zip(ids["greedy"], ids["lookup"])) if a != b), None),
                greedy_s=[round(x, 4) for x in res["greedy"]], lookup_s=[round(x, 4) for x in res["lookup"]],
                greedy_tok_s=round(tokens / best["greedy"], 1), lookup_tok_s=round(tokens / best["lookup"], 1),
                rounds=len(st), matched_share=round(matched / max(1, len(st)), 3),
                acceptance=round(accepted / proposed, 3) if proposed else None,
                ms_per_round=round(best["lookup"] * 1e3 / max(1, len(st)), 3))


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--tokens", type=int, default=128)
    ap.add_argument("--skip-long", action="store_true", help="leave out the 32K-token case (c)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = {"card": card(), "kernel": kernel_rows()}
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV, num_hidden_layers=args.layers)
    model = Qwen3ModelWeek3(ns, page_size=128)
    model.prefill_graph_len = 0  # greedy and prompt lookup prefill the prompt through the same path
    g = torch.Generator().manual_seed(1)
    passage = torch.randint(0, V, (300,), generator=g).tolist()
    cases = {"a_repeated": (passage * 4)[:1000], "b_random": torch.randint(0, V, (1000,), generator=g).tolist()}
    for name, prompt in cases.items():
        for k, ngram in ((4, (2, 3)), (7, (2, 3)), (4, (1, 3))):
            result[f"{name}_k{k}_n{ngram[0]}{ngram[1]}"] = e2e(model, prompt, args.tokens, k, ngram)
            print(name, result[f"{name}_k{k}_n{ngram[0]}{ngram[1]}"], flush=True)
    # control: draft-model speculation with the target's own weights on case (a), same verify graph, every proposal accepted
    draft = Qwen3ModelWeek3(ns, page_size=128)
    draft.prefill_graph_len = 0
    want = greedy_generate_ids(model, cases["a_repeated"], args.tokens, device=DEV)
    got, _ = speculative_generate_ids(draft, model, cases["a_repeated"], args.tokens, proposal_length=4, device=DEV)
    result["control_draft_same_weights"] = dict(same_ids=got == want, first_difference=next(
        (i for i, (a, b) in enumerate(zip(want, got)) if a != b), None))
    print("control", result["control_draft_same_weights"], flush=True)
    del draft
    if not args.skip_long:
        model = Qwen3ModelWeek3(ns, page_size=128)  # a fresh model: the window is set before its first graph engine
        model.prefill_graph_len = 0
        model.set_max_context(65536)
        long_passage = torch.randint(0, V, (2000,), generator=g).tolist()
        result["c_repeated_32k"] = e2e(model, (long_passage * 17)[:32768], args.tokens, 4, (2, 3))
        print("c", result["c_repeated_32k"], flush=True)
    result["card_after"] = card()
    print(json.dumps(result, indent=1))
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))
    return 0


if __name__ == "__main__":
    sys.exit(main())
