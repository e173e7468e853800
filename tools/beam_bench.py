"""Beam search on one GPU (DESIGN.md section 15), on the Qwen3-4B-shaped synthetic model (``--layers``, default 36):

* ``tl_beam_select`` alone: microseconds per launch at W = 1 / 2 / 4 / 8 with 4 EOS ids, CUDA events over 200 launches
  captured in one graph;
* ``beam_search_ids`` at W = 1 / 2 / 4 / 8, contexts 128 and 4,096, ``--tokens`` (256) new tokens with no EOS, so
  every search runs all its steps: per step the wall time (host clock around the whole search, which ends in the
  final read) and the device time (CUDA events around it), the copy-on-write records per step, their bytes and their
  device time (CUDA events around each copy call), and the host-to-device bytes of the beam step graph;
* greedy decoding at B = 1 (``greedy_generate_ids``) and at B = W (``decode_on_device`` over W copies of the prompt),
  alternated with the beam runs in the same process (greedy, beam, greedy, beam).

The card's name and power limit are read in the same run.

  python tools/beam_bench.py [--layers 36] [--tokens 256] [--out tools_out/beam_bench.json]
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
from tiny_llm_b200 import Qwen3ModelWeek3, beam_search_ids, greedy_generate_ids  # noqa: E402
from tiny_llm_b200 import paged_kv_cache as pkv  # noqa: E402
from tiny_llm_b200.kv_cache import BatchingKvCache  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
WIDTHS = (1, 2, 4, 8)
CONTEXTS = (128, 4096)


def select_us(W: int, reps: int = 200) -> float:
    eos = (0, 1, 2, 3)
    N = W + len(eos)
    lp = -torch.rand((W, N), device=DEV).sort(dim=1).values
    ids = torch.randint(4, 1000, (W, N), dtype=torch.int32, device=DEV)
    cum = torch.zeros(W, device=DEV)
    out = torch.zeros(ext.BEAM_RESULT_WORDS, dtype=torch.int32, device=DEV)
    run = graphed(lambda: ext.beam_select(lp, ids, cum, W, eos, out), reps)
    run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    run()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) * 1e3 / reps


class CopyMeter:
    """Counts the copy records of every ``paged_cache_copy_prefix`` call and times each call with CUDA events."""

    def __init__(self):
        self.records = self.slots = 0
        self.events = []
        self._inner = ext.paged_cache_copy_prefix

    def __call__(self, key_slabs, value_slabs, copies, stream=None):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        self._inner(key_slabs, value_slabs, copies, stream)
        b.record()
        self.events.append((a, b))
        self.records += len(copies)
        self.slots += sum(int(c[3]) for c in copies)

    def device_ms(self) -> float:
        torch.cuda.synchronize()
        return sum(a.elapsed_time(b) for a, b in self.events)


def beam_run(model, prompt, W, tokens):
    meter = CopyMeter()
    ext.paged_cache_copy_prefix = meter
    engine = model.decode_engine(W)
    h2d0 = engine.h2d_bytes
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    a.record()
    try:
        hyps = beam_search_ids(model, prompt, tokens, num_beams=W, device=DEV)
    finally:
        ext.paged_cache_copy_prefix = meter._inner
    b.record()
    b.synchronize()
    wall = time.perf_counter() - t0
    steps = tokens  # no EOS: every search runs all its steps
    attn = model.layers_inner[0].self_attn
    per_slot = 2 * attn.num_kv_heads * attn.head_dim * 2  # K and V rows, bf16
    return {
        "wall_ms_per_step": 1e3 * wall / steps,
        "device_ms_per_step": a.elapsed_time(b) / steps,
        "cow_records_per_step": meter.records / steps,
        "cow_bytes_per_step": meter.slots * per_slot / steps,
        "cow_device_ms_per_step": meter.device_ms() / steps,
        "h2d_bytes_per_step": (engine.h2d_bytes - h2d0) / max(1, steps - 1),
        "kernels_per_beam_step": engine.kernels_per_beam_step,
        "best_len": len(hyps[0].ids),
    }


def greedy_b1(model, prompt, tokens) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    greedy_generate_ids(model, prompt, tokens, device=DEV)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / tokens


def greedy_bw(model, prompt, W, tokens) -> float:
    """B = W greedy steps on the device over W copies of the prompt (one prefill, W - 1 forks)."""
    cache = model.create_kv_cache()
    logits = model(torch.tensor([prompt], dtype=torch.int32, device=DEV), 0, cache, logits_to_keep=1)
    first = int(logits[0, -1].argmax())
    kids = pkv.fork([(cache, W - 1)])[0] if W > 1 else []
    groups = [cache, *kids]
    slots = [BatchingKvCache(W) for _ in range(model.num_hidden_layers)]
    for b, caches in enumerate(groups):
        for layer, c in enumerate(caches):
            slots[layer].kv_caches[b] = c
    engine = model.decode_engine(W)
    try:
        engine.decode_on_device([first] * W, [len(prompt)] * W, slots, 2)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = engine.decode_on_device([first] * W, [len(prompt) + 2] * W, slots, tokens)
        out.cpu()
        return 1e3 * (time.perf_counter() - t0) / tokens
    finally:
        for caches in groups:
            for c in caches:
                c.release()


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=36)
    ap.add_argument("--tokens", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    result = {"card": card(), "select_us": {W: select_us(W) for W in WIDTHS}, "runs": []}
    print(json.dumps({"card": result["card"], "select_us": result["select_us"]}), flush=True)
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV, num_hidden_layers=args.layers)
    model = Qwen3ModelWeek3(ns, page_size=128)
    g = torch.Generator().manual_seed(0)
    for ctx in CONTEXTS:
        prompt = torch.randint(0, model.vocab_size, (ctx,), generator=g).tolist()
        for W in WIDTHS:
            beam_run(model, prompt, W, 8)  # warm-up: captures and first launches
            greedy_bw(model, prompt, W, 8)
            row = {"context": ctx, "W": W, "greedy_b1_ms": [], "greedy_bw_ms": [], "beam": []}
            for _ in range(2):
                row["greedy_b1_ms"].append(greedy_b1(model, prompt, args.tokens))
                row["greedy_bw_ms"].append(greedy_bw(model, prompt, W, args.tokens))
                row["beam"].append(beam_run(model, prompt, W, args.tokens))
            print(json.dumps(row), flush=True)
            result["runs"].append(row)
    result["card_after"] = card()
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
