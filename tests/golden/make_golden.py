"""Regenerate the committed fixtures under tests/golden/.

Run from the repo root:  python tests/golden/make_golden.py

Two kinds of file live here (see README.md in this directory):
  * reference_literals.json - known-answer values TRANSCRIBED from the
    reference's own tests (file:line given per entry); never regenerated.
  * *_checksums.json / *_trace.json - outputs of the CPU oracle on
    deterministic inputs.  They are self-generated regression anchors (MLX, and
    therefore the reference itself, cannot run in this container), useful to
    notice when the oracle or the product drifts, not an independent truth.
"""

import json
import sys
from math import prod
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200")]
HERE = Path(__file__).resolve().parent

from oracle import ops  # noqa: E402
from oracle.model import ReferenceCpuModel, greedy_decode  # noqa: E402


def decode_attention_checksums():
    """Fixture sweep of tests_refsol/test_week_2_day_5.py:119-163."""
    D, Hq = 128, 4

    def fixture(shape, phase):
        return torch.sin(torch.arange(prod(shape), dtype=torch.float32) * 0.017 + phase).reshape(shape).to(torch.bfloat16)

    out = {}
    shapes = [(1, s) for s in (1, 31, 32, 127, 128, 129, 255, 256)] + [(8, s) for s in (8, 31, 32, 127, 128, 129, 255, 256)]
    for L, S in shapes:
        for ratio in (1, 4):
            Hkv = Hq // ratio
            q = fixture((Hq, L, D), 0.1)
            k = fixture((Hkv, S, D), 0.7)
            v = fixture((Hkv, S, D), 1.3)
            explicit = torch.where(torch.arange(S) % 5 == 0, -2.0, 0.0).reshape(1, 1, S).expand(Hq, L, S).contiguous()
            for name, causal, mask in (("causal", True, torch.zeros(1)), ("mask", False, explicit)):
                got = ops.decode_attention(q, k, v, mask, D**-0.5, causal, not causal, Hq, Hkv)
                out[f"L{L}_S{S}_g{ratio}_{name}"] = float(got.float().sum())
    (HERE / "decode_attention_fixture_checksums.json").write_text(json.dumps(out, indent=1, sort_keys=True))


def tiny_model_trace():
    """Config-1 style plumbing trace on a tiny Qwen3-shaped model: greedy tokens
    and per-step log-probabilities of the reference's CPU path (oracle.model)."""
    from tiny_llm_b200.synthetic import synthetic_qwen3

    torch.manual_seed(0)
    model_ns = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)
    model = ReferenceCpuModel(model_ns)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11]
    tokens, logprobs = greedy_decode(model, prompt, 12, return_logprobs=True)
    top = [[int(i) for i in torch.topk(lp, 4).indices] for lp in logprobs]
    vals = [[round(float(x), 4) for x in torch.topk(lp, 4).values] for lp in logprobs]
    (HERE / "tiny_d128_greedy_trace.json").write_text(
        json.dumps({"config": "tiny-d128", "seed": 0, "realistic": True, "prompt": prompt, "tokens": tokens, "top4_ids": top, "top4_logprobs": vals}, indent=1)
    )


def qwen3_0p6b_trace():
    """BASELINE config 1 (SURVEY 8d): Qwen3-0.6B-shaped random W4 weights (the benchmark's direct
    code/scale draw, seed 0), 16-token prompt, 128 greedy tokens through the reference's CPU path
    (oracle.model = Qwen3ModelWeek2(checkpoint="kv-cache") + simple_generate_with_kv_cache,
    generate.py:49-81).  Stored: the tokens and, per step, the ids and log-probabilities of the four
    most likely tokens (full 151,936-wide rows would be 78 MB)."""
    import random

    from tiny_llm_b200.synthetic import synthetic_qwen3

    model_ns = synthetic_qwen3("qwen3-0.6b", seed=0)
    model = ReferenceCpuModel(model_ns)
    rng = random.Random(16)
    prompt = [rng.randint(256, model.args.vocab_size - 1) for _ in range(16)]
    tokens, logprobs = greedy_decode(model, prompt, 128, return_logprobs=True)
    top = [[int(i) for i in torch.topk(lp, 4).indices] for lp in logprobs]
    vals = [[round(float(x), 4) for x in torch.topk(lp, 4).values] for lp in logprobs]
    (HERE / "qwen3_0p6b_greedy_trace.json").write_text(
        json.dumps({"config": "qwen3-0.6b", "seed": 0, "realistic": False, "prompt": prompt, "tokens": tokens, "top4_ids": top, "top4_logprobs": vals})
    )


if __name__ == "__main__":
    decode_attention_checksums()
    tiny_model_trace()
    if "--config1" in sys.argv:  # ~5 minutes of CPU time
        qwen3_0p6b_trace()
    print("golden fixtures written to", HERE)
