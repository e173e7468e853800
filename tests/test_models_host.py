"""Model wiring on CPU: the product's Week-2/Week-3 model code is driven through
the CPU stand-in of the extension and compared with the reference's CPU path
(oracle.model) and with itself across cache implementations.  CPU-only."""

import json
from pathlib import Path

import pytest
import torch

from oracle.model import ReferenceCpuModel, greedy_decode
from tiny_llm_b200 import (
    WEEK2_CHECKPOINTS,
    BatchingKvCache,
    FastRMSNorm,
    FastRoPE,
    QuantizedEmbedding,
    QuantizedWeights,
    Qwen3ModelWeek2,
    Qwen3ModelWeek3,
    RMSNorm,
    RoPE,
    dequantize_weights,
    dispatch_model,
    greedy_generate_ids,
    quantized_linear,
    quantized_matvec_custom,
)
from tiny_llm_b200.synthetic import quantize_w4, synthetic_qwen3

GOLDEN = Path(__file__).parent / "golden"


def logprobs(logits):
    x = logits.to(torch.float32)
    return x - torch.logsumexp(x, dim=-1, keepdim=True)


@pytest.fixture(scope="module")
def tiny():
    return synthetic_qwen3("tiny", seed=0, realistic=True, max_position_embeddings=128, rope_theta=10000, rms_norm_eps=1e-5)


def test_quantizer_round_trip_is_within_half_a_step():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(16, 256, generator=g)
    packed, scales, biases = quantize_w4(w)
    assert packed.dtype == torch.uint32 and tuple(packed.shape) == (16, 32) and tuple(scales.shape) == (16, 2)
    back = dequantize_weights(packed, scales, biases, 128, 4).float()
    step = scales.float().repeat_interleave(128, 1)
    assert bool(((back - w).abs() <= 0.51 * step + 0.02).all())


def test_week2_checkpoints_are_cumulative(tiny):
    with pytest.raises(ValueError, match="unknown Week 2 checkpoint"):
        Qwen3ModelWeek2(tiny, checkpoint="nope")
    for name in WEEK2_CHECKPOINTS:
        model = Qwen3ModelWeek2(tiny, checkpoint=name)
        layer = model.layers_inner[0]
        level = WEEK2_CHECKPOINTS.index(name)
        assert isinstance(layer.self_attn.wq, QuantizedWeights) is (level >= 1)
        assert isinstance(layer.input_layernorm, FastRMSNorm) is (level >= 2)
        assert isinstance(layer.input_layernorm, (FastRMSNorm, RMSNorm))
        assert isinstance(layer.self_attn.rope, FastRoPE) is (level >= 3)
        assert isinstance(layer.self_attn.rope, (FastRoPE, RoPE))
        assert layer.mlp.use_fast_swiglu is (level >= 4)
        assert layer.self_attn.use_decode_attention is (level >= 5)
        if level >= 1:
            assert isinstance(model.embedding, QuantizedEmbedding) and not model.embedding.use_custom_kernel
            assert layer.self_attn.wk.use_simdgroup_matmul is (level >= 6)
            assert layer.self_attn.wk.use_split_k_matmul is (level >= 7)


def test_week3_defaults_and_pool_sharing(tiny, cpu_ext):
    model = Qwen3ModelWeek3(tiny, page_size=4, enable_paged_attention=False)
    assert model.embedding.use_custom_kernel and model.embedding.weight.use_simdgroup_matmul
    assert all(l.self_attn.wq.use_simdgroup_matmul and l.self_attn.wq.use_split_k_matmul for l in model.layers_inner)
    a, b = model.create_kv_cache(), model.create_kv_cache()
    assert len(a) == model.num_hidden_layers
    for layer in range(model.num_hidden_layers):
        assert a[layer].pool is model.page_pools[layer] and b[layer].pool is model.page_pools[layer]
    assert a[0].pool is not a[1].pool and a[0].page_ids is not a[1].page_ids
    model(torch.tensor([[1, 5, 7, 3, 9]], dtype=torch.int32), 0, a)
    assert a[0].page_ids == [0, 1] and a[0].page_lens == [4, 1]
    for layer in range(1, model.num_hidden_layers):
        assert a[layer].page_ids == a[0].page_ids and a[layer].page_lens == a[0].page_lens


def test_packed_layers_are_built_once_per_model(cpu_ext):
    """The graph engines' fused q|k|v and gate|up weights: one copy per model, asked for by every engine."""
    model = Qwen3ModelWeek3(synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512), page_size=64)
    packed = model.packed_layers()
    assert model.packed_layers() is packed and len(packed) == model.num_hidden_layers
    as_i32 = lambda w: w.view(torch.int32) if w.dtype == torch.uint32 else w
    for block, pk in zip(model.layers_inner, packed, strict=True):
        at, mlp = block.self_attn, block.mlp
        assert torch.equal(pk.qkv.weight, torch.cat([as_i32(at.wq.weight), as_i32(at.wk.weight), as_i32(at.wv.weight)]))
        for field in ("scales", "biases"):
            assert torch.equal(getattr(pk.qkv, field), torch.cat([getattr(w, field) for w in (at.wq, at.wk, at.wv)]))
        assert torch.equal(pk.gate_up.weight, cpu_ext.interleave_gate_up(as_i32(mlp.w_gate.weight), as_i32(mlp.w_up.weight)))
        for field in ("scales", "biases"):
            assert torch.equal(getattr(pk.gate_up, field), cpu_ext.interleave_gate_up(getattr(mlp.w_gate, field), getattr(mlp.w_up, field)))


def test_week2_offset_mismatch_and_logits_to_keep(tiny, cpu_ext):
    model = Qwen3ModelWeek2(tiny)
    cache = model.create_kv_cache()
    out = model(torch.tensor([[1, 2, 3, 4]], dtype=torch.int32), 0, cache, logits_to_keep=1)
    assert tuple(out.shape) == (1, 1, 128)
    with pytest.raises(ValueError, match="does not match model offset"):
        model(torch.tensor([[1]], dtype=torch.int32), 2, cache)
    with pytest.raises(ValueError, match="logits_to_keep must be positive"):
        model(torch.tensor([[1]], dtype=torch.int32), 4, cache, logits_to_keep=0)
    # the rejected call above had already appended its token (the check runs after the layers, as in the reference)
    assert tuple(model(torch.tensor([[1, 2]], dtype=torch.int32), 5, cache).shape) == (1, 2, 128)


@pytest.mark.parametrize("paged", [False, True], ids=["dense-gather", "paged-attention"])
def test_week3_incremental_decode_matches_week2(tiny, cpu_ext, paged):
    # test_week_3_day_3.py:386-402 and test_week_3_day_4.py:325-345 (tolerance 1e-3)
    week2 = Qwen3ModelWeek2(tiny)
    week3 = Qwen3ModelWeek3(tiny, page_size=4, enable_paged_attention=paged)
    inputs = torch.tensor([[1, 5, 7, 3, 9, 11]], dtype=torch.int32)
    c2, c3 = week2.create_kv_cache(), week3.create_kv_cache()
    for offset in range(inputs.shape[1]):
        token = inputs[:, offset : offset + 1]
        torch.testing.assert_close(logprobs(week3(token, offset, c3)), logprobs(week2(token, offset, c2)), rtol=1e-3, atol=1e-3)


def test_kv_cache_checkpoint_is_the_reference_cpu_path(tiny):
    """Product `kv-cache` checkpoint (pure readable torch ops) == oracle.model:
    two independent restatements of qwen3_week2.py's CPU-capable path."""
    product = Qwen3ModelWeek2(tiny, checkpoint="kv-cache")
    oracle = ReferenceCpuModel(tiny)
    prompt = torch.tensor([[3, 14, 15, 92, 65, 35, 89]], dtype=torch.int32)
    pc, oc = product.create_kv_cache(), oracle.create_kv_cache()
    torch.testing.assert_close(product(prompt, 0, pc).float(), oracle(prompt, 0, oc).float(), rtol=0, atol=0)
    nxt = torch.tensor([[79]], dtype=torch.int32)
    torch.testing.assert_close(product(nxt, 7, pc).float(), oracle(nxt, 7, oc).float(), rtol=0, atol=0)


def test_full_kernel_path_tracks_the_reference_cpu_path(cpu_ext):
    """Week-3 paged model through (oracle-backed) kernels vs the reference CPU
    path on the committed tiny-d128 trace: same greedy tokens, close log-probs."""
    golden = json.loads((GOLDEN / "tiny_d128_greedy_trace.json").read_text())
    ns = synthetic_qwen3(golden["config"], seed=golden["seed"], realistic=True, max_position_embeddings=512)
    oracle_tokens, oracle_lp = greedy_decode(ReferenceCpuModel(ns), golden["prompt"], len(golden["tokens"]), return_logprobs=True)
    assert oracle_tokens == golden["tokens"]
    for lp, ids, vals in zip(oracle_lp, golden["top4_ids"], golden["top4_logprobs"]):
        assert [int(i) for i in torch.topk(lp, 4).indices] == ids
        torch.testing.assert_close(torch.topk(lp, 4).values, torch.tensor(vals), rtol=0, atol=2e-3)
    # Teacher-forced comparison (random weights produce near-ties, so free-running
    # greedy decoding may legitimately fork): feed the reference's tokens and compare
    # the log-probs of its top-4 candidates; demand the same argmax wherever the
    # reference's own top-2 margin is clear.
    model = Qwen3ModelWeek3(ns, page_size=8)
    cache = model.create_kv_cache()
    feed, offset = golden["prompt"], 0
    for step, (ids, vals, ref_tok) in enumerate(zip(golden["top4_ids"], golden["top4_logprobs"], golden["tokens"])):
        lp = logprobs(model(torch.tensor([feed], dtype=torch.int32), offset, cache, logits_to_keep=1)[0, -1])
        torch.testing.assert_close(lp[ids], torch.tensor(vals), rtol=0, atol=0.25)
        if vals[0] - vals[1] > 0.5:
            assert int(torch.argmax(lp)) == ref_tok, f"step {step}"
        offset += len(feed)
        feed = [ref_tok]
    for c in cache:
        c.release()
    assert all(pool.used_page_ids == set() for pool in model.page_pools)
    produced = greedy_generate_ids(model, golden["prompt"], 4)
    assert len(produced) == 4 and produced[0] == golden["tokens"][0]


def test_batched_decode_with_idle_slot_matches_single_requests(tiny, cpu_ext):
    """Continuous-batching step: B=3 slots (one idle) through BatchingKvCache ==
    each request alone (rows independent, idle row ignored)."""
    model = Qwen3ModelWeek3(tiny, page_size=4)
    prompts = {0: [1, 5, 7], 2: [9, 2, 4, 6, 8]}
    tables = [BatchingKvCache(3, max_seq_len=64) for _ in range(model.num_hidden_layers)]
    solo_logits = {}
    for slot, ids in prompts.items():
        cache = model.create_kv_cache()
        model(torch.tensor([ids], dtype=torch.int32), 0, cache, logits_to_keep=1)
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, slot)
        # reference answer: the same request continued alone
        alone = model.create_kv_cache()
        model(torch.tensor([ids], dtype=torch.int32), 0, alone, logits_to_keep=1)
        solo_logits[slot] = model(torch.tensor([[11]], dtype=torch.int32), len(ids), alone, logits_to_keep=1)
        for c in alone:
            c.release()
    batch_tokens = torch.tensor([[11], [0], [11]], dtype=torch.int32)
    out = model(batch_tokens, [3, 0, 5], tables, logits_to_keep=1)
    assert tuple(out.shape) == (3, 1, 128)
    for slot in prompts:
        torch.testing.assert_close(logprobs(out[slot]), logprobs(solo_logits[slot][0]), rtol=1e-3, atol=1e-3)


def test_dispatch_model_and_operator_dispatch_rules(tiny, cpu_ext, monkeypatch):
    assert isinstance(dispatch_model("qwen3-4b", tiny, week=2), Qwen3ModelWeek2)
    assert isinstance(dispatch_model("Qwen/Qwen3-0.6B-MLX-4bit", tiny, week=3, page_size=16), Qwen3ModelWeek3)
    with pytest.raises(ValueError, match="not supported"):
        dispatch_model("llama", tiny, week=3)
    # quantized_linear: rows <= 8 -> matvec entry (extension default use_simdgroup=True), else flags of the weight
    seen = []
    real = cpu_ext.quantized_matmul

    def spy(scales, biases, group_size, bits, a, b, transpose_b=False, use_simdgroup=True, use_split_k=False, stream=None):
        seen.append((a.shape[0], use_simdgroup, use_split_k))
        return real(scales, biases, group_size, bits, a, b, transpose_b, use_simdgroup, use_split_k)

    monkeypatch.setattr(cpu_ext, "quantized_matmul", spy)
    layer = tiny.model.layers[0].self_attn.q_proj
    w = QuantizedWeights.from_mlx_layer(layer, use_simdgroup_matmul=True, use_split_k_matmul=True)
    quantized_linear(torch.zeros(2, 4, 128, dtype=torch.bfloat16), w)
    quantized_linear(torch.zeros(3, 3, 128, dtype=torch.bfloat16), w)
    assert seen == [(8, True, False), (9, True, True)]
    with pytest.raises(ValueError, match="at most 8 input rows"):
        quantized_matvec_custom(w.scales, w.biases, 128, 4, torch.zeros(9, 128, dtype=torch.bfloat16), w.weight, True)
