"""Qwen3-MoE host logic without a GPU: the reference's day-6 tests restated on torch through the CPU stand-ins of the
extension, the bf16 oracle against a float64 referee, the sparse-layer rule, the synthetic MoE layout and the C ABI's
argument checks (which run before any device access)."""

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import moe as omoe
from oracle.model import greedy_decode
from tiny_llm_b200 import Moe, QuantizedWeights, grouped_expert_linear, route_topk
from tiny_llm_b200.qwen3_week3 import is_qwen3_moe_sparse_layer
from tiny_llm_b200.synthetic import make_args, quantize_w4, synthetic_qwen3


@pytest.fixture
def moe_ext(cpu_ext, monkeypatch):
    omoe.install(cpu_ext, monkeypatch)
    return cpu_ext


def quantized_experts(w: torch.Tensor) -> QuantizedWeights:
    parts = [quantize_w4(w[e]) for e in range(w.shape[0])]
    return QuantizedWeights(scales=torch.stack([p[1] for p in parts]), biases=torch.stack([p[2] for p in parts]), group_size=128, bits=4,
                            weight=torch.stack([p[0].view(torch.int32) for p in parts]).view(torch.uint32))


def quantized(w: torch.Tensor) -> QuantizedWeights:
    words, s, b = quantize_w4(w)
    return QuantizedWeights(scales=s, biases=b, group_size=128, bits=4, weight=words)


def dense(q: QuantizedWeights) -> torch.Tensor:
    return omoe.dense_experts(q) if q.weight.dim() == 3 else omoe.ops.dequantize_weights(q.weight, q.scales, q.biases, 128, 4).to(torch.bfloat16)


def test_task_1_grouped_expert_linear(moe_ext):
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(2, 3, 128, generator=g) * 0.25).to(torch.bfloat16)
    w = quantized_experts((torch.randn(3, 64, 128, generator=g) * 0.25).to(torch.bfloat16))
    ids = torch.tensor([[2, 0, 1], [1, 2, 0]], dtype=torch.int32)
    out = grouped_expert_linear(x, w, ids)
    assert out.shape == (2, 3, 64)
    wd = dense(w).to(torch.float32)
    expected = torch.einsum("abh,abkh->abk", x.to(torch.float32), wd[ids.to(torch.int64)])
    torch.testing.assert_close(out.to(torch.float32), expected, atol=2e-2, rtol=1.6e-2)


def test_task_2_router_topk(moe_ext):
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(2, 2, 128, generator=g) * 0.25).to(torch.bfloat16)
    router = quantized((torch.randn(4, 128, generator=g) * 0.25).to(torch.bfloat16))
    probs, ids, scores = route_topk(x, router, top_k=2)
    _, _, normalized = route_topk(x, router, top_k=2, norm_topk_prob=True)
    logits = (x.to(torch.float32) @ dense(router).to(torch.float32).T).to(torch.bfloat16)
    expected = torch.softmax(logits.to(torch.float32), dim=-1)
    assert probs.shape == (2, 2, 4) and ids.shape == (2, 2, 2) and scores.shape == (2, 2, 2)
    assert ids.tolist() == torch.sort(-expected, dim=-1, stable=True).indices[..., :2].tolist()
    exp_scores = torch.gather(expected, -1, ids.to(torch.int64))
    torch.testing.assert_close(probs.to(torch.float32), expected, atol=1e-2, rtol=1.6e-2)
    torch.testing.assert_close(scores.to(torch.float32), exp_scores, atol=1e-2, rtol=1.6e-2)
    torch.testing.assert_close(normalized.to(torch.float32), exp_scores / exp_scores.sum(-1, keepdim=True), atol=1e-2, rtol=1.6e-2)
    assert bool((torch.diff(scores.to(torch.float32), dim=-1) <= 0).all()), "descending order"


def moe_shapes(seed, E=3, I=128, H=128, k=2):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: (torch.randn(*s, generator=g) * 0.25).to(torch.bfloat16)
    return (quantized(r(E, H)), quantized_experts(r(E, I, H)), quantized_experts(r(E, I, H)), quantized_experts(r(E, H, I)), r(2, 3, H))


def test_task_3_moe(moe_ext):
    router, wg, wu, wd, x = moe_shapes(3)
    moe = Moe(router, wg, wu, wd, num_experts_per_tok=2, norm_topk_prob=True)
    out = moe(x)
    assert out.shape == x.shape
    # dense float oracle (Qwen3MoeSparseMoeBlock): silu(gate) * up, scores renormalised, all in fp32
    h = x.reshape(-1, 128).to(torch.float32)
    probs = torch.softmax((h @ dense(router).to(torch.float32).T).to(torch.bfloat16).to(torch.float32), dim=-1)
    top = torch.topk(probs, 2, dim=-1)
    scores = top.values / top.values.sum(-1, keepdim=True)
    expected = torch.zeros_like(h)
    for j in range(2):
        e = top.indices[:, j]
        gg = torch.einsum("th,tih->ti", h, dense(wg).to(torch.float32)[e])
        uu = torch.einsum("th,tih->ti", h, dense(wu).to(torch.float32)[e])
        expected += torch.einsum("ti,thi->th", gg * torch.sigmoid(gg) * uu, dense(wd).to(torch.float32)[e]) * scores[:, j : j + 1]
    torch.testing.assert_close(out.reshape(-1, 128).to(torch.float32), expected, atol=2e-2, rtol=1.6e-2)


def test_moe_block_tracks_the_bf16_oracle_on_the_stand_ins(moe_ext):
    router, wg, wu, wd, x = moe_shapes(4, E=8, I=128, H=256, k=2)
    moe = Moe(router, wg, wu, wd, num_experts_per_tok=2, norm_topk_prob=True)
    h = x.reshape(-1, 256)
    expected = omoe.moe_ref(h, dense(router), dense(wg), dense(wu), dense(wd), 2, True)
    torch.testing.assert_close(moe(h).to(torch.float32), expected.to(torch.float32), atol=3e-2, rtol=2e-2)


@pytest.mark.parametrize("norm", [False, True])
def test_bf16_oracle_within_a_bf16_bound_of_the_float64_referee(norm):
    g = torch.Generator().manual_seed(5)
    T, E, H, I, k = 32, 16, 256, 128, 4
    h = torch.randn(T, H, generator=g).to(torch.bfloat16)
    wg, wu = [(torch.randn(E, I, H, generator=g) * H**-0.5).to(torch.bfloat16) for _ in range(2)]
    wd = (torch.randn(E, H, I, generator=g) * I**-0.5).to(torch.bfloat16)
    logits = torch.randn(T, E, generator=g).to(torch.bfloat16)
    _, ids, scores = omoe.route_ref(logits, k, norm)
    ours = omoe.experts_ref(h, ids, scores, wg, wu, wd).to(torch.float64)
    ref = omoe.moe_f64(h, ids, scores, wg, wu, wd)
    # bf16 roundings of g, u, a, y, y*s and the sum: a few units of 2^-8 relative to the terms' magnitude
    assert float((ours - ref).abs().max()) <= 0.05 * float(ref.abs().max())
    if norm:
        torch.testing.assert_close(scores.to(torch.float64).sum(-1), torch.ones(T, dtype=torch.float64), atol=2e-2, rtol=0)


def test_route_ref_breaks_ties_to_the_lower_expert():
    logits = torch.tensor([[1.0, 3.0, 3.0, 0.0, 3.0]], dtype=torch.bfloat16)
    _, ids, _ = omoe.route_ref(logits, 3, False)
    assert ids.tolist() == [[1, 2, 4]]


def test_sparse_layer_rule():
    args = make_args("tiny-moe-d128")
    assert [is_qwen3_moe_sparse_layer(args, i) for i in range(2)] == [False, True]
    args = make_args("qwen3-30b-a3b")
    assert all(is_qwen3_moe_sparse_layer(args, i) for i in range(48))
    args = make_args("tiny-moe-d128", decoder_sparse_step=2, mlp_only_layers=[], num_hidden_layers=4)
    assert [is_qwen3_moe_sparse_layer(args, i) for i in range(4)] == [False, True, False, True]
    assert not any(is_qwen3_moe_sparse_layer(make_args("tiny-d128"), i) for i in range(2))
    assert not hasattr(make_args("qwen3-4b"), "num_experts"), "dense configs keep their keys"


def test_synthetic_moe_layout():
    m = synthetic_qwen3("tiny-moe-d128")
    assert hasattr(m.model.layers[0].mlp, "gate_proj")
    mlp = m.model.layers[1].mlp
    assert tuple(mlp.gate.weight.shape) == (8, 256 // 8)
    assert tuple(mlp.switch_mlp.gate_proj.weight.shape) == (8, 128, 256 // 8)
    assert tuple(mlp.switch_mlp.down_proj.scales.shape) == (8, 256, 1)
    assert mlp.switch_mlp.up_proj.weight.dtype == torch.uint32


def test_dense_synthetic_draws_are_unchanged():
    a, b = synthetic_qwen3("tiny-d128", seed=3), synthetic_qwen3("tiny-d128", seed=3)
    assert torch.equal(a.model.layers[1].mlp.down_proj.scales, b.model.layers[1].mlp.down_proj.scales)


def test_reference_moe_model_runs_a_dense_and_a_sparse_layer():
    ref = omoe.ReferenceCpuMoeModel(synthetic_qwen3("tiny-moe-d128", realistic=True, max_position_embeddings=64))
    assert isinstance(ref.blocks[1], omoe._MoeBlock) and not isinstance(ref.blocks[0], omoe._MoeBlock)
    out = greedy_decode(ref, [1, 2, 3, 4], 3)
    assert len(out) == 3 and all(0 <= t < 512 for t in out)


def test_week3_model_builds_moe_layers_on_the_stand_ins(moe_ext):
    from tiny_llm_b200 import Qwen3ModelWeek3

    model = Qwen3ModelWeek3(synthetic_qwen3("tiny-moe-d128"))
    assert isinstance(model.layers_inner[1].mlp, Moe) and not isinstance(model.layers_inner[0].mlp, Moe)
    moe = model.layers_inner[1].mlp
    assert tuple(moe.w_gate_up.weight.shape) == (8, 256, 256 // 8)


# ------------------------------------------------------------------ C ABI argument checks (no device) --
@pytest.mark.parametrize("E, k", [(257, 2), (300, 8), (8, 9), (4, 5), (0, 1), (8, 0)])
def test_moe_abi_rejects_expert_and_top_k_limits_without_a_device(E, k):
    assert ext._lib.tl_moe_topk(None, None, None, None, 4, E, k, 0, 2, None) == -1
    assert "moe_topk" in ext._lib.tl_last_error().decode()
    assert ext._lib.tl_moe_grouped_matmul(*([None] * 8), 4, k, E, 128, 128, 0, 2, None) == -1


def test_moe_abi_rejects_bad_shapes_without_a_device():
    lib = ext._lib
    assert lib.tl_moe_topk(None, None, None, None, 1, 8, 2, 0, 7, None) == -2  # dtype
    assert lib.tl_moe_group(None, -1, 8, 0, None, None, None, None) == -1
    assert lib.tl_moe_group(None, 4, 257, 0, None, None, None, None) == -1
    assert lib.tl_moe_gather(None, None, None, 0.0, None, 4, 0, 128, 2, None) == -1
    assert lib.tl_moe_combine(None, None, None, None, 0.0, None, None, 2, 9, 128, 2, None) == -1
    assert lib.tl_moe_grouped_matmul(*([None] * 8), 2, 2, 8, 100, 128, 0, 2, None) == -1  # N % 128
    assert lib.tl_moe_grouped_matmul(*([None] * 8), 2, 2, 8, 128, 136, 2, 2, None) == -1  # swiglu pairs need K % 16
    assert lib.tl_moe_grouped_matmul(*([None] * 8), 2, 2, 8, 128, 128, 0, 0, None) == -2  # fp32
    assert lib.tl_moe_tile_table_size(4, 300, 16) == -1


def test_moe_grouped_route_rule():
    bf = torch.bfloat16
    assert ext.moe_grouped_matmul_route(1, 8, 128, 2048, 1536, ext.EPI_SWIGLU_PAIRS, bf, 0, 0) == (ext.MOE_WGMMA, 16, 8)
    assert ext.moe_grouped_matmul_route(64, 8, 128, 2048, 1536, ext.EPI_SWIGLU_PAIRS, bf, 0, 0)[:2] == (ext.MOE_WGMMA, 16)
    assert ext.moe_grouped_matmul_route(512, 8, 128, 768, 2048, ext.EPI_NONE, bf, 0, 0)[:2] == (ext.MOE_WGMMA, 32)
    assert ext.moe_grouped_matmul_route(4096, 8, 128, 2048, 1536, ext.EPI_SWIGLU_PAIRS, bf, 0, 0)[:2] == (ext.MOE_WGMMA, 128)
    assert ext.moe_grouped_matmul_route(2, 3, 3, 128, 64, ext.EPI_NONE, bf, 0, 0) == (ext.MOE_CONTROL, 0, 0)  # 64-wide experts
    assert ext.moe_grouped_matmul_route(2, 2, 8, 128, 128, ext.EPI_NONE, bf, 8, 0)[0] == ext.MOE_CONTROL  # misaligned a
    assert ext.moe_grouped_matmul_route(2, 2, 8, 128, 128, ext.EPI_NONE, torch.float16, 0, 0)[0] == ext.MOE_WGMMA
    with pytest.raises(RuntimeError, match="top-k"):
        ext.moe_grouped_matmul_route(1, 4, 3, 128, 128, 0, bf, 0, 0)


def test_moe_shim_checks_run_before_the_device_check():
    with pytest.raises(RuntimeError, match="at most 256 experts"):
        ext.moe_topk(torch.zeros(2, 300, dtype=torch.bfloat16), 2)
    with pytest.raises(RuntimeError, match="top-k"):
        ext.moe_topk(torch.zeros(2, 8, dtype=torch.bfloat16), 9)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.moe_topk(torch.zeros(2, 8, dtype=torch.bfloat16), 2)
    with pytest.raises(RuntimeError, match="y must be"):
        ext.moe_combine(torch.zeros(5, 128, dtype=torch.bfloat16), torch.zeros(2, 2, dtype=torch.bfloat16))
    with pytest.raises(RuntimeError, match="incompatible"):
        ext.moe_grouped_matmul(torch.zeros(2, 64, 2), torch.zeros(2, 64, 2), torch.zeros(2, 64, 16, dtype=torch.int32),
                               torch.zeros(4, 128, dtype=torch.bfloat16), torch.zeros(3, dtype=torch.int32), None, 2)
