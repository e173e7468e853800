"""Synthetic Qwen3-shaped W4A16 checkpoints in the ``mlx_model`` duck type.

There is no network here, so benchmarks and tests run on random weights of the
right architecture (SURVEY.md section 8d).  The object mirrors what
``mlx_lm.load`` returns as far as the models look at it
(``src/tiny_llm_ref/qwen3_week3.py:225-313``; minimal fake at
``tests/utils.py:12-69``): ``.args`` plus
``.model.{embed_tokens, layers[i].{self_attn, mlp, *_layernorm}, norm}`` where
every quantised layer carries ``weight`` (packed u32), ``scales``, ``biases``,
``group_size`` and ``bits``.

Tensors are always generated on the CPU from a seeded generator (so the CPU
oracle and every GPU rank see identical bytes) and then moved to ``device``.
"""

from __future__ import annotations

from types import SimpleNamespace

import torch

GROUP_SIZE = 128
BITS = 4

# Published Qwen3 dense configs (hidden, layers, heads, kv heads, head dim, mlp).
CONFIGS = {
    "qwen3-4b": dict(hidden_size=2560, num_hidden_layers=36, num_attention_heads=32, num_key_value_heads=8, head_dim=128, intermediate_size=9728, vocab_size=151936),
    "qwen3-1.7b": dict(hidden_size=2048, num_hidden_layers=28, num_attention_heads=16, num_key_value_heads=8, head_dim=128, intermediate_size=6144, vocab_size=151936),
    "qwen3-0.6b": dict(hidden_size=1024, num_hidden_layers=28, num_attention_heads=16, num_key_value_heads=8, head_dim=128, intermediate_size=3072, vocab_size=151936),
    # small shapes for tests (same structure, every kernel family exercised)
    "tiny": dict(hidden_size=128, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=32, intermediate_size=256, vocab_size=128),
    "tiny-d128": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=128, intermediate_size=384, vocab_size=512),
    # Qwen3-MoE (published Qwen3-30B-A3B config: every layer sparse, untied head)
    "qwen3-30b-a3b": dict(hidden_size=2048, num_hidden_layers=48, num_attention_heads=32, num_key_value_heads=4, head_dim=128, intermediate_size=6144,
                          vocab_size=151936, num_experts=128, num_experts_per_tok=8, moe_intermediate_size=768, norm_topk_prob=True,
                          decoder_sparse_step=1, mlp_only_layers=[], tie_word_embeddings=False),
    # a dense layer and a sparse layer in one small model
    "tiny-moe-d128": dict(hidden_size=256, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, head_dim=128, intermediate_size=384,
                          vocab_size=512, num_experts=8, num_experts_per_tok=2, moe_intermediate_size=128, norm_topk_prob=True,
                          decoder_sparse_step=1, mlp_only_layers=[0]),
}


def make_args(name_or_dims, **overrides) -> SimpleNamespace:
    dims = dict(CONFIGS[name_or_dims]) if isinstance(name_or_dims, str) else dict(name_or_dims)
    dims.setdefault("rms_norm_eps", 1e-6)
    dims.setdefault("max_position_embeddings", 40960)
    dims.setdefault("rope_theta", 1000000)
    dims.setdefault("tie_word_embeddings", True)
    dims.update(overrides)
    if dims.get("num_experts", 0) > 0:  # Qwen3-MoE keys (mlx_lm qwen3_moe.ModelArgs)
        dims.setdefault("num_experts_per_tok", 8)
        dims.setdefault("moe_intermediate_size", dims["intermediate_size"])
        dims.setdefault("norm_topk_prob", True)
        dims.setdefault("decoder_sparse_step", 1)
        dims.setdefault("mlp_only_layers", [])
    return SimpleNamespace(**dims)


def quantize_w4(weight: torch.Tensor, group_size: int = GROUP_SIZE):
    """Plain affine min/max 4-bit quantiser (our own; ``mx.quantize`` is not in
    the reference tree).  Returns (packed uint32 [K, N/8], scales, biases) in
    the layout ``dequantize_weights`` decodes."""
    K, N = weight.shape
    assert N % group_size == 0
    groups = weight.to(torch.float32).reshape(K, N // group_size, group_size)
    lo = groups.amin(dim=-1, keepdim=True)
    hi = groups.amax(dim=-1, keepdim=True)
    scale = ((hi - lo) / 15.0).clamp_min(1e-8)
    scale_b = scale.to(torch.bfloat16)
    bias_b = lo.to(torch.bfloat16)
    codes = torch.round((groups - bias_b.to(torch.float32)) / scale_b.to(torch.float32)).clamp_(0, 15).to(torch.int64)
    codes = codes.reshape(K, N // 8, 8)
    shifts = torch.arange(0, 32, 4, dtype=torch.int64)
    words = (codes << shifts).sum(dim=-1)  # < 2^32
    words = torch.where(words >= 2**31, words - 2**32, words).to(torch.int32)
    return words.view(torch.uint32), scale_b.squeeze(-1).contiguous(), bias_b.squeeze(-1).contiguous()


def _random_layer(out_dim: int, in_dim: int, gen: torch.Generator) -> SimpleNamespace:
    """Random codes + signed scales; dequantised weights ~ N(0, 1/in_dim)
    (value = (q-7.5)*s + e with q uniform: var = 22.25*sigma^2)."""
    sigma = 1.0 / (4.717 * in_dim**0.5)
    words = torch.randint(-(2**31), 2**31, (out_dim, in_dim // 8), dtype=torch.int64, generator=gen).to(torch.int32)
    scales = (torch.randn(out_dim, in_dim // GROUP_SIZE, generator=gen) * sigma).to(torch.bfloat16)
    biases = (-7.5 * scales.to(torch.float32) + torch.randn(out_dim, in_dim // GROUP_SIZE, generator=gen) * sigma).to(torch.bfloat16)
    return SimpleNamespace(weight=words.view(torch.uint32), scales=scales, biases=biases, group_size=GROUP_SIZE, bits=BITS)


def _quantized_layer(out_dim: int, in_dim: int, gen: torch.Generator, std: float) -> SimpleNamespace:
    dense = torch.randn(out_dim, in_dim, generator=gen) * std
    words, scales, biases = quantize_w4(dense)
    return SimpleNamespace(weight=words, scales=scales, biases=biases, group_size=GROUP_SIZE, bits=BITS)


def _norm_weight(dim: int, gen: torch.Generator) -> SimpleNamespace:
    return SimpleNamespace(weight=(1.0 + 0.1 * torch.randn(dim, generator=gen)).to(torch.bfloat16))


def _empty_norm(dim: int, device) -> SimpleNamespace:
    return SimpleNamespace(weight=torch.empty((dim,), dtype=torch.bfloat16, device=device))


def _empty_layer(out_dim: int, in_dim: int, device) -> SimpleNamespace:
    return SimpleNamespace(
        weight=torch.empty((out_dim, in_dim // 8), dtype=torch.int32, device=device).view(torch.uint32),
        scales=torch.empty((out_dim, in_dim // GROUP_SIZE), dtype=torch.bfloat16, device=device),
        biases=torch.empty((out_dim, in_dim // GROUP_SIZE), dtype=torch.bfloat16, device=device),
        group_size=GROUP_SIZE,
        bits=BITS,
    )


def synthetic_qwen3(name_or_dims="qwen3-4b", seed: int = 0, device="cpu", realistic: bool = False, empty: bool = False,
                    **overrides) -> SimpleNamespace:
    """Random Qwen3-shaped model.  ``realistic=True`` quantises Gaussian dense
    weights with ``quantize_w4`` (slow, for small models); the default draws
    codes/scales directly, which is what the 4B-sized benchmarks use.
    ``empty=True`` only allocates (uninitialised, directly on ``device``): the
    receive side of the data-parallel weight broadcast."""
    args = make_args(name_or_dims, **overrides)
    gen = torch.Generator().manual_seed(seed)

    def layer(out_dim: int, in_dim: int) -> SimpleNamespace:
        if empty:
            return _empty_layer(out_dim, in_dim, device)
        if realistic:
            return _quantized_layer(out_dim, in_dim, gen, std=in_dim**-0.5)
        return _random_layer(out_dim, in_dim, gen)

    def norm(dim: int) -> SimpleNamespace:
        return _empty_norm(dim, device) if empty else _norm_weight(dim, gen)

    def experts(out_dim: int, in_dim: int) -> SimpleNamespace:
        """SwitchLinear layout: [E, out, in/8] codes, [E, out, in/128] scales and biases."""
        parts = [layer(out_dim, in_dim) for _ in range(args.num_experts)]
        stacked = {key: torch.stack([getattr(p, key).view(torch.int32) if key == "weight" else getattr(p, key) for p in parts])
                   for key in ("weight", "scales", "biases")}
        stacked["weight"] = stacked["weight"].view(torch.uint32)
        return SimpleNamespace(**stacked, group_size=GROUP_SIZE, bits=BITS)

    def mlp(index: int) -> SimpleNamespace:
        sparse = (getattr(args, "num_experts", 0) > 0 and index not in args.mlp_only_layers
                  and (index + 1) % args.decoder_sparse_step == 0)  # qwen3_week3.is_qwen3_moe_sparse_layer
        if sparse:
            inter = args.moe_intermediate_size
            return SimpleNamespace(
                gate=layer(args.num_experts, args.hidden_size),
                switch_mlp=SimpleNamespace(gate_proj=experts(inter, args.hidden_size), up_proj=experts(inter, args.hidden_size),
                                           down_proj=experts(args.hidden_size, inter)),
            )
        return SimpleNamespace(
            gate_proj=layer(args.intermediate_size, args.hidden_size),
            up_proj=layer(args.intermediate_size, args.hidden_size),
            down_proj=layer(args.hidden_size, args.intermediate_size),
        )

    q_width = args.num_attention_heads * args.head_dim
    kv_width = args.num_key_value_heads * args.head_dim
    layers = []
    for index in range(args.num_hidden_layers):
        layers.append(
            SimpleNamespace(
                self_attn=SimpleNamespace(
                    q_proj=layer(q_width, args.hidden_size),
                    k_proj=layer(kv_width, args.hidden_size),
                    v_proj=layer(kv_width, args.hidden_size),
                    o_proj=layer(args.hidden_size, q_width),
                    q_norm=norm(args.head_dim),
                    k_norm=norm(args.head_dim),
                ),
                mlp=mlp(index),
                input_layernorm=norm(args.hidden_size),
                post_attention_layernorm=norm(args.hidden_size),
            )
        )
    model = SimpleNamespace(
        args=args,
        model=SimpleNamespace(embed_tokens=layer(args.vocab_size, args.hidden_size), layers=layers, norm=norm(args.hidden_size)),
    )
    if not args.tie_word_embeddings:
        model.lm_head = layer(args.vocab_size, args.hidden_size)
    return model if empty else to_device(model, device)


def to_device(node, device):
    """Move every tensor of the namespace tree to ``device`` (in place)."""
    if isinstance(node, SimpleNamespace):
        for key, value in vars(node).items():
            setattr(node, key, to_device(value, device))
        return node
    if isinstance(node, list):
        return [to_device(item, device) for item in node]
    if isinstance(node, torch.Tensor):
        return node.to(device)
    return node


def named_tensors(node, prefix=""):
    """Depth-first (name, tensor) walk in a deterministic order - the order the
    data-parallel launcher broadcasts weights in."""
    if isinstance(node, SimpleNamespace):
        for key in sorted(vars(node)):
            yield from named_tensors(getattr(node, key), f"{prefix}{key}.")
    elif isinstance(node, list):
        for index, item in enumerate(node):
            yield from named_tensors(item, f"{prefix}{index}.")
    elif isinstance(node, torch.Tensor):
        yield prefix[:-1], node


def weight_stream_bytes(args) -> int:
    """Packed bytes one decode token must stream (projections of every layer +
    tied head): 0.53125 B per weight = N/2 codes + 4 B of scale/bias per 128
    (book/src/week2-03-quantize-model.md:179-181)."""
    q_width = args.num_attention_heads * args.head_dim
    kv_width = args.num_key_value_heads * args.head_dim
    per_layer = args.hidden_size * (q_width + 2 * kv_width) + q_width * args.hidden_size + 3 * args.hidden_size * args.intermediate_size
    weights = args.num_hidden_layers * per_layer + args.vocab_size * args.hidden_size
    return weights * 17 // 32
