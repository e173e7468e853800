"""Week-2 Qwen3 model with its cumulative optimisation checkpoints
(``src/tiny_llm_ref/qwen3_week2.py``).

``checkpoint`` selects how far along the course the model is: ``"kv-cache"``
runs dense bf16 weights through the readable operators, each later name turns
on one more CUDA kernel family (``WEEK2_CHECKPOINTS``, qwen3_week2.py:19-28).
The KV cache is the dense concat cache; the fused decode-attention kernel is
used only for ``L <= 2`` and ``S <= 256`` (qwen3_week2.py:30-31,124-136),
everything else takes the fp32 readable attention (:138-144).
"""

from __future__ import annotations

from typing import Any

import torch

from .attention import scaled_dot_product_attention_grouped
from .basics import linear, silu
from .embedding import Embedding, QuantizedEmbedding
from .kv_cache import TinyKvCache
from .layer_norm import RMSNorm
from .positional_encoding import RoPE
from .quantize import QuantizedWeights, dequantize_linear, quantized_linear
from .rope_scaling import parse_rope_scaling
from .week2_kernels import FastRMSNorm, FastRoPE, decode_attention_custom, swiglu

WEEK2_CHECKPOINTS = (
    "kv-cache",
    "quantized-matvec",
    "rmsnorm",
    "rope",
    "swiglu",
    "decode-attention",
    "simd-matmul",
    "split-k",
)

DECODE_ATTENTION_MAX_CONTEXT = 256
DECODE_ATTENTION_MAX_QUERY = 2


def _linear(x: torch.Tensor, weight: torch.Tensor | QuantizedWeights) -> torch.Tensor:
    return quantized_linear(x, weight) if isinstance(weight, QuantizedWeights) else linear(x, weight)


def _readable_rope_offset(offset, sequence_length: int):
    """Readable RoPE wants slices (qwen3_week2.py:39-50)."""
    if isinstance(offset, int):
        return slice(offset, offset + sequence_length)
    values = offset if isinstance(offset, list) else offset.tolist()
    if not isinstance(values, list):
        values = [values]
    return [slice(v, v + sequence_length) for v in values]


class Qwen3MultiHeadAttention:
    """qwen3_week2.py:53-146."""

    def __init__(
        self,
        hidden_size: int,
        num_heads: int,
        num_kv_heads: int,
        head_dim: int,
        wq,
        wk,
        wv,
        wo,
        q_norm: torch.Tensor,
        k_norm: torch.Tensor,
        max_seq_len: int = 32768,
        theta: int = 1000000,
        rms_norm_eps: float = 1e-5,
        use_fast_rms_norm: bool = True,
        use_fast_rope: bool = True,
        use_decode_attention: bool = True,
    ):
        assert hidden_size % num_heads == 0, f"hidden_size {hidden_size} must be divisible by num_heads {num_heads}"
        assert num_heads % num_kv_heads == 0, f"num_heads {num_heads} must be divisible by num_kv_heads {num_kv_heads}"
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.num_kv_heads = num_kv_heads
        self.head_dim = head_dim
        self.scale = head_dim**-0.5
        self.wq, self.wk, self.wv, self.wo = wq, wk, wv, wo
        self.use_fast_rope = use_fast_rope
        self.use_decode_attention = use_decode_attention
        norm = FastRMSNorm if use_fast_rms_norm else RMSNorm
        self.rope = (FastRoPE if use_fast_rope else RoPE)(head_dim, max_seq_len, theta)
        self.q_norm = norm(head_dim, q_norm, eps=rms_norm_eps)
        self.k_norm = norm(head_dim, k_norm, eps=rms_norm_eps)

    def __call__(self, x, offsets, cache: TinyKvCache, mask=None):
        B, L, _ = x.shape
        q = self.q_norm(_linear(x, self.wq).reshape(B, L, self.num_heads, self.head_dim))
        k = self.k_norm(_linear(x, self.wk).reshape(B, L, self.num_kv_heads, self.head_dim))
        v = _linear(x, self.wv).reshape(B, L, self.num_kv_heads, self.head_dim)
        where = offsets if self.use_fast_rope else _readable_rope_offset(offsets, L)
        q = self.rope(q, offset=where).transpose(1, 2)
        k = self.rope(k, offset=where).transpose(1, 2)
        v = v.transpose(1, 2)
        k, v, _, mask = cache.update_and_fetch(k, v, mask_length=L, mask=mask)
        fused = (
            self.use_decode_attention
            and L <= DECODE_ATTENTION_MAX_QUERY
            and k.shape[-2] <= DECODE_ATTENTION_MAX_CONTEXT
            and not isinstance(mask, torch.Tensor)
        )
        if fused:
            y = decode_attention_custom(q, k, v, scale=self.scale, mask=mask)
        else:
            y = scaled_dot_product_attention_grouped(
                q.to(torch.float32), k.to(torch.float32), v.to(torch.float32), scale=self.scale, mask=mask
            ).to(x.dtype)
        return _linear(y.transpose(1, 2).reshape(B, L, self.num_heads * self.head_dim), self.wo)


class Qwen3MLP:
    """qwen3_week2.py:149-170."""

    def __init__(self, dim: int, hidden_dim: int, w_gate, w_up, w_down, use_fast_swiglu: bool = True):
        self.dim = dim
        self.hidden_dim = hidden_dim
        self.w_gate, self.w_up, self.w_down = w_gate, w_up, w_down
        self.use_fast_swiglu = use_fast_swiglu

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        gate, up = _linear(x, self.w_gate), _linear(x, self.w_up)
        return _linear(swiglu(gate, up) if self.use_fast_swiglu else silu(gate) * up, self.w_down)


class Qwen3TransformerBlock:
    """qwen3_week2.py:173-248."""

    def __init__(
        self,
        num_attention_heads: int,
        num_kv_heads: int,
        hidden_size: int,
        head_dim: int,
        intermediate_size: int,
        rms_norm_eps: float,
        wq,
        wk,
        wv,
        wo,
        q_norm: torch.Tensor,
        k_norm: torch.Tensor,
        w_gate,
        w_up,
        w_down,
        w_input_layernorm: torch.Tensor,
        w_post_attention_layernorm: torch.Tensor,
        max_seq_len: int = 32768,
        theta: int = 1000000,
        use_fast_rms_norm: bool = True,
        use_fast_rope: bool = True,
        use_fast_swiglu: bool = True,
        use_decode_attention: bool = True,
    ):
        self.num_attention_heads = num_attention_heads
        self.hidden_size = hidden_size
        self.mlp = Qwen3MLP(hidden_size, intermediate_size, w_gate, w_up, w_down, use_fast_swiglu=use_fast_swiglu)
        norm = FastRMSNorm if use_fast_rms_norm else RMSNorm
        self.input_layernorm = norm(hidden_size, w_input_layernorm, eps=rms_norm_eps)
        self.post_attention_layernorm = norm(hidden_size, w_post_attention_layernorm, eps=rms_norm_eps)
        self.self_attn = Qwen3MultiHeadAttention(
            hidden_size=hidden_size,
            num_heads=num_attention_heads,
            num_kv_heads=num_kv_heads,
            head_dim=head_dim,
            wq=wq,
            wk=wk,
            wv=wv,
            wo=wo,
            q_norm=q_norm,
            k_norm=k_norm,
            max_seq_len=max_seq_len,
            theta=theta,
            rms_norm_eps=rms_norm_eps,
            use_fast_rms_norm=use_fast_rms_norm,
            use_fast_rope=use_fast_rope,
            use_decode_attention=use_decode_attention,
        )

    def __call__(self, x, offset, cache: TinyKvCache, mask=None):
        h = x + self.self_attn(self.input_layernorm(x), offset, cache, mask)
        return h + self.mlp(self.post_attention_layernorm(h))


class Qwen3ModelWeek2:
    """qwen3_week2.py:251-392."""

    def __init__(self, mlx_model: Any, checkpoint: str = "split-k"):
        if checkpoint not in WEEK2_CHECKPOINTS:
            raise ValueError(f"unknown Week 2 checkpoint {checkpoint!r}; choose one of {WEEK2_CHECKPOINTS}")
        level = WEEK2_CHECKPOINTS.index(checkpoint)

        def reached(name: str) -> bool:
            return level >= WEEK2_CHECKPOINTS.index(name)

        self.checkpoint = checkpoint
        args = mlx_model.args
        if parse_rope_scaling(getattr(args, "rope_scaling", None), args.max_position_embeddings) is not None:
            raise ValueError("the Week 2 model does not implement RoPE scaling (YaRN); load this config with Qwen3ModelWeek3")
        self.num_hidden_layers = args.num_hidden_layers
        self.hidden_size = args.hidden_size
        self.vocab_size = args.vocab_size
        self.use_fast_rope = reached("rope")
        self.precision = torch.bfloat16
        packed_weights = reached("quantized-matvec")
        fast_norm = reached("rmsnorm")

        def weight_of(layer: Any):
            if packed_weights:
                return QuantizedWeights.from_mlx_layer(
                    layer, use_simdgroup_matmul=reached("simd-matmul"), use_split_k_matmul=reached("split-k")
                )
            return dequantize_linear(layer).to(torch.bfloat16)

        table = weight_of(mlx_model.model.embed_tokens)
        emb_cls = QuantizedEmbedding if isinstance(table, QuantizedWeights) else Embedding
        self.embedding = emb_cls(vocab_size=self.vocab_size, embedding_dim=self.hidden_size, weight=table)
        self.layers_inner = []
        for layer in mlx_model.model.layers[: self.num_hidden_layers]:
            attn, mlp = layer.self_attn, layer.mlp
            self.layers_inner.append(
                Qwen3TransformerBlock(
                    num_attention_heads=args.num_attention_heads,
                    num_kv_heads=args.num_key_value_heads,
                    hidden_size=args.hidden_size,
                    head_dim=args.head_dim,
                    intermediate_size=args.intermediate_size,
                    rms_norm_eps=args.rms_norm_eps,
                    wq=weight_of(attn.q_proj),
                    wk=weight_of(attn.k_proj),
                    wv=weight_of(attn.v_proj),
                    wo=weight_of(attn.o_proj),
                    q_norm=attn.q_norm.weight,
                    k_norm=attn.k_norm.weight,
                    w_gate=weight_of(mlp.gate_proj),
                    w_up=weight_of(mlp.up_proj),
                    w_down=weight_of(mlp.down_proj),
                    w_input_layernorm=layer.input_layernorm.weight,
                    w_post_attention_layernorm=layer.post_attention_layernorm.weight,
                    max_seq_len=args.max_position_embeddings,
                    theta=args.rope_theta,
                    use_fast_rms_norm=fast_norm,
                    use_fast_rope=self.use_fast_rope,
                    use_fast_swiglu=reached("swiglu"),
                    use_decode_attention=reached("decode-attention"),
                )
            )
        self.norm = (FastRMSNorm if fast_norm else RMSNorm)(args.hidden_size, weight=mlx_model.model.norm.weight, eps=args.rms_norm_eps)
        self.w_lm_head = None if args.tie_word_embeddings else weight_of(mlx_model.lm_head)
        self.mlx_model = mlx_model

    def create_kv_cache(self) -> list[TinyKvCache]:
        from .kv_cache import TinyKvFullCache

        return [TinyKvFullCache() for _ in range(self.num_hidden_layers)]

    def __call__(self, inputs, offset, cache: list[TinyKvCache], logits_to_keep: int | None = None):
        if isinstance(offset, int):
            for index, layer_cache in enumerate(cache):
                have = getattr(layer_cache, "offset", None)
                if have is not None and have != offset:
                    raise ValueError(f"layer {index} cache offset {have} does not match model offset {offset}")
        h = self.embedding(inputs)
        mask = None if inputs.shape[1] == 1 else "causal"
        if not getattr(self, "use_fast_rope", True):
            where = offset
        elif isinstance(offset, int):
            where = torch.full((inputs.shape[0],), offset, dtype=torch.int32, device=h.device)
        elif isinstance(offset, list):
            where = torch.tensor(offset, dtype=torch.int32, device=h.device)
        else:
            where = offset
        for block, layer_cache in zip(self.layers_inner, cache):
            h = block(h, where, layer_cache, mask=mask)
        if logits_to_keep is not None:
            if logits_to_keep <= 0:
                raise ValueError("logits_to_keep must be positive")
            h = h[:, -logits_to_keep:, :]
        h = self.norm(h)
        return _linear(h, self.w_lm_head) if self.w_lm_head is not None else self.embedding.as_linear(h)
