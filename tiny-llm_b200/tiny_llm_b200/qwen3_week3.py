"""Week-3 Qwen3 model: W4A16 projections, fused norm/RoPE/SwiGLU kernels and
paged-KV attention (``src/tiny_llm_ref/qwen3_week3.py``).

Constructor, ``create_kv_cache`` and ``__call__(inputs, offset, cache,
logits_to_keep)`` keep the reference's contract; the only contact with weights
is the ``mlx_model`` duck type (``.args`` + ``.model.layers[i]...`` with each
quantised layer exposing ``weight, scales, biases, group_size, bits``;
qwen3_week3.py:225-313), so synthetic ``SimpleNamespace`` models are first
class inputs.  Tensors are torch tensors living on the GPU.
"""

from __future__ import annotations

from typing import Any

import torch

from .attention import paged_attention
from .embedding import QuantizedEmbedding
from .kv_cache import TinyKvCache
from .moe import Moe
from .paged_kv_cache import TinyKvPagedCache, TinyKvPagedPool
from .quantize import QuantizedWeights, quantized_linear
from .week2_kernels import (
    FastRMSNorm,
    FastRoPE,
    decode_attention_custom,
    residual_add,
    scaled_dot_product_attention,
    swiglu,
)


class Qwen3MultiHeadAttention:
    """qwen3_week3.py:20-121."""

    def __init__(
        self,
        hidden_size: int,
        num_heads: int,
        num_kv_heads: int,
        head_dim: int,
        wq: QuantizedWeights,
        wk: QuantizedWeights,
        wv: QuantizedWeights,
        wo: QuantizedWeights,
        q_norm: torch.Tensor,
        k_norm: torch.Tensor,
        max_seq_len: int = 32768,
        theta: int = 1000000,
        rms_norm_eps: float = 1e-5,
        use_paged_attention: bool = True,
    ):
        assert num_heads % num_kv_heads == 0, f"num_heads {num_heads} must be divisible by num_kv_heads {num_kv_heads}"
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.num_kv_heads = num_kv_heads
        self.head_dim = head_dim
        self.scale = head_dim**-0.5
        self.wq, self.wk, self.wv, self.wo = wq, wk, wv, wo
        self.rope = FastRoPE(head_dim, max_seq_len, theta)
        self.q_norm = FastRMSNorm(head_dim, q_norm, eps=rms_norm_eps)
        self.k_norm = FastRMSNorm(head_dim, k_norm, eps=rms_norm_eps)
        self.use_paged_attention = use_paged_attention

    def __call__(self, x, offsets, cache: TinyKvCache, mask=None):
        B, L, _ = x.shape
        q = quantized_linear(x, self.wq).reshape(B, L, self.num_heads, self.head_dim)
        k = quantized_linear(x, self.wk).reshape(B, L, self.num_kv_heads, self.head_dim)
        q = self.q_norm(q)
        k = self.k_norm(k)
        v = quantized_linear(x, self.wv).reshape(B, L, self.num_kv_heads, self.head_dim)
        q = self.rope(q, offset=offsets)
        k = self.rope(k, offset=offsets)
        q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)  # [B, H, L, D]

        if self.use_paged_attention:
            # Append first, attend second: context_lens is the post-append length.
            meta = cache.update_and_fetch_paged(k, v, mask_length=L, mask=mask)
            y = paged_attention(
                q,
                meta.key_pages,
                meta.value_pages,
                meta.block_table,
                meta.context_lens,
                meta.page_size,
                scale=self.scale,
                mask=meta.mask,
                block_table_host=meta.block_table_host,
                context_lens_host=meta.context_lens_host,
            )
        else:
            keys, values, _, mask = cache.update_and_fetch(k, v, mask_length=L, mask=mask)
            if L <= 8 and keys.shape[-2] <= 256:
                y = decode_attention_custom(q, keys, values, scale=self.scale, mask=mask)
            else:
                y = scaled_dot_product_attention(q, keys, values, scale=self.scale, mask=mask)
        y = y.transpose(1, 2).reshape(B, L, self.num_heads * self.head_dim)
        return quantized_linear(y, self.wo)


class Qwen3MLP:
    """qwen3_week3.py:124-146 - down(swiglu(gate(x), up(x)))."""

    def __init__(self, dim: int, hidden_dim: int, w_gate: QuantizedWeights, w_up: QuantizedWeights, w_down: QuantizedWeights):
        self.dim = dim
        self.hidden_dim = hidden_dim
        self.w_gate, self.w_up, self.w_down = w_gate, w_up, w_down

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        return quantized_linear(swiglu(quantized_linear(x, self.w_gate), quantized_linear(x, self.w_up)), self.w_down)


class Qwen3TransformerBlock:
    """qwen3_week3.py:149-207."""

    def __init__(
        self,
        num_attention_heads: int,
        num_kv_heads: int,
        hidden_size: int,
        head_dim: int,
        rms_norm_eps: float,
        wq: QuantizedWeights,
        wk: QuantizedWeights,
        wv: QuantizedWeights,
        wo: QuantizedWeights,
        q_norm: torch.Tensor,
        k_norm: torch.Tensor,
        w_input_layernorm: torch.Tensor,
        w_post_attention_layernorm: torch.Tensor,
        mlp: Qwen3MLP | Moe,
        max_seq_len: int = 32768,
        theta: int = 1000000,
        use_paged_attention: bool = True,
    ):
        self.num_attention_heads = num_attention_heads
        self.hidden_size = hidden_size
        self.mlp = mlp
        self.input_layernorm = FastRMSNorm(hidden_size, w_input_layernorm, eps=rms_norm_eps)
        self.post_attention_layernorm = FastRMSNorm(hidden_size, w_post_attention_layernorm, eps=rms_norm_eps)
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
            use_paged_attention=use_paged_attention,
        )

    def __call__(self, x, offset, cache: TinyKvCache, mask=None):
        h = residual_add(x, self.self_attn(self.input_layernorm(x), offset, cache, mask))
        return residual_add(h, self.mlp(self.post_attention_layernorm(h)))


def is_qwen3_moe_sparse_layer(args: Any, layer_idx: int) -> bool:
    """qwen3_week3.py:210-215."""
    return (
        getattr(args, "num_experts", 0) > 0
        and layer_idx not in getattr(args, "mlp_only_layers", [])
        and (layer_idx + 1) % getattr(args, "decoder_sparse_step", 1) == 0
    )


class Qwen3ModelWeek3:
    """qwen3_week3.py:218-338."""

    def __init__(self, mlx_model: Any, page_size: int = 128, enable_paged_attention: bool = True):
        args = mlx_model.args
        self.num_hidden_layers = args.num_hidden_layers
        self.hidden_size = args.hidden_size
        self.vocab_size = args.vocab_size
        self.page_size = page_size
        # One physical pool per layer; page ids are layer-local (as in the kernels).
        self.page_pools = [TinyKvPagedPool(page_size=page_size) for _ in range(self.num_hidden_layers)]
        self.precision = torch.bfloat16

        def packed(layer: Any) -> QuantizedWeights:
            return QuantizedWeights.from_mlx_layer(layer, use_simdgroup_matmul=True, use_split_k_matmul=True)

        self.embedding = QuantizedEmbedding(
            vocab_size=self.vocab_size,
            embedding_dim=self.hidden_size,
            weight=packed(mlx_model.model.embed_tokens),
            use_custom_kernel=True,
        )
        self.layers_inner = []
        for index, layer in enumerate(mlx_model.model.layers[: self.num_hidden_layers]):
            attn = layer.self_attn
            if is_qwen3_moe_sparse_layer(args, index):
                switch = layer.mlp.switch_mlp
                mlp = Moe(
                    w_router=packed(layer.mlp.gate),
                    w_gate=packed(switch.gate_proj),
                    w_up=packed(switch.up_proj),
                    w_down=packed(switch.down_proj),
                    num_experts_per_tok=args.num_experts_per_tok,
                    norm_topk_prob=args.norm_topk_prob,
                )
            else:
                mlp = Qwen3MLP(
                    args.hidden_size,
                    args.intermediate_size,
                    packed(layer.mlp.gate_proj),
                    packed(layer.mlp.up_proj),
                    packed(layer.mlp.down_proj),
                )
            self.layers_inner.append(
                Qwen3TransformerBlock(
                    num_attention_heads=args.num_attention_heads,
                    num_kv_heads=args.num_key_value_heads,
                    hidden_size=args.hidden_size,
                    head_dim=args.head_dim,
                    rms_norm_eps=args.rms_norm_eps,
                    wq=packed(attn.q_proj),
                    wk=packed(attn.k_proj),
                    wv=packed(attn.v_proj),
                    wo=packed(attn.o_proj),
                    q_norm=attn.q_norm.weight,
                    k_norm=attn.k_norm.weight,
                    w_input_layernorm=layer.input_layernorm.weight,
                    w_post_attention_layernorm=layer.post_attention_layernorm.weight,
                    mlp=mlp,
                    max_seq_len=args.max_position_embeddings,
                    theta=args.rope_theta,
                    use_paged_attention=enable_paged_attention,
                )
            )
        self.norm = FastRMSNorm(args.hidden_size, weight=mlx_model.model.norm.weight, eps=args.rms_norm_eps)
        self.w_lm_head = None if args.tie_word_embeddings else packed(mlx_model.lm_head)
        self.mlx_model = mlx_model
        # CUDA runtime: decode steps (L == 1) of CUDA-resident paged requests are replayed
        # from a captured CUDA graph instead of ~500 per-operator dispatches (engine.py).
        # None = automatic (on for CUDA inputs), False = always operator by operator.
        self.use_decode_graph: bool | None = None
        self.decode_graph_max_seq_len = 8192
        self._decode_engines: dict = {}
        self._applies_memo = None
        # CUDA runtime: chunked-prefill steps (B == 1, 1 < L <= prefill_graph_len) of CUDA-resident paged requests
        # replay a captured chunk graph too (engine.PrefillEngine).  0 disables; None = automatic (128, the scheduler's
        # default prefill_step) once a decode engine exists, i.e. once the page slabs have been reserved.
        self.prefill_graph_len: int | None = None
        self._prefill_engines: dict = {}
        self._verify_engines: dict = {}
        self._packed_layers: list | None = None
        self._paged = enable_paged_attention

    def create_kv_cache(self) -> list[TinyKvCache]:
        """One logical cache per layer, all sharing that layer's pool."""
        return [TinyKvPagedCache(pool=pool) for pool in self.page_pools]

    # ---- CUDA-graph decode path ------------------------------------------------
    def packed_layers(self) -> list:
        """Per layer, the q|k|v and gate|up weights of the graph engines' fused launches (``engine.pack_layers``).  Built on
        first use and shared by every engine of this model: one copy is 1.25 GB at Qwen3-4B."""
        if self._packed_layers is None:
            from .engine import pack_layers

            self._packed_layers = pack_layers(self)
        return self._packed_layers

    def decode_engine(self, batch_size: int, max_seq_len: int | None = None, device=None):
        """The (cached) graph engine for ``batch_size`` decode slots."""
        from .engine import DecodeEngine

        limit = max_seq_len or self.decode_graph_max_seq_len
        key = (batch_size, limit)
        if key not in self._decode_engines:
            dev = device if device is not None else self.embedding.weight.scales.device
            engine = DecodeEngine(self, batch_size, limit, dev)
            engine.reserve_pools((batch_size + 1) * engine.max_pages + 1)
            self._decode_engines[key] = engine
        return self._decode_engines[key]

    def verify_applies(self, device=None) -> bool:
        """Whether ``verify_engine`` runs on this model: CUDA paged caches and the shapes of the fused decode path."""
        from .engine import VerifyEngine

        dev = device if device is not None else self.embedding.weight.scales.device
        return (self._paged and self.use_decode_graph is not False and torch.device(dev).type == "cuda"
                and VerifyEngine.supported(self, dev, self.decode_graph_max_seq_len))

    def verify_engine(self, rows: int, device=None):
        """The (cached) graph of one speculative verify pass over ``rows`` tokens of one request (``engine.VerifyEngine``).
        It uses the ``max_seq_len`` of the B = 1 decode engine that ``model(...)`` runs a single request with (so the
        attention splits match) and that engine's page reservation (the slabs do not move when the two alternate)."""
        from .engine import VerifyEngine

        limit = self.decode_graph_max_seq_len
        key = (rows, limit)
        if key not in self._verify_engines:
            dev = device if device is not None else self.embedding.weight.scales.device
            self.decode_engine(1, limit, dev)
            self._verify_engines[key] = VerifyEngine(self, rows, limit, dev)
        return self._verify_engines[key]

    def _graph_decode_applies(self, inputs, cache) -> bool:
        if self.use_decode_graph is False or not self._paged or inputs.dim() != 2 or inputs.shape[1] != 1 or not inputs.is_cuda:
            return False
        from .kv_cache import BatchingKvCache

        B = inputs.shape[0]
        first = cache[0]
        if isinstance(first, BatchingKvCache):
            slots0 = first.kv_caches
        elif type(first) is TinyKvPagedCache and B == 1:
            slots0 = [first]
        else:
            return False
        # Deep check (every layer, every slot) only when the set of requests changed; afterwards one
        # identity comparison plus the length limit on the layer-0 objects (layers advance in lockstep).
        memo = self._applies_memo
        if memo is None or memo[0] is not cache or memo[1] != slots0 or memo[2] != B:
            for entry, pool in zip(cache, self.page_pools):
                if isinstance(entry, BatchingKvCache):
                    slots = entry.kv_caches
                    if entry.max_active_requests != B:
                        return False
                elif type(entry) is TinyKvPagedCache and B == 1:
                    slots = [entry]
                else:
                    return False
                for slot in slots:
                    if slot is None:
                        continue
                    if type(slot) is not TinyKvPagedCache or slot.pool is not pool:
                        return False
                    if pool._key_pages is not None and pool._key_pages.dtype != torch.bfloat16:
                        return False
            self._applies_memo = (cache, list(slots0), B)
        limit = self._graph_limit(cache)
        for slot in slots0:
            if slot is not None and slot.logical_offset() + 1 > limit:
                return False
        return True

    def _graph_limit(self, cache) -> int:
        """Longest request the decode engine of this call must hold: the scheduler's own
        ``max_seq_len`` when it states one (rounded up to whole pages), capped by
        ``decode_graph_max_seq_len``.  Round 1 always reserved for 8192 tokens per slot: 76 GB of
        pages for 64 slots of Qwen3-4B regardless of the batcher's limit (ADVICE round 1)."""
        from .kv_cache import BatchingKvCache

        limit = self.decode_graph_max_seq_len
        first = cache[0]
        if isinstance(first, BatchingKvCache) and first.max_seq_len is not None:
            pages = (first.max_seq_len + self.page_size - 1) // self.page_size
            limit = min(limit, pages * self.page_size)
        return limit

    def _graph_decode(self, inputs, offset, cache, logits_to_keep):
        from .kv_cache import BatchingKvCache

        if logits_to_keep is not None and logits_to_keep <= 0:
            raise ValueError("logits_to_keep must be positive")
        B = inputs.shape[0]
        if isinstance(offset, int):
            offsets = [offset] * B
        elif isinstance(offset, torch.Tensor):
            offsets = offset.reshape(-1).tolist()
            offsets = offsets * B if len(offsets) == 1 else offsets
        else:
            offsets = list(offset)
        first = cache[0]
        if isinstance(first, BatchingKvCache):
            if not any(slot is not None for slot in first.kv_caches):
                raise ValueError("Cannot build paged metadata without active requests")
            if first.max_seq_len is not None and any(s is not None and s.logical_offset() + 1 > first.max_seq_len for s in first.kv_caches):
                raise ValueError("Paged batch append exceeds max_seq_len")
        engine = self.decode_engine(B, self._graph_limit(cache))
        logits, _ = engine.step(inputs, offsets, cache)
        attn = self.layers_inner[0].self_attn
        for entry in cache:
            if isinstance(entry, BatchingKvCache):
                entry.HD = (attn.num_kv_heads, attn.head_dim)
                entry.last_batch_bytes = 0
        return logits.clone()

    def prefill_engine(self, chunk: int, max_seq_len: int | None = None, device=None):
        from .engine import PrefillEngine

        limit = max_seq_len or self.decode_graph_max_seq_len
        key = (chunk, limit)
        if key not in self._prefill_engines:
            dev = device if device is not None else self.embedding.weight.scales.device
            self._prefill_engines[key] = PrefillEngine(self, chunk, limit, dev)
        return self._prefill_engines[key]

    def _graph_prefill(self, inputs, offset, cache, logits_to_keep):
        """Route a B == 1 prefill chunk through the captured chunk graph when it applies; None otherwise."""
        from .engine import PrefillEngine

        chunk = self.prefill_graph_len
        if chunk == 0 or self.use_decode_graph is False or not self._paged or logits_to_keep != 1:
            return None
        if inputs.dim() != 2 or inputs.shape[0] != 1 or not inputs.is_cuda:
            return None
        if chunk is None:
            if not self._decode_engines:
                return None
            chunk = 128
        L = inputs.shape[1]
        # 2 <= L: tail chunks of a few tokens replay the graph too (right-aligned in its rows).  On the operator path they
        # are ~700 host-bound launches each, and their cost follows the load of the host.
        if not (1 < L <= chunk) or not PrefillEngine.supported(self, inputs.device):
            return None
        if isinstance(offset, torch.Tensor):
            off = int(offset.reshape(-1)[0])
        elif isinstance(offset, int):
            off = offset
        else:
            off = int(list(offset)[0])
        engine = self.prefill_engine(chunk)
        if not engine.applies(L, off, cache):
            return None
        logits, _ = engine.prefill_chunk(inputs.reshape(-1), off, cache)
        return logits.clone()

    def __call__(self, inputs, offset, cache: list[TinyKvCache], logits_to_keep: int | None = None):
        if self._graph_decode_applies(inputs, cache):
            return self._graph_decode(inputs, offset, cache, logits_to_keep)
        if inputs.dim() == 2 and inputs.shape[1] > 1 and inputs.is_cuda:
            out = self._graph_prefill(inputs, offset, cache, logits_to_keep)
            if out is not None:
                return out
        h = self.embedding(inputs)
        for block, layer_cache in zip(self.layers_inner, cache):
            h = block(h, offset, layer_cache, mask="causal")
        if logits_to_keep is not None:
            if logits_to_keep <= 0:
                raise ValueError("logits_to_keep must be positive")
            h = h[:, -logits_to_keep:, :]
        h = self.norm(h)
        if self.w_lm_head is not None:
            return quantized_linear(h, self.w_lm_head)
        return self.embedding.as_linear(h)
