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

from extensions_b200 import tiny_llm_ext_b200 as ext

from .attention import paged_attention
from .embedding import QuantizedEmbedding
from .kv_cache import TinyKvCache
from .moe import Moe
from .paged_kv_cache import TinyKvPagedCache, TinyKvPagedPool
from .quantize import QuantizedWeights, quantized_linear
from .rope_scaling import parse_rope_scaling, rope_inv_freq
from .week2_kernels import (
    FastRMSNorm,
    FastRoPE,
    decode_attention_custom,
    residual_add,
    scaled_dot_product_attention,
    swiglu,
)


def kv_reservation_pages(window: int, page_size: int, batch_size: int = 1) -> int:
    """Pages per layer a decode engine of ``batch_size`` slots and context window ``window`` reserves."""
    return (batch_size + 1) * (-(-window // page_size)) + 1


def kv_reservation_bytes(layers: int, num_kv_heads: int, head_dim: int, page_size: int, window: int, batch_size: int = 1,
                         dtype_bytes: int = 2) -> int:
    """Bytes of bf16 K and V pages for ``kv_reservation_pages`` pages in each of ``layers`` layers."""
    page_bytes = 2 * num_kv_heads * page_size * head_dim * dtype_bytes
    return layers * kv_reservation_pages(window, page_size, batch_size) * page_bytes


def check_kv_reservation(need: int, free: int, window: int, batch_size: int) -> None:
    """Refuse a reservation of ``need`` bytes that does not fit ``free`` bytes."""
    if need > free:
        gib = 1 << 30
        raise MemoryError(f"context window {window} for {batch_size} slot(s) needs {need} bytes ({need / gib:.2f} GiB) of KV pages, "
                          f"but only {max(free, 0)} bytes ({max(free, 0) / gib:.2f} GiB) of device memory are free")


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
        rope_inv_freq: torch.Tensor | None = None,
        rope_mscale: float = 1.0,
    ):
        """``rope_inv_freq``: the model's scaled RoPE table (``rope_scaling.rope_inv_freq``), None for plain RoPE.
        ``rope_mscale``: YaRN's ``m``; q and k are each scaled by it, which is folded into ``scale`` as ``m^2`` (so
        every engine, which reads ``scale``, applies it and the K pages hold unscaled keys)."""
        assert num_heads % num_kv_heads == 0, f"num_heads {num_heads} must be divisible by num_kv_heads {num_kv_heads}"
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.num_kv_heads = num_kv_heads
        self.head_dim = head_dim
        self.scale = head_dim**-0.5
        if rope_mscale != 1.0:
            self.scale *= rope_mscale * rope_mscale
        self.wq, self.wk, self.wv, self.wo = wq, wk, wv, wo
        self.rope = FastRoPE(head_dim, max_seq_len, theta, inv_freq=rope_inv_freq)
        self.q_norm = FastRMSNorm(head_dim, q_norm, eps=rms_norm_eps)
        self.k_norm = FastRMSNorm(head_dim, k_norm, eps=rms_norm_eps)
        self.use_paged_attention = use_paged_attention

    def __call__(self, x, offsets, cache: TinyKvCache, mask=None, lora=None):
        """``lora``: ``(sites, row_ids)``, the layer's ``AdapterSet`` sites and one adapter id per row of ``x``: each
        targeted projection's output takes its row's adapter (``ext.lora_apply``) before anything reads it."""
        B, L, _ = x.shape
        q, k, v = quantized_linear(x, self.wq), quantized_linear(x, self.wk), quantized_linear(x, self.wv)
        if lora is not None and lora[0].qkv is not None:
            ext.lora_apply(x, [q, k, v], lora[1], lora[0].qkv)
        q = q.reshape(B, L, self.num_heads, self.head_dim)
        k = k.reshape(B, L, self.num_kv_heads, self.head_dim)
        q = self.q_norm(q)
        k = self.k_norm(k)
        v = v.reshape(B, L, self.num_kv_heads, self.head_dim)
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
        out = quantized_linear(y, self.wo)
        if lora is not None and lora[0].o is not None:
            ext.lora_apply(y, out, lora[1], lora[0].o)
        return out


class Qwen3MLP:
    """qwen3_week3.py:124-146 - down(swiglu(gate(x), up(x)))."""

    def __init__(self, dim: int, hidden_dim: int, w_gate: QuantizedWeights, w_up: QuantizedWeights, w_down: QuantizedWeights):
        self.dim = dim
        self.hidden_dim = hidden_dim
        self.w_gate, self.w_up, self.w_down = w_gate, w_up, w_down

    def __call__(self, x: torch.Tensor, lora=None) -> torch.Tensor:
        if lora is None:
            return quantized_linear(swiglu(quantized_linear(x, self.w_gate), quantized_linear(x, self.w_up)), self.w_down)
        sites, row_ids = lora
        gate, up = quantized_linear(x, self.w_gate), quantized_linear(x, self.w_up)
        if sites.gate_up is not None:
            ext.lora_apply(x, [gate, up], row_ids, sites.gate_up)
        act = swiglu(gate, up)
        out = quantized_linear(act, self.w_down)
        if sites.down is not None:
            ext.lora_apply(act, out, row_ids, sites.down)
        return out


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
        rope_inv_freq: torch.Tensor | None = None,
        rope_mscale: float = 1.0,
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
            rope_inv_freq=rope_inv_freq,
            rope_mscale=rope_mscale,
        )

    def __call__(self, x, offset, cache: TinyKvCache, mask=None, lora=None):
        if lora is None:
            h = residual_add(x, self.self_attn(self.input_layernorm(x), offset, cache, mask))
            return residual_add(h, self.mlp(self.post_attention_layernorm(h)))
        h = residual_add(x, self.self_attn(self.input_layernorm(x), offset, cache, mask, lora=lora))
        return residual_add(h, self.mlp(self.post_attention_layernorm(h), lora=lora))


def is_qwen3_moe_sparse_layer(args: Any, layer_idx: int) -> bool:
    """qwen3_week3.py:210-215."""
    return (
        getattr(args, "num_experts", 0) > 0
        and layer_idx not in getattr(args, "mlp_only_layers", [])
        and (layer_idx + 1) % getattr(args, "decoder_sparse_step", 1) == 0
    )


class Qwen3ModelWeek3:
    """qwen3_week3.py:218-338."""

    def __init__(self, mlx_model: Any, page_size: int = 128, enable_paged_attention: bool = True, max_context: int | None = None):
        """``max_context``: the graph engines' context window (``set_max_context``); None keeps the default 8,192."""
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
        # One RoPE frequency table for the whole model when the config scales RoPE (YaRN): every site - operator path,
        # decode, prefill and verify graphs - reads this tensor, so keys written at prefill and queries rotated at
        # decode use identical angles.  None: plain RoPE, every site keeps its inline base^(-i/half).
        self.rope_scaling = parse_rope_scaling(getattr(args, "rope_scaling", None), args.max_position_embeddings)
        self.rope_inv_freq = None
        if self.rope_scaling is not None:
            self.rope_inv_freq = rope_inv_freq(args.head_dim, args.rope_theta, self.rope_scaling, self.embedding.weight.scales.device)
        mscale = 1.0 if self.rope_scaling is None else self.rope_scaling.mscale
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
                    rope_inv_freq=self.rope_inv_freq,
                    rope_mscale=mscale,
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
        self.prefix_cache = None  # prefix_cache.PrefixCache over page_pools, once enable_prefix_cache() is called
        self.adapters = None  # lora.AdapterSet, once load_adapters() is called
        if max_context is not None:
            self.set_max_context(max_context)

    @property
    def max_context(self) -> int:
        """The graph engines' context window: the longest request a decode, prefill or verify graph holds (requests
        beyond it run operator by operator).  Backed by ``decode_graph_max_seq_len``."""
        return self.decode_graph_max_seq_len

    def set_max_context(self, tokens: int, batch_size: int = 1, device=None) -> None:
        """Set the graph engines' context window to ``tokens`` (rounded up to whole pages).  A decode engine of
        ``batch_size`` slots reserves ``(B + 1) * ceil(W / page) + 1`` pages per layer; a window whose reservation does
        not fit the device's free memory is refused here, before anything is allocated or captured.  Only before the
        first graph engine exists: captured graphs do not change their page tables."""
        tokens = int(tokens)
        if tokens <= 0:
            raise ValueError(f"max_context must be positive (got {tokens})")
        if self._decode_engines or self._prefill_engines or self._verify_engines:
            raise RuntimeError("set_max_context: call it before the first decode, prefill or verify graph engine exists")
        window = -(-tokens // self.page_size) * self.page_size
        self._check_reservation(window, batch_size, device)
        self.decode_graph_max_seq_len = window

    def kv_reservation_bytes(self, window: int, batch_size: int = 1) -> int:
        """Bytes of K and V pages a ``batch_size``-slot decode engine with context window ``window`` reserves."""
        attn = self.layers_inner[0].self_attn
        return kv_reservation_bytes(self.num_hidden_layers, attn.num_kv_heads, attn.head_dim, self.page_size, window, batch_size)

    def _check_reservation(self, window: int, batch_size: int, device=None) -> None:
        """Refuse (``MemoryError``, with the bytes needed) a decode-engine page reservation that does not fit the
        device's free memory.  Slabs that already hold enough pages need nothing; a growing slab is allocated whole
        while the old one is still alive, so the whole new size must be free."""
        dev = torch.device(device if device is not None else self.embedding.weight.scales.device)
        pages = kv_reservation_pages(window, self.page_size, batch_size)
        if dev.type != "cuda" or all(p.capacity >= pages for p in self.page_pools):
            return
        free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
        check_kv_reservation(self.kv_reservation_bytes(window, batch_size), free, window, batch_size)

    def create_kv_cache(self) -> list[TinyKvCache]:
        """One logical cache per layer, all sharing that layer's pool."""
        return [TinyKvPagedCache(pool=pool) for pool in self.page_pools]

    def enable_prefix_cache(self):
        """The model's prefix index (``prefix_cache.PrefixCache``), created over ``page_pools`` on first call: requests
        whose prompts share a prefix with one prefilled before share its KV pages.  Off until called."""
        if self.prefix_cache is None:
            from .prefix_cache import PrefixCache

            self.prefix_cache = PrefixCache(self.page_pools)
        return self.prefix_cache

    def load_adapters(self, adapters):
        """Pack ``adapters`` (``lora.LoraAdapter``s) for this model and return the ``lora.AdapterSet``.  From then on a
        call may name one adapter per batch row (``adapter_ids``), and the graph engines this model builds are the LoRA
        engines (``engine.py``).  Once, and before any engine exists: captured graphs do not change their launches."""
        from .lora import AdapterSet

        if self.adapters is not None:
            raise RuntimeError("load_adapters: this model already has its adapter set (adapters cannot be swapped after loading)")
        if self._decode_engines or self._prefill_engines or self._verify_engines:
            raise RuntimeError("load_adapters: call it before the first decode or prefill graph engine exists")
        if any(isinstance(b.mlp, Moe) for b in self.layers_inner):
            raise ValueError("load_adapters: adapters on Qwen3-MoE models are not supported")
        self.adapters = AdapterSet(self.mlx_model.args, adapters, self.embedding.weight.scales.device)
        return self.adapters

    def _adapter_rows(self, adapter_ids, B: int):
        """``adapter_ids`` of a call as a list of ``B`` ids, or None when every row runs the base model."""
        if adapter_ids is None:
            return None
        ids = [int(i) for i in adapter_ids]
        if len(ids) != B:
            raise ValueError(f"adapter_ids must hold one id per batch row ({B})")
        if all(i < 0 for i in ids):
            return None
        if self.adapters is None:
            raise ValueError("adapter_ids name an adapter but the model has none loaded (load_adapters)")
        if any(i >= len(self.adapters.names) for i in ids):
            raise ValueError(f"adapter_ids {ids} exceed the {len(self.adapters.names)} loaded adapters")
        return ids

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
            self._check_reservation(limit, batch_size, dev)
            engine = DecodeEngine(self, batch_size, limit, dev)
            engine.reserve_pools((batch_size + 1) * engine.max_pages + 1)
            self._decode_engines[key] = engine
        return self._decode_engines[key]

    def verify_applies(self, device=None) -> bool:
        """Whether ``verify_engine`` runs on this model: CUDA paged caches and the shapes of the fused decode path."""
        from .engine import VerifyEngine

        dev = device if device is not None else self.embedding.weight.scales.device
        return (self._paged and self.use_decode_graph is not False and torch.device(dev).type == "cuda"
                and VerifyEngine.supported(self, dev, self.decode_graph_max_seq_len))  # False with adapters loaded

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

    def _graph_decode(self, inputs, offset, cache, logits_to_keep, adapter_ids=None):
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
        logits, _ = engine.step(inputs, offsets, cache) if self.adapters is None else engine.step(inputs, offsets, cache, adapter_ids=adapter_ids)
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

    def _graph_prefill(self, inputs, offset, cache, logits_to_keep, adapter_id: int = -1):
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
        logits, _ = engine.prefill_chunk(inputs.reshape(-1), off, cache) if self.adapters is None else \
            engine.prefill_chunk(inputs.reshape(-1), off, cache, adapter_id=adapter_id)
        return logits.clone()

    # Operator-path calls are run as they come up to ONE_CALL_MAX_TOKENS rows while every activation and logits tensor
    # stays below 2^31 elements (the kernels index elements with 32-bit ints there).  A longer prompt - a 131,072-token
    # prefill under YaRN - is run as consecutive PREFILL_PIECE_TOKENS-row calls on the same cache: chunked prefill.
    ONE_CALL_MAX_TOKENS = 32768
    PREFILL_PIECE_TOKENS = 8192

    def _needs_pieces(self, B: int, L: int, logits_to_keep: int | None) -> bool:
        args = self.mlx_model.args
        attn = self.layers_inner[0].self_attn
        width = max(args.hidden_size, attn.num_heads * attn.head_dim, args.intermediate_size,
                    getattr(args, "moe_intermediate_size", 0) * getattr(args, "num_experts_per_tok", 0))
        keep = L if logits_to_keep is None else min(logits_to_keep, L)
        return L > self.PREFILL_PIECE_TOKENS and (L > self.ONE_CALL_MAX_TOKENS or B * L * width >= 2**31 or B * keep * self.vocab_size >= 2**31)

    def _prefill_in_pieces(self, inputs, offset, cache, logits_to_keep, adapter_ids):
        """``self(inputs, ...)`` as consecutive calls of at most ``PREFILL_PIECE_TOKENS`` rows; returns the same rows."""
        L = inputs.shape[1]
        keep = L if logits_to_keep is None else logits_to_keep
        if keep <= 0:
            raise ValueError("logits_to_keep must be positive")
        outs = []
        for a in range(0, L, self.PREFILL_PIECE_TOKENS):
            b = min(a + self.PREFILL_PIECE_TOKENS, L)
            want = min(b - a, max(0, b - (L - keep)))  # rows of this piece among the last `keep`
            if isinstance(offset, int):
                off = offset + a
            elif isinstance(offset, torch.Tensor):
                off = offset + a
            else:
                off = [int(o) + a for o in offset]
            out = self(inputs[:, a:b], off, cache, logits_to_keep=max(want, 1), adapter_ids=adapter_ids)
            if want:
                outs.append(out[:, -want:])
        return outs[0] if len(outs) == 1 else torch.cat(outs, dim=1)

    def __call__(self, inputs, offset, cache: list[TinyKvCache], logits_to_keep: int | None = None, adapter_ids=None):
        """``adapter_ids``: one ``AdapterSet`` id per batch row (-1: the base model), after ``load_adapters``."""
        ids = self._adapter_rows(adapter_ids, inputs.shape[0])
        if self._graph_decode_applies(inputs, cache):
            return self._graph_decode(inputs, offset, cache, logits_to_keep, ids)
        if inputs.dim() == 2 and inputs.shape[1] > 1 and inputs.is_cuda:
            out = self._graph_prefill(inputs, offset, cache, logits_to_keep, -1 if ids is None else ids[0])
            if out is not None:
                return out
        if inputs.dim() == 2 and self._needs_pieces(inputs.shape[0], inputs.shape[1], logits_to_keep):
            return self._prefill_in_pieces(inputs, offset, cache, logits_to_keep, adapter_ids)
        h = self.embedding(inputs)
        row_ids = None if ids is None else self.adapters.row_ids(ids, inputs.shape[1])
        for index, (block, layer_cache) in enumerate(zip(self.layers_inner, cache)):
            if row_ids is None:
                h = block(h, offset, layer_cache, mask="causal")
            else:
                h = block(h, offset, layer_cache, mask="causal", lora=(self.adapters.sites[index], row_ids))
        if logits_to_keep is not None:
            if logits_to_keep <= 0:
                raise ValueError("logits_to_keep must be positive")
            h = h[:, -logits_to_keep:, :]
        h = self.norm(h)
        if self.w_lm_head is not None:
            return quantized_linear(h, self.w_lm_head)
        return self.embedding.as_linear(h)
