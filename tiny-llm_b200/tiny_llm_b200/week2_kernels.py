"""Fused model operators: signatures of
``src/tiny_llm_ref/week2_kernels.py`` over the CUDA extension."""

from __future__ import annotations

import torch

from extensions_b200 import tiny_llm_ext_b200

from .basics import softmax

_NO_MASK: dict = {}


def _no_attention_mask(device) -> torch.Tensor:
    """The dummy fp32 ``[1]`` mask handed to the kernel when ``has_mask`` is
    false (week2_kernels.py:7,134)."""
    key = str(device)
    if key not in _NO_MASK:
        _NO_MASK[key] = torch.zeros((1,), dtype=torch.float32, device=device)
    return _NO_MASK[key]


class FastRMSNorm:
    """week2_kernels.py:10-19."""

    def __init__(self, dim: int, weight: torch.Tensor, eps: float = 1e-5):
        self.dim = dim
        self.weight = weight
        self.eps = eps
        self._cast: dict = {}

    def _weight_as(self, dtype, device) -> torch.Tensor:
        key = (dtype, str(device))
        if key not in self._cast:
            self._cast[key] = self.weight.to(device=device, dtype=dtype).contiguous()
        return self._cast[key]

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        return tiny_llm_ext_b200.rms_norm(x.contiguous(), self._weight_as(x.dtype, x.device), self.eps)


class FastRoPE:
    """week2_kernels.py:22-53 - ``offset`` may be an int, one int per batch
    row, a 0-d tensor or a ``[B]`` tensor.  ``inv_freq``: a float64 ``[dims / 2]`` device table of a scaled RoPE
    (``rope_scaling.rope_inv_freq``) that replaces ``base``; None rotates by ``base^(-i / (dims / 2))``."""

    def __init__(self, dims: int, seq_len: int, base: int = 10000, traditional: bool = False, inv_freq: torch.Tensor | None = None):
        self.dims = dims
        self.seq_len = seq_len
        self.base = base
        self.traditional = traditional
        self.inv_freq = inv_freq

    def __call__(self, x: torch.Tensor, offset: int | list[int] | torch.Tensor = 0) -> torch.Tensor:
        batch = x.shape[0]
        if isinstance(offset, int):
            offsets = torch.full((batch,), offset, dtype=torch.int32, device=x.device)
        elif isinstance(offset, list):
            if len(offset) != batch:
                raise ValueError("FastRoPE needs one offset per batch row")
            offsets = torch.tensor(offset, dtype=torch.int32, device=x.device)
        elif offset.dim() == 0:
            offsets = offset.to(device=x.device, dtype=torch.int32).expand(batch)
        elif tuple(offset.shape) != (batch,):
            raise ValueError("FastRoPE needs one offset per batch row")
        else:
            offsets = offset.to(device=x.device, dtype=torch.int32)
        if self.inv_freq is not None:
            return tiny_llm_ext_b200.rope_table(x.contiguous(), offsets.contiguous(), self.dims, self.inv_freq, self.traditional)
        return tiny_llm_ext_b200.rope(x.contiguous(), offsets.contiguous(), self.dims, self.base, self.traditional)


def swiglu(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    """week2_kernels.py:56-57."""
    return tiny_llm_ext_b200.swiglu(gate.contiguous(), up.contiguous())


def residual_add(x: torch.Tensor, r: torch.Tensor) -> torch.Tensor:
    """``x + r`` of the transformer block (qwen3_week3.py:204-206) as one
    vectorised launch of the extension (not in the reference module)."""
    if x.shape != r.shape or x.dtype != r.dtype:
        return x + r
    return tiny_llm_ext_b200.add(x.contiguous(), r.contiguous())


def scaled_dot_product_attention(
    query: torch.Tensor,
    key: torch.Tensor,
    value: torch.Tensor,
    scale: float,
    mask: torch.Tensor | str | None = None,
) -> torch.Tensor:
    """Grouped-query attention in the query dtype (week2_kernels.py:60-95);
    the dense fallback of the Week-3 model for long or wide chunks."""
    out_shape = query.shape
    lead = tuple(query.shape[:-3])
    n_heads, q_len, head_dim = query.shape[-3:]
    n_kv, ctx_len, _ = key.shape[-3:]
    if key.shape != value.shape or n_heads % n_kv != 0:
        raise ValueError("incompatible grouped-query attention shapes")
    reps = n_heads // n_kv
    q = query.reshape(*lead, -1, n_kv, reps, q_len, head_dim)
    k = key.reshape(*lead, -1, n_kv, 1, ctx_len, head_dim)
    v = value.reshape(*lead, -1, n_kv, 1, ctx_len, head_dim)
    scores = torch.matmul(q, k.transpose(-1, -2)) * torch.tensor(scale, dtype=query.dtype, device=query.device)
    if isinstance(mask, str):
        if mask != "causal":
            raise ValueError(f"unsupported attention mask: {mask}")
        keep = torch.tril(torch.ones((q_len, ctx_len), device=query.device), diagonal=ctx_len - q_len).bool()
        scores = scores + torch.where(keep, 0.0, float("-inf")).to(scores.dtype)
    elif mask is not None:
        wide = torch.broadcast_to(mask, (*lead, n_heads, q_len, ctx_len))
        scores = scores + wide.reshape(*lead, -1, n_kv, reps, q_len, ctx_len).to(scores.dtype)
    return torch.matmul(softmax(scores, axis=-1), v).reshape(out_shape)


def decode_attention_custom(
    query: torch.Tensor,
    key: torch.Tensor,
    value: torch.Tensor,
    scale: float,
    mask: torch.Tensor | str | None = None,
) -> torch.Tensor:
    """week2_kernels.py:98-147 - dense-KV decode kernel, ``[B,H,L,D]`` in/out."""
    batch, n_heads, q_len, head_dim = query.shape
    k_batch, n_kv, ctx_len, k_dim = key.shape
    if batch != k_batch or key.shape != value.shape:
        raise ValueError("query, key, and value batch dimensions must match")
    if head_dim != k_dim or n_heads % n_kv != 0:
        raise ValueError("incompatible grouped-query attention shapes")
    if isinstance(mask, str) and mask != "causal":
        raise ValueError(f"unsupported attention mask: {mask}")
    q3 = query.reshape(batch * n_heads, q_len, head_dim).contiguous()
    k3 = key.reshape(batch * n_kv, ctx_len, head_dim).contiguous()
    v3 = value.reshape(batch * n_kv, ctx_len, head_dim).contiguous()
    causal = isinstance(mask, str) and mask == "causal"
    explicit = isinstance(mask, torch.Tensor)
    if explicit:
        wide = torch.broadcast_to(mask, (batch, n_heads, q_len, ctx_len))
        mask_arg = wide.to(torch.float32).reshape(batch * n_heads, q_len, ctx_len).contiguous()
    else:
        mask_arg = _no_attention_mask(query.device)
    out = tiny_llm_ext_b200.decode_attention(q3, k3, v3, mask_arg, scale, causal, explicit, n_heads, n_kv)
    return out.reshape(batch, n_heads, q_len, head_dim)
