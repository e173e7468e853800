"""Attention operators (``src/tiny_llm_ref/attention.py``).

``paged_attention`` keeps the reference's model-facing contract - query
``[B, H_q, L, D]``, page storage ``[P, H_kv, page_size, D]``, int32
``block_table [B, max_pages]`` padded with ``-1`` and int32 post-append
``context_lens [B]`` - and its metadata validation, message for message
(attention.py:85-158).  The reference validates through ``.tolist()`` on the
device arrays, one host sync per layer (attention.py:131-132); here callers
that built the tables on the host pass those host copies along
(``block_table_host`` / ``context_lens_host``) and no sync happens.  The
integer checks themselves are done on the host either way and are bit-exact.
"""

from __future__ import annotations

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200

from .basics import linear, softmax


def scaled_dot_product_attention_simple(query, key, value, scale=None, mask=None):
    """attention.py:6-21 - equal head counts, additive float mask."""
    factor = query.shape[-1] ** -0.5 if scale is None else scale
    scores = torch.matmul(query, key.transpose(-1, -2)) * factor
    if mask is not None:
        scores = scores + mask
    return torch.matmul(softmax(scores, axis=-1), value)


def causal_mask(L: int, S: int, dtype: torch.dtype, device=None) -> torch.Tensor:
    """attention.py:24-27 - bottom-right aligned: row l sees keys <= l + (S-L)."""
    keep = torch.tril(torch.ones((L, S), device=device), diagonal=S - L).bool()
    zero = torch.zeros((), device=device)
    return torch.where(keep, zero, zero - float("inf")).to(dtype)


def scaled_dot_product_attention_grouped(query, key, value, scale=None, mask=None):
    """attention.py:30-66 - grouped-query attention in the operand dtype."""
    head_dim = query.shape[-1]
    factor = torch.tensor(head_dim**-0.5 if scale is None else float(scale), device=query.device).to(query.dtype)
    out_shape = query.shape
    n_q, L, _ = query.shape[-3:]
    n_kv, S, _ = key.shape[-3:]
    lead = tuple(query.shape[:-3])
    assert n_q % n_kv == 0
    reps = n_q // n_kv
    q = query.reshape(*lead, -1, n_kv, reps, L, head_dim)
    k = key.reshape(*lead, -1, n_kv, 1, S, head_dim)
    v = value.reshape(*lead, -1, n_kv, 1, S, head_dim)
    scores = torch.matmul(q, k.transpose(-1, -2)) * factor
    if mask is not None:
        if isinstance(mask, str):
            if mask != "causal":
                raise ValueError(f"unsupported attention mask: {mask}")
            scores = scores + causal_mask(L, S, scores.dtype, device=scores.device)
        else:
            wide = torch.broadcast_to(mask, (*lead, n_q, L, S)).reshape(*lead, 1, n_kv, reps, L, S)
            scores = scores + wide.to(scores.dtype)
    return torch.matmul(softmax(scores, axis=-1), v).reshape(out_shape)


def _raise_first_metadata_error(ctx_rows, table_rows, page_size, max_pages, num_physical_pages, L) -> None:
    """The reference's row-by-row scan (attention.py:133-158); run only after the
    vectorised pre-check found a violation, to raise the identical first error.
    A page may be live in several rows (a prompt prefix shared through the prefix
    cache), never twice in one row."""
    for b, (ctx, row) in enumerate(zip(ctx_rows, table_rows)):
        seen: set[int] = set()
        if ctx < 0:
            raise ValueError(f"context_lens[{b}] must be nonnegative")
        live = (ctx + page_size - 1) // page_size
        if live > max_pages:
            raise ValueError(f"context_lens[{b}] is not covered by block_table")
        for slot, page_id in enumerate(row):
            if slot < live:
                if page_id < 0 or page_id >= num_physical_pages:
                    raise ValueError(f"Live page id {page_id} at [{b}, {slot}] is outside physical page storage")
                if page_id in seen:
                    raise ValueError(f"Live page id {page_id} is aliased")
                seen.add(page_id)
            elif page_id != -1:
                raise ValueError(f"Unused block_table entry [{b}, {slot}] must use the -1 sentinel")
        if 0 < ctx < L:
            raise ValueError(f"context_lens[{b}] must be zero or at least query length {L}")


def validate_paged_metadata(ctx: np.ndarray, table: np.ndarray, page_size: int, num_physical_pages: int, L: int) -> None:
    """Integer validation of the paged metadata; vectorised fast path, exact
    reference error on failure."""
    max_pages = table.shape[1]
    ctx64 = ctx.astype(np.int64)
    live_pages = (ctx64 + page_size - 1) // page_size
    live = np.arange(max_pages, dtype=np.int64)[None, :] < live_pages[:, None]
    ids = table[live]
    in_row = np.nonzero(live)[0].astype(np.int64) * max(num_physical_pages, 1) + ids  # distinct while ids are in range
    clean = (
        not (ctx64 < 0).any()
        and not (live_pages > max_pages).any()
        and not ((ids < 0) | (ids >= num_physical_pages)).any()
        and np.unique(in_row).size == in_row.size
        and not (table[~live] != -1).any()
        and not ((ctx64 > 0) & (ctx64 < L)).any()
    )
    if not clean:
        _raise_first_metadata_error(ctx.tolist(), table.tolist(), page_size, max_pages, num_physical_pages, L)
        raise AssertionError("paged metadata pre-check and scan disagree")  # pragma: no cover


def paged_attention(
    query: torch.Tensor,
    key_pages: torch.Tensor,
    value_pages: torch.Tensor,
    block_table: torch.Tensor,
    context_lens: torch.Tensor,
    page_size: int,
    scale: float | None = None,
    mask: torch.Tensor | str | None = None,
    *,
    block_table_host: np.ndarray | None = None,
    context_lens_host: np.ndarray | None = None,
) -> torch.Tensor:
    """Paged attention backed by the sm_90a extension (attention.py:69-178)."""
    if isinstance(mask, torch.Tensor):
        raise NotImplementedError("Paged attention only supports mask=None or causal")
    if mask is not None and mask != "causal":
        raise NotImplementedError

    if query.dim() != 4:
        raise ValueError("query must be 4D [B, H_q, L, D]")
    if key_pages.dim() != 4 or value_pages.dim() != 4:
        raise ValueError("page tensors must be 4D [P, H_kv, page_size, D]")
    if key_pages.shape != value_pages.shape:
        raise ValueError("key pages and value pages must have the same shape")
    if block_table.dim() != 2 or context_lens.dim() != 1:
        raise ValueError("block_table must be 2D and context_lens must be 1D")
    if block_table.dtype != torch.int32 or context_lens.dtype != torch.int32:
        raise ValueError("block_table and context_lens must be int32")
    if not isinstance(page_size, int) or page_size <= 0:
        raise ValueError("page_size must be a positive integer")

    factor = query.shape[-1] ** -0.5 if scale is None else float(scale)
    B, n_q, L, D = query.shape
    num_physical_pages, n_kv, stored_page_size, stored_dim = key_pages.shape
    if min(B, n_q, L, D, n_kv, stored_page_size, stored_dim) <= 0:
        raise ValueError("paged attention dimensions must be positive")
    if num_physical_pages <= 0:
        raise ValueError("paged attention requires nonempty physical page storage")
    if n_q % n_kv != 0:
        raise ValueError("query heads must be divisible by K/V heads")
    if stored_dim != D:
        raise ValueError("query and page tensors must have the same head dimension")
    if stored_page_size != page_size:
        raise ValueError(f"page_size={page_size} does not match page storage {stored_page_size}")
    if block_table.shape[0] != B or context_lens.shape[0] != B:
        raise ValueError("query, block_table, and context_lens batch sizes must match")
    if block_table.shape[1] <= 0:
        raise ValueError("block_table must provide at least one page slot")
    if query.dtype != key_pages.dtype or query.dtype != value_pages.dtype:
        raise ValueError("query, key pages, and value pages must have the same dtype")
    if query.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError("paged attention supports float32 or bfloat16 inputs")

    # Small integer metadata is checked on the host before any dispatch.
    if context_lens_host is None:
        context_lens_host = context_lens.detach().cpu().numpy()
    if block_table_host is None:
        block_table_host = block_table.detach().cpu().numpy()
    validate_paged_metadata(
        np.asarray(context_lens_host).reshape(B), np.asarray(block_table_host).reshape(B, -1), page_size, num_physical_pages, L
    )

    out = tiny_llm_ext_b200.paged_attention(
        query.reshape(B * n_q, L, D).contiguous(),
        key_pages.contiguous(),
        value_pages.contiguous(),
        block_table.contiguous(),
        context_lens.contiguous(),
        factor,
        is_causal=(mask == "causal"),
        num_kv_heads=n_kv,
        num_heads=n_q,
    )
    return out.reshape(B, n_q, L, D)


class SimpleMultiHeadAttention:
    """attention.py:181-237 - Week-1 dense multi-head attention."""

    def __init__(self, hidden_size: int, num_heads: int, wq, wk, wv, wo):
        assert hidden_size % num_heads == 0
        self.hidden_size = hidden_size
        self.num_heads = num_heads
        self.head_dim = hidden_size // num_heads
        self.scale = self.head_dim**-0.5
        assert tuple(wq.shape) == (num_heads * self.head_dim, hidden_size)
        assert tuple(wk.shape) == (num_heads * self.head_dim, hidden_size)
        assert tuple(wv.shape) == (num_heads * self.head_dim, hidden_size)
        assert tuple(wo.shape) == (hidden_size, num_heads * self.head_dim)
        self.wq, self.wk, self.wv, self.wo = wq, wk, wv, wo

    def _split(self, x, w):
        N, L, _ = x.shape
        return linear(x, w).reshape(N, L, self.num_heads, self.head_dim).transpose(1, 2)

    def __call__(self, query, key, value, mask=None):
        N, L, _ = query.shape
        assert query.shape == key.shape == value.shape
        heads = scaled_dot_product_attention_simple(
            self._split(query, self.wq), self._split(key, self.wk), self._split(value, self.wv), scale=self.scale, mask=mask
        )
        return linear(heads.transpose(1, 2).reshape(N, L, self.hidden_size), self.wo)
