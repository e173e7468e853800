"""KV-cache interfaces and the dense caches
(``src/tiny_llm_ref/kv_cache.py``).

``BatchingKvCache`` is the decode-slot table of the continuous-batching
scheduler: a fixed number of slots, each holding one request's cache (or
nothing).  ``update_and_fetch`` is the Week-3-day-1 dense path (right-aligned
padding + additive mask); ``update_and_fetch_paged`` appends one chunk per
active slot into the shared page pool and returns block-table metadata.  Here
the per-slot appends of a decode step (one token per request) are
collapsed into a single device-driven launch; all integer bookkeeping stays on
the host and is identical to the reference's.
"""

from __future__ import annotations

from abc import ABC, abstractmethod
from typing import TYPE_CHECKING, Optional

import numpy as np
import torch

from .attention import causal_mask

if TYPE_CHECKING:
    from .paged_kv_cache import PagedKvMetadata


def _nbytes(t: torch.Tensor) -> int:
    return t.numel() * t.element_size()


class TinyKvCache(ABC):
    """kv_cache.py:11-72."""

    @abstractmethod
    def update_and_fetch(
        self,
        key: torch.Tensor,
        value: torch.Tensor,
        mask_length: int | None = None,
        mask: torch.Tensor | str | None = None,
    ) -> tuple[torch.Tensor, torch.Tensor, int, Optional[torch.Tensor]]:
        """Append ``key``/``value`` and return (keys, values, seq_len, mask)."""

    def release(self):
        """Give back whatever this cache owns (pages for paged caches)."""
        return None

    def materialize(self):
        """MLX evaluates lazy storage here; torch is eager, so nothing to do -
        the hook stays because schedulers call it and tests override it."""
        return None

    def update_and_fetch_paged(self, key, value, mask_length=None, mask=None) -> "PagedKvMetadata":
        raise NotImplementedError("This KV cache does not support paged attention")

    def rewind(self, n: int):
        raise NotImplementedError("This KV cache does not support rewind")


class TinyKvFullCache(TinyKvCache):
    """Dense concat-growth cache (kv_cache.py:246-287)."""

    def __init__(self):
        self.key_values = None
        self.offset = 0
        self.growth_copy_bytes = 0

    def update_and_fetch(self, key, value, mask_length=None, mask=None):
        if self.key_values is None:
            assert self.offset == 0
            self.key_values = (key, value)
            self.offset = key.shape[2]
            return key, value, self.offset, mask
        B, H, S, D = key.shape
        assert key.shape == value.shape
        old_k, old_v = self.key_values
        assert tuple(old_k.shape) == (B, H, self.offset, D)
        assert tuple(old_v.shape) == (B, H, self.offset, D)
        self.growth_copy_bytes += _nbytes(old_k) + _nbytes(old_v)
        self.key_values = (torch.cat([old_k, key], dim=2), torch.cat([old_v, value], dim=2))
        self.offset += S
        return self.key_values[0], self.key_values[1], self.offset, mask

    def rewind(self, n: int):
        self.offset -= n
        self.key_values = (self.key_values[0][:, :, : self.offset], self.key_values[1][:, :, : self.offset])


class BatchingKvCache(TinyKvCache):
    """Slot table of the decode batch (kv_cache.py:75-243)."""

    def __init__(self, max_active_requests: int, max_seq_len: int | None = None):
        self.max_active_requests = max_active_requests
        self.max_seq_len = max_seq_len
        self.kv_caches: list[TinyKvCache] = [None] * max_active_requests
        self.HD = None
        self.last_batch_bytes = 0
        self.staging_copy_bytes = 0

    # -- dense Week-3-day-1 path ------------------------------------------
    def update_and_fetch(self, keys, values, mask_length=None, mask=None):
        B, H, S, D = keys.shape
        assert keys.shape == values.shape
        if self.max_seq_len is not None:
            assert S <= self.max_seq_len
        if self.HD is None:
            self.HD = (H, D)
        else:
            assert self.HD == (H, D), f"expect {self.HD} but got {H, D}"
        assert B == self.max_active_requests
        dtype, device = keys.dtype, keys.device
        fetched = []
        for b, slot in enumerate(self.kv_caches):
            if slot is None:
                fetched.append(None)
                continue
            k, v, length, slot_mask = slot.update_and_fetch(keys[b : b + 1], values[b : b + 1])
            fetched.append((k[0], v[0], length, slot_mask))
        seq_len = max((item[2] for item in fetched if item is not None), default=0)
        batch_k = torch.zeros((B, H, seq_len, D), dtype=dtype, device=device)
        batch_v = torch.zeros((B, H, seq_len, D), dtype=dtype, device=device)
        masks = torch.full((B, mask_length, seq_len), float("-inf"), dtype=dtype, device=device)
        for b, item in enumerate(fetched):
            if item is None:
                continue
            k, v, length, slot_mask = item
            self.staging_copy_bytes += _nbytes(k) + _nbytes(v)
            batch_k[b, :, seq_len - length :, :] = k
            batch_v[b, :, seq_len - length :, :] = v
            if slot_mask is None or (isinstance(slot_mask, str) and slot_mask == "causal"):
                masks[b, :, seq_len - length :] = causal_mask(mask_length, length, dtype=dtype, device=device)
            elif isinstance(slot_mask, torch.Tensor):
                masks[b, :, seq_len - length :] = slot_mask
            else:
                raise NotImplementedError
        self.last_batch_bytes = _nbytes(batch_k) + _nbytes(batch_v)
        return batch_k, batch_v, None, masks.reshape(B, 1, mask_length, seq_len)

    # -- paged path ---------------------------------------------------------
    def update_and_fetch_paged(self, keys, values, mask_length=None, mask=None) -> "PagedKvMetadata":
        from .paged_kv_cache import PagedKvMetadata, TinyKvPagedCache

        if keys.dim() != 4 or values.dim() != 4:
            raise ValueError("Batched K/V chunks must be 4D [B, H, S, D]")
        if keys.shape != values.shape:
            raise ValueError("Batched K/V chunks must have the same shape")
        B, H, S, D = keys.shape
        if B != self.max_active_requests:
            raise ValueError(f"Expected batch size {self.max_active_requests}, got {B}")
        if self.HD is not None and self.HD != (H, D):
            raise ValueError(f"expect {self.HD} but got {H, D}")

        # Whole-batch validation before any request or allocator is touched
        # (kv_cache.py:163-183): mixed pools must fail before row zero appends.
        pool = None
        active: list[tuple[int, TinyKvPagedCache]] = []
        for b, slot in enumerate(self.kv_caches):
            if slot is None:
                continue
            if not isinstance(slot, TinyKvPagedCache):
                raise ValueError("BatchingKvCache contains a non-paged request cache")
            if pool is None:
                pool = slot.pool
            elif pool is not slot.pool:
                raise ValueError("Paged batch caches must share one page pool")
            if self.max_seq_len is not None and slot.offset + S > self.max_seq_len:
                raise ValueError("Paged batch append exceeds max_seq_len")
            slot.validate_append(keys[b : b + 1], values[b : b + 1])
            active.append((b, slot))
        if pool is None:
            raise ValueError("Cannot build paged metadata without active requests")

        pool_state = pool._snapshot_state()
        slot_states = [(slot, slot._snapshot_state()) for _, slot in active]
        old_hd = self.HD
        try:
            if pool.can_batch_decode_append(keys, [slot for _, slot in active]):
                # One launch for the whole decode batch: host bookkeeping per
                # request, then a single device-driven scatter.
                for b, slot in active:
                    slot._append_chunk(keys[b : b + 1], values[b : b + 1], device_write=False)
                context = [0] * B
                for b, slot in active:
                    context[b] = slot.offset
                width = max(slot.num_pages for _, slot in active)
                table_host, ctx_host = self._metadata_host(width, context)
                table = torch.from_numpy(table_host).to(keys.device, non_blocking=True)
                ctx_dev = torch.from_numpy(ctx_host).to(keys.device, non_blocking=True)
                pool.append_decode_batch(keys, values, table, ctx_dev)
            else:
                for b, slot in active:
                    slot.update_and_fetch_paged(keys[b : b + 1], values[b : b + 1], mask_length=mask_length, mask=mask)
                context = [0] * B
                for b, slot in active:
                    context[b] = slot.offset
                width = max(slot.num_pages for _, slot in active)
                table_host, ctx_host = self._metadata_host(width, context)
                table = torch.from_numpy(table_host).to(keys.device)
                ctx_dev = torch.from_numpy(ctx_host).to(keys.device)
            self.HD = (H, D)
        except Exception:
            pool._restore_state(pool_state)
            for slot, state in slot_states:
                slot._restore_state(state)
            self.HD = old_hd
            raise

        self.last_batch_bytes = 0
        return PagedKvMetadata(
            key_pages=pool.key_pages,
            value_pages=pool.value_pages,
            block_table=table,
            context_lens=ctx_dev,
            page_size=pool.page_size,
            mask=mask,
            block_table_host=table_host,
            context_lens_host=ctx_host,
        )

    def _metadata_host(self, width: int, context: list[int]) -> tuple[np.ndarray, np.ndarray]:
        """Rows of page ids padded with -1 (idle slots are all -1) and the
        post-append context lengths (kv_cache.py:210-221)."""
        table = np.full((self.max_active_requests, width), -1, dtype=np.int32)
        for b, slot in enumerate(self.kv_caches):
            if slot is not None:
                table[b, : slot.num_pages] = slot.page_ids
        return table, np.asarray(context, dtype=np.int32)

    def add_request(self, prefilled: TinyKvCache, id: int):
        if id >= self.max_active_requests:
            raise ValueError(f"Request id {id} is out of range")
        if isinstance(prefilled, TinyKvFullCache) and prefilled.key_values is not None:
            B, H, _, D = prefilled.key_values[0].shape
            assert B == 1
            if self.HD is None:
                self.HD = (H, D)
            else:
                assert self.HD == (H, D)
        self.kv_caches[id] = prefilled

    def remove_request(self, id: int):
        if self.kv_caches[id] is None:
            raise ValueError(f"Request id {id} is not in the cache")
        self.kv_caches[id].release()
        self.kv_caches[id] = None
