"""Paged KV storage (``src/tiny_llm_ref/paged_kv_cache.py``).

One ``TinyKvPagedPool`` per transformer layer owns the physical page slab
``[capacity, H_kv, page_size, D]`` for keys and for values; every request holds
one ``TinyKvPagedCache`` per layer, a purely logical object (page ids, page
fill levels, offset).  At the Qwen3-4B shape a (page, head) is 128 x 128 bf16 =
32 KiB of contiguous HBM, the unit the attention kernels stream.

All allocator behaviour is integer, host-side and identical to the reference,
counters included: LIFO free list (:135-142), storage growth to
``max(4, num_pages, 2*capacity)`` copying ``num_pages-1`` old pages (:154-182),
fill-the-tail-then-allocate appends with snapshot/rollback (:271-312),
``block_table`` objects cached per (page ids, width) (:364-377).
"""

from __future__ import annotations

import itertools
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200

# Every (re)allocation of a pool's K/V slabs takes a fresh number: the graph engines compare 36 integers per step
# instead of 72 data_ptr() calls to learn whether the addresses baked into their captured graphs are still valid.
_SLAB_VERSIONS = itertools.count(1)

from .kv_cache import TinyKvCache

_PAGE_DTYPES = (torch.float32, torch.bfloat16)


@dataclass
class PagedKvMetadata:
    """What paged attention needs for one layer (paged_kv_cache.py:11-18).  The
    two ``*_host`` fields are the host copies the tables were built from; they
    let ``paged_attention`` validate without a device round trip."""

    key_pages: torch.Tensor
    value_pages: torch.Tensor
    block_table: torch.Tensor
    context_lens: torch.Tensor
    page_size: int
    mask: torch.Tensor | str | None = None
    block_table_host: np.ndarray | None = None
    context_lens_host: np.ndarray | None = None


class TinyKvPagedPool:
    """Layer-local physical page storage shared by all requests of that layer."""

    def __init__(self, page_size: int = 128):
        assert page_size > 0
        self.page_size = page_size
        self._key_pages: torch.Tensor | None = None
        self._value_pages: torch.Tensor | None = None
        self.free_page_ids: list[int] = []
        self.used_page_ids: set[int] = set()
        self.num_allocated_pages = 0
        self.reused_page_allocations = 0
        self.storage_growths = 0
        self.slab_version = 0  # no slab yet
        self.copied_pages_on_growth = 0
        self.copied_bytes_on_growth = 0

    # ---- views and sizes ---------------------------------------------------
    @property
    def key_pages(self) -> torch.Tensor | None:
        return None if self._key_pages is None else self._key_pages[: self.num_pages]

    @property
    def value_pages(self) -> torch.Tensor | None:
        return None if self._value_pages is None else self._value_pages[: self.num_pages]

    @property
    def capacity(self) -> int:
        return 0 if self._key_pages is None else self._key_pages.shape[0]

    @property
    def num_pages(self) -> int:
        return self.num_allocated_pages

    @property
    def num_free_pages(self) -> int:
        return len(self.free_page_ids)

    @property
    def storage_nbytes(self) -> int:
        if self._key_pages is None or self._value_pages is None:
            return 0
        return sum(t.numel() * t.element_size() for t in (self._key_pages, self._value_pages))

    # ---- validation --------------------------------------------------------
    def validate_page_chunk(self, key: torch.Tensor, value: torch.Tensor) -> None:
        """paged_kv_cache.py:74-104 - nothing is mutated here."""
        if key.dim() != 4 or value.dim() != 4:
            raise ValueError("Paged K/V chunks must be 4D [1, H, S, D]")
        if key.shape != value.shape:
            raise ValueError("Paged K/V chunks must have the same shape")
        B, H, S, D = key.shape
        if B != 1:
            raise ValueError("Paged request cache only supports one request")
        if H <= 0 or D <= 0 or S <= 0:
            raise ValueError("Paged K/V chunks must have positive valid dimensions")
        if key.dtype != value.dtype or key.dtype not in _PAGE_DTYPES:
            raise ValueError("Paged K/V chunks must have the same float32 or bfloat16 dtype")
        if (self._key_pages is None) != (self._value_pages is None):
            raise ValueError("Paged K/V storage is incomplete")
        if self._key_pages is not None:
            if tuple(self._key_pages.shape[1:]) != (H, self.page_size, D):
                raise ValueError("Paged K/V chunks must match the existing page storage shape")
            if self._value_pages.shape != self._key_pages.shape:
                raise ValueError("Paged key and value storage must have the same shape")
            if self._key_pages.dtype != key.dtype or self._value_pages.dtype != value.dtype:
                raise ValueError("Paged K/V chunks must match the existing page storage dtype")

    # ---- transactional state ------------------------------------------------
    def _snapshot_state(self) -> tuple:
        return (
            self._key_pages,
            self._value_pages,
            list(self.free_page_ids),
            set(self.used_page_ids),
            self.num_allocated_pages,
            self.reused_page_allocations,
            self.storage_growths,
            self.copied_pages_on_growth,
            self.copied_bytes_on_growth,
        )

    def _restore_state(self, state: tuple) -> None:
        (
            self._key_pages,
            self._value_pages,
            self.free_page_ids,
            self.used_page_ids,
            self.num_allocated_pages,
            self.reused_page_allocations,
            self.storage_growths,
            self.copied_pages_on_growth,
            self.copied_bytes_on_growth,
        ) = state

    # ---- allocator ----------------------------------------------------------
    def allocate_page(self) -> int:
        """Newest freed page first, else the next never-used id (:132-142)."""
        if self.free_page_ids:
            page_id = self.free_page_ids.pop()
            self.reused_page_allocations += 1
        else:
            page_id = self.num_pages
            self.num_allocated_pages += 1
        self.used_page_ids.add(page_id)
        return page_id

    def free_page(self, page_id: int) -> None:
        """Ids stay stable; stale bytes are masked by page_lens (:236-242)."""
        if page_id not in self.used_page_ids:
            raise ValueError(f"Page {page_id} is already free")
        self.used_page_ids.remove(page_id)
        self.free_page_ids.append(page_id)

    def read_page(self, page_id: int) -> tuple[torch.Tensor, torch.Tensor]:
        if self._key_pages is None or self._value_pages is None:
            raise ValueError(f"Page {page_id} has no storage")
        if page_id >= self.num_pages:
            raise ValueError(f"Page {page_id} is out of range")
        return self._key_pages[page_id : page_id + 1], self._value_pages[page_id : page_id + 1]

    def _ensure_page_storage(self, key: torch.Tensor, value: torch.Tensor) -> None:
        """Grow the slab geometrically when ``num_pages`` outruns it (:154-182)."""
        B, H, _, D = key.shape
        assert B == 1
        if self._key_pages is not None and self._value_pages is not None:
            assert tuple(self._key_pages.shape[1:]) == (H, self.page_size, D)
            assert self._value_pages.shape == self._key_pages.shape
            assert self._key_pages.dtype == key.dtype
            assert self._value_pages.dtype == value.dtype
            if self.capacity >= self.num_pages:
                return
        self._grow(max(4, self.num_pages, self.capacity * 2), H, D, key.dtype, key.device)

    def _grow(self, new_capacity: int, H: int, D: int, dtype, device) -> None:
        shape = (new_capacity, H, self.page_size, D)
        new_k = torch.zeros(shape, dtype=dtype, device=device)
        new_v = torch.zeros(shape, dtype=dtype, device=device)
        self.storage_growths += 1
        if self._key_pages is not None and self._value_pages is not None:
            carried = self.num_pages - 1  # the newest page has not been written yet
            self.copied_pages_on_growth += carried
            old_k, old_v = self._key_pages[:carried], self._value_pages[:carried]
            self.copied_bytes_on_growth += (old_k.numel() + old_v.numel()) * old_k.element_size()
            new_k[:carried] = old_k
            new_v[:carried] = old_v
        self._key_pages, self._value_pages = new_k, new_v
        self.slab_version = next(_SLAB_VERSIONS)

    def reserve(self, num_pages: int, heads: int, head_dim: int, dtype=torch.bfloat16, device="cuda") -> None:
        """CUDA extension: size the slab once (one counted growth) so that page
        base addresses stay fixed, which CUDA-graph replay of the decode step
        needs.  Logical page accounting is unchanged."""
        if self.capacity >= num_pages:
            return
        if self._key_pages is None:
            self._key_pages = torch.zeros((num_pages, heads, self.page_size, head_dim), dtype=dtype, device=device)
            self._value_pages = torch.zeros_like(self._key_pages)
            self.storage_growths += 1
            self.slab_version = next(_SLAB_VERSIONS)
            return
        shape = (num_pages, heads, self.page_size, head_dim)
        new_k = torch.zeros(shape, dtype=dtype, device=device)
        new_v = torch.zeros(shape, dtype=dtype, device=device)
        self.storage_growths += 1
        live = self.num_pages
        self.copied_pages_on_growth += live
        self.copied_bytes_on_growth += 2 * self._key_pages[:live].numel() * self._key_pages.element_size()
        new_k[:live] = self._key_pages[:live]
        new_v[:live] = self._value_pages[:live]
        self._key_pages, self._value_pages = new_k, new_v
        self.slab_version = next(_SLAB_VERSIONS)

    def reset(self) -> None:
        if self.used_page_ids:
            raise ValueError("Cannot reset a page pool with live requests")
        self._key_pages = None
        self._value_pages = None
        self.slab_version = next(_SLAB_VERSIONS)
        self.free_page_ids.clear()
        self.num_allocated_pages = 0
        self.reused_page_allocations = 0
        self.storage_growths = 0
        self.copied_pages_on_growth = 0
        self.copied_bytes_on_growth = 0

    # ---- writes -------------------------------------------------------------
    def _prepare_slice(self, page_id: int, start: int, key: torch.Tensor, value: torch.Tensor) -> None:
        """Every check of write_page_slice plus storage growth (:196-222)."""
        self.validate_page_chunk(key, value)
        if key.shape[2] > self.page_size:
            raise ValueError("Paged K/V writes cannot exceed one physical page")
        if page_id not in self.used_page_ids:
            raise ValueError(f"Page {page_id} is free")
        if page_id < 0 or page_id >= self.num_pages:
            raise ValueError(f"Page {page_id} is out of range")
        if start < 0 or start + key.shape[2] > self.page_size:
            raise ValueError("Paged K/V write is outside page storage")
        self._ensure_page_storage(key, value)
        H, slots, D = self._key_pages.shape[1:]
        assert self._value_pages.shape == self._key_pages.shape
        assert slots == self.page_size
        assert tuple(key.shape[:2]) == (1, H) and key.shape[3] == D

    def write_page_slice(self, page_id: int, start: int, key: torch.Tensor, value: torch.Tensor) -> None:
        """One request, one page, K then V: two in-place kernel launches (:224-234)."""
        self._prepare_slice(page_id, start, key, value)
        self._key_pages = tiny_llm_ext_b200.paged_cache_update(self._key_pages, key.contiguous(), page_id, start)
        self._value_pages = tiny_llm_ext_b200.paged_cache_update(self._value_pages, value.contiguous(), page_id, start)

    def reserve_page_slice(self, page_id: int, start: int, key: torch.Tensor, value: torch.Tensor) -> None:
        """Host half of ``write_page_slice``: checks and storage, no launch.  The
        bytes follow in one batched ``append_decode_batch`` call."""
        self._prepare_slice(page_id, start, key, value)

    def can_batch_chunk_append(self, key: torch.Tensor, value: torch.Tensor) -> bool:
        """True when a multi-page chunk may be written by ONE launch (``write_page_spans``) instead of
        two ``paged_cache_update`` launches plus two slice copies per page."""
        if not key.is_cuda or key.dtype not in _PAGE_DTYPES or key.shape[2] < 2:
            return False
        if "write_page_slice" in vars(self) or type(self).write_page_slice is not TinyKvPagedPool.write_page_slice:
            return False  # overridden writer (fault injection, instrumentation): keep the per-page calls
        return key.stride(3) == 1 and value.stride() == key.stride()

    def write_page_spans(self, spans: list, key: torch.Tensor, value: torch.Tensor) -> None:
        tiny_llm_ext_b200.paged_cache_append_chunk(self._key_pages, self._value_pages, key, value, spans)

    def can_batch_decode_append(self, keys: torch.Tensor, slots: list) -> bool:
        """True when a decode batch (one token per request) may be written with
        a single device-driven launch instead of 2 launches per request."""
        if keys.shape[2] != 1 or not keys.is_cuda or keys.dtype not in _PAGE_DTYPES:
            return False
        if "write_page_slice" in vars(self):  # instance-level override (fault injection)
            return False
        return all(type(s)._append_chunk is TinyKvPagedCache._append_chunk for s in slots)

    def append_decode_batch(self, keys, values, block_table, context_lens) -> None:
        tiny_llm_ext_b200.paged_cache_append_decode(
            self.key_pages, self.value_pages, keys.contiguous(), values.contiguous(), block_table, context_lens
        )


class TinyKvPagedCache(TinyKvCache):
    """Request-and-layer-local logical cache backed by a layer pool (:245-443)."""

    def __init__(self, pool: TinyKvPagedPool):
        self.pool = pool
        self.page_size = pool.page_size
        self.page_ids: list[int] = []
        self._page_lens: list[int] = []
        self._offset = 0
        # CUDA runtime (engine.py): while a request decodes inside the CUDA-graph engine, one-token
        # appends that fit in the tail page are DEFERRED - counted once per request instead of once
        # per layer object - and folded into page_lens / offset the moment anybody looks at them.
        self._lazy = None
        self.epoch = 0  # bumped by rewind() / release(): the page-id list changed other than by appending
        self._cached_block_table: torch.Tensor | None = None
        self._cached_block_table_key: tuple[tuple[int, ...], int] | None = None

    # page_lens / offset are the reference's plain attributes (paged_kv_cache.py:245-262); here they
    # are properties so that deferred appends are settled before any read or write.
    @property
    def page_lens(self) -> list[int]:
        if self._lazy is not None:
            self._lazy.settle()
        return self._page_lens

    @page_lens.setter
    def page_lens(self, value: list[int]) -> None:
        if self._lazy is not None:
            self._lazy.settle()
        self._page_lens = value

    @property
    def offset(self) -> int:
        if self._lazy is not None:
            self._lazy.settle()
        return self._offset

    @offset.setter
    def offset(self, value: int) -> None:
        if self._lazy is not None:
            self._lazy.settle()
        self._offset = value

    def logical_offset(self) -> int:
        """``offset`` without settling deferred appends (hot-path reads of the decode runtime)."""
        lazy = self._lazy
        return self._offset if lazy is None else self._offset + lazy.pending

    @property
    def num_pages(self) -> int:
        return len(self.page_ids)

    @property
    def key_values(self) -> tuple[torch.Tensor, torch.Tensor] | None:
        return None if self.offset == 0 else self.gather_dense()

    def _device(self):
        return self.pool._key_pages.device if self.pool._key_pages is not None else torch.device("cpu")

    # ---- append -------------------------------------------------------------
    def _append_chunk(self, key: torch.Tensor, value: torch.Tensor, device_write: bool = True) -> None:
        """Fill the tail page, then take fresh pages; all-or-nothing (:271-312)."""
        self.pool.validate_page_chunk(key, value)
        total = key.shape[2]
        mine = self._snapshot_state()
        theirs = self.pool._snapshot_state()
        # CUDA: when nothing overrides the per-page writer, the host bookkeeping below runs with the
        # launch-free reserve_page_slice and ALL page slices are written by one device launch at the
        # end (same bytes, same page/offset evolution, same all-or-nothing behaviour: the launch
        # happens only after every check and allocation has succeeded)
        batched = device_write and self.pool.can_batch_chunk_append(key, value)
        put = self.pool.write_page_slice if (device_write and not batched) else self.pool.reserve_page_slice
        spans = []
        done = 0
        try:
            if self.page_ids and self.page_lens[-1] < self.page_size:
                room = self.page_size - self.page_lens[-1]
                take = min(room, total)
                put(self.page_ids[-1], self.page_lens[-1], key[:, :, :take, :], value[:, :, :take, :])
                spans.append((self.page_ids[-1], self.page_lens[-1], take, 0))
                self.page_lens[-1] += take
                done = take
            while done < total:
                stop = min(done + self.page_size, total)
                page_id = self.pool.allocate_page()
                put(page_id, 0, key[:, :, done:stop, :], value[:, :, done:stop, :])
                spans.append((page_id, 0, stop - done, done))
                self.page_ids.append(page_id)
                self.page_lens.append(stop - done)
                done = stop
            if batched:
                self.pool.write_page_spans(spans, key, value)
            self.offset += total
        except Exception:
            self.pool._restore_state(theirs)
            self._restore_state(mine)
            raise

    def append_slots(self, count: int) -> None:
        """Host bookkeeping of a ``count``-token append whose bytes are written by a device-driven kernel
        (prefill-chunk engine): the page / offset evolution of ``_append_chunk`` (fill the tail page, then
        take fresh pages), all-or-nothing, no launch.  The pool slab must cover the pages (``pool.reserve``)."""
        if count <= 0:
            return
        tail_room = self.page_size - self.page_lens[-1] if self.page_ids else 0
        fresh = max(0, -(-(count - tail_room) // self.page_size))
        if fresh > len(self.pool.free_page_ids) + (self.pool.capacity - self.pool.num_pages):
            raise RuntimeError("page pool slab exhausted: reserve() more pages before prefilling")
        take = min(tail_room, count)
        if take:
            self.page_lens[-1] += take
        left = count - take
        while left > 0:
            n = min(self.page_size, left)
            self.page_ids.append(self.pool.allocate_page())
            self.page_lens.append(n)
            left -= n
        self.offset += count

    def append_token_slot(self) -> tuple[int, int]:
        """Host bookkeeping of a ONE-token append whose bytes are written by a
        device-driven kernel (decode engine): same page/offset evolution as
        ``_append_chunk`` with S == 1, minus the device write and the snapshot
        (nothing can fail once the page is allocated).  Returns (page id, slot).
        The pool slab must already cover the page (``pool.reserve``)."""
        if self.page_ids and self.page_lens[-1] < self.page_size:
            slot = self.page_lens[-1]
            self.page_lens[-1] += 1
            page_id = self.page_ids[-1]
        else:
            if not self.pool.free_page_ids and self.pool.num_pages >= self.pool.capacity:
                raise RuntimeError("page pool slab exhausted: reserve() more pages before decoding")
            page_id = self.pool.allocate_page()
            self.page_ids.append(page_id)
            self.page_lens.append(1)
            slot = 0
        self.offset += 1
        return page_id, slot

    def validate_append(self, key: torch.Tensor, value: torch.Tensor) -> None:
        self.pool.validate_page_chunk(key, value)

    def _snapshot_state(self) -> tuple:
        return (list(self.page_ids), list(self.page_lens), self.offset, self._cached_block_table, self._cached_block_table_key)

    def _restore_state(self, state: tuple) -> None:
        (self.page_ids, self.page_lens, self.offset, self._cached_block_table, self._cached_block_table_key) = state

    # ---- dense compatibility --------------------------------------------------
    def gather_dense(self) -> tuple[torch.Tensor, torch.Tensor]:
        """Concatenate the valid prefix of every page (tests / dense fallback)."""
        assert self.offset > 0
        ks, vs = [], []
        for page_id, fill in zip(self.page_ids, self.page_lens):
            k_page, v_page = self.pool.read_page(page_id)
            assert k_page.shape[2] == self.page_size and v_page.shape[2] == self.page_size
            ks.append(k_page[:, :, :fill, :])
            vs.append(v_page[:, :, :fill, :])
        if len(ks) == 1:
            return ks[0], vs[0]
        return torch.cat(ks, dim=2), torch.cat(vs, dim=2)

    def update_and_fetch(self, key, value, mask_length=None, mask=None):
        self._append_chunk(key, value)
        dense_k, dense_v = self.gather_dense()
        return dense_k, dense_v, self.offset, mask

    # ---- paged metadata -------------------------------------------------------
    def block_table_host(self, max_pages: int | None = None) -> np.ndarray:
        width = self.num_pages if max_pages is None else max_pages
        assert width >= self.num_pages
        row = np.full((1, width), -1, dtype=np.int32)
        row[0, : self.num_pages] = self.page_ids
        return row

    def block_table(self, max_pages: int | None = None) -> torch.Tensor:
        """int32 ``[1, max_pages]``; the SAME tensor object is handed out until
        the page-id list (or the width) changes (:364-377)."""
        width = self.num_pages if max_pages is None else max_pages
        assert width >= self.num_pages
        tag = (tuple(self.page_ids), width)
        if self._cached_block_table is not None and self._cached_block_table_key == tag:
            return self._cached_block_table
        self._cached_block_table = torch.from_numpy(self.block_table_host(width)).to(self._device())
        self._cached_block_table_key = tag
        return self._cached_block_table

    def context_lens(self) -> torch.Tensor:
        return torch.tensor([self.offset], dtype=torch.int32, device=self._device())

    def paged_metadata(self, max_pages: int | None = None, mask=None) -> PagedKvMetadata:
        assert self.pool.key_pages is not None
        assert self.pool.value_pages is not None
        return PagedKvMetadata(
            key_pages=self.pool.key_pages,
            value_pages=self.pool.value_pages,
            block_table=self.block_table(max_pages=max_pages),
            context_lens=self.context_lens(),
            page_size=self.page_size,
            mask=mask,
            block_table_host=self.block_table_host(max_pages),
            context_lens_host=np.asarray([self.offset], dtype=np.int32),
        )

    def update_and_fetch_paged(self, key, value, mask_length=None, mask=None) -> PagedKvMetadata:
        self._append_chunk(key, value)
        return self.paged_metadata(mask=mask)

    def materialize(self):
        """Eager backend: page storage is already materialised (batch.py:65-68
        still calls this after every prefill chunk, and tests override it)."""
        return None

    # ---- shrinking ------------------------------------------------------------
    def rewind(self, n: int):
        """Drop the newest ``n`` tokens; whole pages go back to the pool (:414-434)."""
        assert 0 <= n <= self.offset
        keep = self.offset - n
        if keep == self.offset:
            return
        if keep == 0:
            self.release()
            return
        self.epoch += 1
        pages_needed = (keep + self.page_size - 1) // self.page_size
        while len(self.page_ids) > pages_needed:
            self.page_lens.pop()
            self.pool.free_page(self.page_ids.pop())
        self.page_lens[-1] = keep - self.page_size * (pages_needed - 1)
        self.offset = keep

    def release(self):
        """Return every page, in page order, to the pool's free list (:436-443)."""
        self.epoch += 1
        lens = self.page_lens  # settles deferred appends first
        for page_id in self.page_ids:
            self.pool.free_page(page_id)
        self.page_ids.clear()
        lens.clear()
        self.offset = 0
