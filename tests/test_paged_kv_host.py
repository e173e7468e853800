"""Paged-KV host logic (allocator, block tables, counters, validation): integer
results, bit-exact against the literals of the reference's own tests
(tests/golden/reference_literals.json cites them).  CPU-only: the extension's
entry points are routed to the CPU oracle by the ``cpu_ext`` fixture."""

import json
from pathlib import Path

import numpy as np
import pytest
import torch

from tiny_llm_b200 import (
    BatchingKvCache,
    TinyKvFullCache,
    TinyKvPagedCache,
    TinyKvPagedPool,
    paged_attention,
    scaled_dot_product_attention_grouped,
)

LIT = json.loads((Path(__file__).parent / "golden" / "reference_literals.json").read_text())


def chunk(length, heads=2, dim=4, dtype=torch.float32, seed=None):
    g = torch.Generator().manual_seed(length * 131 + (seed or 0))
    return (torch.randn(1, heads, length, dim, generator=g).to(dtype), torch.randn(1, heads, length, dim, generator=g).to(dtype))


def state(cache):
    pool = cache.pool
    return (
        tuple(cache.page_ids), tuple(cache.page_lens), cache.offset, tuple(pool.free_page_ids), frozenset(pool.used_page_ids),
        pool.num_pages, pool.capacity, pool.reused_page_allocations, pool.storage_growths, pool.copied_pages_on_growth,
        pool.copied_bytes_on_growth,
    )


def test_dense_batching_cache_known_answer():
    lit = LIT["batching_kv_cache_dense"]
    col = lambda xs: torch.tensor(xs, dtype=torch.float32).reshape(1, 1, -1, 1)  # noqa: E731
    cache = BatchingKvCache(max_active_requests=3)
    assert cache.max_seq_len is None
    slot0, slot2 = TinyKvFullCache(), TinyKvFullCache()
    slot0.update_and_fetch(col(lit["slot0_prefill"]["keys"]), col(lit["slot0_prefill"]["values"]))
    slot2.update_and_fetch(col(lit["slot2_prefill"]["keys"]), col(lit["slot2_prefill"]["values"]))
    cache.add_request(slot0, 0)
    cache.add_request(slot2, 2)
    keys = torch.tensor(lit["step_keys"], dtype=torch.float32).reshape(3, 1, 2, 1)
    values = torch.tensor(lit["step_values"], dtype=torch.float32).reshape(3, 1, 2, 1)
    k, v, seq_len, mask = cache.update_and_fetch(keys, values, mask_length=2)
    assert seq_len is None
    assert torch.equal(k, torch.tensor(lit["expected_keys"], dtype=torch.float32).reshape(3, 1, 4, 1))
    assert torch.equal(v, torch.tensor(lit["expected_values"], dtype=torch.float32).reshape(3, 1, 4, 1))
    visible = torch.tensor(lit["expected_mask_is_visible"]).reshape(3, 1, 2, 4).bool()
    assert tuple(mask.shape) == (3, 1, 2, 4)
    assert torch.equal(mask == 0, visible) and torch.equal(torch.isinf(mask) & (mask < 0), ~visible)
    assert cache.last_batch_bytes == lit["last_batch_bytes"]
    assert cache.staging_copy_bytes == lit["staging_copy_bytes"]


def test_paged_cache_matches_full_cache(cpu_ext):
    full, paged = TinyKvFullCache(), TinyKvPagedCache(pool=TinyKvPagedPool(page_size=4))
    total = 0
    for length in (3, 2, 5):
        key, value = chunk(length)
        fk, fv, flen, _ = full.update_and_fetch(key, value)
        pk, pv, plen, _ = paged.update_and_fetch(key, value)
        total += length
        assert flen == plen == total
        assert paged.num_pages == (total + 3) // 4
        assert [paged.pool.read_page(p)[0].shape[2] for p in paged.page_ids] == [4] * paged.num_pages
        assert sum(paged.page_lens) == total
        assert torch.equal(pk, fk) and torch.equal(pv, fv)


def test_pool_reuses_freed_pages_lifo(cpu_ext):
    lit = LIT["paged_pool_reuse"]
    pool = TinyKvPagedPool(page_size=4)
    first, second = TinyKvPagedCache(pool), TinyKvPagedCache(pool)
    first.update_and_fetch(*chunk(lit["first_append"]))
    assert first.page_ids == lit["first_page_ids"] and pool.num_pages == 2 and pool.num_free_pages == 0
    first.release()
    assert first.offset == 0 and pool.num_pages == 2 and pool.num_free_pages == 2
    key, value = chunk(lit["second_append"])
    gk, gv, n, _ = second.update_and_fetch(key, value)
    assert n == 5 and pool.num_pages == 2 and pool.num_free_pages == 0
    assert set(second.page_ids) == set(lit["second_page_id_set"])
    assert second.page_ids == [1, 0]  # LIFO: release appends [0,1], pop() hands out 1 first (paged_kv_cache.py:135-137)
    assert pool.reused_page_allocations == 2
    assert torch.equal(gk, key) and torch.equal(gv, value)


def test_growth_counters_known_answer(cpu_ext):
    lit = LIT["paged_pool_growth"]
    pool = TinyKvPagedPool(page_size=lit["page_size"])
    cache = TinyKvPagedCache(pool)
    cache.update_and_fetch_paged(*chunk(lit["append_tokens"], lit["heads"], lit["head_dim"]))
    assert pool.num_pages == lit["num_pages"]
    assert pool.capacity == lit["capacity"]
    assert pool.key_pages.shape[0] == pool.num_pages and pool.value_pages.shape[0] == pool.num_pages
    assert pool.storage_growths == lit["storage_growths"]
    assert pool.copied_pages_on_growth == lit["copied_pages_on_growth"]
    assert pool.copied_bytes_on_growth == lit["copied_bytes_on_growth"]
    cache.release()
    assert pool.capacity == 8 and pool.num_free_pages == 5
    pool.reset()
    assert (pool.capacity, pool.num_pages, pool.num_free_pages, pool.storage_nbytes) == (0, 0, 0, 0)
    assert (pool.storage_growths, pool.copied_pages_on_growth, pool.copied_bytes_on_growth) == (0, 0, 0)


def test_dtype_and_shape_mismatch_leave_state_untouched(cpu_ext):
    cache = TinyKvPagedCache(TinyKvPagedPool(page_size=4))
    cache.update_and_fetch_paged(*chunk(4))
    before = state(cache)
    key, value = chunk(1)
    with pytest.raises(ValueError, match="existing page storage dtype"):
        cache.update_and_fetch_paged(key.to(torch.bfloat16), value.to(torch.bfloat16))
    assert state(cache) == before
    with pytest.raises(ValueError, match="same shape"):
        cache.update_and_fetch_paged(key, torch.cat([value, value], dim=2))
    assert state(cache) == before


def test_append_rolls_back_when_a_later_page_write_fails(cpu_ext, monkeypatch):
    cache = TinyKvPagedCache(TinyKvPagedPool(page_size=4))
    before = state(cache)
    real = cache.pool.write_page_slice
    calls = []

    def second_write_fails(*args, **kwargs):
        calls.append(1)
        if len(calls) == 2:
            raise RuntimeError("injected page write failure")
        return real(*args, **kwargs)

    monkeypatch.setattr(cache.pool, "write_page_slice", second_write_fails)
    with pytest.raises(RuntimeError, match="injected page write failure"):
        cache.update_and_fetch_paged(*chunk(5))
    assert len(calls) == 2 and state(cache) == before


def test_mixed_pools_fail_before_any_row_mutates(cpu_ext):
    first, second = TinyKvPagedCache(TinyKvPagedPool(4)), TinyKvPagedCache(TinyKvPagedPool(4))
    batch = BatchingKvCache(max_active_requests=2, max_seq_len=8)
    batch.add_request(first, 0)
    batch.add_request(second, 1)
    keys = torch.zeros(2, 2, 1, 4)
    before = (state(first), state(second))
    with pytest.raises(ValueError, match="share one page pool"):
        batch.update_and_fetch_paged(keys, keys, mask_length=1)
    assert (state(first), state(second)) == before and batch.HD is None


def test_block_table_object_is_cached_until_page_ids_change(cpu_ext):
    cache = TinyKvPagedCache(TinyKvPagedPool(page_size=4))
    cache.update_and_fetch_paged(*chunk(3))
    first = cache.block_table()
    assert cache.block_table() is first
    cache.update_and_fetch_paged(*chunk(1))  # fills the tail page: only context_lens changes
    assert cache.block_table() is first
    cache.update_and_fetch_paged(*chunk(1))  # new physical page
    assert cache.block_table() is not first
    assert cache.block_table().dtype == torch.int32 and cache.block_table().tolist() == [[0, 1]]


def test_rewind_known_answer(cpu_ext):
    lit = LIT["paged_rewind"]
    pool = TinyKvPagedPool(page_size=4)
    paged, full = TinyKvPagedCache(pool), TinyKvFullCache()
    for n in lit["appends"]:
        key, value = chunk(n)
        paged.update_and_fetch(key, value)
        full.update_and_fetch(key, value)
    assert paged.page_lens == lit["page_lens_before"]
    paged.rewind(lit["rewind"])
    full.rewind(lit["rewind"])
    assert paged.offset == full.offset == lit["offset_after"]
    assert paged.page_lens == lit["page_lens_after"] and paged.num_pages == 2
    assert pool.num_pages == lit["pool_num_pages"] and pool.num_free_pages == lit["pool_num_free_pages"]
    pk, pv = paged.gather_dense()
    assert torch.equal(pk, full.key_values[0]) and torch.equal(pv, full.key_values[1])


def test_noncontiguous_page_ids_with_a_blocker(cpu_ext):
    lit = LIT["noncontiguous_pages"]
    pool = TinyKvPagedPool(page_size=lit["page_size"])
    cache, blocker = TinyKvPagedCache(pool), TinyKvPagedCache(pool)
    cache.update_and_fetch(*chunk(lit["first_append"], dim=8))
    blocker.update_and_fetch(*chunk(lit["blocker_append"], dim=8))
    meta = cache.update_and_fetch_paged(*chunk(9, dim=8), mask="causal")
    assert cache.page_ids[:2] == lit["page_ids_prefix"] and cache.page_ids[2] == lit["third_page_id"]
    assert meta.block_table.tolist() == [[0, 1, 3]] and meta.context_lens.tolist() == [73]
    assert np.array_equal(meta.block_table_host, np.array([[0, 1, 3]], dtype=np.int32))


def test_batched_metadata_with_an_idle_slot_known_answer(cpu_ext):
    lit = LIT["batched_paged_metadata"]
    pool = TinyKvPagedPool(page_size=lit["page_size"])
    first, second = TinyKvPagedCache(pool), TinyKvPagedCache(pool)
    first.update_and_fetch(*chunk(lit["first_len"]))
    second.update_and_fetch(*chunk(lit["second_len"]))
    batch = BatchingKvCache(max_active_requests=3, max_seq_len=16)
    batch.add_request(first, lit["slots"][0])
    batch.add_request(second, lit["slots"][1])
    keys, values = torch.zeros(3, 2, 1, 4), torch.zeros(3, 2, 1, 4)
    keys[0:1], values[0:1] = chunk(1, seed=1)
    keys[2:3], values[2:3] = chunk(1, seed=2)
    meta = batch.update_and_fetch_paged(keys, values, mask_length=1, mask="causal")
    assert meta.context_lens.tolist() == lit["context_lens"]
    assert list(meta.block_table.shape) == lit["block_table_shape"]
    assert meta.block_table.tolist()[1] == lit["idle_row"]
    assert list(meta.key_pages.shape) == lit["key_pages_shape"]
    assert meta.block_table.dtype == torch.int32 and meta.context_lens.dtype == torch.int32
    g = torch.Generator().manual_seed(5)
    query = torch.randn(3, 4, 1, 4, generator=g)
    out = paged_attention(query, meta.key_pages, meta.value_pages, meta.block_table, meta.context_lens, meta.page_size, mask=meta.mask,
                          block_table_host=meta.block_table_host, context_lens_host=meta.context_lens_host)
    for slot, cache in ((0, first), (2, second)):
        k, v = cache.gather_dense()
        want = scaled_dot_product_attention_grouped(query[slot : slot + 1], k, v, mask="causal")
        torch.testing.assert_close(out[slot : slot + 1], want, rtol=1e-5, atol=1e-6)
    assert torch.count_nonzero(out[1]) == 0


@pytest.mark.parametrize("query_length", [1, 9, 65])
@pytest.mark.parametrize("case", LIT["paged_metadata_errors"]["cases"], ids=lambda c: c["match"].replace(" ", "-")[:24])
def test_invalid_metadata_is_rejected_before_dispatch(cpu_ext, monkeypatch, query_length, case):
    monkeypatch.setattr(cpu_ext, "paged_attention", lambda *a, **k: pytest.fail("dispatched despite invalid metadata"))
    head_dim = 4 if query_length == 1 else 128
    dtype = torch.float32 if query_length == 1 else torch.bfloat16
    query = torch.zeros(1, 4, query_length, head_dim, dtype=dtype)
    pages = torch.zeros(3, 2, 32, head_dim, dtype=dtype)
    with pytest.raises(ValueError, match=case["match"]):
        paged_attention(query, pages, pages.clone(), torch.tensor(case["block_table"], dtype=torch.int32),
                        torch.tensor(case["context_lens"], dtype=torch.int32), case["page_size"], mask="causal")


@pytest.mark.parametrize("case", LIT["paged_metadata_errors"]["short_context"], ids=lambda c: f"L{c['query_length']}")
def test_active_context_shorter_than_query_is_rejected(cpu_ext, case):
    L, ctx = case["query_length"], case["context_len"]
    head_dim = 4 if L == 2 else 128
    dtype = torch.float32 if L == 2 else torch.bfloat16
    query = torch.zeros(1, 4, L, head_dim, dtype=dtype)
    pages = torch.zeros(3, 2, 32, head_dim, dtype=dtype)
    live = (ctx + 31) // 32
    table = [[*range(live), *([-1] * (3 - live))]]
    with pytest.raises(ValueError, match=LIT["paged_metadata_errors"]["short_context_match"]):
        paged_attention(query, pages, pages.clone(), torch.tensor(table, dtype=torch.int32), torch.tensor([ctx], dtype=torch.int32), 32, mask="causal")


def test_array_masks_are_not_supported():
    q = torch.zeros(1, 4, 1, 4)
    p = torch.zeros(1, 2, 4, 4)
    with pytest.raises(NotImplementedError):
        paged_attention(q, p, p, torch.zeros(1, 1, dtype=torch.int32), torch.ones(1, dtype=torch.int32), 4, mask=torch.zeros(1))


def test_decode_batch_append_matches_per_request_writes(cpu_ext):
    """The single-launch decode append (CUDA extension) must leave pools and
    metadata exactly as the reference's per-request loop does."""
    def run(batched: bool):
        pool = TinyKvPagedPool(page_size=4)
        caches = [TinyKvPagedCache(pool) for _ in range(3)]
        for i, c in enumerate(caches):
            c.update_and_fetch(*chunk(3 + 2 * i, seed=i))
        batch = BatchingKvCache(max_active_requests=4, max_seq_len=64)
        for slot, c in zip((0, 1, 3), caches):
            batch.add_request(c, slot)
        metas = []
        for step in range(6):
            g = torch.Generator().manual_seed(100 + step)
            keys, values = torch.randn(4, 2, 1, 4, generator=g), torch.randn(4, 2, 1, 4, generator=g)
            if batched:
                keys, values = _FakeCuda(keys), _FakeCuda(values)
            metas.append(batch.update_and_fetch_paged(keys, values, mask_length=1, mask="causal"))
        return pool, caches, metas

    class _FakeCuda(torch.Tensor):
        """CPU tensor that claims to be on the GPU so the batched branch is taken."""

        @staticmethod
        def __new__(cls, t):
            return torch.Tensor._make_subclass(cls, t)

        @property
        def is_cuda(self):
            return True

    ref_pool, ref_caches, ref_metas = run(False)
    new_pool, new_caches, new_metas = run(True)
    assert [state(c) for c in new_caches] == [state(c) for c in ref_caches]
    assert torch.equal(new_pool.key_pages, ref_pool.key_pages) and torch.equal(new_pool.value_pages, ref_pool.value_pages)
    for a, b in zip(new_metas, ref_metas):
        assert a.block_table.tolist() == b.block_table.tolist() and a.context_lens.tolist() == b.context_lens.tolist()


# ---------------------------------------------------------------------------------------------
# CUDA runtime additions to the cache objects (engine.py): deferred one-token appends and bulk slot appends must be
# indistinguishable from the reference's per-token bookkeeping (paged_kv_cache.py:279-306).
def _pool_with_capacity(pages, page_size=4):
    pool = TinyKvPagedPool(page_size=page_size)
    pool.reserve(pages, 2, 8, dtype=torch.float32, device="cpu")
    return pool


def test_deferred_appends_settle_on_first_read_and_match_per_token_bookkeeping():
    from tiny_llm_b200.engine import _LockstepGroup

    pools = [_pool_with_capacity(8) for _ in range(3)]
    lazy = [TinyKvPagedCache(p) for p in pools]
    plain = [TinyKvPagedCache(_pool_with_capacity(8)) for _ in range(3)]
    for c in (*lazy, *plain):
        c.append_slots(5)  # pages [4, 1]
    group = _LockstepGroup(lazy)
    for c in lazy:
        c._lazy = group
    group.pending += 3  # three decode steps that fit in the tail page: nothing touched yet
    assert lazy[1]._page_lens == [4, 1] and lazy[1]._offset == 5
    assert lazy[0].logical_offset() == 8
    for c in plain:
        for _ in range(3):
            c.append_token_slot()
    assert lazy[2].offset == 8  # first read settles the whole group
    assert group.pending == 0
    for a, b in zip(lazy, plain):
        assert (a.page_ids, a.page_lens, a.offset) == (b.page_ids, b.page_lens, b.offset) == ([0, 1], [4, 4], 8)
    group.pending += 0
    lazy[0].rewind(3)
    assert lazy[0].page_lens == [4, 1] and lazy[0].epoch == 1
    group2 = _LockstepGroup(lazy[1:])
    for c in lazy[1:]:
        c._lazy = group2
    for c in lazy[1:]:
        c.append_token_slot()  # page boundary: [4, 4] -> new page, through the settled properties
    group2.pending += 2
    lazy[1].release()  # settles (both), frees the pages in page order, bumps the epoch
    assert lazy[1].page_ids == [] and lazy[1].offset == 0 and pools[1].used_page_ids == set()
    assert lazy[2].page_lens == [4, 4, 3] and lazy[2].offset == 11


def test_append_slots_equals_repeated_token_slots_and_is_all_or_nothing():
    a, b = TinyKvPagedCache(_pool_with_capacity(6)), TinyKvPagedCache(_pool_with_capacity(6))
    for count in (1, 3, 4, 9):
        a.append_slots(count)
        for _ in range(count):
            b.append_token_slot()
        assert (a.page_ids, a.page_lens, a.offset) == (b.page_ids, b.page_lens, b.offset)
    before = (list(a.page_ids), list(a.page_lens), a.offset, a.pool.num_pages)
    with pytest.raises(RuntimeError, match="slab exhausted"):
        a.append_slots(100)
    assert (a.page_ids, a.page_lens, a.offset, a.pool.num_pages) == before
