"""Prefix caching through the host layers, on the CPU stand-in of the extension (``cpu_ext``) plus the CPU stand-in of
``paged_cache_copy_prefix`` (``prefix_cache_ref``): the radix index (lookup, insert, LRU eviction), shared pages in
the pool (reference counts, the write guard, ``pages_available``), the batcher's lifecycle, generate, the CLI flag
and the shim's argument checks."""

import ctypes
import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.paged_kv_cache import TinyKvPagedCache, TinyKvPagedPool
from tiny_llm_b200.prefix_cache import PrefixCache
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load_ref():
    """The helper next to this file, by path: `tests` is no package of this project."""
    name = "tiny_llm_b200_prefix_cache_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("prefix_cache_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


pcref = _load_ref()
P = 4  # page size of the hand-built trees


@pytest.fixture
def cpu_pc(cpu_ext, monkeypatch):
    pcref.install(cpu_ext, monkeypatch)
    return cpu_ext


def _kv(ids, start, layer):
    """[1, 1, n, 2] float32 K/V rows that name their token, position and layer exactly."""
    t = torch.tensor([[float(tok) + (start + i) / 1024 + layer * 4096] for i, tok in enumerate(ids)])
    k = torch.cat([t, t + 0.5], dim=1)[None, None]
    return k.contiguous(), (-k).contiguous()


def _pools(layers=2, page=P):
    return [TinyKvPagedPool(page_size=page) for _ in range(layers)]


def _request(pools, index, ids):
    """A request that reuses what the index offers, writes the rest of its prompt and indexes it."""
    caches = [TinyKvPagedCache(pool) for pool in pools]
    m = index.adopt(index.lookup(ids), caches) if index is not None else 0
    if m < len(ids):
        for layer, c in enumerate(caches):
            c._append_chunk(*_kv(ids[m:], m, layer))
    if index is not None:
        index.insert(ids, caches)
    return caches, m


def _assert_holds(caches, ids):
    """Every layer's cache holds exactly the K/V rows of ``ids`` at their positions."""
    for layer, c in enumerate(caches):
        k, v = c.gather_dense()
        want_k, want_v = _kv(ids, 0, layer)
        assert torch.equal(k, want_k) and torch.equal(v, want_v)


def _release(*requests):
    for caches in requests:
        for c in caches:
            c.release()


# ------------------------------------------------------------------ index --
def test_lookup_full_chain_mid_page_partial_siblings_and_cap(cpu_pc):
    pools = _pools()
    index = PrefixCache(pools)
    a = list(range(10, 20))                # pages [10..13] [14..17], partial tail [18, 19]
    donor, _ = _request(pools, index, a)
    sib = a[:6] + [90, 91, 92]             # diverges mid page 1: page 1 of a stays, a sibling partial [14, 15, 90, 91] + ...
    other, m = _request(pools, index, sib)
    assert m == 6                          # page 0 shared, 2 slots of page 1 copied
    # exact full-page chain, then a partial page: longest common prefix 2 of the tail [18, 19]
    got = index.lookup(a + [1, 2])
    assert [n.tokens for n in got.shared] == [tuple(a[:4]), tuple(a[4:8])] and got.cow.tokens == (18, 19) and got.cow_slots == 2
    assert got.reused == 10
    # divergence inside the partial tail
    got = index.lookup(a[:9] + [77, 78])
    assert got.cow.tokens == (18, 19) and got.cow_slots == 1 and got.reused == 9
    # divergence inside a full page: the sibling with the longest common prefix wins
    got = index.lookup(a[:4] + [14, 15, 90, 5, 5])
    assert got.cow.tokens == (14, 15, 90, 91) and got.cow_slots == 3 and got.reused == 7
    got = index.lookup(a[:4] + [14, 15, 16, 5, 5])
    assert got.cow.tokens == tuple(a[4:8]) and got.cow_slots == 3
    # the last prompt token is always recomputed: a cached prompt reuses n - 1 tokens
    got = index.lookup(a[:8])
    assert len(got.shared) == 1 and got.cow.tokens == tuple(a[4:8]) and got.cow_slots == 3 and got.reused == 7
    assert index.lookup(a[:1]).reused == 0 and index.lookup([]).reused == 0
    _release(donor, other)
    index.clear()


def test_adopted_request_holds_the_donor_rows_and_copies_on_write(cpu_pc):
    pools = _pools()
    index = PrefixCache(pools)
    a = list(range(10, 21))
    donor, _ = _request(pools, index, a)
    b = a[:7] + [50, 51, 52]
    taker, m = _request(pools, index, b)
    assert m == 7
    for layer, (cd, ct) in enumerate(zip(donor, taker)):
        assert ct.page_ids[0] == cd.page_ids[0]                      # shared
        assert ct.page_ids[1] not in cd.page_ids                     # the copy-on-write page is private
        assert pools[layer].refcount(cd.page_ids[0]) == 3            # donor, taker, index
        assert pools[layer].refcount(cd.page_ids[1]) == 2            # donor, index
    _assert_holds(donor, a)
    _assert_holds(taker, b)
    s = index.stats()
    assert (s["hits"], s["reused_tokens"], s["cow_copies"], s["cow_slots"]) == (1, 7, 1, 3)
    _release(donor, taker)
    index.clear()
    for pool in pools:
        assert not pool.used_page_ids and not pool.extra_refs and not pool.indexed


def test_duplicate_insert_keeps_the_existing_node(cpu_pc):
    pools = _pools()
    index = PrefixCache(pools)
    a = list(range(30, 39))
    first, _ = _request(pools, index, a)
    before = index.stats()["cached_pages"]
    second, _ = _request(pools, None, a)                 # computed without the index, then inserted
    assert index.insert(a, second) == 0
    assert index.stats()["cached_pages"] == before == 3
    for layer, c in enumerate(second):
        assert all(pools[layer].refcount(p) == 1 and p not in pools[layer].indexed for p in c.page_ids)
    got = index.lookup(a + [1])
    assert [n.pages for n in got.shared] == [[c.page_ids[0] for c in first], [c.page_ids[1] for c in first]]
    _release(first, second)
    index.clear()


def test_eviction_takes_unreferenced_leaves_least_recently_used_first(cpu_pc):
    pools = _pools()
    index = PrefixCache(pools)
    a, b = [1, 2, 3, 4, 5, 6], [1, 2, 3, 4, 7, 8]
    ra, _ = _request(pools, index, a)          # nodes: [1..4] -> [5, 6]
    rb, _ = _request(pools, index, b)          # [1..4] shared -> [7, 8]
    _release(ra)
    index.lookup(a + [9])                      # touches [1..4] and the [5, 6] leaf
    assert index.evictable_pages() == 1        # [5, 6]: [1..4] and [7, 8] are held by b
    held = set(rb[0].page_ids)
    assert index.evict_one() and index.stats()["evictions"] == 1
    assert {tuple(n.tokens) for n in index._nodes} == {(1, 2, 3, 4), (7, 8)}
    assert not index.evict_one()               # everything left is held
    _release(rb)
    assert index.evictable_pages() == 2
    index.lookup([1, 2, 3, 4, 7, 8, 0])        # the parent is touched last, but only a leaf can go
    assert index.evict_one()
    assert {tuple(n.tokens) for n in index._nodes} == {(1, 2, 3, 4)}
    assert held - set(pools[0].free_page_ids) == {next(iter(index._nodes)).pages[0]}
    assert index.evict_one() and not index._nodes
    for pool in pools:
        assert not pool.used_page_ids


def test_allocation_evicts_before_taking_a_new_id_and_pages_available_counts_it(cpu_pc):
    pools = _pools(layers=1)
    index = PrefixCache(pools)
    a = list(range(100, 109))
    ra, _ = _request(pools, index, a)
    pool = pools[0]
    assert pool.pages_available() == pool.capacity - pool.num_pages + len(pool.free_page_ids)
    _release(ra)
    assert pool.pages_available() == pool.capacity - pool.num_pages + 3
    n = pool.num_pages
    other, _ = _request(pools, None, [7] * 5)   # two pages, free list empty: the two newest leaves go
    assert pool.num_pages == n and index.stats()["evictions"] == 2
    assert [tuple(x.tokens) for x in index._nodes] == [tuple(a[:4])]
    _release(other)
    index.clear()


# ------------------------------------------------------------------ pool --
def test_reference_counts_through_release_and_rewind(cpu_pc):
    pools = _pools(layers=1)
    index = PrefixCache(pools)
    pool = pools[0]
    a = list(range(12))                         # three full pages
    donor, _ = _request(pools, index, a)
    taker, m = _request(pools, index, a[:8] + [40, 41])
    assert m == 8
    shared = donor[0].page_ids[:2]
    assert [pool.refcount(p) for p in shared] == [3, 3]
    taker[0].rewind(6)                          # drops its own page and the shared second page
    assert taker[0].page_ids == shared[:1] and pool.refcount(shared[1]) == 2
    _release(donor)
    assert [pool.refcount(p) for p in shared] == [2, 1]
    _release(taker)
    assert all(pool.refcount(p) == 1 for p in shared)
    index.clear()
    assert not pool.used_page_ids and sorted(pool.free_page_ids) == list(range(pool.num_pages))


def test_write_guard(cpu_pc):
    pools = _pools(layers=1)
    index = PrefixCache(pools)
    pool = pools[0]
    a = list(range(10))                         # pages [0..3] [4..7], partial [8, 9] indexed with length 2
    donor, _ = _request(pools, index, a)
    taker, _ = _request(pools, index, a[:8] + [1])
    c = donor[0]
    # the donor keeps decoding into its own indexed tail, at slots beyond the indexed length
    c._append_chunk(*_kv([5], 10, 0))
    page, slot = c.append_token_slot()
    assert (page, slot) == (c.page_ids[2], 3)
    # a write into a page another request holds raises, as does one below a partial node's indexed length
    with pytest.raises(RuntimeError, match="requests share"):
        pool.check_write(c.page_ids[1], 0)
    with pytest.raises(RuntimeError, match="below its 2 slots"):
        pool.check_write(c.page_ids[2], 1)
    with pytest.raises(RuntimeError, match="below its 2 slots"):
        c.rewind(3)                             # would leave the next append at slot 1 of the indexed tail
    with pytest.raises(RuntimeError, match="requests share"):
        c.rewind(6)                             # would leave the next append inside the shared second page
    assert c.offset == 12
    c.rewind(2)                                 # back to the indexed length: allowed
    t = taker[0]
    t.rewind(1)                                 # the taker's copy-on-write page is its own
    assert t.offset == 8
    with pytest.raises(RuntimeError, match="requests share"):
        t.rewind(1)
    _release(donor, taker)
    index.clear()


def test_write_guard_covers_every_append_path(cpu_pc):
    pools = _pools(layers=1)
    index = PrefixCache(pools)
    a = list(range(6))
    donor, _ = _request(pools, index, a)        # full [0..3], partial [4, 5]
    c = donor[0]
    c.rewind(0)
    # fake a request that holds the partial page below its length (not reachable through adopt_prefix)
    pool = pools[0]
    partial = c.page_ids[1]
    c._page_lens[-1] = 1
    c._offset = 5
    with pytest.raises(RuntimeError, match="below its 2 slots"):
        c._append_chunk(*_kv([9], 5, 0))
    with pytest.raises(RuntimeError, match="below its 2 slots"):
        c.append_slots(1)
    with pytest.raises(RuntimeError, match="below its 2 slots"):
        c.append_token_slot()
    assert c.page_lens == [4, 1] and pool.refcount(partial) == 2
    c._page_lens[-1], c._offset = 2, 6
    _release(donor)
    index.clear()


def test_adopt_prefix_checks(cpu_pc):
    pools = _pools(layers=1)
    ra, _ = _request(pools, None, list(range(9)))
    c = TinyKvPagedCache(pools[0])
    with pytest.raises(ValueError, match="only full pages"):
        c.adopt_prefix(ra[0].page_ids[2:], [1], 1)
    with pytest.raises(ValueError, match="do not fit"):
        c.adopt_prefix(ra[0].page_ids[:1], [P], P + P)
    with pytest.raises(ValueError, match="fresh cache"):
        ra[0].adopt_prefix([], [], 1)
    free = TinyKvPagedPool(P)
    with pytest.raises(ValueError, match="is free"):
        TinyKvPagedCache(free).adopt_prefix([0], [P], P)
    assert c.page_ids == [] and all(pools[0].refcount(p) == 1 for p in ra[0].page_ids)
    _release(ra)


def test_cache_off_allocator_is_unchanged(cpu_pc):
    """Scripted appends / rewinds / releases: page ids, counters and the LIFO free list, written out by hand."""
    pool = TinyKvPagedPool(page_size=P)
    a, b = TinyKvPagedCache(pool), TinyKvPagedCache(pool)
    a._append_chunk(*_kv(range(9), 0, 0))          # a: 0 1 2
    b._append_chunk(*_kv(range(5), 0, 0))          # b: 3 4
    a.rewind(6)                                    # frees 2 then 1
    assert pool.free_page_ids == [2, 1] and a.page_ids == [0]
    b._append_chunk(*_kv(range(4), 5, 0))          # b fills page 4, then takes 1
    assert b.page_ids == [3, 4, 1] and pool.free_page_ids == [2]
    a.release()
    b._append_chunk(*_kv(range(12), 9, 0))         # fills page 1, then LIFO: 0, 2, then the next new id
    assert b.page_ids == [3, 4, 1, 0, 2, 5] and pool.free_page_ids == []
    # slabs of 4 then 8 pages (the second growth carries the 4 pages written before it)
    assert (pool.num_allocated_pages, pool.reused_page_allocations, pool.storage_growths) == (6, 3, 2)
    assert pool.copied_pages_on_growth == 4 and pool.pages_available() == 2
    assert pool.extra_refs == {} and pool.indexed == {}
    b.release()
    assert pool.free_page_ids == [3, 4, 1, 0, 2, 5]


# ------------------------------------------------------------------ batcher --
@pytest.fixture(scope="module")
def ns():
    return synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)


BASE = [(7 * i + 3) % 500 + 1 for i in range(40)]
PROMPTS = [
    BASE,                                   # 2 full pages + 8 tokens
    BASE + [9] * 5,                         # reuses all 40: pages 0, 1 shared, 8 slots copied
    BASE[:20] + [11] * 10,                  # page 0 shared, 4 slots of page 1 copied
    BASE[:32],                              # cached as a prefix: 31 reused, 15 slots of page 1 copied
    [13] * 20,                              # no hit
]
PLAN = {0: 0, 1: 40, 2: 20, 3: 31, 4: 0}


def test_batcher_reuses_as_planned_and_returns_every_page(cpu_pc, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    b = ContinuousBatcher(model, None, PROMPTS, max_seq_len=96, batch_size=5, prefill_step=16, verbose=False,
                          max_new_tokens=[12] * len(PROMPTS), prefix_cache=True)
    b.record_timing = True
    b.run()
    assert b.reused_tokens == PLAN and b.reused_total == 91
    assert b.prefill_tokens == sum(len(p) - PLAN[i] for i, p in enumerate(PROMPTS))
    s = model.prefix_cache.stats()
    assert (s["lookups"], s["hits"], s["reused_tokens"], s["cow_copies"], s["cow_slots"]) == (5, 3, 91, 3, 8 + 4 + 15)
    assert s["evictions"] == 0 and s["cached_pages"] > 0
    model.prefix_cache.clear()
    for pool in model.page_pools:
        assert not pool.used_page_ids and len(pool.free_page_ids) == pool.num_pages
        assert not pool.extra_refs and not pool.indexed
    assert 0 < b.peak_live_pages


def test_batcher_counts_shared_pages_once(cpu_pc, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    b = ContinuousBatcher(model, None, PROMPTS[:2], max_seq_len=96, batch_size=2, prefill_step=64, verbose=False,
                          max_new_tokens=[8, 8], prefix_cache=True)
    b.record_timing = True
    try:
        while not b.idle():
            b.step()
            live = [s for s in b.slots if s is not None]
            if len(live) == 2:
                distinct = len(set(live[0].kv_cache[0].page_ids) | set(live[1].kv_cache[0].page_ids))
                assert distinct < sum(len(s.kv_cache[0].page_ids) for s in live)
                b.peak_live_pages = 0
                b._record_cache_state()
                assert b.peak_live_pages == distinct * model.num_hidden_layers
    finally:
        b.release_all()
    model.prefix_cache.clear()


def test_cache_off_batcher_has_no_index(cpu_pc, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    b = ContinuousBatcher(model, None, PROMPTS[:2], max_seq_len=96, batch_size=2, prefill_step=16, verbose=False, max_new_tokens=[3, 3])
    b.run()
    assert model.prefix_cache is None and b.reused_tokens == {} and b.prefill_tokens == 85
    assert all(p.prefix_index is None and not p.extra_refs for p in model.page_pools)


def test_generate_with_prefix_cache(cpu_pc, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    first = greedy_generate_ids(model, PROMPTS[0], 4, prefix_cache=True)
    assert model.prefix_cache.stats()["cached_pages"] == 3
    again = greedy_generate_ids(model, PROMPTS[1], 4, prefix_cache=True)
    s = model.prefix_cache.stats()
    assert (s["hits"], s["reused_tokens"], s["cow_copies"]) == (1, 40, 1)
    assert len(first) == len(again) == 4
    model.prefix_cache.clear()
    assert all(not p.used_page_ids for p in model.page_pools)


def test_cli_prefix_cache_flag(cpu_pc, capsys):
    ids = ";".join(",".join(map(str, p)) for p in PROMPTS[:2])
    argv = ["batch", "--synthetic", "tiny-d128", "--prompt-ids", ids, "--max-new-tokens", "3", "--device", "cpu",
            "--batch-size", "2", "--max-seq-len", "96", "--prefill-step", "16", "--quiet"]
    assert cli_main(argv) == 0
    plain = capsys.readouterr().out
    assert "reused" not in plain and "prefix cache" not in plain
    assert cli_main(argv + ["--prefix-cache"]) == 0  # 128-slot pages: the second request copies 40 slots of the first
    out = capsys.readouterr().out
    assert "reused tokens: 0" in out and "reused tokens: 40" in out and "prefix cache: lookups 2, hits 1" in out


# ------------------------------------------------------------------ shim --
def _slabs(layers=3, pages=4, dtype=torch.float32):
    g = torch.Generator().manual_seed(0)
    ks = [torch.randn(pages, 2, 8, 8, generator=g).to(dtype) for _ in range(layers)]
    vs = [torch.randn(pages, 2, 8, 8, generator=g).to(dtype) for _ in range(layers)]
    return ks, vs


@pytest.mark.parametrize("copies, message", [
    ([(3, 0, 1, 4)], "layer 3 outside the 3 slabs"),
    ([(-1, 0, 1, 4)], "layer -1"),
    ([(0, 4, 1, 4)], "page outside the 4 pages"),
    ([(0, 0, -1, 4)], "page outside"),
    ([(0, 0, 1, 0)], r"slots 0 outside \[1, 8\]"),
    ([(0, 0, 1, 9)], r"slots 9 outside \[1, 8\]"),
    ([(1, 2, 2, 3)], "copied onto itself"),
    ([(1, 0, 2, 3), (1, 1, 2, 3)], "destination page 2 named twice in layer 1"),
    ([(1, 0, 2, 3), (1, 2, 3, 3)], "both a source and a destination"),
    ([(1, 0, 2, 3), (1, 3, 0, 3)], "both a source and a destination"),
])
def test_shim_refuses_bad_records_before_the_device(copies, message):
    ks, vs = _slabs()
    with pytest.raises(RuntimeError, match=message):
        ext.paged_cache_copy_prefix(ks, vs, copies)


def test_shim_refuses_bad_slabs_then_cpu_tensors():
    ks, vs = _slabs()
    with pytest.raises(RuntimeError, match="float32 or bfloat16"):
        ext.paged_cache_copy_prefix([k.half() for k in ks], [v.half() for v in vs], [(0, 0, 1, 1)])
    with pytest.raises(RuntimeError, match="same float32 or bfloat16 dtype"):
        ext.paged_cache_copy_prefix(ks, [vs[0].bfloat16(), *vs[1:]], [(0, 0, 1, 1)])
    with pytest.raises(RuntimeError, match="one key and one value slab"):
        ext.paged_cache_copy_prefix(ks, vs[:2], [(0, 0, 1, 1)])
    with pytest.raises(RuntimeError, match="one H, page_size and D"):
        ext.paged_cache_copy_prefix([ks[0], ks[1][:, :1].contiguous(), ks[2]], vs, [(0, 0, 1, 1)])
    # the same layer and destination in different layers are fine; the device check comes last
    with pytest.raises(RuntimeError, match="paged_cache_copy_prefix: the course extension is GPU-only"):
        ext.paged_cache_copy_prefix(ks, vs, [(0, 0, 1, 8), (1, 0, 1, 8), (2, 3, 2, 1)])
    assert "tl_paged_cache_copy_prefix" in ext.EXPORTED_SYMBOLS and "paged_cache_copy_prefix" in ext.__all__


def test_records_fit_the_kernel_parameter_limit():
    assert ctypes.sizeof(ext.KvSlabTable) + ctypes.sizeof(ext.PrefixCopyList) + 4 * 4 <= 4096
    assert ext.PREFIX_COPIES >= 2 * 36 and ext.PREFIX_COPY_LAYERS == 64


def test_cpu_stand_in_copies_only_the_slots():
    ks, vs = _slabs()
    before_k, before_v = [k.clone() for k in ks], [v.clone() for v in vs]
    copies = [(0, 1, 2, 3), (2, 0, 3, 8), (2, 1, 2, 1)]
    pcref.copy_prefix_like_ext(ks, vs, copies)
    for layer, src, dst, slots in copies:
        for now, was in ((ks, before_k), (vs, before_v)):
            assert torch.equal(now[layer][dst, :, :slots], was[layer][src, :, :slots])
            assert torch.equal(now[layer][dst, :, slots:], was[layer][dst, :, slots:])
            assert torch.equal(now[layer][src], was[layer][src])
    assert torch.equal(ks[1], before_k[1]) and torch.equal(vs[1], before_v[1])
