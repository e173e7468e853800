"""Host-only parts of tests/engine_plan.py, the eager statement of the graph engines' steps: the packing of the fused
weights and the metadata built from request caches.  No GPU needed."""

import importlib.util
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import BatchingKvCache
from tiny_llm_b200.paged_kv_cache import TinyKvPagedCache, TinyKvPagedPool


def _load(name, file):
    """A helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


plan = _load("tiny_llm_b200_engine_plan", "engine_plan.py")


def labelled(K, N, tag):
    """Weights whose every entry names its row: word = tag * 2^20 + row, scale / bias = row + 1 (exact in bf16 up to 256)."""
    rows = torch.arange(K, dtype=torch.int32)
    return SimpleNamespace(weight=(tag * 2**20 + rows)[:, None].expand(K, N // 8).contiguous().view(torch.uint32),
                           scales=(rows + 1).to(torch.bfloat16)[:, None].expand(K, N // 128).contiguous(),
                           biases=(-(rows + 1)).to(torch.bfloat16)[:, None].expand(K, N // 128).contiguous())


def test_gate_up_pairs_layout_is_the_headers_and_the_extensions():
    K, N = 48, 256
    gate, up = labelled(K, N, 1), labelled(K, N, 2)
    packed = plan.pack_gate_up(gate, up)
    words = packed.weight[:, 0].tolist()
    for c in range(K // 8):
        for j in range(8):
            assert words[16 * c + j] == 1 * 2**20 + 8 * c + j, "rows 16c..16c+7 are gate rows 8c..8c+7"
            assert words[16 * c + 8 + j] == 2 * 2**20 + 8 * c + j, "rows 16c+8..16c+15 are up rows 8c..8c+7"
    assert packed.scales[:, 0].tolist() == [float(8 * (r // 16) + r % 8 + 1) for r in range(2 * K)]
    for name in ("weight", "scales", "biases"):
        a, b = getattr(gate, name), getattr(up, name)
        a, b = (a.view(torch.int32), b.view(torch.int32)) if a.dtype == torch.uint32 else (a, b)
        assert torch.equal(getattr(packed, name), ext.interleave_gate_up(a, b)), name


def test_qkv_rows_are_q_then_k_then_v():
    wq, wk, wv = labelled(64, 256, 1), labelled(16, 256, 2), labelled(16, 256, 3)
    packed = plan.pack_qkv(wq, wk, wv)
    tags = (packed.weight[:, 0] >> 20).tolist()
    assert tags == [1] * 64 + [2] * 16 + [3] * 16
    assert (packed.weight[:, 0] & 0xFFFFF).tolist() == list(range(64)) + list(range(16)) * 2
    assert packed.biases.shape == (96, 2) and packed.weight.dtype == torch.int32


def pools(layers, page, capacity):
    out = []
    for _ in range(layers):
        p = TinyKvPagedPool(page_size=page)
        p.reserve(capacity, 1, 8, dtype=torch.bfloat16, device="cpu")
        out.append(p)
    return out


def test_decode_metadata_from_request_caches():
    """Slots 0 and 3 hold requests, 1 and 2 are idle; slot 3's append ends exactly on a page boundary."""
    page, B, layers, max_pages = 4, 4, 2, 5
    ps = pools(layers, page, 32)
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=page * max_pages) for _ in range(layers)]
    burn = [TinyKvPagedCache(p) for p in ps]  # take pages 0, 1 so the requests' ids differ from their logical pages
    for c in burn:
        c.append_slots(5)
    lens = {0: 5, 3: 7}
    for b, n in lens.items():
        for layer, p in enumerate(ps):
            c = TinyKvPagedCache(p)
            c.append_slots(n)
            tables[layer].add_request(c, b)
    for t in tables:  # the engine's own bookkeeping of the step: one token per request
        for b in lens:
            t.kv_caches[b].append_token_slot()
    meta = plan.decode_metadata(tables, [11, 12, 13, 14], max_pages)
    assert meta.tokens == [11, 0, 0, 14]
    assert meta.offsets == [5, 0, 0, 7]
    assert meta.context_lens == [6, 0, 0, 8]
    want = np.array([[2, 3, -1, -1, -1], [-1] * 5, [-1] * 5, [4, 5, -1, -1, -1]], dtype=np.int32)
    assert meta.tables.dtype == np.int32 and meta.tables.shape == (layers, B, max_pages)
    for layer in range(layers):
        assert (meta.tables[layer] == want).all(), meta.tables[layer]
    # three steps accounted for ahead (decode_on_device): the metadata is the first step's, the table holds every page
    for t in tables:
        for b in lens:
            for _ in range(2):
                t.kv_caches[b].append_token_slot()
    ahead = plan.decode_metadata(tables, [11, 12, 13, 14], max_pages, steps=3)
    assert ahead.offsets == [5, 0, 0, 7] and ahead.context_lens == [6, 0, 0, 8]
    assert ahead.tables[0, 3].tolist() == [4, 5, 6, -1, -1]


def test_decode_metadata_of_a_single_request_cache_list():
    ps = pools(2, 16, 8)
    cache = [TinyKvPagedCache(p) for p in ps]
    for c in cache:
        c.append_slots(16)
        c.append_token_slot()  # token 16 opens page 1
    meta = plan.decode_metadata(cache, [9], 3)
    assert (meta.tokens, meta.offsets, meta.context_lens) == ([9], [16], [17])
    assert meta.tables.tolist() == [[[0, 1, -1]], [[0, 1, -1]]]


def test_right_aligned_prefill_rows():
    assert plan.prefill_rows(8, 3, 10) == (5, [5, 6, 7, 8, 9, 10, 11, 12], [0, 0, 0, 0, 0, 11, 12, 13], 13)
    # a 2-token first chunk: the padding rows in front of position 0 carry negative positions and context 0
    assert plan.prefill_rows(6, 2, 0) == (4, [-4, -3, -2, -1, 0, 1], [0, 0, 0, 0, 1, 2], 2)
    assert plan.prefill_rows(4, 4, 64) == (0, [64, 65, 66, 67], [65, 66, 67, 68], 68)


def test_prefill_metadata_from_request_caches():
    ps = pools(2, 4, 8)
    cache = [TinyKvPagedCache(p) for p in ps]
    for c in cache:
        c.append_slots(3)
        c.append_slots(3)  # the chunk: fills page 0's last slot, opens page 1
    meta = plan.prefill_metadata(cache, [7, 8, 9], 3, 5, 4)
    assert meta.tokens == [0, 0, 7, 8, 9]
    assert meta.offsets == [1, 2, 3, 4, 5]
    assert meta.context_lens == [0, 0, 4, 5, 6]
    assert meta.ctx_after == 6
    assert meta.tables.tolist() == [[0, 1, -1, -1], [0, 1, -1, -1]]
