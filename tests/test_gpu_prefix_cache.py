"""Prefix caching on the H100: ``tl_paged_cache_copy_prefix`` bit for bit against torch slicing, model calls on a reused
prefix bit for bit against an independent "rewind fork" (the donor's prompt run on a second model, its caches rewound to
the reused length, the new suffix run from there), the batcher with the cache on against the cache off, and the shared
page ids themselves."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, batch_generate
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load_ref():
    name = "tiny_llm_b200_prefix_cache_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("prefix_cache_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


pcref = _load_ref()


# ------------------------------------------------------------------ kernel --
def _records(layers, per_layer, pages, slots, g):
    """``per_layer`` copies in each of ``layers`` layers: sources from the first half of the pages, destinations from
    the second, never the same page twice."""
    out = []
    for layer in range(layers):
        src = torch.randperm(pages // 2, generator=g)[:per_layer].tolist()
        dst = (pages // 2 + torch.randperm(pages // 2, generator=g)[:per_layer]).tolist()
        out += [(layer, s, d, slots) for s, d in zip(src, dst)]
    return out


def _slabs(layers, pages, H, page, D, dtype, dev, g):
    ks = [torch.randn(pages, H, page, D, generator=g).to(dtype).to(dev) for _ in range(layers)]
    vs = [torch.randn(pages, H, page, D, generator=g).to(dtype).to(dev) for _ in range(layers)]
    sentinel = torch.tensor(-77.25, dtype=dtype)
    for s in (*ks, *vs):
        s[pages // 2 :] = sentinel.to(dev)  # destination tails keep this value
    return ks, vs


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("page", [16, 64, 128])
def test_copy_prefix_equals_torch_slicing(cuda_device, dtype, page):
    g = torch.Generator().manual_seed(page)
    H, D = 8, 128
    for slots in (1, 63, 64, 127, 128):
        if slots > page:
            continue
        # one record; one per layer over 36 layers; the most one launch takes (128), mixing layers
        for layers, per_layer in ((1, 1), (36, 1), (32, 4)):
            pages = 2 * per_layer + 2
            ks, vs = _slabs(layers, pages, H, page, D, dtype, cuda_device, g)
            copies = _records(layers, per_layer, pages, slots, g)
            want_k, want_v = pcref.expected_after(ks, vs, copies)
            launches = ext.launch_count()
            ext.paged_cache_copy_prefix(ks, vs, copies)
            torch.cuda.synchronize()
            assert ext.launch_count() - launches == 1
            for got, want in zip((*ks, *vs), (*want_k, *want_v)):
                assert torch.equal(got, want), (slots, layers, per_layer)


def test_copy_prefix_scalar_path_and_split_launches(cuda_device):
    g = torch.Generator().manual_seed(1)
    # D = 12 bf16 rows are 24 bytes: the scalar kernel
    ks, vs = _slabs(3, 6, 2, 16, 12, torch.bfloat16, cuda_device, g)
    copies = _records(3, 2, 6, 7, g)
    want_k, want_v = pcref.expected_after(ks, vs, copies)
    ext.paged_cache_copy_prefix(ks, vs, copies)
    assert all(torch.equal(a, b) for a, b in zip((*ks, *vs), (*want_k, *want_v)))
    # 280 records over 70 layers: two slab tables, three copy lists
    ks, vs = _slabs(70, 12, 2, 16, 64, torch.float32, cuda_device, g)
    copies = [(layer, s, 6 + s, 1 + (layer + s) % 16) for layer in range(70) for s in range(4)]
    want_k, want_v = pcref.expected_after(ks, vs, copies)
    launches = ext.launch_count()
    ext.paged_cache_copy_prefix(ks, vs, copies)
    torch.cuda.synchronize()
    assert ext.launch_count() - launches == 3  # layers 0-63: 256 records in two launches; layers 64-69: 24 in one
    assert all(torch.equal(a, b) for a, b in zip((*ks, *vs), (*want_k, *want_v)))


# ------------------------------------------------------------------ model calls --
@pytest.fixture(scope="module")
def ns(cuda_device):
    return synthetic_qwen3("tiny-d128", seed=3, realistic=True, max_position_embeddings=8192, device=cuda_device)


def _model(ns):
    model = Qwen3ModelWeek3(ns, page_size=64)
    model.decode_engine(1)  # the graph engines are active: reserved slabs, decode graph, 128-row prefill graph
    model.prefill_graph_len = 128
    return model


def _run(model, ids, start, cache, dev, chunk=128):
    """Prefill ``ids[start:]`` in ``chunk``-token calls; the last call's logits row."""
    logits = None
    for s in range(start, len(ids), chunk):
        logits = model(torch.tensor([ids[s : s + chunk]], dtype=torch.int32, device=dev), s, cache, logits_to_keep=1)
    return logits[0, -1].clone()


def _decode(model, cache, token, offset, steps, dev):
    out = []
    for i in range(steps):
        logits = model(torch.tensor([[token]], dtype=torch.int32, device=dev), offset + i, cache, logits_to_keep=1)
        token = int(ext.argmax(logits[:, -1, :].contiguous())[0])
        out.append(token)
    return out


def _release(cache):
    for c in cache:
        c.release()


BASE = [(37 * i + 11) % 500 + 1 for i in range(300)]  # ids below the 512-token vocabulary of tiny-d128
OTHER = [(53 * i + 7) % 500 + 1 for i in range(300)]


@pytest.mark.parametrize("case", ["page_boundary", "mid_page", "whole_prompt", "donor_decoding"])
def test_reused_prefix_equals_rewind_fork(cuda_device, ns, case):
    dev = cuda_device
    donor = BASE[:150]                    # pages of 64: [0, 64), [64, 128), a 22-token tail
    new = {"page_boundary": BASE[:128] + OTHER[:40], "mid_page": BASE[:100] + OTHER[:45], "whole_prompt": BASE[:150],
           "donor_decoding": BASE[:140] + OTHER[:20]}[case]
    m_want = {"page_boundary": 128, "mid_page": 100, "whole_prompt": 149, "donor_decoding": 140}[case]
    early = 2 if case == "donor_decoding" else 0
    late = 5 if case == "donor_decoding" else 0

    # warm run: the donor through the prefix cache, then the new prompt on what it left
    a = _model(ns)
    index = a.enable_prefix_cache()
    dc = a.create_kv_cache()
    first = int(ext.argmax(_run(a, donor, 0, dc, dev)[None].contiguous())[0])
    index.insert(donor, dc)
    donor_tokens = [first] + _decode(a, dc, first, len(donor), early, dev)
    nc = a.create_kv_cache()
    match = index.lookup(new)
    m = index.adopt(match, nc)
    assert m == m_want
    full = len(match.shared)
    for layer, (pool, d, c) in enumerate(zip(a.page_pools, dc, nc)):
        assert c.page_ids[:full] == d.page_ids[:full]          # the donor's pages, in every layer
        assert all(pool.refcount(p) == 3 for p in c.page_ids[:full])  # donor, new request, index
        if m % 64:
            assert c.page_ids[full] not in d.page_ids and pool.refcount(c.page_ids[full]) == 1
    if late:
        donor_tokens += _decode(a, dc, donor_tokens[-1], len(donor) + early, late, dev)
    got_logits = _run(a, new, m, nc, dev)

    # reference: the donor's prompt with the same calls on a second model, rewound to m, then the suffix from m
    b = _model(ns)
    rc = b.create_kv_cache()
    ref_first = int(ext.argmax(_run(b, donor, 0, rc, dev)[None].contiguous())[0])
    ref_tokens = [ref_first] + _decode(b, rc, ref_first, len(donor), early, dev)
    for c in rc:
        c.rewind(c.offset - m)
    want_logits = _run(b, new, m, rc, dev)

    assert torch.equal(got_logits, want_logits)
    assert int(ext.argmax(got_logits[None].contiguous())[0]) == int(ext.argmax(want_logits[None].contiguous())[0])
    for layer, (c, r) in enumerate(zip(nc, rc)):
        assert c.offset == r.offset == len(new)
        gk, gv = c.gather_dense()
        wk, wv = r.gather_dense()
        assert torch.equal(gk, wk) and torch.equal(gv, wv), layer
    if late:  # the donor, decoding on while the new request copied from its tail, gives the tokens of a run alone
        c3 = _model(ns)
        alone = c3.create_kv_cache()
        t0 = int(ext.argmax(_run(c3, donor, 0, alone, dev)[None].contiguous())[0])
        assert donor_tokens == [t0] + _decode(c3, alone, t0, len(donor), early + late, dev)
        _release(alone)
    assert ref_tokens == donor_tokens[: 1 + early]
    _release(dc)
    _release(nc)
    _release(rc)
    index.clear()
    assert all(not p.used_page_ids for p in a.page_pools)


# ------------------------------------------------------------------ batcher --
def test_batcher_cache_on_equals_cache_off(cuda_device, ns):
    g = torch.Generator().manual_seed(0)
    system = BASE[:192]                   # three full pages
    prompts = []
    for i in range(24):
        keep = (192, 128, 150, 100, 64, 37)[i % 6]          # page boundaries and mid-page
        tail = torch.randint(1, 500, (3 + int(torch.randint(0, 60, (1,), generator=g)),), generator=g).tolist()
        if (keep + len(tail)) % 128 == 1:
            tail.append(7)
        prompts.append(system[:keep] + tail)
    # A 1-token chunk is a decode step, whose bits follow the decode graph rather than a prefill chunk: no suffix is
    # that short with the cache on, and with it off no prompt ends in a 1-token chunk of 128 (n % 128 == 1).
    prompts.append(OTHER[:90])                              # no hit
    params = [None if i % 3 == 0 else SamplingParams(0.8, top_p=0.95, seed=i, repetition_penalty=1.2 if i % 3 == 2 else 1.0,
                                                      presence_penalty=0.5 if i % 3 == 2 else 0.0) for i in range(len(prompts))]
    budgets = [6 + i % 9 for i in range(len(prompts))]

    def run(prefix_cache):
        model = _model(ns)
        batch_generate(model, None, [OTHER[100:140], OTHER[150:230]], max_seq_len=384, batch_size=8, prefill_step=128, verbose=False,
                       device=cuda_device, max_new_tokens=[4, 4])  # warm the 8-slot decode graph
        from tiny_llm_b200.batch import ContinuousBatcher

        b = ContinuousBatcher(model, None, prompts, max_seq_len=384, batch_size=8, prefill_step=128, verbose=False, device=cuda_device,
                              max_new_tokens=budgets, sampling=[p if p is not None else SamplingParams(0.0) for p in params], logprobs=2,
                              prefix_cache=prefix_cache)
        out = dict(b.run())
        return out, b.logprobs, b

    off, lp_off, b_off = run(False)
    on, lp_on, b_on = run(True)
    assert on == off
    assert lp_on == lp_off
    assert b_on.reused_total > 0 and b_off.reused_total == 0
    assert b_on.prefill_tokens == sum(len(p) for p in prompts) - b_on.reused_total
    assert b_on.reused_tokens[len(prompts) - 1] == 0 and b_on.reused_tokens[1] >= 128 and b_on.reused_tokens[3] >= 100
    assert all(len(p) - b_on.reused_tokens[i] >= 2 for i, p in enumerate(prompts))
    s = b_on.model.prefix_cache.stats()
    assert s["cow_copies"] > 0 and s["hits"] >= 23
    b_on.model.prefix_cache.clear()
    assert all(not p.used_page_ids for p in b_on.model.page_pools)
