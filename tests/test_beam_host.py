"""Beam search on the host: the plain-loop rule (``beam_ref.py``) on hand-built cases, the protocol of
``beam_search_ids`` with scripted models on CPU page pools and the references in place of ``tl_logprobs`` and
``tl_beam_select``, the fork's page bookkeeping, the refusals, the CLI and the C ABI's argument checks."""

import ctypes
import importlib.util
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import BeamHypothesis, beam_search_ids, greedy_generate_ids
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.kv_cache import BatchingKvCache
from tiny_llm_b200.paged_kv_cache import TinyKvPagedCache, TinyKvPagedPool, fork


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_beam_ref", "beam_ref.py")
LP = _load("tiny_llm_b200_logprobs_ref", "logprobs_ref.py")
PC = _load("tiny_llm_b200_prefix_cache_ref", "prefix_cache_ref.py")
NINF = -math.inf


# ------------------------------------------------------------------ the rule --
def test_ties_within_a_row_go_to_the_lower_rank():
    live, fin = R.select([[-1.0, -1.0, -2.0]], [[7, 3, 9]], [0.0], 2, ())
    assert live == [(0, 7, -1.0), (0, 3, -1.0)] and fin == []


def test_ties_across_rows_go_to_the_lower_row():
    live, _ = R.select([[-1.0, -3.0], [-0.5, -3.0]], [[4, 5], [6, 7]], [-1.0, -1.5], 2, ())
    assert live == [(0, 4, -2.0), (1, 6, -2.0)]


def test_eos_below_w_finishes_and_eos_at_or_beyond_w_is_skipped():
    # order: (0, 9) eos p=0, (0, 1) p=1, (1, 9) eos p=2 >= W, (1, 2) p=3
    live, fin = R.select([[-0.1, -0.2, -5], [-0.3, -0.4, -5]], [[9, 1, 8], [9, 2, 8]], [0.0, 0.0], 2, (9,))
    assert fin == [(0, 9, np.float32(-0.1), 0)]
    assert live == [(0, 1, np.float32(-0.2)), (1, 2, np.float32(-0.4))]


def test_several_eos_ids():
    live, fin = R.select([[-0.1, -0.2, -0.3, -0.4]], [[5, 6, 1, 2]], [0.0], 2, (6, 5))
    assert [f[1] for f in fin] == [5, 6] and [f[3] for f in fin] == [0, 1]
    assert [t for _, t, _ in live] == [1, 2]


def test_fewer_takeable_candidates_than_w():
    live, fin = R.select([[-0.5, NINF, NINF], [NINF, NINF, NINF]], [[3, -1, -1], [0, 1, 2]], [0.0, 0.0], 3, ())
    assert live == [(0, 3, -0.5)] and fin == []
    live, _ = R.select([[-0.5, -0.1]], [[3, 4]], [NINF], 2, ())
    assert live == [], "a row with cum -inf is never taken"
    live, _ = R.select([[math.nan, -0.1]], [[3, 4]], [0.0], 2, ())
    assert live == [(0, 4, np.float32(-0.1))]


def test_score_is_one_fp32_rounding_of_cum_plus_lp():
    cum, lp = np.float32(-1.0000001), np.float32(-3e-8)
    live, _ = R.select([[lp]], [[1]], [cum], 1, ())
    assert live[0][2] == np.float32(cum + lp)


def test_the_walk_stops_at_w_live():
    live, fin = R.select([[-0.1, -0.2, -0.3, -0.4]], [[1, 2, 3, 9]], [0.0], 2, (9,))
    assert [t for _, t, _ in live] == [1, 2] and fin == []


def _table_tops(table, V):
    """``tops`` for ``search``: each beam's logits are ``table(ids)``; the top-N lists come from the float64 reference
    rounded to fp32, as ``logprobs_like_ext`` gives them."""

    def tops(beams, n):
        rows = np.stack([np.asarray(table(tuple(ids)), dtype=np.float32) for ids in beams])
        _, _, _, ids, lps = LP.logprobs(rows, None, None, n)
        return lps, ids

    return tops


def _logits_table(V, seed, step=0.5):
    """Deterministic logits of a context, on a coarse grid so that exact ties are common."""

    def table(ctx):
        g = np.random.default_rng(abs(hash((seed, ctx))) % (2**32))
        return g.integers(0, 6, V).astype(np.float32) * np.float32(step)

    return table


def _search(table, V, W, max_new, eos=(), **kw):
    tops = _table_tops(table, V)
    n = W + len(set(eos))
    return R.search(lambda beams: tops(beams, n), max_new, W, eos=eos, **kw)


@pytest.mark.parametrize("alpha", [0.0, 1.0, 2.0])
def test_length_penalty_scores(alpha):
    hyps = _search(_logits_table(7, 1), 7, 3, 5, eos=(2,), length_penalty=alpha, num_return_sequences=3)
    for ids, total, score, finished in hyps:
        L = len(ids) + int(finished)
        assert score == total / L**alpha
    assert [h[2] for h in hyps] == sorted((h[2] for h in hyps), reverse=True)


def test_max_new_tokens_zero_and_one():
    assert _search(_logits_table(7, 1), 7, 2, 0) == []
    hyps = _search(_logits_table(7, 1), 7, 2, 1, num_return_sequences=2)
    assert all(len(ids) == 1 and not fin for ids, _, _, fin in hyps)


def test_early_stopping_both_ways():
    table = _logits_table(5, 3)
    a = _search(table, 5, 2, 12, eos=(0,), early_stopping=True, num_return_sequences=2)
    b = _search(table, 5, 2, 12, eos=(0,), early_stopping=False, num_return_sequences=2)
    assert all(len(h) == 4 for h in a + b)
    assert max(len(h[0]) for h in a) <= max(len(h[0]) for h in b)


def test_num_return_sequences():
    table = _logits_table(9, 4)
    three = _search(table, 9, 4, 4, num_return_sequences=3)
    one = _search(table, 9, 4, 4, num_return_sequences=1)
    assert len(three) == 3 and one == three[:1]


# ------------------------------------------------------------------ scripted models on CPU page pools --
class PagedScripted:
    """A model whose logits are ``table(context ids)``, where the context is read back from its own layer caches: each
    appended K row names its token and position, so a fork that copies the wrong slots changes the logits."""

    def __init__(self, table, V, layers=2, page=4, fail_at=None):
        self.table, self.V, self.page = table, V, page
        self.pools = [TinyKvPagedPool(page_size=page) for _ in range(layers)]
        self.calls = 0
        self.fail_at = fail_at

    def create_kv_cache(self):
        return [TinyKvPagedCache(pool) for pool in self.pools]

    def _append(self, caches, ids, start):
        for layer, c in enumerate(caches):
            t = torch.tensor([[float(tok), float(start + i) + layer * 4096] for i, tok in enumerate(ids)])[None, None]
            c._append_chunk(t.contiguous(), (-t).contiguous())

    def _row(self, caches):
        ctx = None
        for layer, c in enumerate(caches):
            k, v = c.gather_dense()
            assert torch.equal(k[0, 0, :, 1], torch.arange(c.offset, dtype=torch.float32) + layer * 4096), "positions"
            assert torch.equal(v, -k)
            toks = tuple(int(x) for x in k[0, 0, :, 0])
            assert ctx is None or toks == ctx, "layers disagree"
            ctx = toks
        return torch.from_numpy(np.asarray(self.table(ctx), dtype=np.float32))

    def __call__(self, inputs, offset, cache, logits_to_keep=None):
        self.calls += 1
        if self.fail_at is not None and self.calls == self.fail_at:
            raise RuntimeError("injected failure")
        if isinstance(cache[0], BatchingKvCache):
            rows = []
            for b, slot in enumerate(cache[0].kv_caches):
                if slot is None:
                    rows.append(torch.zeros(self.V))
                    continue
                caches = [layer.kv_caches[b] for layer in cache]
                assert caches[0].offset == offset[b]
                self._append(caches, [int(inputs[b, 0])], offset[b])
                rows.append(self._row(caches))
            return torch.stack(rows)[:, None]
        ids = [int(t) for t in inputs.reshape(-1)]
        self._append(cache, ids, offset)
        return self._row(cache)[None, None]


@pytest.fixture
def kernels_ref(cpu_ext, monkeypatch):
    """The float64 ``tl_logprobs`` and the plain-loop ``tl_beam_select`` in place of the kernels, the torch copy in
    place of ``tl_paged_cache_copy_prefix`` (which records every call's records)."""
    monkeypatch.setattr(ext, "logprobs", LP.logprobs_like_ext)
    monkeypatch.setattr(ext, "beam_select", R.beam_select_like_ext)
    calls = []

    def copy(key_slabs, value_slabs, copies, stream=None):
        calls.append(list(copies))
        PC.copy_prefix_like_ext(key_slabs, value_slabs, copies)

    monkeypatch.setattr(ext, "paged_cache_copy_prefix", copy)
    return calls


def _all_free(model):
    return all(not p.used_page_ids and not p.extra_refs for p in model.pools)


def _run(model, prompt, max_new, W, **kw):
    hyps = beam_search_ids(model, prompt, max_new, num_beams=W, **kw)
    return [(h.ids, h.sum_logprob, h.score, h.finished) for h in hyps]


CASES = [
    dict(V=7, seed=1, W=3, max_new=6, eos=(2,)),
    dict(V=5, seed=2, W=4, max_new=9, eos=(0, 4)),
    dict(V=11, seed=3, W=8, max_new=5, eos=()),
    dict(V=3, seed=4, W=8, max_new=4, eos=(1,)),  # fewer takeable candidates than W
    dict(V=9, seed=5, W=2, max_new=12, eos=(3,), length_penalty=2.0, early_stopping=True),
    dict(V=9, seed=6, W=5, max_new=7, eos=(3, 4, 5, 6), length_penalty=0.0),
]


@pytest.mark.parametrize("case", CASES, ids=[str(i) for i in range(len(CASES))])
@pytest.mark.parametrize("prompt", [[1, 2, 3], [1, 2, 3, 4], [5] * 9])
def test_protocol_gives_the_references_hypotheses(kernels_ref, case, prompt):
    case = dict(case)
    V, seed, W, max_new, eos = (case.pop(k) for k in ("V", "seed", "W", "max_new", "eos"))
    table = _logits_table(V, seed)
    W_ret = min(W, 3)
    model = PagedScripted(table, V)
    want = _search(lambda ids: table(tuple(prompt) + ids), V, W, max_new, eos=eos,
                   num_return_sequences=W_ret, **case)
    got = _run(model, prompt, max_new, W, eos_token_ids=eos, num_return_sequences=W_ret, **case)
    assert got == [(list(i), float(s), sc, f) for i, s, sc, f in want]
    assert _all_free(model)


def test_one_beam_with_early_stopping_is_greedy(kernels_ref):
    table = _logits_table(13, 7, step=0.25)
    prompt = [3, 1, 4]
    for eos in (None, 5):
        model = PagedScripted(table, 13)
        greedy = greedy_generate_ids(model, prompt, 20, eos_token_id=eos)
        hyps = beam_search_ids(model, prompt, 20, num_beams=1, early_stopping=True, eos_token_ids=() if eos is None else (eos,))
        assert hyps[0].ids == greedy
        assert _all_free(model)


def test_an_exception_mid_search_returns_every_page(kernels_ref):
    for fail_at in (2, 3, 5):
        model = PagedScripted(_logits_table(6, 8), 6, fail_at=fail_at)
        with pytest.raises(RuntimeError, match="injected"):
            beam_search_ids(model, [1, 2, 3, 4, 5], 10, num_beams=4)
        assert _all_free(model)


def test_result_block_round_trip():
    from tiny_llm_b200.generate import unpack_beam_result

    live, fin = [(0, 5, -1.5), (2, 7, -2.25)], [(1, 9, -0.75, 0)]
    assert unpack_beam_result(R.pack(live, fin).tolist()) == (live, fin)


# ------------------------------------------------------------------ fork bookkeeping --
def _filled(pools, n):
    caches = [TinyKvPagedCache(p) for p in pools]
    for layer, c in enumerate(caches):
        t = torch.arange(2 * n, dtype=torch.float32).view(1, 1, n, 2) + layer * 1000
        c._append_chunk(t.contiguous(), (-t).contiguous())
    return caches


def test_fork_shares_full_pages_and_copies_the_tail(kernels_ref):
    pools = [TinyKvPagedPool(page_size=4) for _ in range(3)]
    parent = _filled(pools, 10)  # two full pages and a tail of 2
    (kids,) = fork([(parent, 2)])
    assert len(kids) == 2 and len(kernels_ref) == 1
    records = kernels_ref[0]
    assert len(records) == 2 * 3
    for layer, pool in enumerate(pools):
        full, tail = parent[layer].page_ids[:2], parent[layer].page_ids[2]
        assert all(pool.refcount(p) == 3 for p in full)
        assert pool.refcount(tail) == 1
        for kid in kids:
            c = kid[layer]
            assert c.page_ids[:2] == full and c.page_ids[2] != tail and c.offset == 10 and c.page_lens == [4, 4, 2]
            assert (layer, tail, c.page_ids[2], 2) in records
            assert all(torch.equal(a, b) for a, b in zip(c.gather_dense(), parent[layer].gather_dense()))
    for caches in (parent, *kids):
        for c in caches:
            c.release()
    assert all(not p.used_page_ids and not p.extra_refs for p in pools)


def test_a_page_boundary_tail_needs_no_copy(kernels_ref):
    pools = [TinyKvPagedPool(page_size=4) for _ in range(2)]
    parent = _filled(pools, 8)
    (kids,) = fork([(parent, 3)])
    assert kernels_ref == []
    for layer, pool in enumerate(pools):
        assert all(pool.refcount(p) == 4 for p in parent[layer].page_ids)
        assert all(k[layer].page_ids == parent[layer].page_ids for k in kids)
    kid = kids[0]
    with pytest.raises(RuntimeError, match="share"):
        pools[0].check_write(kid[0].page_ids[-1], 3)
    for caches in (parent, *kids):
        for c in caches:
            c.release()
    assert all(not p.used_page_ids and not p.extra_refs for p in pools)


def test_several_parents_fork_in_one_copy_call(kernels_ref):
    pools = [TinyKvPagedPool(page_size=4) for _ in range(2)]
    a, b = _filled(pools, 5), _filled(pools, 7)
    kids = fork([(a, 1), (b, 2)])
    assert [len(k) for k in kids] == [1, 2] and len(kernels_ref) == 1 and len(kernels_ref[0]) == 2 * 3
    for caches in (a, b, *kids[0], *kids[1]):
        for c in caches:
            c.release()
    assert all(not p.used_page_ids for p in pools)


def test_a_failing_fork_gives_back_what_it_took(kernels_ref, monkeypatch):
    pools = [TinyKvPagedPool(page_size=4) for _ in range(2)]
    parent = _filled(pools, 6)
    monkeypatch.setattr(ext, "paged_cache_copy_prefix", lambda *a, **k: (_ for _ in ()).throw(RuntimeError("copy failed")))
    with pytest.raises(RuntimeError, match="copy failed"):
        fork([(parent, 3)])
    for layer, pool in enumerate(pools):
        assert pool.used_page_ids == set(parent[layer].page_ids) and not pool.extra_refs
    for c in parent:
        c.release()


# ------------------------------------------------------------------ refusals --
@pytest.mark.parametrize("kw, msg", [
    (dict(num_beams=0), "num_beams"), (dict(num_beams=9), "num_beams"), (dict(num_beams=2.0), "num_beams"),
    (dict(eos_token_ids=(1, 2, 3, 4, 5)), "EOS"), (dict(num_return_sequences=3, num_beams=2), "num_return_sequences"),
    (dict(num_return_sequences=0), "num_return_sequences"), (dict(length_penalty=math.inf), "length_penalty"),
    (dict(length_penalty=math.nan), "length_penalty"), (dict(max_new_tokens=-1), "max_new_tokens"),
])
def test_bad_arguments_are_refused_before_any_work(kernels_ref, kw, msg):
    model = PagedScripted(_logits_table(5, 0), 5)
    args = dict(max_new_tokens=4, num_beams=2)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        beam_search_ids(model, [1, 2], **args)
    assert model.calls == 0 and _all_free(model)


def test_an_empty_prompt_and_non_paged_caches_are_refused(kernels_ref):
    model = PagedScripted(_logits_table(5, 0), 5)
    with pytest.raises(ValueError, match="prompt"):
        beam_search_ids(model, [], 4)

    class Dense(PagedScripted):
        def create_kv_cache(self):
            from tiny_llm_b200.kv_cache import TinyKvFullCache

            return [TinyKvFullCache() for _ in self.pools]

    with pytest.raises(ValueError, match="paged"):
        beam_search_ids(Dense(_logits_table(5, 0), 5), [1, 2], 4)


def test_zero_new_tokens_returns_nothing(kernels_ref):
    model = PagedScripted(_logits_table(5, 0), 5)
    assert beam_search_ids(model, [1, 2], 0) == [] and model.calls == 0 and _all_free(model)


def test_hypotheses_are_the_public_type(kernels_ref):
    model = PagedScripted(_logits_table(5, 0), 5)
    (h,) = beam_search_ids(model, [1, 2], 3, num_beams=2)
    assert isinstance(h, BeamHypothesis) and len(h.ids) == 3 and not h.finished


# ------------------------------------------------------------------ CLI --
def test_cli_prints_every_hypothesis(kernels_ref, capsys):
    assert cli_main(["generate", "--synthetic", "tiny-d128", "--device", "cpu", "--prompt-ids", "5,17,3", "--max-new-tokens", "3",
                     "--num-beams", "3", "--num-return-sequences", "2", "--length-penalty", "0.5"]) == 0
    out = capsys.readouterr().out.splitlines()
    heads = [line for line in out if line.startswith("beam ")]
    texts = [line for line in out if line.startswith("[")]
    assert len(heads) == 2 and len(texts) == 2
    assert all("length 3" in h and "unfinished" in h for h in heads)
    assert all(len(t.split()[1:]) == 3 for t in texts)


@pytest.mark.parametrize("extra, msg", [
    (["--sampler-temp", "0.7"], "sampler-temp"), (["--repetition-penalty", "1.2"], "penalties"), (["--min-p", "0.1"], "penalties"),
    (["--regex", "[0-9]+"], "regex"), (["--logprobs", "2"], "logprobs"), (["--prompt-lookup", "3"], "prompt-lookup"),
    (["--draft-synthetic", "tiny-d128"], "draft"), (["--synthetic-lora", "a=8"], "adapters"),
])
def test_cli_refuses_what_beam_search_does_not_take(kernels_ref, extra, msg):
    with pytest.raises(SystemExit, match=msg):
        cli_main(["generate", "--synthetic", "tiny-d128", "--device", "cpu", "--prompt-ids", "5,17,3", "--max-new-tokens", "2",
                  "--num-beams", "2", *extra])


def test_cli_reports_bad_beam_arguments(kernels_ref):
    with pytest.raises(SystemExit, match="num_return_sequences"):
        cli_main(["generate", "--synthetic", "tiny-d128", "--device", "cpu", "--prompt-ids", "5,17,3", "--num-beams", "2",
                  "--num-return-sequences", "3"])


# ------------------------------------------------------------------ C ABI --
def _abi(*args):
    return ext._lib.tl_beam_select(*args)


@pytest.mark.parametrize("rows, n, W, eos, msg", [
    (1, 1, 0, [], "num_beams must be in"), (1, 9, 9, [], "num_beams must be in"), (1, 7, 2, [1, 2, 3, 4, 5], "at most 4 EOS"),
    (3, 2, 2, [], "rows must be in"), (0, 2, 2, [], "rows must be in"), (1, 3, 2, [], "n must be num_beams"),
    (1, 4, 2, [-1, 3], "non-negative"), (1, 4, 2, [3, 3], "given twice"),
])
def test_the_c_abi_refuses_bad_shapes_without_a_device(rows, n, W, eos, msg):
    ids = (ctypes.c_int32 * 8)(*eos)
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    assert _abi(p, p, p, rows, n, W, ids, len(eos), p, None) != 0
    assert msg in ext._lib.tl_last_error().decode()


def test_the_c_abi_refuses_null_pointers():
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    assert _abi(None, p, p, 1, 2, 2, None, 0, p, None) != 0
    assert "null pointer" in ext._lib.tl_last_error().decode()
    assert _abi(p, p, p, 1, 3, 2, None, 1, p, None) != 0
    assert "null pointer" in ext._lib.tl_last_error().decode()


def test_the_binding_checks_its_tensors():
    lp, ids, cum, out = torch.zeros(1, 3), torch.zeros(1, 3, dtype=torch.int32), torch.zeros(2), torch.zeros(ext.BEAM_RESULT_WORDS, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.beam_select(lp, ids, cum, 2, (9,), out)
    with pytest.raises(RuntimeError, match="top_lp must be float32"):
        ext.beam_select(lp.double(), ids, cum, 2, (9,), out)
    with pytest.raises(RuntimeError, match="top_lp must be float32"):
        ext.beam_select(lp, ids, cum, 2, (), out)
    with pytest.raises(RuntimeError, match="top_ids must be int32"):
        ext.beam_select(lp, ids.long(), cum, 2, (9,), out)
    with pytest.raises(RuntimeError, match="cum must be float32"):
        ext.beam_select(lp, ids, torch.zeros(3), 2, (9,), out)
    with pytest.raises(RuntimeError, match="out must be int32"):
        ext.beam_select(lp, ids, cum, 2, (9,), out[:-1])
    with pytest.raises(RuntimeError, match="rows must be in"):
        ext.beam_select(torch.zeros(3, 3), torch.zeros(3, 3, dtype=torch.int32), cum, 2, (9,), out)
    with pytest.raises(RuntimeError, match="contiguous"):
        ext.beam_select(torch.zeros(1, 6)[:, ::2], ids, cum, 2, (9,), out)
