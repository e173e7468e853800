"""Parallel sampling on the host: the protocol of ``parallel_sample_ids`` against plain-loop independent runs with a
scripted model on CPU page pools (it reads its context back from its own K/V pages, so a bad fork or a write into a
shared page changes the result), seed derivation, EOS and budget truncation across rounds, group detection from
block tables, pages after an injected exception, every refusal, the CLI and the C entry's argument errors."""

import ctypes
import importlib.util
import sys
from dataclasses import replace
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import SamplingParams, parallel_sample_ids
from tiny_llm_b200 import generate as gen
from tiny_llm_b200.engine import shared_prefix_attention_applies, shared_run


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


BH = _load("tiny_llm_b200_beam_host_helpers", "test_beam_host.py")
kernels_ref = BH.kernels_ref


def fake_sample(rows, params, positions, state=None, constraints=None):
    """A deterministic stand-in for ``tl_sample``: a pure function of (row, seed, position)."""
    out = [(int(torch.argmax(r)) + int(p.seed) % 7 + int(pos)) % r.numel() for r, p, pos in zip(rows, params, positions)]
    return torch.tensor(out, dtype=torch.int32)


@pytest.fixture
def scripted(kernels_ref, monkeypatch):
    monkeypatch.setattr(gen, "sample_tokens", fake_sample)
    return kernels_ref


def _table(V, seed):
    def table(ctx):
        g = np.random.default_rng(hash((seed, ctx)) % (1 << 32))
        return g.normal(size=V)
    return table


def _independent(model, prompt, sampling, n, max_new, eos):
    """Plain loop: sample j alone on a fresh cache, drawing with seed + j at each position."""
    out = []
    for j in range(n):
        p = replace(sampling, seed=gen.sample_seed(sampling.seed, j))
        cache = model.create_kv_cache()
        ids, reason = [], "length"
        row = model(torch.tensor([prompt]), 0, cache)[:, -1, :]
        pos = len(prompt)
        while True:
            tok = int(fake_sample(row, [p], [pos])[0])
            if tok in eos:
                reason = "stop"
                break
            ids.append(tok)
            if len(ids) >= max_new:
                break
            row = model(torch.tensor([[tok]]), pos, cache)[:, -1, :]
            pos += 1
        gen._release_kv_cache(cache)
        out.append((ids, reason))
    return out


@pytest.mark.parametrize("prompts", [[[1, 2, 3]], [[1, 2, 3, 4], [5] * 9], [[2], [3, 1, 4, 1, 5], [9, 2, 6, 5, 3, 5, 8]]])
@pytest.mark.parametrize("n, max_new, eos", [(1, 5, ()), (3, 20, (0,)), (4, 37, (1, 2)), (16, 3, ())])
def test_protocol_equals_independent_runs(scripted, prompts, n, max_new, eos):
    if len(prompts) * n > 64:
        pytest.skip("over the slot limit")
    V = 9
    model = BH.PagedScripted(_table(V, 11), V, page=4)
    sampling = SamplingParams(0.7, seed=5)
    got = parallel_sample_ids(model, prompts, n, sampling, max_new, eos_token_ids=eos)
    for i, prompt in enumerate(prompts):
        want = _independent(model, prompt, sampling, n, max_new, set(eos))
        assert [(s.ids, s.finish_reason) for s in got[i]] == want
    assert BH._all_free(model)


def test_per_prompt_sampling_and_logprobs(scripted):
    V = 7
    model = BH.PagedScripted(_table(V, 3), V, page=4)
    per = [SamplingParams(0.5, seed=1), SamplingParams(0.9, seed=100)]
    got = parallel_sample_ids(model, [[1, 2], [3, 4, 5, 6]], 2, per, 6, logprobs=2)
    for i, prompt in enumerate([[1, 2], [3, 4, 5, 6]]):
        want = _independent(model, prompt, per[i], 2, 6, set())
        assert [s.ids for s in got[i]] == [w[0] for w in want]
        for s in got[i]:
            assert [e.token for e in s.logprobs] == s.ids
            assert all(len(e.top) == 2 for e in s.logprobs)
    assert BH._all_free(model)


def test_finishing_across_round_boundaries(scripted, monkeypatch):
    monkeypatch.setattr(gen, "PARALLEL_ROUND", 3)
    V = 5
    model = BH.PagedScripted(_table(V, 8), V, page=4)
    sampling = SamplingParams(1.0, seed=2)
    for max_new in (1, 3, 4, 7, 12):
        got = parallel_sample_ids(model, [[1, 2, 3]], 5, sampling, max_new, eos_token_ids=(4,))
        assert [(s.ids, s.finish_reason) for s in got[0]] == _independent(model, [1, 2, 3], sampling, 5, max_new, {4})
        assert all(len(s.ids) <= max_new for s in got[0])
    assert BH._all_free(model)


def test_budget_zero_returns_empty_samples(scripted):
    model = BH.PagedScripted(_table(5, 1), 5)
    got = parallel_sample_ids(model, [[1]], 3, SamplingParams(1.0), 0)
    assert [(s.ids, s.finish_reason) for s in got[0]] == [([], "length")] * 3
    assert model.calls == 0 and BH._all_free(model)


@pytest.mark.parametrize("fail_at", [1, 2, 3, 5])
def test_an_exception_returns_every_page(scripted, fail_at):
    model = BH.PagedScripted(_table(5, 4), 5, page=4, fail_at=fail_at)
    with pytest.raises(RuntimeError, match="injected"):
        parallel_sample_ids(model, [[1, 2, 3, 4, 5], [2, 3]], 3, SamplingParams(1.0, seed=9), 8)
    assert BH._all_free(model)


def test_seed_derivation_wraps_around():
    assert gen.sample_seed(3, 0) == 3 and gen.sample_seed(3, 5) == 8
    assert gen.sample_seed((1 << 63) - 1, 1) == -(1 << 63)
    assert gen.sample_seed(-1, 1) == 0
    assert gen.sample_seed(-2, 3) == 1


@pytest.mark.parametrize("kw, match", [
    (dict(num_samples=0), "num_samples"), (dict(num_samples=17), "num_samples"), (dict(num_samples=True), "num_samples"),
    (dict(prompts=[[1]] * 5, num_samples=16), "prompts x num_samples"), (dict(prompts=[]), "prompts x num_samples"),
    (dict(prompts=[[1], []]), "at least one token"), (dict(max_new_tokens=-1), "max_new_tokens"),
    (dict(sampling=SamplingParams(0.0)), "temperature 0"), (dict(adapter="a"), "adapter"),
    (dict(sampling=[SamplingParams(1.0)] * 3), "one per prompt"), (dict(logprobs=21), "logprobs"),
])
def test_refusals_before_any_work(scripted, kw, match):
    model = BH.PagedScripted(_table(5, 1), 5)
    args = dict(prompts=[[1, 2]], num_samples=2, sampling=SamplingParams(1.0), max_new_tokens=4) | kw
    with pytest.raises(ValueError, match=match):
        parallel_sample_ids(model, **args)
    assert model.calls == 0 and BH._all_free(model)


def test_greedy_single_sample_is_allowed(scripted):
    model = BH.PagedScripted(_table(5, 1), 5)
    got = parallel_sample_ids(model, [[1, 2]], 1, SamplingParams(0.0), 3)
    assert len(got[0]) == 1 and BH._all_free(model)


def test_non_paged_caches_are_refused():
    class Dense:
        calls = 0

        def create_kv_cache(self):
            return [gen.BatchingKvCache(1)]

    with pytest.raises(ValueError, match="paged"):
        parallel_sample_ids(Dense(), [[1]], 2, SamplingParams(1.0), 2)


# ------------------------------------------------------------------ group detection --
def _tables(prompt_tokens, n, page, layers=2, generated=0, diverge_layer=None):
    """Block tables of n forks of one prompt: full prompt pages shared, the tail and generated pages private."""
    full = prompt_tokens // page
    total = -(-(prompt_tokens + generated) // page)
    t = np.full((layers, n, total + 2), -1, dtype=np.int32)
    nxt = 1000
    for layer in range(layers):
        t[layer, :, :full] = np.arange(full) + 100 * layer
        for b in range(n):
            for p in range(full, total):
                t[layer, b, p] = nxt
                nxt += 1
    if diverge_layer is not None and full > 0:
        t[diverge_layer, 1, full - 1] = 7777
    return t


@pytest.mark.parametrize("prompt_tokens", [3, 4, 5, 8, 63, 64, 65, 200])
def test_shared_run_of_forks(prompt_tokens):
    page = 4 if prompt_tokens < 60 else 64
    t = _tables(prompt_tokens, 3, page, generated=9)
    assert shared_run(t, 0, 3, prompt_tokens, page) == prompt_tokens // page
    # the run stops before the page holding the first position a slot may still write
    assert shared_run(t, 0, 3, page, page) == min(1, prompt_tokens // page)
    # one slot alone shares every page it has filled
    assert shared_run(t, 1, 1, prompt_tokens + 9, page) == (prompt_tokens + 9) // page


def test_a_group_whose_layers_disagree_is_refused():
    t = _tables(16, 3, 4, diverge_layer=1)
    with pytest.raises(ValueError, match="same pages"):
        shared_run(t, 0, 3, 16, 4)
    assert shared_run(t, 0, 1, 16, 4) == 4  # one slot alone shares its own pages


class _Shape:
    def __init__(self, Hq, Hkv, D=128, page=64, dtype=torch.bfloat16):
        from types import SimpleNamespace

        self.layers_inner = [SimpleNamespace(self_attn=SimpleNamespace(num_heads=Hq, num_kv_heads=Hkv, head_dim=D))]
        self.page_size = page
        self.embedding = SimpleNamespace(weight=SimpleNamespace(scales=torch.zeros(1, dtype=dtype)))


def test_selection_rule_limits():
    m = _Shape(32, 8)
    assert shared_prefix_attention_applies(8, 4096, m)
    assert not shared_prefix_attention_applies(1, 4096, m)
    assert not shared_prefix_attention_applies(33, 4096, m)  # count x G > 128
    assert not shared_prefix_attention_applies(8, 4096, _Shape(32, 8, D=64))
    assert not shared_prefix_attention_applies(8, 4096, _Shape(32, 8, page=16))
    assert not shared_prefix_attention_applies(8, 4096, _Shape(32, 8, dtype=torch.float16))


# ------------------------------------------------------------------ the C entry --
def _call(groups, num_groups=None, batch=8, D=128, page=64, max_pages=16, Hq=32, Hkv=8, dtype=2, ws=1 << 30, null=False):
    arr = (ctypes.c_int * max(1, 3 * len(groups)))(*[v for g in groups for v in g])
    ptr = ctypes.cast(arr, ctypes.c_void_p)
    p = None if null else 1
    code = ext._lib.tl_shared_prefix_attention(p, 1, 1, 1, 1, 1, ptr, len(groups) if num_groups is None else num_groups, 1, batch, D,
                                               100, page, max_pages, 1.0, Hkv, Hq, dtype, 1, ws, None)
    return code, ext._lib.tl_last_error().decode()


@pytest.mark.parametrize("kw, match", [
    (dict(groups=[(0, 4, 2)], dtype=0), "bfloat16"),
    (dict(groups=[(0, 4, 2)], D=64), "head dimension"),
    (dict(groups=[(0, 4, 2)], page=32), "multiple of 64"),
    (dict(groups=[(0, 4, 2)], Hq=24, Hkv=8), "divisor of 128"),
    (dict(groups=[(6, 4, 2)]), "leaves the slots"),
    (dict(groups=[(-1, 2, 2)]), "leaves the slots"),
    (dict(groups=[(0, 4, 2), (3, 2, 1)]), "two groups"),
    (dict(groups=[(0, 8, 2)], Hq=64, Hkv=2), "more than 128"),
    (dict(groups=[(0, 4, 17)]), "outside"),
    (dict(groups=[(0, 4, 2)], num_groups=9), "num_groups"),
    (dict(groups=[(0, 4, 2)], null=True), "null pointer"),
    (dict(groups=[(0, 4, 2)], ws=16), "workspace too small"),
])
def test_c_entry_refuses_bad_arguments(kw, match):
    code, msg = _call(**kw)
    assert code != 0 and match in msg


def test_workspace_size_follows_the_split_counts():
    assert ext.shared_prefix_attention_workspace(8, 32, 8, 64, 16) > 0
    assert ext.shared_prefix_attention_workspace(0, 32, 8, 64, 16) == 0
    # the size does not depend on any grouping, only on the shapes
    a = ext.shared_prefix_attention_workspace(16, 32, 8, 64, 128)
    assert a % (16 * 32 * 130 * 4) == 0 and a // (16 * 32 * 130 * 4) <= 32  # PAGED_MAX_SPLITS partials per row


# ------------------------------------------------------------------ the CLI --
def test_cli_refuses_num_samples_with_beams_and_proposers(capsys):
    from tiny_llm_b200 import cli

    base = ["generate", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3", "--device", "cpu", "--num-samples", "2"]
    for extra, match in [(["--num-beams", "2"], "not both"), (["--prompt-lookup", "2"], "prompt-lookup"),
                         (["--draft-synthetic", "tiny-d128"], "draft"), ([], "CUDA")]:
        with pytest.raises(SystemExit, match=match):
            cli.main(base + extra)
