"""Continuous-batching scheduler against fake models: exact call traces,
EOS/max_seq_len handling and release-exactly-once, pinned by the literals of
tests_refsol/test_week_3_day_2.py (tests/golden/reference_literals.json).
CPU-only."""

import json
from pathlib import Path

import pytest
import torch

from tiny_llm_b200 import BatchingKvCache, ContinuousBatcher, Request, TinyKvFullCache, TinyKvPagedCache, TinyKvPagedPool, batch_generate

LIT = json.loads((Path(__file__).parent / "golden" / "reference_literals.json").read_text())["scheduler_traces"]


class FakeDetokenizer:
    def __init__(self, _):
        self.text = ""

    def add_token(self, token):
        self.text += str(token)


class FakeTokenizer:
    eos_token_id = 99
    _tokenizer = object()
    detokenizer = FakeDetokenizer(_tokenizer)

    def encode(self, prompt, add_special_tokens=False):
        assert not add_special_tokens
        return list(range(1, len(prompt) + 1))


def one_hot_logits(rows, vocab, token):
    logits = torch.zeros(rows, 1, vocab)
    logits[..., token] = 1
    return logits


class FakeModel:
    num_hidden_layers = 1

    def __init__(self):
        self.calls = []

    def create_kv_cache(self):
        return [TinyKvFullCache()]

    def __call__(self, inputs, offsets, cache, logits_to_keep=1):
        offset = offsets[0] if isinstance(offsets, list) else int(offsets)
        self.calls.append((offset, inputs.shape[1]))
        key = torch.zeros(1, 1, inputs.shape[1], 1)
        cache[0].update_and_fetch(key, key)
        return one_hot_logits(1, 4, 1)


class FailingMaterializePagedCache(TinyKvPagedCache):
    def materialize(self):
        super().materialize()
        raise RuntimeError("injected materialization failure")


class PagedFakeModel:
    num_hidden_layers = 1

    def __init__(self, output_token=1, fail_at=None):
        self.pool = TinyKvPagedPool(page_size=4)
        self.output_token = output_token
        self.fail_at = fail_at
        self.calls = []
        self.cache_creations = 0

    def create_kv_cache(self):
        self.cache_creations += 1
        kind = FailingMaterializePagedCache if self.fail_at == "materialize" else TinyKvPagedCache
        return [kind(self.pool)]

    def __call__(self, inputs, offsets, cache, logits_to_keep=1):
        offset = offsets[0] if isinstance(offsets, list) else int(offsets)
        call_number = len(self.calls) + 1
        self.calls.append((offset, inputs.shape[1]))
        key = torch.zeros(inputs.shape[0], 1, inputs.shape[1], 1)
        if isinstance(cache[0], BatchingKvCache):
            cache[0].update_and_fetch_paged(key, key, mask_length=inputs.shape[1])
        else:
            cache[0].update_and_fetch_paged(key, key)
        if self.fail_at == "prefill" and call_number == 1:
            raise RuntimeError("injected prefill failure")
        if self.fail_at == "decode" and call_number == 2:
            raise RuntimeError("injected decode failure")
        return one_hot_logits(inputs.shape[0], 128, self.output_token)


class FailingTextDetokenizer:
    def __init__(self, _):
        self._text = ""

    def add_token(self, token):
        self._text += str(token)

    @property
    def text(self):
        raise RuntimeError("injected detokenization failure")


class FailingTextTokenizer(FakeTokenizer):
    detokenizer = FailingTextDetokenizer(FakeTokenizer._tokenizer)


def as_tuples(pairs):
    return [tuple(p) for p in pairs]


def test_chunked_prefill_bounds_work_and_advances_cache():
    lit = LIT["chunked_prefill"]
    model = FakeModel()
    request = Request(model, FakeTokenizer(), "x" * lit["prompt_len"], prefill_max_step=lit["prefill_step"])
    for expected_offset, done in ((3, False), (6, False), (7, True)):
        request.try_prefill()
        assert request.offset == expected_offset and request.kv_cache[0].offset == expected_offset
        assert request.is_prefill_done is done
    assert request.next_token == lit["next_token"]
    assert model.calls == as_tuples(lit["calls"])
    with pytest.raises(ValueError, match="after done"):
        request.try_prefill()


def test_request_uses_the_model_cache_factory():
    model = FakeModel()
    sentinel = [TinyKvFullCache()]
    model.create_kv_cache = lambda: sentinel
    assert Request(model, FakeTokenizer(), "1").kv_cache is sentinel


def test_lone_multi_chunk_prefill_then_decode(cpu_ext):
    lit = LIT["lone_multichunk"]
    model = PagedFakeModel()
    result = batch_generate(model, FakeTokenizer(), ["x" * lit["prompt_len"]], max_seq_len=lit["max_seq_len"], batch_size=1,
                            prefill_step=lit["prefill_step"], verbose=False)
    assert result == as_tuples(lit["result"])
    assert model.calls == as_tuples(lit["calls"])
    assert model.pool.used_page_ids == set() and model.pool.num_free_pages == model.pool.num_pages


def test_eos_at_prefill_needs_no_decode(cpu_ext):
    lit = LIT["eos_at_prefill"]
    model = PagedFakeModel(output_token=FakeTokenizer.eos_token_id)
    result = batch_generate(model, FakeTokenizer(), ["x" * lit["prompt_len"]], max_seq_len=10, batch_size=1, prefill_step=10)
    assert result == as_tuples(lit["result"]) and model.calls == as_tuples(lit["calls"])
    assert model.pool.used_page_ids == set() and model.pool.num_free_pages == model.pool.num_pages


@pytest.mark.parametrize("lit", LIT["max_seq_len_3"], ids=lambda c: f"len{c['prompt_len']}")
def test_max_seq_len_is_enforced_before_emission_or_allocation(cpu_ext, lit):
    model = PagedFakeModel()
    prompt = "x" * lit["prompt_len"]
    if lit["result"] is None:
        with pytest.raises(ValueError, match="exceeds max_seq_len"):
            batch_generate(model, FakeTokenizer(), [prompt], max_seq_len=3)
    else:
        assert batch_generate(model, FakeTokenizer(), [prompt], max_seq_len=3, batch_size=1, verbose=False) == as_tuples(lit["result"])
    assert model.calls == as_tuples(lit["calls"])
    assert model.cache_creations == lit["creations"]
    assert model.pool.used_page_ids == set()


@pytest.mark.parametrize(
    ("failure_point", "tokenizer"),
    [("prefill", FakeTokenizer()), ("materialize", FakeTokenizer()), ("decode", FakeTokenizer()), ("detokenize", FailingTextTokenizer())],
)
def test_every_paged_cache_is_released_on_exception(cpu_ext, failure_point, tokenizer):
    model = PagedFakeModel(fail_at=failure_point)
    with pytest.raises(RuntimeError, match="injected"):
        batch_generate(model, tokenizer, ["1"], max_seq_len=4, batch_size=1, prefill_step=4)
    assert model.pool.used_page_ids == set() and model.pool.num_free_pages == model.pool.num_pages


def test_argument_validation():
    for kwargs in (dict(max_seq_len=0), dict(batch_size=0), dict(prefill_step=0)):
        with pytest.raises(ValueError, match="must be positive"):
            batch_generate(FakeModel(), FakeTokenizer(), ["1"], **kwargs)


def test_token_id_prompts_and_decode_slot_reuse(cpu_ext):
    """Synthetic-serving form: prompts are id lists, no tokenizer, per-request
    output budgets; 5 requests through 2 decode slots with one prefill at a time."""
    model = PagedFakeModel(output_token=7)
    prompts = [[3] * n for n in (5, 9, 2, 6, 4)]
    batcher = ContinuousBatcher(model, None, prompts, max_seq_len=64, batch_size=2, prefill_step=4, verbose=False,
                                max_new_tokens=[3, 2, 4, 1, 3])
    results = dict(batcher.run())
    assert sorted(results) == [0, 1, 2, 3, 4]
    assert [len(results[i].split()) for i in range(5)] == [3, 2, 4, 1, 3]
    assert all(tok == "7" for text in results.values() for tok in text.split())
    assert batcher.prefill_tokens == sum(len(p) for p in prompts)
    assert model.pool.used_page_ids == set() and model.pool.num_free_pages == model.pool.num_pages
    # prefill calls are B=1 chunks of <= 4 tokens at increasing offsets; decode calls are B=2, L=1
    assert all(length <= 4 for _, length in model.calls)
