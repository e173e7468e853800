"""Seeded sampling through the host layers, on the CPU stand-in of the extension (``cpu_ext``) plus the float64
sampling reference in place of ``tl_sample``: ``SamplingParams`` validation, the shim's argument checks, and the batcher
and CLI with ``sampling``."""

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as ref
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, batch_generate
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.synthetic import synthetic_qwen3


@pytest.mark.parametrize("kwargs", [
    dict(temperature=-0.1), dict(temperature=float("nan")), dict(temperature=float("inf")), dict(temperature="1"),
    dict(temperature=True), dict(temperature=1.0, top_k=-1), dict(temperature=1.0, top_k=2.5), dict(temperature=1.0, top_k=True),
    dict(temperature=1.0, top_p=float("nan")), dict(temperature=1.0, top_p=float("-inf")), dict(temperature=1.0, seed=-1),
    dict(temperature=1.0, seed=1 << 64), dict(temperature=1.0, seed=1.0),
])
def test_sampling_params_reject_bad_values(kwargs):
    with pytest.raises(ValueError):
        SamplingParams(**kwargs)


def test_sampling_params_accept_the_contract_range():
    SamplingParams(0)
    SamplingParams(0.7, top_k=0, top_p=0.0, seed=(1 << 64) - 1)
    SamplingParams(1.5, top_k=151936, top_p=2.0, seed=0)
    with pytest.raises(AttributeError):
        SamplingParams(1.0).temperature = 2.0  # frozen


def _args(rows=2, vocab=16, **over):
    a = dict(logits=torch.zeros(rows, vocab, dtype=torch.bfloat16), temperature=torch.zeros(rows), top_k=torch.zeros(rows, dtype=torch.int32),
             top_p=torch.zeros(rows), seed=torch.zeros(rows, dtype=torch.int64), positions=torch.zeros(rows, dtype=torch.int32))
    a.update(over)
    return a


@pytest.mark.parametrize("over,message", [
    (dict(logits=torch.zeros(2, 16, dtype=torch.int32)), "expected 2D float logits"),
    (dict(logits=torch.zeros(16, dtype=torch.bfloat16)), "expected 2D float logits"),
    (dict(temperature=torch.zeros(2, dtype=torch.float64)), "temperature must be float32"),
    (dict(top_k=torch.zeros(3, dtype=torch.int32)), r"top_k must be int32 \[2\]"),
    (dict(top_p=torch.zeros(2, 1)), "top_p must be float32"),
    (dict(seed=torch.zeros(2, dtype=torch.int32)), "seed must be int64"),
    (dict(positions=torch.zeros(2, dtype=torch.int64)), "positions must be int32"),
    (dict(logits=torch.zeros(16, 2, dtype=torch.bfloat16).t()), "logits must be contiguous"),
])
def test_shim_checks_arguments_before_the_device(over, message):
    with pytest.raises(RuntimeError, match=message):
        ext.sample(**_args(**over))


def test_shim_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="sample: the course extension is GPU-only"):
        ext.sample(**_args())


def test_sample_is_bound_in_the_library():
    assert "tl_sample" in ext.EXPORTED_SYMBOLS and "sample" in ext.__all__


# ------------------------------------------------------------------ batcher --
@pytest.fixture
def cpu_sample(cpu_ext, monkeypatch):
    """``cpu_ext`` and, for ``tl_sample``, the float64 reference (``oracle.sampling``)."""
    monkeypatch.setattr(cpu_ext, "sample", ref.sample_like_ext)
    return cpu_ext


PROMPTS = [[5, 17, 3, 250], [9, 2, 4, 6, 8, 11], [300, 1, 77], [42] * 9, [8, 8, 1, 2, 3]]


@pytest.fixture(scope="module")
def ns():
    return synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)


def _run(ns, prompts, sampling=None, batch_size=3, **kw):
    model = Qwen3ModelWeek3(ns, page_size=16)
    out = batch_generate(model, None, prompts, max_seq_len=64, batch_size=batch_size, prefill_step=4, verbose=False,
                         max_new_tokens=[6] * len(prompts), sampling=sampling, **kw)
    return dict(out)


def test_batcher_with_greedy_sampling_returns_todays_output(cpu_sample, ns):
    today = _run(ns, PROMPTS)
    assert _run(ns, PROMPTS, sampling=None) == today
    assert _run(ns, PROMPTS, sampling=SamplingParams(0.0, top_k=3, top_p=0.5, seed=9)) == today
    assert _run(ns, PROMPTS, sampling=[SamplingParams(0.0, seed=i) for i in range(len(PROMPTS))]) == today


def test_sampled_tokens_do_not_depend_on_queue_position_or_slot(cpu_sample, ns):
    params = [SamplingParams(0.9, top_k=None if i % 2 else 20, top_p=0.95 if i % 3 else None, seed=100 + i) for i in range(len(PROMPTS))]
    params[2] = SamplingParams(0.0)  # a greedy request in the same batch
    first = _run(ns, PROMPTS, sampling=params)
    order = [3, 0, 4, 2, 1]
    second = _run(ns, [PROMPTS[i] for i in order], sampling=[params[i] for i in order], batch_size=2)
    assert {i: first[i] for i in range(len(PROMPTS))} == {i: second[j] for j, i in enumerate(order)}
    assert first[2] == _run(ns, PROMPTS)[2]


def test_different_seeds_give_different_outputs(cpu_sample, ns):
    a = _run(ns, PROMPTS, sampling=SamplingParams(1.0, seed=1))
    b = _run(ns, PROMPTS, sampling=SamplingParams(1.0, seed=2))
    assert a != b
    assert a == _run(ns, PROMPTS, sampling=SamplingParams(1.0, seed=1))


def test_batcher_refuses_a_wrong_number_of_params(cpu_sample, ns):
    with pytest.raises(ValueError, match="one per prompt"):
        _run(ns, PROMPTS, sampling=[SamplingParams(1.0)] * 2)


def test_cli_batch_sampling_is_seeded(cpu_sample, capsys):
    argv = ["batch", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3;9,2,4,6,8;300,1", "--max-new-tokens", "5", "--device", "cpu",
            "--batch-size", "2", "--max-seq-len", "64", "--prefill-step", "4", "--quiet", "--sampler-temp", "0.7", "--seed", "3"]
    assert cli_main(argv) == 0
    first = capsys.readouterr().out
    assert cli_main(argv) == 0
    assert capsys.readouterr().out == first and "--- request 2" in first
    assert cli_main(argv[:-1] + ["4"]) == 0
    assert capsys.readouterr().out != first
