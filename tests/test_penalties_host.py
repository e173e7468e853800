"""Token-history penalties and min-p through the host layers, on the CPU stand-in of the extension (``cpu_ext``) plus
the penalised sampling reference (``penalties_ref``) in place of ``tl_sample_penalized``: ``SamplingParams``, the fp32
penalty restatement on hand-worked values, the shim's argument checks, the batcher's token-state lifecycle and the CLI
flags."""

import importlib.util
import sys
from collections import Counter
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as ref
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, batch_generate, greedy_generate_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.sampler import penalty_tensors, sampling_tensors, token_state_row
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load_penalties_ref():
    """The helper next to this file, by path: `tests` is no package of this project."""
    name = "tiny_llm_b200_penalties_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("penalties_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


pref = _load_penalties_ref()


# ------------------------------------------------------------------ params --
def test_fields_follow_seed_and_default_to_off():
    p = SamplingParams(0.7, 50, 0.9, 3)
    assert (p.temperature, p.top_k, p.top_p, p.seed) == (0.7, 50, 0.9, 3)
    assert (p.repetition_penalty, p.presence_penalty, p.frequency_penalty, p.min_p) == (1.0, 0.0, 0.0, 0.0)
    assert not p.penalized
    assert SamplingParams(0.7, 50, 0.9, 3, 1.1).repetition_penalty == 1.1
    for kw in (dict(repetition_penalty=0.8), dict(presence_penalty=-0.5), dict(frequency_penalty=0.3), dict(min_p=1.0)):
        assert SamplingParams(0.0, **kw).penalized


@pytest.mark.parametrize("kwargs", [
    dict(repetition_penalty=0.0), dict(repetition_penalty=-1.0), dict(repetition_penalty=float("inf")), dict(repetition_penalty=float("nan")),
    dict(repetition_penalty=True), dict(presence_penalty=float("nan")), dict(presence_penalty=float("-inf")), dict(presence_penalty="1"),
    dict(frequency_penalty=float("inf")), dict(min_p=-0.01), dict(min_p=1.01), dict(min_p=float("nan")),
])
def test_bad_penalties_are_refused(kwargs):
    with pytest.raises(ValueError):
        SamplingParams(0.7, **kwargs)


def test_penalty_tensors_and_state_row():
    params = [None, SamplingParams(1.0, repetition_penalty=1.3, presence_penalty=-0.5, frequency_penalty=0.25, min_p=0.05)]
    r, pres, f, mp = penalty_tensors(params, "cpu")
    assert r.tolist() == [1.0, pytest.approx(1.3)] and pres.tolist() == [0.0, -0.5] and f.tolist() == [0.0, 0.25]
    assert mp.tolist() == [0.0, pytest.approx(0.05)] and all(t.dtype == torch.float32 for t in (r, pres, f, mp))
    assert len(sampling_tensors(params, "cpu")) == 4  # unchanged
    row = token_state_row([3, 5, 3], [5, 7, 7, 7], 10)
    want = [0] * 10
    want[3] = 1 << 30
    want[5] = (1 << 30) + 1
    want[7] = 3
    assert row.dtype == torch.int32 and row.tolist() == want
    slab = torch.full((2, 10), 99, dtype=torch.int32)
    token_state_row([1], [], 10, out=slab[1])
    assert slab[1].tolist() == [0, 1 << 30] + [0] * 8 and slab[0].tolist() == [99] * 10
    with pytest.raises(ValueError):
        token_state_row([10], [], 10)


# ---------------------------------------------------------------- penalize --
def _state(prompt=(), counts=None, V=8):
    s = np.zeros(V, dtype=np.int32)
    for i in prompt:
        s[i] |= pref.PROMPT
    for i, c in (counts or {}).items():
        s[i] += c
    return s


def test_penalize_hand_worked_values():
    x = np.array([3.0, -2.0, 0.75, 4.0, 0.75, 1.0, 0.0, np.nan], dtype=np.float32)
    s = _state(prompt=[0, 1, 3, 7], counts={0: 3, 6: 1})
    y = pref.penalize(x, s, 1.5, 0.5, 0.25)
    # token 0: in the prompt and drawn 3 times: 3 / 1.5 = 2, 2 - 0.25 * 3 = 1.25, 1.25 - 0.5 = 0.75
    assert y[0] == np.float32(0.75)
    assert y[1] == np.float32(-3.0)  # prompt only, negative: times r; no presence or frequency term
    assert y[3] == np.float32(4.0 / 1.5)  # prompt only, positive: divided once
    assert y[2] == y[4] == np.float32(0.75) and y[5] == np.float32(1.0)
    assert y[6] == np.float32(-0.75)  # drawn once: 0 * 1.5 = 0, - 0.25, - 0.5
    assert np.isnan(y[7])
    # token 0 now ties token 2: the first maximum after 3 and 5 is the lower id
    z = y.copy()
    z[3] = z[5] = -1
    assert ref.greedy(z) == 0


def test_penalize_rounds_each_step_on_its_own():
    # f * c and the subtractions are separate fp32 roundings (no fused multiply-add)
    x = np.array([1.0], dtype=np.float32)
    s = _state(counts={0: 3}, V=1)
    f = np.float32(0.1)
    fc = np.float32(f * np.float32(3))
    want = np.float32(np.float32(x[0] - fc) - np.float32(0.2))
    assert pref.penalize(x, s, 1.0, 0.2, 0.1)[0] == want
    # r on a token seen only in the prompt: x / r, rounded once
    assert pref.penalize(np.float32([1.0]), _state(prompt=[0], V=1), 3.0, 0.0, 0.0)[0] == np.float32(1.0) / np.float32(3.0)


def test_everything_off_is_the_identity_and_min_p_bounds():
    g = np.random.default_rng(0)
    x = g.standard_normal(64).astype(np.float32)
    s = g.integers(0, 4, 64).astype(np.int32) | np.where(g.random(64) < 0.3, pref.PROMPT, 0).astype(np.int32)
    assert np.array_equal(pref.penalize(x, s, 1.0, 0.0, 0.0), x)
    # min_p = 1 keeps the maximum's ties only
    x[[5, 9]] = 7.0
    keep = pref.keep_set(x, None, None, 1.0, 0.8)
    assert np.flatnonzero(keep).tolist() == [5, 9]
    thr = pref.min_p_threshold(7.0, 1.0, 0.1)
    assert thr == np.float32(np.float32(7.0) + np.float32(np.log(0.1)))


# ------------------------------------------------------------------- shim --
def _args(rows=2, vocab=16, **over):
    a = dict(logits=torch.zeros(rows, vocab, dtype=torch.bfloat16), temperature=torch.zeros(rows), top_k=torch.zeros(rows, dtype=torch.int32),
             top_p=torch.zeros(rows), seed=torch.zeros(rows, dtype=torch.int64), positions=torch.zeros(rows, dtype=torch.int32),
             repetition=torch.ones(rows), presence=torch.zeros(rows), frequency=torch.zeros(rows), min_p=torch.zeros(rows),
             state=torch.zeros(rows, vocab, dtype=torch.int32))
    a.update(over)
    return a


@pytest.mark.parametrize("over,message", [
    (dict(logits=torch.zeros(2, 16, dtype=torch.int32)), "expected 2D float logits"),
    (dict(temperature=torch.zeros(2, dtype=torch.float64)), "temperature must be float32"),
    (dict(positions=torch.zeros(2, dtype=torch.int64)), "positions must be int32"),
    (dict(repetition=torch.ones(3)), r"repetition must be float32 \[2\]"),
    (dict(presence=torch.zeros(2, dtype=torch.float16)), "presence must be float32"),
    (dict(frequency=torch.zeros(2, 1)), "frequency must be float32"),
    (dict(min_p=torch.zeros(2, dtype=torch.float64)), "min_p must be float32"),
    (dict(state=torch.zeros(2, 16, dtype=torch.int64)), r"state must be int32 \[2, 16\]"),
    (dict(state=torch.zeros(2, 15, dtype=torch.int32)), r"state must be int32 \[2, 16\]"),
    (dict(state=torch.zeros(16, 2, dtype=torch.int32).t()), "state must be contiguous"),
])
def test_shim_checks_arguments_before_the_device(over, message):
    with pytest.raises(RuntimeError, match=message):
        ext.sample_penalized(**_args(**over))


def test_shim_refuses_cpu_tensors_and_is_bound():
    with pytest.raises(RuntimeError, match="sample_penalized: the course extension is GPU-only"):
        ext.sample_penalized(**_args())
    assert "tl_sample_penalized" in ext.EXPORTED_SYMBOLS and "sample_penalized" in ext.__all__


# ------------------------------------------------------------ batcher, CLI --
@pytest.fixture
def cpu_pen(cpu_ext, monkeypatch):
    monkeypatch.setattr(cpu_ext, "sample", ref.sample_like_ext)
    monkeypatch.setattr(cpu_ext, "sample_penalized", pref.sample_penalized_like_ext)
    return cpu_ext


@pytest.fixture(scope="module")
def ns():
    return synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)


PROMPTS = [[5, 17, 3, 250], [9, 2, 4, 6, 8, 11], [300, 1, 77], [42] * 9, [8, 8, 1, 2, 3]]


def _params(n):
    out = []
    for i in range(n):
        if i == 2:
            out.append(SamplingParams(0.9, top_k=20, seed=100 + i))  # plain sampled, in the same batch
        else:
            out.append(SamplingParams((0.0, 0.9, 1.2)[i % 3], top_p=0.95 if i % 2 else None, seed=100 + i, repetition_penalty=1.3,
                                      presence_penalty=0.5 * (i % 2), frequency_penalty=0.4, min_p=0.02 * (i % 3)))
    return out


def test_batcher_token_state_follows_each_request(cpu_pen, ns):
    params = _params(len(PROMPTS))
    model = Qwen3ModelWeek3(ns, page_size=16)
    b = ContinuousBatcher(model, None, PROMPTS, max_seq_len=64, batch_size=2, prefill_step=4, verbose=False,
                          max_new_tokens=[6] * len(PROMPTS), sampling=params)
    seen_slots = {}
    try:
        while not b.idle():
            b.step()
            for i, s in enumerate(b.slots):
                if s is None:
                    continue
                seen_slots.setdefault(i, set()).add(s.prompt_idx)
                if s.sampling.penalized:  # prompt bits and a count per generated id, nothing from the slot's earlier requests
                    want = token_state_row(PROMPTS[s.prompt_idx], s.detokenizer.tokens, model.vocab_size)
                    assert torch.equal(b.token_state[i], want), (i, s.prompt_idx)
                    row = b.token_state[i]
                    assert Counter({t: int(row[t]) & pref.COUNT for t in set(s.detokenizer.tokens)}) == Counter(s.detokenizer.tokens)
                    assert all(int(row[t]) & pref.PROMPT for t in PROMPTS[s.prompt_idx])
    finally:
        b.release_all()
    assert any(len(v) > 1 for v in seen_slots.values())  # a slot was reused
    assert b.token_state.shape == (2, model.vocab_size)


def _run(ns, prompts, sampling, batch_size=3):
    model = Qwen3ModelWeek3(ns, page_size=16)
    out = batch_generate(model, None, prompts, max_seq_len=64, batch_size=batch_size, prefill_step=4, verbose=False,
                         max_new_tokens=[6] * len(prompts), sampling=sampling)
    return dict(out)


def test_penalised_tokens_do_not_depend_on_queue_position_or_slot(cpu_pen, ns):
    params = _params(len(PROMPTS))
    first = _run(ns, PROMPTS, params)
    order = [3, 0, 4, 2, 1]
    second = _run(ns, [PROMPTS[i] for i in order], [params[i] for i in order], batch_size=2)
    assert {i: first[i] for i in range(len(PROMPTS))} == {i: second[j] for j, i in enumerate(order)}
    plain = _run(ns, PROMPTS, [SamplingParams(p.temperature, p.top_k, p.top_p, p.seed) for p in params])
    assert first[2] == plain[2]  # the unpenalised request is unaffected by its penalised neighbours
    assert first != plain


def test_generate_keeps_the_state_across_steps(cpu_pen, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    prompt = [5, 17, 3, 250, 5, 5]
    p = SamplingParams(0.0, repetition_penalty=1.5, frequency_penalty=2.0)
    got = greedy_generate_ids(model, prompt, 10, sampling=p)
    # the same loop by hand on the reference: one state, counted at every draw
    state = token_state_row(prompt, [], model.vocab_size)[None]
    cache = model.create_kv_cache()
    ids, toks, offset = [], torch.tensor(prompt, dtype=torch.int32), 0
    try:
        for _ in range(10):
            logits = model(toks[None], offset, cache, logits_to_keep=1)[:, -1, :]
            t = pref.sample_penalized_like_ext(logits, *sampling_tensors([p], "cpu"), torch.tensor([offset + toks.numel()], dtype=torch.int32),
                                               *penalty_tensors([p], "cpu"), state)
            ids.append(int(t[0]))
            offset += toks.numel()
            toks = t.to(torch.int32)
    finally:
        for c in cache:
            c.release()
    assert got == ids
    assert got != greedy_generate_ids(model, prompt, 10)


def test_cli_penalty_flags(cpu_pen, ns, capsys):
    base = ["generate", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3,5,5", "--max-new-tokens", "8", "--device", "cpu"]
    assert cli_main(base) == 0
    greedy = capsys.readouterr().out
    assert cli_main(base + ["--sampler-temp", "0", "--repetition-penalty", "1.2", "--frequency-penalty", "3"]) == 0
    penalised = capsys.readouterr().out
    model = Qwen3ModelWeek3(synthetic_qwen3("tiny-d128", seed=0, realistic=True), page_size=16)
    want = greedy_generate_ids(model, [5, 17, 3, 5, 5], 8, sampling=SamplingParams(0.0, repetition_penalty=1.2, frequency_penalty=3.0))
    assert penalised.split() == [str(t) for t in want] and penalised != greedy
    argv = ["batch", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3;9,2,4,6,8;300,1", "--max-new-tokens", "5", "--device", "cpu",
            "--batch-size", "2", "--max-seq-len", "64", "--prefill-step", "4", "--quiet", "--sampler-temp", "0.7", "--seed", "3"]
    assert cli_main(argv) == 0
    plain = capsys.readouterr().out
    pen = argv + ["--presence-penalty", "1.5", "--min-p", "0.05"]
    assert cli_main(pen) == 0
    first = capsys.readouterr().out
    assert cli_main(pen) == 0
    assert capsys.readouterr().out == first and first != plain and "--- request 2" in first
