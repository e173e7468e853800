"""Speculative sampling on the host: the float64 rule (``spec_sample_ref.py``) against the target's distribution,
analytically and over seeds, the sampled protocol of ``_speculate`` with a scripted runner, the refusals of
``speculative_generate_ids(sampling=...)`` and the CLI flags."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import stats

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as S
from tiny_llm_b200 import generate as gen
from tiny_llm_b200 import speculative_generate_ids
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.sampler import SamplingParams


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_spec_sample_ref", "spec_sample_ref.py")

# A chi-square test of 20,000 draws at a significance level of 0.01; the seeds are fixed, so the outcome is too.  The
# rule gives p = 0.12.  Reusing the draft's Philox stream 0 for the acceptance uniform gives p = 0.0014, for the
# residual noise p = 7e-19: both fail.
CHI2_ALPHA = 1e-2
SEEDS = 20_000


def _pairs():
    rng = np.random.default_rng(7)
    for case in range(200):
        V = int(rng.integers(2, 9))
        x, y = rng.normal(0, 2, V), rng.normal(0, 2, V)
        T = float(rng.choice([0.0, 0.5, 1.0, 1.7]))
        top_k = int(rng.integers(0, V + 1))
        top_p = float(rng.choice([0.0, 0.5, 0.8, 1.0]))
        yield case, x, y, T, top_k, top_p
    # disjoint supports: top-k 2 on rows whose two largest entries differ
    x = np.array([5.0, 4.0, 0.0, 0.0, 0.0])
    y = np.array([0.0, 0.0, 0.0, 4.0, 5.0])
    yield "disjoint", x, y, 1.0, 2, 0.0
    # non-finite maxima: point masses
    yield "point", np.array([1.0, np.inf, 0.0]), np.array([0.0, 1.0, 2.0]), 1.0, 0, 0.0


@pytest.mark.parametrize("case,x,y,T,top_k,top_p", list(_pairs()), ids=lambda v: None)
def test_rule_output_distribution_is_the_target_distribution(case, x, y, T, top_k, top_p):
    p = R.row_dist(x, T, top_k, top_p)
    q = R.row_dist(y, T, top_k, top_p)
    assert abs(p.sum() - 1) < 1e-12 and abs(q.sum() - 1) < 1e-12
    np.testing.assert_allclose(R.output_distribution(p, q), p, rtol=0, atol=1e-12)


def _empirical(accept_stream=R.STREAM_ACCEPT, residual_stream=R.STREAM_RESIDUAL):
    x = np.array([1.2, 0.3, -0.5, 2.0, 0.9, -1.1, 0.0, 1.5])
    y = np.array([0.1, 1.4, 0.8, 1.9, -0.3, 0.5, 1.1, -0.8])
    T, top_k, top_p, pos = 0.9, 7, 0.97, 11
    p = R.row_dist(x, T, top_k, top_p)
    q = R.row_dist(y, T, top_k, top_p)
    counts = np.zeros(len(x))
    for seed in range(SEEDS):
        d = S.sample_row(y, T, top_k, top_p, seed, pos)
        counts[R.decide(p, q, d, seed, pos, S.greedy(x), accept_stream=accept_stream, residual_stream=residual_stream).token] += 1
    return counts, p


def test_rule_over_seeds_passes_a_chi_square_test_against_the_target():
    counts, p = _empirical()
    assert counts[p == 0].sum() == 0
    live = p > 0
    assert stats.chisquare(counts[live], SEEDS * p[live]).pvalue > CHI2_ALPHA


def test_greedy_rows_are_greedy_verification():
    rng = np.random.default_rng(3)
    for _ in range(50):
        x, y = rng.normal(size=6), rng.normal(size=6)
        d = S.greedy(y)
        dec = R.rule_row(x, y, d, 0.0, 0, 0.0, 5, 9)
        assert dec.token == S.greedy(x) and dec.accepted == (d == S.greedy(x))


def test_identical_rows_accept_every_drawn_proposal():
    rng = np.random.default_rng(4)
    for seed in range(200):
        x = rng.normal(size=7)
        d = S.sample_row(x, 0.8, 5, 0.9, seed, 3)
        dec = R.rule_row(x, x, d, 0.8, 5, 0.9, seed, 3)
        assert dec.accepted and dec.token == d


def test_a_rejected_proposal_never_comes_back_as_the_residual():
    rng = np.random.default_rng(5)
    for seed in range(2000):
        x, y = rng.normal(size=5), rng.normal(size=5)
        d = S.sample_row(y, 1.0, 0, 0.0, seed, 2)
        dec = R.rule_row(x, y, d, 1.0, 0, 0.0, seed, 2)
        assert dec.accepted == (dec.token == d)


def test_empty_residual_set_falls_back_to_the_target_argmax():
    # q as a rounded row could hold it (not summing to 1): p <= q everywhere, and p_d < u q_d rejects d
    p = np.array([0.5, 0.25, 0.25])
    q = np.array([0.5, 0.25, 0.3])
    seed = next(s for s in range(100) if R.accept_uniform(s, 4) * q[2] > p[2])
    dec = R.decide(p, q, 2, seed, 4, fallback=0)
    assert not dec.accepted and dec.token == 0


# ------------------------------------------------------------------ protocol --
class Layer:
    def __init__(self):
        self.offset = 0

    def rewind(self, n):
        assert 0 <= n <= self.offset
        self.offset -= n

    def release(self):
        pass


class Model:
    def create_kv_cache(self):
        return [Layer(), Layer()]


def _grow(cache, n):
    for layer in cache:
        layer.offset += n


class ScriptedRunner:
    """Rounds scripted as (proposals, out): ``out`` plays ``tl_speculative_sample``'s tokens for the T rows."""

    def __init__(self, first, rounds, target_steps=(), fits=True):
        self.first, self.rounds, self.target_steps, self.fits = first, list(rounds), list(target_steps), fits
        self.calls = []

    def round_fits(self, offset, k):
        return self.fits

    def prefill(self, model, ids, cache):
        _grow(cache, len(ids))
        return self.first

    def target_step(self, token, offset, cache):
        _grow(cache, 1)
        self.calls.append(("target", token, offset))
        return self.target_steps.pop(0)

    def draft(self, token, offset, cache, k, eos):
        self.calls.append(("draft", token, offset, k))
        if k == 1 and not self.rounds:  # the draft's catch-up after a fully accepted last round
            _grow(cache, 1)
            return [0]
        proposals = self.rounds[0][0] if eos != () else [0]
        _grow(cache, len(proposals))
        return list(proposals)

    def verify(self, token, proposals, offset, cache):
        _, out = self.rounds.pop(0)
        _grow(cache, len(proposals) + 1)
        self.calls.append(("verify", token, offset))
        return list(out), list(proposals)


def _run(runner, n=30, k=4, eos=(99,)):
    got = []
    stats = gen._speculate(runner, Model(), Model(), [1, 2, 3], n, k, set(eos), got.extend)
    return got, stats


@pytest.mark.parametrize("j", range(4))
def test_rejection_at_each_index_emits_the_accepted_prefix_and_the_residual(j):
    d = [10, 11, 12, 13]
    out = d[:j] + [50 + j] + [70] * (4 - j)  # rows past the first rejection are discarded
    runner = ScriptedRunner(7, [(d, out), ([20, 21, 22, 23], [20, 21, 22, 23, 99])])
    got, stats = _run(runner)
    assert got == [7, *d[:j], 50 + j, 20, 21, 22, 23]
    assert stats == [(4, j), (4, 4)]
    verifies = [c for c in runner.calls if c[0] == "verify"]
    assert verifies[1] == ("verify", 50 + j, 3 + j + 1)  # the rewind left both caches at the residual's position


def test_a_bonus_eos_ends_the_run():
    runner = ScriptedRunner(7, [([10, 11, 12, 13], [10, 11, 12, 13, 99])])
    assert _run(runner) == ([7, 10, 11, 12, 13], [(4, 4)])


def test_eos_inside_an_accepted_run_ends_it_there():
    runner = ScriptedRunner(7, [([10, 99, 12, 13], [10, 99, 12, 13, 14])])
    assert _run(runner) == ([7, 10], [(4, 2)])  # the EOS proposal counts as accepted, and is not emitted


def test_target_only_fallback_draws_with_target_steps():
    runner = ScriptedRunner(7, [], target_steps=[8, 9, 99], fits=False)
    got, stats = _run(runner)
    assert got == [7, 8, 9] and stats == []
    assert [c[2] for c in runner.calls] == [3, 4, 5]


# ------------------------------------------------------------------ front door --
class _Never:
    def create_kv_cache(self):
        raise AssertionError("no model call before the refusal")


@pytest.mark.parametrize("params,message", [
    (SamplingParams(0.7, presence_penalty=1.0), "no penalties or min-p"),
    (SamplingParams(0.7, min_p=0.1), "no penalties or min-p"),
    (SamplingParams(0.0, repetition_penalty=1.2), "no penalties or min-p"),
])
def test_speculative_sampling_refuses_what_it_does_not_take(params, message):
    with pytest.raises(ValueError, match=message):
        speculative_generate_ids(_Never(), _Never(), [1, 2], 4, sampling=params)


def test_temperature_zero_takes_the_greedy_runner(monkeypatch):
    seen = []
    monkeypatch.setattr(gen, "_speculate", lambda runner, *a: seen.append(runner.sampling) or [])
    speculative_generate_ids(_Never(), _Never(), [1, 2], 4, sampling=SamplingParams(0.0, seed=3))
    speculative_generate_ids(_Never(), _Never(), [1, 2], 4, sampling=SamplingParams(0.5, top_k=3, seed=3))
    assert seen == [None, SamplingParams(0.5, top_k=3, seed=3)]


def test_speculative_sample_is_bound_in_the_library():
    assert "tl_speculative_sample" in ext.EXPORTED_SYMBOLS and "speculative_sample" in ext.__all__
    assert "tl_log_rows" in ext.EXPORTED_SYMBOLS and "log_rows" in ext.__all__


def test_shim_checks_shapes_before_the_device():
    t = torch.zeros(3, 16)
    f, i, l = torch.zeros(3), torch.zeros(3, dtype=torch.int32), torch.zeros(3, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="draft must be"):
        ext.speculative_sample(t, torch.zeros(3, 16), torch.zeros(2, dtype=torch.int32), f, i, f, l, i)
    with pytest.raises(RuntimeError, match="proposals must be"):
        ext.speculative_sample(t, torch.zeros(2, 16), torch.zeros(3, dtype=torch.int32), f, i, f, l, i)
    with pytest.raises(RuntimeError, match="exceeds"):
        big = torch.zeros(1, ext.SPECULATIVE_SAMPLE_MAX_VOCAB + 1)
        ext.speculative_sample(big, big[:0], torch.zeros(0, dtype=torch.int32), f[:1], i[:1], f[:1], l[:1], i[:1])


# ------------------------------------------------------------------ CLI --
@pytest.fixture
def spec_cli(cpu_ext, monkeypatch):
    seen = {}

    def fake(draft, model, ids, n, **kw):
        seen.update(kw)
        return [1] * n, [(4, 4)]

    monkeypatch.setattr(gen, "speculative_generate_ids", fake)
    return seen


BASE = ["generate", "--synthetic", "tiny", "--prompt-ids", "5,17,3", "--max-new-tokens", "4", "--draft-synthetic", "tiny"]


def test_cli_passes_sampling_flags_to_speculative_decoding(spec_cli, capsys):
    assert cli_main(BASE + ["--device", "cpu", "--sampler-temp", "0.7", "--sampler-top-k", "20", "--sampler-top-p", "0.9", "--seed", "3"]) == 0
    assert spec_cli["sampling"] == SamplingParams(0.7, top_k=20, top_p=0.9, seed=3)
    assert "4/4 proposals accepted" in capsys.readouterr().err


@pytest.mark.parametrize("extra,message", [
    (["--presence-penalty", "1.5"], "drop the penalties"),
    (["--min-p", "0.1"], "drop the penalties"),
    (["--logprobs", "2"], "log-probabilities"),
    (["--regex", "a+"], "drop --regex"),
    (["--synthetic-lora", "a=2"], "adapters"),
])
def test_cli_refuses_what_speculative_sampling_does_not_take(spec_cli, extra, message):
    with pytest.raises(SystemExit, match=message):
        cli_main(BASE + ["--device", "cpu", "--sampler-temp", "0.7"] + extra)
