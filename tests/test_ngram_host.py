"""Prompt lookup on the host: the plain-loop proposer (``ngram_ref.py``) on hand-built histories, the protocol of
``prompt_lookup_generate_ids`` with scripted models and the reference proposer in place of the kernel, its refusals,
and the CLI through the CPU stand-in of the extension."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from tiny_llm_b200 import greedy_generate_ids, prompt_lookup_generate_ids
from tiny_llm_b200 import generate as gen
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.sampler import SamplingParams


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_ngram_ref", "ngram_ref.py")


# ------------------------------------------------------------------ the reference --
def test_no_match():
    assert R.propose([1, 2, 3, 4, 5], 4, 1, 3) == (0, -1, [])
    assert R.propose([1, 2, 3, 1], 4, 2, 3) == (0, -1, []), "a 1-token match is below n_min = 2"


@pytest.mark.parametrize("s", [[], [7], [7, 7]])
def test_histories_no_longer_than_n_min(s):
    assert R.propose(s, 3, 2, 4) == (0, -1, [])


def test_single_token_history_has_no_candidate_end():
    assert R.propose([5], 2, 1, 1) == (0, -1, [])
    assert R.propose([5, 5], 2, 1, 1) == (1, 0, [5, 5])


def test_a_tie_goes_to_the_latest_occurrence():
    s = [1, 2, 10, 1, 2, 20, 1, 2]
    assert R.propose(s, 2, 2, 3) == (2, 4, [20, 1])


def test_a_longer_match_beats_a_later_shorter_one():
    s = [3, 1, 2, 10, 0, 1, 2, 20, 3, 1, 2]
    assert R.propose(s, 1, 2, 4) == (3, 2, [10])


def test_the_n_max_cap_makes_equal_lengths_tie_to_the_latest():
    s = [3, 1, 2, 10, 0, 1, 2, 20, 3, 1, 2]
    assert R.propose(s, 1, 2, 2) == (2, 6, [20])


@pytest.mark.parametrize("period", [1, 3])
def test_self_extension_repeats_the_period(period):
    unit = [4, 5, 6][:period]
    s = [9] + unit * 3
    c, e, p = R.propose(s, 7, 1, 8)
    assert (c, e) == {1: (2, 2), 3: (6, 6)}[period], "the latest end of the longest match, one period back"
    assert p == (unit * 8)[:7]


def test_a_continuation_longer_than_the_remaining_history():
    s = [1, 2, 3, 7, 8, 1, 2, 3]
    c, e, p = R.propose(s, 7, 2, 3)
    assert (c, e) == (3, 2)
    assert p == [7, 8, 1, 2, 3, 7, 8]


def test_a_match_overlapping_the_suffix():
    assert R.propose([0, 9, 9, 9, 9], 3, 1, 8) == (3, 3, [9, 9, 9])
    assert R.propose([9, 9, 9, 9], 3, 1, 8) == (3, 2, [9, 9, 9])


def test_appended_tokens_equal_a_history_written_in_one_piece():
    g = torch.Generator().manual_seed(0)
    s = torch.randint(0, 4, (200,), generator=g).tolist()
    prop = RefProposer(None, s[:50], 4, (2, 3))
    committed = list(s[:50])
    i = 50
    while i < len(s):
        token = s[i]
        got = prop(committed, token)
        want = R.propose(s[: i + 1], 4, 2, 3)
        assert got[0] == want[0] and got[1] == want[2]
        step = 1 + i % 8
        committed.extend(s[i : i + step])
        i += step


# ------------------------------------------------------------------ the protocol, scripted --
V = 50
EOS = 49


class FakeLayer:
    def __init__(self, log):
        self.tokens, self.log, self.released = [], log, False

    @property
    def offset(self):
        return len(self.tokens)

    def rewind(self, n):
        assert 0 <= n <= len(self.tokens)
        self.log.append(("rewind", n))
        del self.tokens[len(self.tokens) - n :]

    def release(self):
        self.released = True


class Scripted:
    """A causal model whose greedy next token is ``rule(prefix)`` of the whole prefix in its cache."""

    def __init__(self, rule, layers=2):
        self.rule, self.layers = rule, layers
        self.calls, self.log, self.caches = [], [], []

    def create_kv_cache(self):
        cache = [FakeLayer(self.log) for _ in range(self.layers)]
        self.caches.append(cache)
        return cache

    def __call__(self, inputs, offset, cache, logits_to_keep=None):
        ids = [int(t) for t in inputs.reshape(-1).tolist()]
        assert all(layer.offset == offset for layer in cache)
        self.calls.append((offset, len(ids)))
        rows = []
        for t in ids:
            for layer in cache:
                layer.tokens.append(t)
            logits = torch.zeros(V)
            logits[self.rule(tuple(cache[0].tokens))] = 1.0
            rows.append(logits)
        n = logits_to_keep or len(ids)
        return torch.stack(rows[-n:])[None]


class RefProposer:
    """``NgramProposer`` with the plain-loop reference in place of the kernel (host ids only)."""

    instances: list = []

    def __init__(self, model, prompt_ids, k, ngram, device=None, sampled=False, capacity=0):
        self.k, self.ngram, self.s, self.appends = k, ngram, list(prompt_ids), []
        RefProposer.instances.append(self)

    def __call__(self, committed, token):
        new = [*committed[len(self.s) :], int(token)]
        assert 1 <= len(new) <= 8, "each call appends the ids emitted since the previous one (at most 8)"
        self.s += new
        assert self.s == [*committed, token], "the history is the prompt, the emitted ids and the pending token"
        self.appends.append(len(new))
        c, _, p = R.propose(self.s, self.k, *self.ngram)
        return c, p, p, None


def hash_rule(prefix):
    return (sum((i + 3) * t for i, t in enumerate(prefix)) * 7 + 11) % (V - 1)  # never EOS


def copy_rule(prefix):
    """The token after the latest earlier occurrence of the last token (text that copies itself), else a hash."""
    last = prefix[-1]
    for j in range(len(prefix) - 2, -1, -1):
        if prefix[j] == last:
            return prefix[j + 1]
    return hash_rule(prefix)


def rule_with(overrides, base=copy_rule):
    def rule(prefix):
        o = overrides.get(len(prefix))
        return base(prefix) if o is None else (o(prefix) if callable(o) else o)

    return rule


PROMPT = [3, 9, 4, 7, 1, 3, 9, 4, 7, 2, 6]


@pytest.fixture
def ref_proposer(monkeypatch):
    RefProposer.instances = []
    monkeypatch.setattr(gen, "NgramProposer", RefProposer)
    return RefProposer


def greedy(rule, n, eos=None, prompt=PROMPT):
    return greedy_generate_ids(Scripted(rule), prompt, n, eos_token_id=eos)


def lookup(rule, n, k=4, ngram=(2, 3), eos=(), prompt=PROMPT):
    target = Scripted(rule)
    ids, stats = prompt_lookup_generate_ids(target, prompt, n, proposal_length=k, ngram=ngram, eos_token_ids=eos)
    assert all(layer.released for cache in target.caches for layer in cache), "the cache goes back to its pool"
    assert len(target.caches) == 1, "prompt lookup keeps no second cache"
    return ids, stats, target


@pytest.mark.parametrize("k", [1, 4, 7])
@pytest.mark.parametrize("ngram", [(1, 1), (2, 3), (1, 8)])
@pytest.mark.parametrize("rule", [copy_rule, hash_rule])
def test_greedy_ids_are_unchanged(ref_proposer, k, ngram, rule):
    ids, stats, target = lookup(rule, 40, k=k, ngram=ngram)
    assert ids == greedy(rule, 40)
    assert all(p in (0, k) and 0 <= a <= p for p, a in stats)
    if rule is copy_rule:
        assert sum(a for _, a in stats) > 0, "text that copies itself accepts proposals"


def test_a_mismatch_rewinds_the_cache_exactly(ref_proposer):
    # the prompt's suffix [7, 2, 6] has no earlier occurrence; the copy rule then repeats [3, 9, 4, 7, ...] after a 3
    prompt = [3, 9, 4, 7, 1, 3, 9]
    k = 4
    # first round: pending token 4 (copy of the 3, 9 -> 4), match [3, 9, 4] at e = 2 proposes [7, 1, 3, 9]; the target
    # disagrees at prefix length 9 (the second proposal's slot)
    rule = rule_with({9: 0})
    ids, stats, target = lookup(rule, 12, k=k, prompt=prompt)
    assert ids == greedy(rule, 12, prompt=prompt)
    assert stats[0] == (k, 1)
    assert target.calls[1] == (7, k + 1)
    assert target.log[:2] == [("rewind", k + 1 - 2)] * 2, "both layers drop the rejected rows"
    assert target.calls[2][0] == 9


def test_a_no_match_round_is_exactly_one_target_step(ref_proposer):
    prompt = [1, 2, 3, 4, 5]
    ids, stats, target = lookup(hash_rule, 10, prompt=prompt, ngram=(8, 8))
    assert ids == greedy(hash_rule, 10, prompt=prompt)
    assert stats == [(0, 0)] * 10, "every round is recorded as (0, 0); the last one only emits its pending token"
    assert target.calls == [(0, 5)] + [(5 + i, 1) for i in range(9)]
    assert target.log == []


def test_an_eos_inside_a_proposal_ends_the_run(ref_proposer):
    prompt = [3, 9, EOS, 7, 3]
    rule = rule_with({6: EOS}, base=lambda p: 9 if p[-1] == 3 else hash_rule(p))
    ids, stats, target = lookup(rule, 30, k=4, ngram=(1, 3), prompt=prompt, eos=(EOS,))
    assert ids == greedy(rule, 30, EOS, prompt=prompt) == [9]
    # the pending 9 matches [3, 9] at e = 1: proposals [EOS, 7, 3, 9], the target agrees on EOS
    assert stats == [(4, 1)]
    assert target.calls == [(0, 5), (5, 5)]


def test_an_eos_proposal_the_target_rejects_is_discarded(ref_proposer):
    prompt = [3, 9, EOS, 7, 3]
    rule = lambda p: 9 if p[-1] == 3 else hash_rule(p)  # noqa: E731
    ids, stats, _ = lookup(rule, 20, k=4, ngram=(1, 3), prompt=prompt, eos=(EOS,))
    assert ids == greedy(rule, 20, EOS, prompt=prompt) and len(ids) == 20 and EOS not in ids
    assert stats[0] == (4, 0)


@pytest.mark.parametrize("n", [1, 2, 3, 5, 8, 13, 21])
def test_the_token_budget_is_respected(ref_proposer, n):
    ids, stats, _ = lookup(copy_rule, n, k=7, ngram=(1, 3))
    assert ids == greedy(copy_rule, n) and len(ids) == n


def test_zero_tokens_runs_no_model_call(ref_proposer):
    ids, stats, target = lookup(copy_rule, 0)
    assert ids == [] and stats == [] and target.calls == []


class LimitedGraph(gen._GraphRunner):
    """The graph runner's window rule with the scripted model's calls in place of the engines."""

    verify = gen._GenericRunner.verify
    propose = gen._GenericRunner.propose


@pytest.mark.parametrize("limit", [3, 10, 12, 20, 30])
def test_rounds_past_the_graph_window_run_target_only(ref_proposer, limit):
    prompt = [3, 9, 4, 7, 1, 3, 9]  # the pending 4 matches at once
    target = Scripted(copy_rule)
    target.decode_graph_max_seq_len = limit
    out = []
    proposer = RefProposer(target, prompt, 4, (2, 3))
    gen._speculate(LimitedGraph(target, None, None, proposer=proposer), target, None, prompt, 25, 4, set(), out.extend)
    assert out == greedy(copy_rule, 25, prompt=prompt)
    rows = target.calls[1:]
    assert all(o + n <= limit for o, n in rows if n > 1), "no verify pass reaches past the window"
    assert rows[-1][1] == 1
    calls = len(proposer.appends)
    if limit < len(prompt) + 5:
        assert calls == 0, "a prompt already at the window never runs the proposer"
    else:
        assert calls > 0 and any(n > 1 for _, n in rows)


@pytest.mark.parametrize("k", [0, 8, -1, True, 2.0, "3"])
def test_bad_proposal_lengths_are_refused_before_any_model_call(ref_proposer, k):
    target = Scripted(copy_rule)
    with pytest.raises(ValueError, match=r"proposal_length must be an integer in \[1, 7\]"):
        prompt_lookup_generate_ids(target, PROMPT, 5, proposal_length=k)
    assert target.calls == [] and RefProposer.instances == []


@pytest.mark.parametrize("ngram", [(0, 2), (3, 2), (1, 9), (2,), (1, 2, 3), 3, (True, 2), (1.5, 2)])
def test_bad_ngram_ranges_are_refused_before_any_model_call(ref_proposer, ngram):
    target = Scripted(copy_rule)
    with pytest.raises(ValueError, match="ngram must"):
        prompt_lookup_generate_ids(target, PROMPT, 5, ngram=ngram)
    assert target.calls == []


@pytest.mark.parametrize("sampling,msg", [
    (SamplingParams(0.7, repetition_penalty=1.2), "no penalties or min-p"),
    (SamplingParams(0.7, min_p=0.1), "no penalties or min-p"),
    ("greedy", "sampling must be None or a SamplingParams"),
])
def test_what_draft_speculation_refuses_is_refused(ref_proposer, sampling, msg):
    target = Scripted(copy_rule)
    with pytest.raises(ValueError, match=msg):
        prompt_lookup_generate_ids(target, PROMPT, 5, sampling=sampling)
    assert target.calls == []


def test_an_empty_prompt_is_refused(ref_proposer):
    with pytest.raises(ValueError, match="at least one token"):
        prompt_lookup_generate_ids(Scripted(copy_rule), [], 5)


# ------------------------------------------------------------------ CLI --
CLI = ["generate", "--synthetic", "tiny", "--prompt-ids", "5,17,3,9,5,17,3", "--max-new-tokens", "12", "--device", "cpu"]


def test_cli_prompt_lookup_prints_the_greedy_ids(cpu_ext, ref_proposer, capsys):
    assert cli_main(CLI) == 0
    greedy_out = capsys.readouterr().out.split()
    assert cli_main(CLI + ["--prompt-lookup", "3", "--prompt-lookup-ngram", "1:2"]) == 0
    captured = capsys.readouterr()
    out = captured.out.split()
    # the CPU stand-in's multi-row verify pass does not round like its one-row step, so, as for draft speculation,
    # the shape of the run and the prefilled first token are pinned here and token-for-token equality on the GPU
    assert len(out) == 12 and all(t.isdigit() for t in out) and out[0] == greedy_out[0]
    assert "proposals accepted" in captured.err and "rounds matched" in captured.err
    assert RefProposer.instances and RefProposer.instances[-1].ngram == (1, 2)


def test_cli_prompt_lookup_without_a_match_prints_the_greedy_ids(cpu_ext, ref_proposer, capsys):
    assert cli_main(CLI) == 0
    greedy_out = capsys.readouterr().out.split()
    # an 8-token suffix never recurs in this run, so every round is a one-row target step, as greedy's
    assert cli_main(CLI + ["--prompt-lookup", "4", "--prompt-lookup-ngram", "8:8"]) == 0
    captured = capsys.readouterr()
    assert captured.out.split() == greedy_out
    assert ", 0 rounds matched" in captured.err


@pytest.mark.parametrize("extra,msg", [
    (["--draft-synthetic", "tiny"], "not both"),
    (["--regex", "[0-9]+"], "drop --regex"),
    (["--presence-penalty", "1.0"], "drop the penalties"),
    (["--min-p", "0.1"], "drop the penalties"),
    (["--logprobs", "2"], "drop --logprobs"),
    (["--synthetic-lora", "a=8"], "does not take adapters"),
    (["--prompt-lookup-ngram", "3:2"], "1 <= n_min <= n_max <= 8"),
    (["--prompt-lookup-ngram", "x"], "--prompt-lookup-ngram"),
])
def test_cli_refuses_what_speculation_refuses(cpu_ext, ref_proposer, extra, msg):
    with pytest.raises(SystemExit, match=msg):
        cli_main(CLI + ["--prompt-lookup", "4", *extra])


@pytest.mark.parametrize("k", ["0", "8"])
def test_cli_refuses_a_bad_proposal_count(cpu_ext, ref_proposer, k):
    with pytest.raises(SystemExit, match=r"in \[1, 7\]"):
        cli_main(CLI + ["--prompt-lookup", k])


@pytest.mark.parametrize("alphabet", [2, 3, 50])
def test_the_vectorised_reference_equals_the_loops(alphabet):
    g = torch.Generator().manual_seed(alphabet)
    for i in range(300):
        L = int(torch.randint(0, 60, (1,), generator=g))
        s = torch.randint(0, alphabet, (L,), generator=g).tolist()
        n_max = 1 + i % 8
        n_min = 1 + (i // 8) % n_max
        k = 1 + i % 7
        assert R.propose_np(s, k, n_min, n_max) == R.propose(s, k, n_min, n_max), (s, k, n_min, n_max)
