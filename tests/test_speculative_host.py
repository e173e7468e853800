"""Speculative decoding on the host: the protocol of ``speculative_generate`` / ``speculative_generate_ids`` with scripted
models and fake caches, the fast path's acceptance rule (proposals past a draft EOS are verified, then discarded), the
CLI through the CPU stand-in of the extension, and the builder checks of ``decode_attention_fused(rows_per_request=)``."""

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import greedy_generate_ids, speculative_generate, speculative_generate_ids
from tiny_llm_b200 import generate as gen
from tiny_llm_b200.cli import main as cli_main

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
    """A causal model whose greedy next token is a function of the whole prefix in its cache: ``rule(prefix)``."""

    def __init__(self, rule, layers=2):
        self.rule, self.layers = rule, layers
        self.calls, self.log, self.caches = [], [], []

    def create_kv_cache(self):
        cache = [FakeLayer(self.log) for _ in range(self.layers)]
        self.caches.append(cache)
        return cache

    def __call__(self, inputs, offset, cache, logits_to_keep=None):
        ids = [int(t) for t in inputs.reshape(-1).tolist()]
        assert all(layer.offset == offset for layer in cache), "the call's offset is the cache's"
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


def base_rule(prefix):
    return (sum((i + 3) * t for i, t in enumerate(prefix)) * 7 + 11) % (V - 1)  # never EOS


def rule_with(overrides, base=base_rule):
    """``base``, except at the prefix lengths in ``overrides`` (length -> token or callable(prefix))."""

    def rule(prefix):
        o = overrides.get(len(prefix))
        if o is None:
            return base(prefix)
        return o(prefix) if callable(o) else o

    return rule


def wrong(prefix):
    return (base_rule(prefix) + 1) % (V - 1)


PROMPT = [3, 9, 4]


def greedy(rule, n, eos=None, prompt=PROMPT):
    return greedy_generate_ids(Scripted(rule), prompt, n, eos_token_id=eos)


def spec(draft_rule, target_rule, n, k=4, eos=(), prompt=PROMPT):
    draft, target = Scripted(draft_rule), Scripted(target_rule)
    ids, stats = speculative_generate_ids(draft, target, prompt, n, proposal_length=k, eos_token_ids=eos)
    for m in (draft, target):
        assert all(layer.released for cache in m.caches for layer in cache), "every cache goes back to its pool"
    return ids, stats, draft, target


def test_target_prefill_eos_ends_the_run_before_the_draft_runs():
    ids, stats, draft, target = spec(base_rule, rule_with({3: EOS}), 20, eos=(EOS,))
    assert ids == [] and stats == [] and draft.calls == [] and target.calls == [(0, 3)]


def test_proposal_length_zero_is_target_only():
    ids, stats, draft, target = spec(base_rule, base_rule, 12, k=0)
    assert ids == greedy(base_rule, 12) and draft.calls == [] and stats == []
    assert [n for _, n in target.calls] == [3] + [1] * 11


def test_draft_prefill_eos_falls_back_to_target_only():
    ids, stats, draft, target = spec(rule_with({3: EOS}), base_rule, 10, eos=(EOS,))
    assert ids == greedy(base_rule, 10, EOS) and draft.calls == [(0, 3)] and stats == []
    assert all(n == 1 for _, n in target.calls[1:])


@pytest.mark.parametrize("index", [1, 2, 4])
def test_a_mismatch_rewinds_each_cache_exactly(index):
    # the draft's proposal `index` (1-based) of the first round is wrong: it is predicted at prefix length 3 + index
    k = 4
    ids, stats, draft, target = spec(rule_with({3 + index: wrong}), base_rule, 7, k=k)
    assert ids == greedy(base_rule, 7)
    assert stats[0] == (k, index - 1)
    assert target.calls[1] == (3, k + 1)
    assert target.log[0] == ("rewind", k + 1 - index) and len([e for e in target.log[:2] if e == target.log[0]]) == 2  # both layers
    draft_rewind = k - index
    if draft_rewind:
        assert draft.log[0] == ("rewind", draft_rewind)
    else:
        assert not draft.log or draft.calls.index((3 + index, 1)) >= 0
    # the next round starts at the target's correction, one position after the accepted prefix
    assert target.calls[2][0] == 3 + index


def test_low_acceptance_equals_the_target_only_output():
    ids, stats, _, _ = spec(lambda p: wrong(p), base_rule, 30, k=3)
    assert ids == greedy(base_rule, 30)
    assert all(acc == 0 for _, acc in stats)


def test_a_bonus_eos_ends_the_run_with_no_follow_up_call():
    # full acceptance of [t, d1, d2]; the bonus prediction (prefix length 3 + 3) is EOS
    target_rule = rule_with({6: EOS})
    ids, stats, draft, target = spec(target_rule, target_rule, 40, k=2, eos=(EOS,))
    assert ids == greedy(target_rule, 40, EOS) and len(ids) == 3
    assert target.calls == [(0, 3), (3, 3)] and draft.calls == [(0, 3), (3, 1), (4, 1)]


def test_an_eos_inside_a_short_proposal_is_terminal():
    target_rule = rule_with({5: EOS})
    ids, stats, draft, target = spec(target_rule, target_rule, 40, k=4, eos=(EOS,))
    assert ids == greedy(target_rule, 40, EOS) and len(ids) == 2
    assert draft.calls == [(0, 3), (3, 1), (4, 1)], "the draft stops after its EOS"
    assert target.calls == [(0, 3), (3, 3)] and stats == [(2, 2)]
    assert target.caches[0][0].offset == 5 and draft.caches[0][0].offset == 5


def test_full_acceptance_catch_up_offsets():
    ids, stats, draft, target = spec(base_rule, base_rule, 6, k=2, prompt=[3, 9])
    assert ids == greedy(base_rule, 6, prompt=[3, 9]) and stats == [(2, 2), (2, 2)]
    assert [o for o, _ in target.calls] == [0, 2, 5]
    assert [o for o, _ in draft.calls] == [0, 2, 3, 4, 5, 6]


def test_a_draft_eos_ends_the_proposal_without_terminating_the_target():
    ids, stats, draft, target = spec(rule_with({4: EOS}), base_rule, 12, k=4, eos=(EOS,))
    assert ids == greedy(base_rule, 12, EOS) and len(ids) == 12
    assert stats[0] == (1, 0) and target.calls[1] == (3, 2)


class FullProposals(gen._GenericRunner):
    """The fast path's draft: always k proposals, whatever they contain (the device cannot stop at a draft EOS)."""

    def draft(self, token, offset, cache, k, eos):
        return super().draft(token, offset, cache, k, ())


@pytest.mark.parametrize("eos_at,target_agrees", [(4, False), (4, True), (5, True), (6, False)])
def test_verifying_past_a_draft_eos_emits_what_the_early_stop_emits(eos_at, target_agrees):
    draft_rule = rule_with({eos_at: EOS})
    target_rule = rule_with({eos_at: EOS}) if target_agrees else base_rule
    runs = []
    for runner_cls in (gen._GenericRunner, FullProposals):
        draft, target = Scripted(draft_rule), Scripted(target_rule)
        out = []
        gen._speculate(runner_cls(target, draft, None), target, draft, PROMPT, 25, 4, {EOS}, out.extend)
        runs.append((out, [c[0].offset for c in target.caches], [c[0].offset for c in draft.caches]))
    assert runs[0] == runs[1]
    assert runs[0][0] == greedy(target_rule, 25, EOS)


class Detok:
    def __init__(self):
        self.ids = []

    def reset(self):
        self.ids = []

    def add_token(self, t):
        self.ids.append(t)

    @property
    def text(self):
        return " ".join(map(str, self.ids))


class Tok:
    def __init__(self, vocab=None, eos=EOS, prompt=PROMPT):
        self.vocab, self.eos_token_id, self.prompt = vocab or {"a": 0}, eos, prompt
        self.detokenizers = []

    def encode(self, text, add_special_tokens=False):
        return list(self.prompt)

    def get_vocab(self):
        return self.vocab

    @property
    def detokenizer(self):
        d = Detok()
        self.detokenizers.append(d)
        return d


def test_speculative_generate_prints_runs_and_returns_the_greedy_text(capsys):
    target_rule = rule_with({12: EOS})
    tok, dtok = Tok(), Tok()
    text = speculative_generate(Scripted(target_rule), Scripted(target_rule), dtok, tok, "hi", proposal_length=3)
    assert text == " ".join(map(str, greedy(target_rule, 100, EOS)))
    lines = capsys.readouterr().out.splitlines()
    assert lines[0].startswith("+") and lines[-1] == text
    text2 = speculative_generate(Scripted(target_rule), Scripted(target_rule), dtok, tok, "hi", proposal_length=3)
    assert text2 == text and len(tok.detokenizers) == 2 and tok.detokenizers[0] is not tok.detokenizers[1]


@pytest.mark.parametrize("case,msg", [
    ("prompt", "encode the prompt differently"),
    ("eos", "different EOS token ids"),
    ("vocab", "use different token ids"),
    ("no-vocab", "comparable vocabularies"),
    ("empty", "at least one token"),
])
def test_incompatible_tokenizers_fail_before_any_model_call(case, msg):
    draft, target = Scripted(base_rule), Scripted(base_rule)
    tok = Tok(prompt=[] if case == "empty" else PROMPT)
    dtok = Tok(prompt=[1, 2] if case == "prompt" else ([] if case == "empty" else PROMPT), eos=7 if case == "eos" else EOS,
               vocab={"b": 0} if case == "vocab" else None)
    if case == "no-vocab":
        dtok.get_vocab = None
    with pytest.raises(ValueError, match=msg):
        speculative_generate(draft, target, dtok, tok, "hi")
    assert draft.calls == [] and target.calls == []


@pytest.mark.parametrize("bad", [True, -1, 2.0, "3"])
def test_invalid_proposal_length_fails_before_any_model_call(bad):
    draft, target = Scripted(base_rule), Scripted(base_rule)
    with pytest.raises(ValueError, match="proposal_length must be a non-negative integer"):
        speculative_generate(draft, target, Tok(), Tok(), "hi", proposal_length=bad)
    with pytest.raises(ValueError, match="proposal_length must be a non-negative integer"):
        speculative_generate_ids(draft, target, PROMPT, 5, proposal_length=bad)
    assert draft.calls == [] and target.calls == []


def test_generic_path_takes_any_proposal_length():
    ids, stats, _, _ = spec(rule_with({7: wrong, 20: wrong}), base_rule, 40, k=9)
    assert ids == greedy(base_rule, 40) and max(p for p, _ in stats) == 9


def test_cli_speculative_run_prints_the_greedy_ids(cpu_ext, capsys):
    common = ["generate", "--synthetic", "tiny", "--prompt-ids", "5,17,3", "--max-new-tokens", "12", "--device", "cpu"]
    assert cli_main(common) == 0
    greedy_out = capsys.readouterr().out.split()
    assert cli_main(common + ["--draft-synthetic", "tiny", "--proposal-length", "3"]) == 0
    captured = capsys.readouterr()
    # the CPU stand-in's multi-row verify pass does not round like its one-row decode step, so only the shape of the
    # run and its prefilled first token are pinned here; token-for-token equality is the CUDA fast path's (GPU suite)
    out = captured.out.split()
    assert len(out) == 12 and all(t.isdigit() for t in out) and out[0] == greedy_out[0] and len(greedy_out) == 12
    assert "proposals accepted" in captured.err


# ----------------------------------------------------------- shim: rows_per_request builder checks --
def _attn_args(rows, R=1, table_rows=None, ctx_rows=None, D=128, Hq=4, Hkv=2):
    bf = torch.bfloat16
    return (torch.zeros(rows, (Hq + 2 * Hkv) * D, dtype=bf), torch.ones(D, dtype=bf), torch.ones(D, dtype=bf),
            torch.zeros(rows, dtype=torch.int32), torch.zeros(table_rows if table_rows is not None else rows // R, 3, dtype=torch.int32),
            torch.ones(ctx_rows if ctx_rows is not None else rows, dtype=torch.int32), torch.zeros(D // 2, dtype=torch.float64),
            torch.zeros(4, Hkv, 16, D, dtype=bf), torch.zeros(4, Hkv, 16, D, dtype=bf), Hq, Hkv, 1e-6, 1.0, 16)


@pytest.mark.parametrize("R", [0, 9, True, 2.0])
def test_rows_per_request_out_of_range_is_refused(R):
    with pytest.raises(RuntimeError, match=r"decode_attention_fused: rows_per_request must be an int in \[1, 8\]"):
        ext.decode_attention_fused(*_attn_args(8, 1), rows_per_request=R)
    with pytest.raises(RuntimeError, match=r"rows_per_request must be an int in \[1, 8\]"):
        ext.decode_attention_fused_workspace(1, 4, 2, rows_per_request=R)


def test_rows_per_request_shapes_are_checked_before_the_device():
    with pytest.raises(RuntimeError, match=r"qkv rows must be a multiple of rows_per_request \(3\)"):
        ext.decode_attention_fused(*_attn_args(8, 1, table_rows=2), rows_per_request=3)
    with pytest.raises(RuntimeError, match=r"block_table must be int32 \[B / rows_per_request, max_pages\] and context_lens int32 \[B\]"):
        ext.decode_attention_fused(*_attn_args(8, 4, table_rows=8), rows_per_request=4)
    with pytest.raises(RuntimeError, match=r"context_lens must hold one entry per row \(\[8\]\)"):
        ext.decode_attention_fused(*_attn_args(8, 4, ctx_rows=2), rows_per_request=4)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.decode_attention_fused(*_attn_args(8, 4), rows_per_request=4)
    with pytest.raises(RuntimeError, match=r"block_table must be int32 \[B, max_pages\] and context_lens int32 \[B\]"):
        ext.decode_attention_fused(*_attn_args(8, 1, table_rows=2))


class LimitedGraph(gen._GraphRunner):
    """The graph runner's length rule with the scripted models' calls in place of the engines."""

    draft = gen._GenericRunner.draft
    verify = gen._GenericRunner.verify


@pytest.mark.parametrize("target_limit,draft_limit", [(12, 40), (40, 13), (3, 40)])
def test_rounds_past_the_graph_length_continue_target_only(target_limit, draft_limit):
    draft, target = Scripted(rule_with({9: wrong})), Scripted(base_rule)
    target.decode_graph_max_seq_len, draft.decode_graph_max_seq_len = target_limit, draft_limit
    out = []
    gen._speculate(LimitedGraph(target, draft, None), target, draft, PROMPT, 20, 4, set(), out.extend)
    assert out == greedy(base_rule, 20)
    limit = min(target_limit, draft_limit)
    rows = [(o, n) for o, n in target.calls[1:]]
    assert all(o + n <= limit for o, n in rows if n > 1), "no verify pass reaches past the engines' length"
    assert all(o + n <= limit for o, n in draft.calls[1:]), "no draft step past the engines' length"
    assert rows[-1][1] == 1 and len(out) == 20
    if limit >= 3 + 5:
        assert any(n > 1 for _, n in rows)
    else:
        assert draft.calls == [], "a prompt already past the limit never runs the draft"


def test_cli_refuses_two_drafts(cpu_ext, tmp_path):
    with pytest.raises(SystemExit, match="not both"):
        cli_main(["generate", "--synthetic", "tiny", "--prompt-ids", "5,17,3", "--device", "cpu", "--draft-synthetic", "tiny",
                  "--draft-model", str(tmp_path)])
