"""Regex-constrained generation on the host: the byte DFA against ``re.fullmatch``, refused syntax, trimming, the
token-mask lifting against a per-token walk, dead-end vocabularies, the GPT-2 byte alphabet, ``SamplingParams`` and
the CLI's argument errors.  No kernel is launched here."""

import importlib.util
import re
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200.constrained import (MAX_STATES, TokenConstraint, TokenVocabulary, check_spellable, compile_dfa, descriptor_values,
                                       gpt2_byte_decoder, token_masks_reference, utf8_sequences)
from tiny_llm_b200.sampler import SamplingParams


def _load_constrained_ref():
    """tests/constrained_ref.py, loaded by path (tests/ is not a package)."""
    name = "tiny_llm_b200_constrained_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("constrained_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


cref = _load_constrained_ref()
PATTERNS, random_strings, token_masks_walk = cref.PATTERNS, cref.random_strings, cref.token_masks_walk


@pytest.mark.parametrize("pattern", PATTERNS)
def test_dfa_accepts_exactly_what_fullmatch_accepts(pattern):
    dfa = compile_dfa(pattern)
    rx = re.compile(pattern, re.ASCII)
    strings = random_strings(pattern, 400, seed=len(pattern))
    matched = 0
    for s in strings:
        want = rx.fullmatch(s) is not None
        matched += want
        assert dfa.matches(s.encode()) == want, (pattern, s)
    # and on strings the pattern matches: every prefix of a match is viable (the walk never dies on it)
    for s in strings:
        if rx.fullmatch(s):
            data = s.encode()
            for k in range(len(data) + 1):
                assert dfa.walk(0, data[:k]) >= 0


@pytest.mark.parametrize("pattern,text", [("[0-9]{4}-[0-9]{2}-[0-9]{2}", "2026-10-16"), (r"\d+(\.\d{1,3})?", "3.141"),
                                          ("é+ж?[α-ω]", "ééжλ"), (r"\w+@\w+\.(com|org)", "a_1@b.org"), ("x{2,4}y{0,2}z{3,}", "xxxyzzzz"),
                                          (r"\{\d\}\.\*\[\]", "{7}.*[]"), (".{0,4}!", "a\tä!")])
def test_known_matches_and_near_misses(pattern, text):
    dfa = compile_dfa(pattern)
    assert dfa.matches(text.encode())
    assert not dfa.matches(text.encode() + b"\x00")
    assert not dfa.matches(text.encode()[:-1]) or re.fullmatch(pattern, text[:-1], re.ASCII)


def test_quantifier_bounds_exactly():
    dfa = compile_dfa("a{2,4}")
    assert [dfa.matches(b"a" * n) for n in range(7)] == [False, False, True, True, True, False, False]
    assert [compile_dfa("a{3}").matches(b"a" * n) for n in range(5)] == [False, False, False, True, False]
    assert [compile_dfa("a{2,}").matches(b"a" * n) for n in (1, 2, 50)] == [False, True, True]
    assert [compile_dfa("a{,2}").matches(b"a" * n) for n in (0, 2, 3)] == [True, True, False]
    assert compile_dfa("a{").matches(b"a{") and compile_dfa("a{x}").matches(b"a{x}")  # not quantifiers: literals, as in re


def test_dot_and_negations_take_whole_utf8_characters():
    for pattern in (".", "[^a]", r"\D", r"\W", r"\S"):
        dfa = compile_dfa(pattern)
        for ch in ("ä", "中", "😀"):
            assert dfa.matches(ch.encode()), (pattern, ch)
            data = ch.encode()
            assert not dfa.matches(data[:1])
        assert not dfa.matches(b"\xff") and not dfa.matches(b"\xc0\x80")  # not well-formed UTF-8
        assert not dfa.matches("\ud800".encode("utf-8", "surrogatepass"))
    assert not compile_dfa(".").matches(b"\n")


def test_utf8_sequences_cover_each_range_exactly():
    for lo, hi in ((0, 0x10FFFF), (0x7F, 0x80), (0x7FF, 0x800), (0xD7FF, 0xE000), (0x10000, 0x10FFF), (0x3B1, 0x3C9)):
        seqs = utf8_sequences(lo, hi)
        for cp in sorted({lo, hi, (lo + hi) // 2, min(hi, lo + 1), 0xD800, 0xDFFF, 0xFFFF, 0x10000}):
            if not lo <= cp <= hi or 0xD800 <= cp <= 0xDFFF:
                continue
            data = chr(cp).encode()
            hits = [s for s in seqs if len(s) == len(data) and all(a <= b <= c for (a, c), b in zip(s, data))]
            assert len(hits) == 1, hex(cp)


@pytest.mark.parametrize("pattern,construct", [("^abc", "anchor '^'"), ("abc$", "anchor '$'"), (r"\bx", r"anchor \b"), (r"\Ax", r"anchor \A"),
                                               (r"(a)\1", r"backreference \1"), ("(?P<n>a)(?P=n)", "backreference (?P=...)"),
                                               ("a(?=b)", "lookaround"), ("a(?!b)", "lookaround"), ("(?<=a)b", "lookaround"),
                                               ("(?<!a)b", "lookaround"), ("(?i)a", "inline flags"), ("(?i:a)", "inline flags"),
                                               ("*a", "nothing to repeat"), ("a**", "multiple repeat"), ("a{3,2}", "min repeat greater"),
                                               ("(ab", "missing )"), ("ab)", "unbalanced parenthesis"), ("[ab", "unterminated character set"),
                                               ("a*+", "possessive"), (r"\q", r"bad escape \q"), ("[z-a]", "bad character range")])
def test_unsupported_or_bad_syntax_raises_naming_the_construct(pattern, construct):
    with pytest.raises(ValueError, match=re.escape(construct)):
        compile_dfa(pattern)


def test_state_limit_and_empty_language():
    with pytest.raises(ValueError, match="above the limit of 10"):
        compile_dfa("[a-z]{20}", max_states=10)
    assert compile_dfa("[a-z]{20}").num_states == 21
    assert MAX_STATES == 4096
    with pytest.raises(ValueError, match="matches nothing"):
        compile_dfa("[^\\x00-\\U0010ffff]")


@pytest.mark.parametrize("pattern", PATTERNS)
def test_trimming_leaves_only_live_states(pattern):
    dfa = compile_dfa(pattern)
    S = dfa.num_states
    assert dfa.table.dtype == np.int32 and dfa.table.shape == (S, 256)
    assert ((dfa.table >= -1) & (dfa.table < S)).all()
    live = dfa.accept.copy()
    for _ in range(S):
        live |= np.array([any(live[t] for t in row if t >= 0) for row in dfa.table])
    assert live.all()
    # every state is reachable from the start
    seen, stack = {0}, [0]
    while stack:
        for t in dfa.table[stack.pop()]:
            if t >= 0 and int(t) not in seen:
                seen.add(int(t))
                stack.append(int(t))
    assert seen == set(range(S))


@pytest.mark.parametrize("V", [128, 512, 3000])
def test_numpy_token_masks_equal_a_per_token_walk(V):
    vocab = TokenVocabulary.synthetic(V, seed=V)
    for pattern in (r"[0-9]{4}-[0-9]{2}-[0-9]{2}", r"(ab|cd)*e?", r"\w+@\w+\.(com|org)", r"[^a-c\n]{1,3}"):
        dfa = compile_dfa(pattern)
        masks, reach = token_masks_reference(dfa, vocab)
        want_m, want_r = token_masks_walk(dfa, vocab)
        assert masks.dtype == np.uint32 and masks.shape == (dfa.num_states + 1, (V + 31) // 32)
        np.testing.assert_array_equal(masks, want_m)
        np.testing.assert_array_equal(reach, want_r)


def test_synthetic_vocabulary_is_deterministic_and_well_formed():
    for V in (128, 512, 151936):
        a, b = TokenVocabulary.synthetic(V), TokenVocabulary.synthetic(V)
        assert a.size == V and a.tokens == b.tokens and a.eos_ids == [V - 1] and a.tokens[V - 1] is None
        assert all(t is None or 1 <= len(t) <= 8 * 2 for t in a.tokens)
    assert TokenVocabulary.synthetic(512).tokens[:256] == [bytes([i]) for i in range(256)]
    assert bytes([ord("7")]) in TokenVocabulary.synthetic(128).tokens
    lengths = [len(t) for t in TokenVocabulary.synthetic(151936).tokens if t is not None]
    assert 2 < np.mean(lengths) < 6 and max(lengths) >= 8
    assert TokenVocabulary.synthetic(512, seed=1).tokens != TokenVocabulary.synthetic(512, seed=2).tokens
    with pytest.raises(ValueError, match="EOS ids"):
        TokenVocabulary([b"a"], [3])


def test_dead_end_vocabularies_are_detected():
    # a vocabulary of "ab" and "a" cannot finish "ab?c" after "a" + "b" ... it has no "c" at all
    vocab = TokenVocabulary([b"a", b"ab", b"b", None], [3])
    dfa = compile_dfa("abc|a")
    masks, reach = token_masks_reference(dfa, vocab)
    with pytest.raises(ValueError, match="cannot continue the text"):
        check_spellable("abc|a", masks, reach, dfa.num_states)
    ok = TokenVocabulary([b"a", b"ab", b"c", None], [3])
    check_spellable("abc|a", *token_masks_reference(dfa, ok), dfa.num_states)
    # without an EOS id an accepting state with no continuation is a dead end too
    vocab = TokenVocabulary([b"x", b"y"], [])
    dfa = compile_dfa("xy")
    with pytest.raises(ValueError, match="cannot continue"):
        check_spellable("xy", *token_masks_reference(dfa, vocab), dfa.num_states)


def test_gpt2_byte_alphabet_round_trips():
    dec = gpt2_byte_decoder()
    assert len(dec) == 256 and sorted(dec.values()) == list(range(256))
    assert dec["Ġ"] == 0x20 and dec["Ċ"] == 0x0A and dec["a"] == ord("a") and dec["!"] == ord("!")
    enc = {b: c for c, b in dec.items()}
    for data in (b"hello world", " 2026-10-16\n".encode(), "ééжλ中😀".encode(), bytes(range(256))):
        assert bytes(dec[c] for c in "".join(enc[b] for b in data)) == data


def test_vocabulary_from_a_byte_level_tokenizer():
    class Added:
        def __init__(self, content, special):
            self.content, self.special = content, special

        def __str__(self):
            return self.content

    class Tok:  # the Hugging Face attributes the builder reads
        all_special_ids = [4]
        added_tokens_decoder = {4: Added("<|endoftext|>", True), 5: Added("<think>", False)}
        eos_token_id = 4

        def __len__(self):
            return 6

        def convert_ids_to_tokens(self, ids):
            return ["a", "Ġb", "ĊĊ", "Ã©", "<|endoftext|>", "<think>"][: len(ids)]

    vocab = TokenVocabulary.from_tokenizer(Tok(), 8)
    assert vocab.tokens == [b"a", b" b", b"\n\n", "é".encode(), None, b"<think>", None, None]
    assert vocab.eos_ids == [4]


def test_sampling_params_validate_the_constraint():
    with pytest.raises(ValueError, match="constraint must be None or a TokenConstraint"):
        SamplingParams(0.0, constraint="[0-9]+")
    assert SamplingParams(0.0).constraint is None
    c = TokenConstraint.__new__(TokenConstraint)
    p = SamplingParams(0.0, constraint=c)
    assert p.constraint is c and not p.penalized and p == SamplingParams(0.0, constraint=c)


def test_descriptor_layout():
    assert descriptor_values(None) == [0] * 5
    assert ext.CONSTRAINT_ROW_WORDS == 5


def test_host_walk_of_a_constraint():
    vocab = TokenVocabulary([b"1", b"2", b"12", b"-", None], [4])
    dfa = compile_dfa(r"\d{2}-?")
    masks, reach = token_masks_reference(dfa, vocab)
    c = TokenConstraint(r"\d{2}-?", vocab, dfa, torch.from_numpy(masks.view(np.int32)), None, None, reach)
    S = c.terminal_state
    assert c.walk(0, [2]) == dfa.walk(0, b"12") and dfa.accept[c.walk(0, [2])]
    assert c.walk(0, [2, 4]) == S and c.walk(0, [2, 4, 4]) == S
    assert c.walk(0, [4]) == -1 and c.walk(0, [2, 4, 0]) == -1 and c.walk(0, [2, 2]) == -1
    assert c.walk(0, [0, 1, 3, 4]) == S


def test_shim_checks_constrained_arguments_before_the_device():
    f32, i32, i64 = torch.float32, torch.int32, torch.int64
    x = torch.zeros(2, 64)
    args = [torch.zeros(2, dtype=f32), torch.zeros(2, dtype=i32), torch.zeros(2, dtype=f32), torch.zeros(2, dtype=i64), torch.zeros(2, dtype=i32)]
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.sample_constrained(x, *args, torch.zeros(2, 5, dtype=i64))
    with pytest.raises(RuntimeError, match=r"constraints must be int64 \[2, 5\]"):
        ext.sample_constrained(x, *args, torch.zeros(2, 4, dtype=i64))
    with pytest.raises(RuntimeError, match="every penalty array and the state, or none"):
        ext.sample_constrained(x, *args, torch.zeros(2, 5, dtype=i64), repetition=torch.ones(2))
    with pytest.raises(RuntimeError, match=r"state must be int32 \[2, 64\]"):
        ext.sample_constrained(x, *args, torch.zeros(2, 5, dtype=i64), *[torch.zeros(2)] * 4, torch.zeros(2, 63, dtype=i32))
    with pytest.raises(RuntimeError, match=r"dfa must be int32 \[S, 256\]"):
        ext.constraint_token_masks(torch.zeros(3, 255, dtype=i32), torch.zeros(3, dtype=torch.uint8), torch.zeros(5, dtype=i32),
                                   torch.zeros(4, dtype=torch.uint8), torch.zeros(1, dtype=i32))
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.constraint_token_masks(torch.zeros(3, 256, dtype=i32), torch.zeros(3, dtype=torch.uint8), torch.zeros(5, dtype=i32),
                                   torch.zeros(4, dtype=torch.uint8), torch.zeros(1, dtype=i32))
    lib = ext._lib
    assert lib.tl_constraint_token_masks(None, None, 0, None, None, 4, None, 0, None, None, None) == -1
    assert b"constraint_token_masks: bad shape" in lib.tl_last_error()
    assert lib.tl_sample_constrained(*[None] * 13, 1, 64, 7, None) == -2


def test_sample_tokens_refuses_a_constraint_without_descriptors_or_of_another_vocabulary():
    from tiny_llm_b200.sampler import sample_tokens

    vocab = TokenVocabulary([b"1", None], [1])
    dfa = compile_dfa("1")
    masks, reach = token_masks_reference(dfa, vocab)
    c = TokenConstraint("1", vocab, dfa, torch.from_numpy(masks.view(np.int32)), None, None, reach)
    with pytest.raises(ValueError, match="needs the request's constraint descriptor"):
        sample_tokens(torch.zeros(1, 2), [SamplingParams(0.0, constraint=c)], [1])
    with pytest.raises(ValueError, match="the constraint's vocabulary has 2 ids, the logits 3"):
        sample_tokens(torch.zeros(1, 3), [SamplingParams(0.0, constraint=c)], [1], constraints=torch.zeros(1, 5, dtype=torch.int64))


def test_speculative_decoding_refuses_a_constraint():
    from tiny_llm_b200.generate import speculative_generate_ids

    with pytest.raises(ValueError, match="greedy and unconstrained"):
        speculative_generate_ids(None, None, [1, 2], 4, constraint=object())


def test_cli_regex_argument_errors(capsys):
    from tiny_llm_b200 import cli

    with pytest.raises(SystemExit, match="speculative decoding is greedy and unconstrained: drop --regex"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--draft-synthetic", "tiny", "--regex", "a+"])
    with pytest.raises(SystemExit, match="--regex runs on the CUDA sampling kernel"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--regex", "a+"])
    with pytest.raises(SystemExit, match="--regex runs on the CUDA sampling kernel"):
        cli.main(["batch", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--regex", "a+", "--quiet"])
    with pytest.raises(SystemExit):
        cli.main(["score", "--synthetic", "tiny", "--regex", "a+"])
    assert "unrecognized arguments: --regex" in capsys.readouterr().err
