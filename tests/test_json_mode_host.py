"""JSON mode on the host (DESIGN.md section 20): the reference language against json.loads, the package walker against
the reference, the vocabulary check, and the refusals of every layer."""

import importlib.util
import json
import re
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200.constrained import TokenVocabulary
from tiny_llm_b200.json_mode import JSON_MAX_DEPTH, JSON_MAX_WS_RUN, JsonConstraint, JsonWalker, check_vocabulary
from tiny_llm_b200.sampler import SamplingParams


def _load(name: str, file: str):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


jref = _load("tiny_llm_b200_json_ref", "json_ref.py")

ALPHABET = b'{}[]:,"\\ua01-.e tn\xc3\xa9'  # structure, digits, escapes, a hex letter, space, literals, one 2-byte character


def _loads_dict(data: bytes) -> bool:
    try:
        value = json.loads(data.decode("utf-8", "strict"))
    except (UnicodeDecodeError, ValueError):
        return False
    return isinstance(value, dict) and jref.caps_hold(data)


def test_reference_complete_iff_json_loads_gives_a_dict_and_witnesses_parse():
    frontier, checked = [b""], 0
    for _ in range(6):
        nxt = []
        for p in frontier:
            for c in ALPHABET:
                s = p + bytes([c])
                kind = jref.classify(s)
                assert (kind == "complete") == _loads_dict(s), s
                if kind != "dead":
                    w = jref.witness(s)
                    assert w.startswith(s) and _loads_dict(w), (s, w)
                    nxt.append(s)
                checked += 1
        frontier = nxt
    assert checked > 100_000


def test_reference_caps():
    assert jref.classify(b" " * JSON_MAX_WS_RUN + b"{}" + b"\n" * JSON_MAX_WS_RUN) == "complete"
    assert jref.classify(b" " * (JSON_MAX_WS_RUN + 1)) == "dead"
    assert jref.classify(b"{}" + b" " * (JSON_MAX_WS_RUN + 1)) == "dead"
    assert jref.classify(b'{"a":' + b" " * (JSON_MAX_WS_RUN + 1)) == "dead"
    assert jref.classify(b'{"' + b" " * 100 + b'":1}') == "complete"  # string content is not whitespace
    deep = b'{"a":' + b"[" * (JSON_MAX_DEPTH - 1) + b"]" * (JSON_MAX_DEPTH - 1) + b"}"
    assert jref.classify(deep) == "complete" and _loads_dict(deep)
    assert jref.classify(b'{"a":' + b"[" * JSON_MAX_DEPTH) == "dead"
    assert not jref.caps_hold(b'{"a":' + b"[" * JSON_MAX_DEPTH + b"]" * JSON_MAX_DEPTH + b"}")


ADVERSARIAL = [b'"},', b"]]]", b'[{"', b"\\u00", b"\xc3", b"\xa9", b"\xe0", b"\xa0", b"\x80", b"\xf0\x9f", b"\x98\x80", b"-0.", b"1e+",
               b"01", b" " * 40, b" " * 20, b"\n\t", b"[" * 8, b"{\"k\":" * 3, b"true", b"fal", b"se", b"nul", b"l", b'\\"', b"\\",
               b"0", b"12", b".5", b"e", b"E-", b",", b":", b'"', b"{", b"}", b"[", b"]", b"a", b"u", b"F", b"\xed\x9f", b"\xed\xa0",
               b"\xf4\x8f", b"\xf4\x90", b'"}', b"}\n", b"}}", b'":"', b" ", b"\t"]


def adversarial_vocabulary() -> TokenVocabulary:
    """Every byte alone, then tokens that cross strings, containers, numbers, characters and both caps."""
    tokens = [bytes([b]) for b in range(256)] + ADVERSARIAL + [None, None]
    return TokenVocabulary(tokens, [len(tokens) - 2])


def _walker_allowed(vocab, walker, eos):
    out = np.zeros(vocab.size, dtype=bool)
    for i, t in enumerate(vocab.tokens):
        if t is None:
            out[i] = i in eos and walker.complete
        else:
            out[i] = walker.copy().walk(t)
    return out


@pytest.mark.parametrize("seed", range(6))
def test_walker_equals_reference_on_random_token_walks(seed):
    vocab = adversarial_vocabulary()
    eos = set(vocab.eos_ids)
    rng = np.random.default_rng(seed)
    heavy = [i for i, t in enumerate(vocab.tokens) if t is not None and (t.strip() == b"" and len(t) > 1 or t.count(b"[") > 2)]
    text, walker = b"", JsonWalker()
    for _ in range(120):
        want = jref.allowed(text, vocab.tokens, vocab.eos_ids)
        got = _walker_allowed(vocab, walker, eos)
        assert np.array_equal(got, want), (text, np.flatnonzero(got != want))
        assert walker.complete == (jref.classify(text) == "complete")
        choices = np.flatnonzero(want)
        assert choices.size, text
        pick_heavy = [i for i in heavy if want[i]]
        t = int(rng.choice(pick_heavy) if pick_heavy and rng.random() < 0.3 else rng.choice(choices))
        if t in eos:
            break
        assert walker.walk(vocab.tokens[t])
        text += vocab.tokens[t]
        assert JsonWalker(walker.words()).words() == walker.words()


def test_walker_state_words_and_caps_within_one_token():
    w = JsonWalker()
    assert w.words() == (0, 1 << 32)
    assert w.walk(b" " * 32 + b"{")
    assert not JsonWalker().walk(b" " * 33)
    w = JsonWalker()
    assert w.walk(b'{"a":' + b"[" * (JSON_MAX_DEPTH - 1))
    assert w.depth == JSON_MAX_DEPTH and w.stack == (1 << JSON_MAX_DEPTH) - 2
    assert not w.copy().walk(b"[") and not w.copy().walk(b"{") and w.copy().walk(b"0")
    stack, word1 = w.words()
    assert stack < 0  # bit 63 set: the word is signed int64 on the device
    assert JsonWalker((stack, word1)).words() == (stack, word1)


def test_json_constraint_walk_and_terminal():
    vocab = adversarial_vocabulary()
    c = JsonConstraint(vocab, device="cpu")
    ids = {t: i for i, t in enumerate(vocab.tokens) if t is not None}
    eos = vocab.eos_ids[0]
    w = c.walk([ids[b"{"], ids[b"}"]])
    assert w is not None and w.complete
    assert c.walk([ids[b"{"], eos]) is None
    w = c.walk([ids[b"{"], ids[b"}"], eos])
    assert w.terminal and not w.complete
    assert c.walk([ids[b"{"], ids[b"}"], eos, eos]).terminal
    assert c.walk([ids[b"{"], ids[b"}"], eos, ids[b" "]]) is None
    assert c.walk([ids[b"["]]) is None
    allowed = c.allowed(w)
    assert np.flatnonzero(allowed).tolist() == [eos]


def test_vocabulary_check():
    check_vocabulary(TokenVocabulary.synthetic(300))
    check_vocabulary(TokenVocabulary.synthetic(151_936))
    check_vocabulary(TokenVocabulary.synthetic(200))  # printable ASCII singles; its merges hold whole characters
    check_vocabulary(adversarial_vocabulary())
    singles = [bytes([b]) for b in range(256)]
    with pytest.raises(ValueError, match="needs a vocabulary with an EOS id"):
        check_vocabulary(TokenVocabulary(singles, []))
    with pytest.raises(ValueError, match=re.escape("one-byte token for each of '}'")):
        check_vocabulary(TokenVocabulary([t for t in singles if t != b"}"] + [b"}}", None], [256]))
    no_a0 = [t for t in singles if not 0xA0 <= t[0] <= 0xBF]
    with pytest.raises(ValueError, match="0xA0-0xBF: token .* UTF-8 lead byte 0xE0"):
        check_vocabulary(TokenVocabulary(no_a0 + [None], [len(no_a0)]))
    whole = [t for t in no_a0 if t != b"\xe0"] + [b"\xe0\xa0\x80", None]  # E0 only inside whole characters
    check_vocabulary(TokenVocabulary(whole, [len(whole) - 1]))
    no_cont = [t for t in singles if not 0x80 <= t[0] <= 0xBF]
    with pytest.raises(ValueError, match="0x80-0xBF"):
        ascii_lead = [t for t in no_cont if t[0] < 0x80] + [b"\xc3", None]
        check_vocabulary(TokenVocabulary(ascii_lead, [len(ascii_lead) - 1]))
    with pytest.raises(ValueError, match="EOS id"):
        JsonConstraint(TokenVocabulary(singles, []), device="cpu")


def test_sampling_params_accept_json_mode_and_refuse_other_types():
    c = JsonConstraint(TokenVocabulary.synthetic(300), device="cpu")
    assert SamplingParams(0.0, constraint=c).constraint is c
    with pytest.raises(ValueError, match="constraint must be None or a TokenConstraint"):
        SamplingParams(0.0, constraint="json")


def test_json_rows_need_constraint_rows_and_keep_logits_and_speculative_refuse_them():
    from tiny_llm_b200.generate import _spec_sampling
    from tiny_llm_b200.sampler import sample_tokens

    c = JsonConstraint(TokenVocabulary.synthetic(300), device="cpu")
    with pytest.raises(ValueError, match="needs the request's constraint descriptor"):
        sample_tokens(torch.zeros(1, 300), [SamplingParams(0.0, constraint=c)], [1])
    with pytest.raises(ValueError, match="needs the request's ConstraintRows"):
        sample_tokens(torch.zeros(1, 300), [SamplingParams(0.0, constraint=c)], [1], constraints=torch.zeros(1, 5, dtype=torch.int64))
    with pytest.raises(ValueError, match="speculative decoding is unconstrained"):
        _spec_sampling(SamplingParams(0.0, constraint=c), None)


def test_c_entries_and_shim_refusals_without_a_device():
    lib = ext._lib
    assert lib.tl_json_token_masks(None, None, -1, 8, None) == -1
    assert b"json_token_masks: bad shape" in lib.tl_last_error()
    assert lib.tl_json_token_masks(None, None, 2, 8, None) == -1
    assert b"json_token_masks: null pointer" in lib.tl_last_error()
    assert lib.tl_json_advance(None, None, None, None, 2, None) == -1
    assert b"json_advance: null pointer" in lib.tl_last_error()
    assert lib.tl_json_token_masks(None, None, 0, 8, None) == 0 and lib.tl_json_advance(None, None, None, None, 0, None) == 0
    i64, i32 = torch.int64, torch.int32
    with pytest.raises(RuntimeError, match=r"constraints must be int64 \[rows, 5\]"):
        ext.json_token_masks(torch.zeros(2, 4, dtype=i64), torch.zeros(2, 2, dtype=i64), 64)
    with pytest.raises(RuntimeError, match=r"json_states must be int64 \[2, 2\]"):
        ext.json_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 3, dtype=i64), 64)
    with pytest.raises(RuntimeError, match="vocab must be a positive int"):
        ext.json_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 2, dtype=i64), 0)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.json_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 2, dtype=i64), 64)
    with pytest.raises(RuntimeError, match=r"tokens must be int32 \[2\]"):
        ext.json_advance(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 2, dtype=i64), torch.zeros(3, dtype=i32), torch.zeros(2, dtype=i32))
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.json_advance(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 2, dtype=i64), torch.zeros(2, dtype=i32), torch.zeros(2, dtype=i32))
    header = (Path(__file__).resolve().parents[1] / "include" / "tiny_llm_b200.h").read_text()
    for name in ("tl_json_token_masks", "tl_json_advance"):
        assert f"int {name}(" in header and name in ext.EXPORTED_SYMBOLS
    assert f"#define TL_JSON_MAX_DEPTH {JSON_MAX_DEPTH}" in header and f"#define TL_JSON_MAX_WS_RUN {JSON_MAX_WS_RUN}" in header


def test_cli_json_argument_errors(capsys):
    from tiny_llm_b200 import cli

    with pytest.raises(SystemExit, match="give --regex or --json, not both"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--regex", "a+", "--json"])
    with pytest.raises(SystemExit, match="speculative decoding is greedy and unconstrained: drop --json"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--draft-synthetic", "tiny", "--json"])
    with pytest.raises(SystemExit, match="speculative decoding is greedy and unconstrained: drop --json"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--prompt-lookup", "3", "--json"])
    with pytest.raises(SystemExit, match="beam search is deterministic and takes no --json"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--num-beams", "2", "--json"])
    with pytest.raises(SystemExit, match="--json runs on the CUDA sampling kernel"):
        cli.main(["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--json"])
    with pytest.raises(SystemExit, match="--json runs on the CUDA sampling kernel"):
        cli.main(["batch", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--json", "--quiet"])
    with pytest.raises(SystemExit):
        cli.main(["score", "--synthetic", "tiny", "--json"])
    assert "unrecognized arguments: --json" in capsys.readouterr().err
