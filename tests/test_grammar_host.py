"""Grammar-constrained generation on the host (DESIGN.md section 23): the GBNF compiler and ``GrammarWalker`` against
the independent Earley recognizer of ``grammar_ref.py`` on every string of up to 6 bytes over a small alphabet that
extends a viable prefix, for ten grammars; the depth and parse caps; a regular grammar against the regex compiler;
every refusal with its message; the vocabulary check; ``SamplingParams``, the refusals of other paths, the C and
shim entries and the CLI."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import grammar as gmod
from tiny_llm_b200.constrained import TokenVocabulary, compile_dfa
from tiny_llm_b200.grammar import (GRAMMAR_MAX_DEPTH, GRAMMAR_MAX_PARSES, GRAMMAR_STATE_WORDS, GrammarConstraint, GrammarWalker,
                                   check_vocabulary, compile_grammar, load_grammar_arg)
from tiny_llm_b200.sampler import SamplingParams


def _load(name: str, file: str):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


gref = _load("tiny_llm_b200_grammar_ref", "grammar_ref.py")

EXPR = '''root ::= expr
expr ::= term | term "+" expr
term ::= num | "(" expr ")"
num  ::= [0-9]+'''

JSONLIKE = r'''# a small JSON
root   ::= value
value  ::= object | array | string | number | "true"
object ::= "{" ( pair ( "," pair )* )? "}"
pair   ::= string ":" value
array  ::= "[" ( value ( "," value )* )? "]"
string ::= "\"" [a]* "\""
number ::= "-"? [0-9]+'''

CLIKE = '''root ::= stmt+
stmt ::= "if" "(" id ")" stmt
       | "while" "(" id ")" stmt
       | id "=" id ";"
       | "{" stmt* "}"
id   ::= [a-z]+'''

CHESS = '''root  ::= move (" " move)*
move  ::= piece? file? rank? "x"? file rank promo? check? | "O-O" | "O-O-O"
piece ::= [KQRBN]
file  ::= [a-h]
rank  ::= [1-8]
promo ::= "=" [QRBN]
check ::= [+#]'''

NULLABLE = '''root ::= a b a "!"
a    ::= "x"* | c
b    ::= "y"?
c    ::= ("z" c)?'''

NESTING = '''root ::= p
p    ::= "(" p ")" | "[" p "]" | "x"'''

UTF8 = r'''root     ::= greek+ "." notlower any
greek    ::= [α-ω]
notlower ::= [^a-z\n]
any      ::= .'''

COUNTED = '''root ::= "a"{2,3} "b"{2} ("c" | "d"){0,2} [0-9]{1,}'''

SEVERAL = '''root ::= r1 | r2 | r3
r1   ::= "x" r1 "1" | "z"
r2   ::= "x" r2 "2" | "z"
r3   ::= "x" r3 "3" | "zz"'''

ESCAPES = r'''root ::= greet ("," " "? greet)*   # a list
greet ::= "h\x69" | "é"
        | [\t\\]'''

GRAMMARS = {
    "expr": (EXPR, b"12+()"),
    "jsonlike": (JSONLIKE, b'{}[]":,a1'),
    "clike": (CLIKE, b"ifx(){}=;"),
    "chess": (CHESS, b"Ne4xO-+"),
    "nullable": (NULLABLE, b"xyz!"),
    "nesting": (NESTING, b"()[]x"),
    "utf8": (UTF8, bytes([0x61, 0x2E, 0x0A, 0xCE, 0xB1, 0xC3, 0xA9, 0xE2, 0x82, 0xAC, 0xED, 0xA0])),
    "counted": (COUNTED, b"abcd1"),
    "several": (SEVERAL, b"xz123"),
    "escapes": (ESCAPES, "hi, é\t\\".encode()),
}


def _enumerate(text: str, alphabet: bytes, max_len: int = 6):
    """Every string of up to ``max_len`` bytes over ``alphabet`` that extends a viable prefix: the walker must agree
    with the reference on viability and completeness.  Returns (strings checked, most parses seen)."""
    g = compile_grammar(text)
    ref = gref.Earley(text)
    sets = ref.initial()
    w0 = GrammarWalker(g)
    assert w0.complete == ref.complete(sets)
    frontier = [(b"", sets, w0)]
    checked, most = 0, 1
    for _ in range(max_len):
        nxt = []
        for s, sets, w in frontier:
            for a in alphabet:
                sets2 = ref.feed(sets, a)
                w2 = w.copy()
                ok = w2.step(a)
                checked += 1
                assert ok == ref.viable(sets2), s + bytes([a])
                if ok:
                    assert w2.complete == ref.complete(sets2), s + bytes([a])
                    most = max(most, len(w2.parses))
                    nxt.append((s + bytes([a]), sets2, w2))
        frontier = nxt
    return checked, most


@pytest.mark.parametrize("name", sorted(GRAMMARS))
def test_walker_equals_the_earley_reference(name):
    text, alphabet = GRAMMARS[name]
    checked, most = _enumerate(text, alphabet)
    assert checked > 50
    assert most <= GRAMMAR_MAX_PARSES
    if name == "several":
        assert most >= 3  # several parses live at once, under the cap


def test_reference_on_hand_picked_texts():
    ref = gref.Earley(EXPR)
    assert ref.check(b"(1+2)+3") == (True, True)
    assert ref.check(b"(1+") == (True, False)
    assert ref.check(b"1)") == (False, False)
    u = gref.Earley(UTF8)
    assert u.check("αβ.Zé".encode()) == (True, True)
    assert u.check("α.a".encode())[0] is False
    assert u.check("α.".encode() + b"\xed")[0] is True  # a lead byte that can still start a non-surrogate character
    assert u.check(b"\xce\xb1.Z\xed\xa0")[0] is False  # a surrogate's encoding


def test_depth_cap_is_exact():
    g = compile_grammar(NESTING)
    ref = gref.Earley(NESTING)
    w = GrammarWalker(g)
    # root calls p at the first "(", each further "(" pushes one entry and the innermost p still needs one more
    assert w.walk(b"(" * (GRAMMAR_MAX_DEPTH - 1))
    assert w.depth == GRAMMAR_MAX_DEPTH - 1
    assert not w.copy().walk(b"(")
    assert not w.copy().walk(b"[")
    assert ref.check(b"(" * GRAMMAR_MAX_DEPTH)[0]  # the grammar has no cap; the walker keeps every text completable
    assert w.walk(b"x" + b")" * (GRAMMAR_MAX_DEPTH - 1)) and w.complete
    w = GrammarWalker(g)
    assert w.walk(b"([" * 15 + b"(") and w.walk(b"x" + b")" + b"])" * 15) and w.complete


def test_parse_cap_refuses_the_token():
    rules = "\n".join(f'r{k} ::= "x" r{k} "{k}" | "z"' for k in range(1, 10))
    text = 'root ::= "ab" tail\ntail ::= ' + " | ".join(f"r{k}" for k in range(1, 10)) + "\n" + rules
    g = compile_grammar(text)
    w = GrammarWalker(g)
    assert w.walk(b"ab")
    assert not w.copy().walk(b"x") and not w.copy().walk(b"z")  # nine parses: one past the cap
    assert gref.Earley(text).check(b"abx")[0]
    eight = text.replace(" | r9", "")
    w = GrammarWalker(compile_grammar(eight))
    assert w.walk(b"abxx") and len(w.parses) == GRAMMAR_MAX_PARSES


def test_regular_grammar_equals_the_regex_dfa():
    g = compile_grammar('root ::= [0-9]{4} "-" [0-9]{2} "-" [0-9]{2}')
    dfa = compile_dfa(r"[0-9]{4}-[0-9]{2}-[0-9]{2}")
    rng = np.random.default_rng(0)
    alphabet = b"0123456789-x"
    for _ in range(400):
        s = bytes(rng.choice(list(alphabet), int(rng.integers(0, 12))))
        w = GrammarWalker(g)
        ok = w.walk(s)
        d = dfa.walk(0, s)
        assert ok == (d >= 0), s
        if ok:
            assert w.complete == bool(dfa.accept[d]) and len(w.parses) == 1
    vocab = TokenVocabulary.synthetic(2000)
    c = GrammarConstraint('root ::= [0-9]{4} "-" [0-9]{2} "-" [0-9]{2}', vocab, device="cpu")
    for text in (b"", b"19", b"2024-", b"2024-01-3", b"2024-01-31"):
        w = c.start()
        assert w.walk(text)
        d0 = dfa.walk(0, text)
        want = np.array([(i in vocab.eos_ids and bool(dfa.accept[d0])) if t is None else dfa.walk(d0, t) >= 0
                         for i, t in enumerate(vocab.tokens)])
        assert np.array_equal(c.allowed(w), want), text


def test_words_round_trip_and_layout():
    g = compile_grammar(SEVERAL)
    w = GrammarWalker(g)
    assert w.walk(b"xxz")
    words = w.words(0x1234)
    assert len(words) == GRAMMAR_STATE_WORDS and words[0] == 0x1234
    assert words[1] & 15 == len(w.parses) and (words[1] >> 32) & 1
    back = GrammarWalker(g, words)
    assert back.parses == w.parses and not back.terminal and not back.failed
    for p, (s, stack) in enumerate(w.parses):
        assert words[2 + p] == s | len(stack) << 16
    w.terminal = True
    assert GrammarWalker(g, w.words(0)).terminal
    failed = GrammarWalker(g)
    failed.parses, failed.failed = (), True
    fw = failed.words(7)
    assert fw[1] == (1 << 32 | 1 << 34) and not any(fw[2:])
    assert gmod.failed_rows(torch.tensor([fw, w.words(7)], dtype=torch.int64)) == [0]


def test_blob_layout():
    g = compile_grammar(EXPR)
    blob = g.blob
    S, C, nbytes, A = np.frombuffer(blob[:16].tobytes(), dtype=np.int32)
    assert (S, C, nbytes) == (g.num_states, g.num_classes, blob.size) and nbytes % 16 == 0
    assert np.array_equal(blob[16:272], g.class_of)
    info = np.frombuffer(blob[272 : 272 + 4 * S].tobytes(), dtype=np.uint32)
    trans = np.frombuffer(blob[272 + 4 * S : 272 + 4 * S + 4 * S * C].tobytes(), dtype=np.uint32).reshape(S, C)
    acts = np.frombuffer(blob[272 + 4 * S + 4 * S * C : 272 + 4 * S + 4 * S * C + 4 * A].tobytes(), dtype=np.uint32)
    for s in range(S):
        assert info[s] & 1 == g.may_end[s] and info[s] >> 8 == g.need[s]
        for k in range(C):
            e = int(trans[s, k])
            got, off = [], e & 0xFFFFFF
            for _ in range(e >> 24):
                word = int(acts[off])
                n = (word >> 16) & 63
                pushes = tuple((int(acts[off + 1 + j // 2]) >> (16 * (j % 2))) & 0xFFFF for j in range(n))
                got.append((word & 0x7FFF, pushes, word >> 24))
                off += 1 + (n + 1) // 2
            assert tuple(got) == g.lists[s][k]
    assert any(len(p) >= 2 for row in g.lists for acts_ in row for _, p, _ in acts_)  # precomposed call chains


REFUSALS = [
    ("root ::= a", r"rule 'root': undefined rule 'a' at line 1, column 10"),
    ('x ::= "a"', "grammar has no 'root' rule"),
    ("root ::= <[12]>", r"rule 'root': token references .* at line 1, column 10"),
    ('root ::= "a" <think>', r"rule 'root': token references .* at line 1, column 14"),
    ('root ::= root "a" | "b"', r"rule 'root': left recursion \(root -> root\)"),
    ('root ::= a\na ::= b "x" | "y"\nb ::= a "z"', r"rule 'a': left recursion \(a -> b -> a\)"),
    ('root ::= a\na ::= n a "x" | "y"\nn ::= "q"?', r"rule 'a': left recursion \(a -> a\)"),
    ('root ::= a\na ::= "x" a', "the language of 'root' is empty"),
    (r"root ::= [^\x00-\U0010FFFF]", "the language of 'root' is empty"),
    ('root ::= "a"{1001}', r"rule 'root': repeat counts above 1000 are not supported at line 1, column 13"),
    ('root ::= "a"{3,2}', "min repeat greater than max repeat"),
    ('root ::= "abc', r"rule 'root': unterminated string literal at line 1, column 10"),
    ("root ::= [a-", "unterminated character class"),
    ('root ::= ("a"', "missing '\\)'"),
    ('root ::= "a"*+', "multiple repeat"),
    (r'root ::= "\q"', r"bad escape \\q"),
    (r'root ::= "\x4"', r"incomplete escape \\x"),
    ("root ::= [z-a]", "bad character range"),
    ('root = "a"', "expected '::=' after rule name 'root'"),
    ('root ::= "a"\nroot ::= "b"', r"rule 'root' is defined twice at line 2, column 1"),
    ('root ::= "a" @', r"rule 'root': unexpected '@'"),
    ("root ::= *", "nothing to repeat"),
]


@pytest.mark.parametrize("text,message", REFUSALS)
def test_refusals_name_the_rule_and_position(text, message):
    with pytest.raises(ValueError, match=message):
        compile_grammar(text)


def test_caps(monkeypatch):
    monkeypatch.setattr(gmod, "GRAMMAR_MAX_STATES", 10)
    with pytest.raises(ValueError, match="the automaton exceeds 10 states"):
        compile_grammar('root ::= "abcdefghijklmnop"')
    monkeypatch.undo()
    monkeypatch.setattr(gmod, "GRAMMAR_MAX_DEPTH", 0)
    with pytest.raises(ValueError, match="no complete text fits the depth cap of 0"):
        compile_grammar(NESTING)
    monkeypatch.undo()
    monkeypatch.setattr(gmod, "GRAMMAR_MAX_TABLE_BYTES", 256)
    with pytest.raises(ValueError, match="the tables take 6.* bytes, above the limit of 256"):
        compile_grammar(EXPR)
    monkeypatch.undo()
    monkeypatch.setattr(gmod, "_MAX_NFA_STATES", 100)
    with pytest.raises(ValueError, match="exceeds 100 automaton states"):
        compile_grammar('root ::= "a"{200}')


def test_syntax_features():
    g = compile_grammar('root ::= ( "a"\n  | "b" )  # comment\n  | "c"\n\n# trailing comment\n')
    for s, ok in ((b"a", True), (b"b", True), (b"c", True), (b"d", False)):
        w = GrammarWalker(g)
        assert w.walk(s) == ok and (not ok or w.complete)
    w = GrammarWalker(compile_grammar(r'root ::= "\U0001F600" [\]\-\^] "\"\\"'))
    assert w.walk("😀]\"\\".encode()) and w.complete
    w = GrammarWalker(compile_grammar("root ::= [^\\n]"))
    assert not w.copy().walk(b"\n") and w.copy().walk("é".encode()) and not w.copy().walk(b"\xc3\x28")
    assert not GrammarWalker(compile_grammar("root ::= .")).walk(b"\xed\xa0\x80")  # a surrogate is not a character
    assert GrammarWalker(compile_grammar('root ::= "" "a"{ 1 , 2 }')).walk(b"aa")


def test_vocabulary_check_and_token_walk():
    singles = [bytes([b]) for b in range(0x20, 0x7F)]
    with pytest.raises(ValueError, match="needs a vocabulary with an EOS id"):
        GrammarConstraint(EXPR, TokenVocabulary(singles, []), device="cpu")
    no_close = [t for t in singles if t != b")"] + [b"1)", None]
    with pytest.raises(ValueError, match=r"one-byte token for one of '\)'"):
        GrammarConstraint(EXPR, TokenVocabulary(no_close, [len(no_close) - 1]), device="cpu")
    vocab = TokenVocabulary(singles + [b"(1", b"+2", b"))", b"1+1", None], [len(singles) + 4])
    check_vocabulary(compile_grammar(EXPR), vocab)
    c = GrammarConstraint(EXPR, vocab, device="cpu")
    ids = {t: i for i, t in enumerate(vocab.tokens) if t is not None}
    eos = vocab.eos_ids[0]
    assert c.walk([ids[b"(1"], ids[b"+2"]]) is not None
    assert c.walk([ids[b"(1"], eos]) is None
    w = c.walk([ids[b"(1"], ids[b"+2"], ids[b")"], eos])
    assert w.terminal and np.flatnonzero(c.allowed(w)).tolist() == [eos]
    w = c.walk([ids[b"(1"], ids[b"+2"]])
    got = c.allowed(w)
    want = [i for i, t in enumerate(vocab.tokens) if t is not None and gref.Earley(EXPR).check(b"(1+2" + t)[0]]
    assert np.flatnonzero(got).tolist() == want


def test_sampling_params_and_refusals_of_other_paths():
    from tiny_llm_b200.generate import _spec_sampling
    from tiny_llm_b200.sampler import sample_tokens

    c = GrammarConstraint(EXPR, TokenVocabulary.synthetic(300), device="cpu")
    p = SamplingParams(0.0, constraint=c)
    assert p.constraint is c and p.grammar and not SamplingParams(0.0).grammar
    with pytest.raises(ValueError, match="take no grammar constraint"):
        SamplingParams(0.0, constraint=c, logit_bias={1: 2.0})
    with pytest.raises(ValueError, match="take no grammar constraint"):
        SamplingParams(0.0, constraint=c, min_tokens=2)
    with pytest.raises(ValueError, match="a grammar SamplingParams needs the request's ConstraintRows"):
        sample_tokens(torch.zeros(1, 300), [p], [1], constraints=torch.zeros(1, 5, dtype=torch.int64))
    with pytest.raises(ValueError, match="speculative decoding and prompt lookup are unconstrained: sampling must carry no grammar"):
        _spec_sampling(p, None)
    with pytest.raises(ValueError, match="speculative decoding is greedy and unconstrained: it takes no grammar"):
        _spec_sampling(None, c)


def test_load_grammar_arg(tmp_path):
    assert load_grammar_arg('root ::= "a"') == 'root ::= "a"'
    (tmp_path / "g.gbnf").write_text(EXPR)
    assert load_grammar_arg(str(tmp_path / "g.gbnf")) == EXPR
    with pytest.raises(OSError):
        load_grammar_arg(str(tmp_path / "missing.gbnf"))


def test_c_entries_and_shim_refusals_without_a_device():
    lib = ext._lib
    assert lib.tl_grammar_token_masks(None, None, -1, 8, 0, None) == -1
    assert b"grammar_token_masks: bad shape" in lib.tl_last_error()
    for smem in (-16, 8, 46 * 1024 + 16):
        assert lib.tl_grammar_token_masks(None, None, 2, 8, smem, None) == -1
        assert b"grammar_token_masks: bad smem_bytes" in lib.tl_last_error()
    assert lib.tl_grammar_token_masks(None, None, 2, 8, 0, None) == -1
    assert b"grammar_token_masks: null pointer" in lib.tl_last_error()
    assert lib.tl_grammar_advance(None, None, None, None, 2, 8, None) == -1
    assert b"grammar_advance: null pointer" in lib.tl_last_error()
    assert lib.tl_grammar_advance(None, None, None, None, 2, 0, None) == -1
    assert b"grammar_advance: bad shape" in lib.tl_last_error()
    assert lib.tl_grammar_token_masks(None, None, 0, 8, 0, None) == 0 and lib.tl_grammar_advance(None, None, None, None, 0, 8, None) == 0
    i64, i32 = torch.int64, torch.int32
    with pytest.raises(RuntimeError, match=r"grammar_states must be int64 \[2, 74\]"):
        ext.grammar_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 10, dtype=i64), 64)
    with pytest.raises(RuntimeError, match="vocab must be a positive int"):
        ext.grammar_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 74, dtype=i64), 0)
    with pytest.raises(RuntimeError, match=r"smem_bytes must be a multiple of 16 in \[0, 47104\]"):
        ext.grammar_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 74, dtype=i64), 64, 100)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.grammar_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 74, dtype=i64), 64)
    with pytest.raises(RuntimeError, match=r"tokens must be int32 \[2\]"):
        ext.grammar_advance(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 74, dtype=i64), torch.zeros(3, dtype=i32), torch.zeros(2, dtype=i32), 64)
    header = (Path(__file__).resolve().parents[1] / "include" / "tiny_llm_b200.h").read_text()
    for name in ("tl_grammar_token_masks", "tl_grammar_advance"):
        assert f"int {name}(" in header and name in ext.EXPORTED_SYMBOLS
    for name, value in (("TL_GRAMMAR_MAX_STATES", gmod.GRAMMAR_MAX_STATES), ("TL_GRAMMAR_MAX_DEPTH", GRAMMAR_MAX_DEPTH),
                        ("TL_GRAMMAR_MAX_PARSES", GRAMMAR_MAX_PARSES), ("TL_GRAMMAR_STATE_WORDS", GRAMMAR_STATE_WORDS),
                        ("TL_GRAMMAR_SMEM_BYTES (46 * 1024)", None), ("TL_GRAMMAR_MAX_TABLE_BYTES (1 << 22)", None)):
        assert f"#define {name}" + ("" if value is None else f" {value}") in header
    assert ext.GRAMMAR_STATE_WORDS == GRAMMAR_STATE_WORDS and ext.GRAMMAR_SMEM_BYTES == gmod.GRAMMAR_SMEM_BYTES


def test_cli_grammar_argument_errors(tmp_path, capsys):
    from tiny_llm_b200 import cli

    base = ["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2"]
    with pytest.raises(SystemExit, match="--grammar takes no --regex, --json or --json-schema: give one constraint"):
        cli.main(base + ["--regex", "a+", "--grammar", EXPR])
    with pytest.raises(SystemExit, match="--grammar takes no --regex, --json or --json-schema: give one constraint"):
        cli.main(base + ["--json", "--grammar", EXPR])
    with pytest.raises(SystemExit, match="speculative decoding and prompt lookup are greedy and unconstrained: drop --grammar"):
        cli.main(base + ["--prompt-lookup", "3", "--grammar", EXPR])
    with pytest.raises(SystemExit, match="beam search is deterministic and takes no --grammar"):
        cli.main(base + ["--num-beams", "2", "--grammar", EXPR])
    with pytest.raises(SystemExit, match="take no --grammar"):
        cli.main(base + ["--logit-bias", "1:2", "--grammar", EXPR])
    with pytest.raises(SystemExit, match="--grammar runs on the CUDA sampling kernel"):
        cli.main(base + ["--grammar", EXPR])
    with pytest.raises(SystemExit, match="--grammar: not a grammar file or inline GBNF grammar"):
        cli.main(base + ["--grammar", str(tmp_path / "missing.gbnf")])
    (tmp_path / "g.gbnf").write_text(EXPR)
    with pytest.raises(SystemExit, match="--grammar runs on the CUDA sampling kernel"):
        cli.main(["batch", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--quiet", "--grammar", str(tmp_path / "g.gbnf")])
    with pytest.raises(SystemExit, match="take no --grammar"):
        cli.main(["batch", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--quiet", "--min-tokens", "2", "--grammar", EXPR])
    with pytest.raises(SystemExit):
        cli.main(["score", "--synthetic", "tiny", "--grammar", EXPR])
    assert "unrecognized arguments: --grammar" in capsys.readouterr().err
