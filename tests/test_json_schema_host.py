"""JSON Schema structured outputs on the host (DESIGN.md section 21): the independent reference against json.loads and
a validator (and jsonschema where it is installed), the package walker against the reference on token walks, the
vocabulary check, and the refusals of the compiler, the C entries, the shim and the CLI."""

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
from tiny_llm_b200.json_schema import (SCHEMA_MAX_DEPTH, SCHEMA_MAX_ITEMS, SCHEMA_MAX_STATES, SCHEMA_SMEM_BYTES, SCHEMA_STATE_WORDS,
                                       JsonSchemaConstraint, SchemaWalker, check_vocabulary, compile_schema)
from tiny_llm_b200.sampler import SamplingParams


def _load(name: str, file: str):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


sref = _load("tiny_llm_b200_json_schema_ref", "json_schema_ref.py")
jhost = _load("tiny_llm_b200_json_mode_host", "test_json_mode_host.py")

TREE = {"$defs": {"node": {"type": "object", "properties": {"v": {"type": "integer"}, "kids": {"type": "array", "items": {"$ref": "#/$defs/node"}}},
                           "required": ["v"]}}, "$ref": "#/$defs/node"}
# name -> (schema, seed prefixes the enumeration grows from, its alphabet)
SCHEMAS = {
    "flat": ({"type": "object", "properties": {"a": {"type": "string"}, "b": {"type": "integer"}}, "required": ["a", "b"]},
             [b"", b'{"a":"', b'{"a":"x","b":', b'{"a":"x","b":1'], b'{}",:ab1-0\\ .'),
    "nested": ({"type": "object", "properties": {"o": {"type": "object", "properties": {"x": {"type": "boolean"}}, "required": ["x"]}},
                "required": ["o"]}, [b'{"o":', b'{"o":{"x":', b'{"o":{"x":t'], b'{}":,otrfx '),
    "optional": ({"type": "object", "properties": {"a": {"type": "number"}, "b": {"type": "null"}, "c": {"type": "integer"}},
                  "required": ["c"]}, [b"{", b'{"a":', b'{"a":1', b'{"b":n', b'{"a":1,"c":'], b'{}":,abcn1.e- '),
    "items": ({"type": "object", "properties": {"r": {"type": "array", "minItems": 1, "maxItems": 2,
                                                        "items": {"type": "object", "properties": {"k": {"type": "integer"}}}}},
               "required": ["r"]}, [b'{"r":', b'{"r":[', b'{"r":[{}', b'{"r":[{},', b'{"r":[{},{}'], b'{}[]":,rk1 '),
    "item_cap": ({"type": "object", "properties": {"n": {"type": "array", "items": {"type": "integer"}, "minItems": SCHEMA_MAX_ITEMS,
                                                           "maxItems": SCHEMA_MAX_ITEMS}}},
                 [b'{"n":[' + b"0," * (SCHEMA_MAX_ITEMS - 2), b'{"n":[' + b"0," * (SCHEMA_MAX_ITEMS - 1)], b'[]},0 '),
    "enum": ({"type": "object", "properties": {"e": {"enum": ["on", "o", 1, 12, None, True, -0.5]}}, "required": ["e"]},
             [b'{"e":', b'{"e":"o', b'{"e":1', b'{"e":-'], b'{}":,eon12ut-.5 '),
    "const": ({"type": "object", "properties": {"c": {"const": "x\"y"}}}, [b'{"c":', b'{"c":"x\\'], b'{}":,cxy\\ '),
    "pattern": ({"type": "object", "properties": {"p": {"type": "string", "pattern": "^[A-Z]{2}-[0-9]{1,2}$"}}, "required": ["p"]},
                [b'{"p":', b'{"p":"A', b'{"p":"AB-'], b'{}":,pAZ-09a\\ '),
    "nullable": ({"type": "object", "properties": {"s": {"type": ["string", "null"]}}, "required": ["s"]}, [b'{"s":', b'{"s":n'],
                 b'{}":,snul\\ '),
    "tree": ({"type": "object", "properties": {"t": TREE}, "$defs": TREE["$defs"]}, [b'{"t":', b'{"t":{"v":1,"kids":[', b'{"t":{"v":0,"kids":[{"v":1'],
             b'{}[]":,vkids01 '),
    "any": ({"type": "object", "properties": {"x": {}}}, [b'{"x":', b'{"x":[', b'{"x":{"'], b'{}[]":,x0tn-\\ '),
    "object": ({"type": "object"}, [b"", b'{"', b'{"k":', b'{"k":[{'], b'{}[]":,k0tn '),
}


def _walker(schema, text: bytes):
    w = SchemaWalker(compile_schema(schema))
    return w if w.walk(text) else None


# --------------------------------------------------------------------------------------- a strict validator --
def _parse(text: bytes):
    """json.loads keeping key order and number spellings (("int" | "float", text)); None when it does not parse."""
    try:
        return json.loads(text.decode("utf-8", "strict"), object_pairs_hook=lambda pairs: ("obj", pairs),
                          parse_int=lambda s: ("int", s), parse_float=lambda s: ("float", s))
    except (UnicodeDecodeError, ValueError):
        return None


def _plain(v):
    if isinstance(v, tuple) and v[0] == "obj":
        return {k: _plain(x) for k, x in v[1]}
    if isinstance(v, tuple):
        return int(v[1]) if v[0] == "int" else float(v[1])
    if isinstance(v, list):
        return [_plain(x) for x in v]
    return v


def _deref(root, s):
    while isinstance(s, dict) and "$ref" in s:
        node = root
        for part in s["$ref"][2:].split("/") if s["$ref"] != "#" else []:
            node = node[part]
        s = node
    return s


def _valid(v, s, root) -> bool:
    """``v`` (from ``_parse``) validates against ``s`` with keys in schema order and enum values in json.dumps form."""
    s = _deref(root, s)
    if "anyOf" in s:
        return any(_valid(v, b, root) for b in s["anyOf"])
    if "enum" in s or "const" in s:
        values = [s["const"]] if "const" in s else s["enum"]
        form = json.dumps(_plain(v), ensure_ascii=False) if not isinstance(v, tuple) or v[0] == "obj" else v[1]
        return any(json.dumps(x, ensure_ascii=False) == form and type(x) is type(_plain(v)) for x in values)
    types = s.get("type", ["object", "array", "string", "number", "boolean", "null"])
    types = [types] if isinstance(types, str) else types
    for t in types:
        if t == "null" and v is None or t == "boolean" and isinstance(v, bool):
            return True
        if t == "integer" and isinstance(v, tuple) and v[0] == "int" or t == "number" and isinstance(v, tuple) and v[0] in ("int", "float"):
            return True
        if t == "string" and isinstance(v, str):
            if "pattern" not in s:
                return True
            return "\\" not in json.dumps(v, ensure_ascii=False) and re.fullmatch(s["pattern"][1:-1], v, re.ASCII) is not None
        if t == "array" and isinstance(v, list):
            if not s.get("minItems", 0) <= len(v) <= s.get("maxItems", len(v)):
                return False
            return all(_valid(x, s.get("items", {}), root) for x in v)
        if t == "object" and isinstance(v, tuple) and v[0] == "obj":
            props, req = s.get("properties"), s.get("required", [])
            if props is None and s.get("additionalProperties") is not False and not req:
                return all(_valid(x, {}, root) for _, x in v[1])
            names = list(props or {})
            keys = [k for k, _ in v[1]]
            if any(k not in names for k in keys) or [names.index(k) for k in keys] != sorted({names.index(k) for k in keys}) \
                    or len(set(keys)) != len(keys) or any(r not in keys for r in req):
                return False
            return all(_valid(x, props[k], root) for k, x in v[1])
    return False


def _canonical(text: bytes, v) -> bool:
    """``text`` is written the way json.dumps writes its value, but for whitespace between tokens."""
    def dump(x):
        if isinstance(x, tuple) and x[0] == "obj":
            return "{" + ",".join(json.dumps(k, ensure_ascii=False) + ":" + dump(y) for k, y in x[1]) + "}"
        if isinstance(x, tuple):
            return json.dumps(_plain(x))
        if isinstance(x, list):
            return "[" + ",".join(dump(y) for y in x) + "]"
        return json.dumps(x, ensure_ascii=False)

    out, in_str, esc = bytearray(), False, False
    for b in text:
        if in_str:
            out.append(b)
            if esc:
                esc = False
            elif b == 0x5C:
                esc = True
            elif b == 0x22:
                in_str = False
        elif b not in b" \t\n\r":
            out.append(b)
            in_str = b == 0x22
    return bytes(out) == dump(v).encode()


def _nesting(text: bytes) -> int:
    """The deepest container nesting of ``text`` (the root object is 1)."""
    depth = best = 0
    in_str = esc = False
    for b in text:
        if in_str:
            esc, in_str = (False, True) if esc else (b == 0x5C, b != 0x22)
        elif b == 0x22:
            in_str = True
        elif b in b"{[":
            depth += 1
            best = max(best, depth)
        elif b in b"}]":
            depth -= 1
    return best


def _caps(text: bytes) -> bool:
    """Whitespace runs and nesting within the language's caps."""
    return max((len(m) for m in re.findall(rb"[ \t\n\r]+", text)), default=0) <= 32 and _nesting(text) <= SCHEMA_MAX_DEPTH + 1


def _enumerate(schema, seeds, alphabet, n, budget=40_000):
    """Every seed + up to n alphabet bytes whose parent is viable: (text, viable, complete, witness); a level that
    would take more than ``budget`` strings (free string content grows fastest) is left out."""
    out = []
    frontier = []
    for s in seeds:
        v = sref.check(schema, s)
        assert v[0], s
        frontier.append(s)
        out.append((s, *v))
    for _ in range(n):
        if len(frontier) * len(alphabet) > budget:
            break
        nxt = []
        for p in frontier:
            for b in alphabet:
                t = p + bytes([b])
                v = sref.check(schema, t)
                out.append((t, *v))
                if v[0]:
                    nxt.append(t)
        frontier = nxt
    return out


@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_reference_complete_iff_valid_and_witnesses_complete(name):
    schema, seeds, alphabet = SCHEMAS[name]
    tables = compile_schema(schema)
    rows = _enumerate(schema, seeds, alphabet, 6)
    assert len(rows) > 100
    for text, viable, complete, witness in rows:
        v = _parse(text)
        valid = v is not None and _valid(v, schema, schema)
        if complete:
            assert valid, text
        elif v is not None and valid and _canonical(text, v):
            assert not _caps(text), text  # canonical and valid within the caps: complete
        if viable:
            full = text + witness
            assert sref.check(schema, full)[1], (text, witness)
            assert _valid(_parse(full), schema, schema), (text, witness)
        w = SchemaWalker(tables)
        ok = w.walk(text)
        assert ok == viable, (text, viable)
        assert (ok and w.complete) == complete, text


@pytest.mark.parametrize("name", sorted(SCHEMAS))
def test_jsonschema_validates_every_complete_text(name):
    jsonschema = pytest.importorskip("jsonschema")
    schema, seeds, alphabet = SCHEMAS[name]
    for text, _, complete, witness in _enumerate(schema, seeds, alphabet, 3):
        if witness is not None:
            jsonschema.validate(json.loads(text + witness), schema)


def _allowed(tables, vocab, walker, eos):
    out = np.zeros(vocab.size, dtype=bool)
    for i, t in enumerate(vocab.tokens):
        if t is None:
            out[i] = i in eos and walker.complete
        else:
            out[i] = walker.copy().walk(t)
    return out


def _ref_allowed(schema, text, vocab, eos):
    out = np.zeros(vocab.size, dtype=bool)
    complete = sref.check(schema, text)[1]
    for i, t in enumerate(vocab.tokens):
        out[i] = (i in eos and complete) if t is None else sref.check(schema, text + t)[0]
    return out


WALK_SCHEMAS = ["flat", "items", "enum", "pattern", "tree", "any", "object"]


@pytest.mark.parametrize("name", WALK_SCHEMAS)
@pytest.mark.parametrize("seed", range(2))
def test_walker_equals_reference_on_random_token_walks(name, seed):
    schema = SCHEMAS[name][0]
    vocab = jhost.adversarial_vocabulary()
    eos = set(vocab.eos_ids)
    c = JsonSchemaConstraint(schema, vocab, device="cpu")
    rng = np.random.default_rng(seed)
    heavy = [i for i, t in enumerate(vocab.tokens) if t is not None and (t.strip() == b"" and len(t) > 1 or len(t) > 2)]
    text, walker = b"", c.start()
    for _ in range(40):
        want = _ref_allowed(schema, text, vocab, eos)
        got = _allowed(c.compiled, vocab, walker, eos)
        assert np.array_equal(got, want), (text, [vocab.tokens[i] for i in np.flatnonzero(got != want)])
        assert np.array_equal(c.allowed(walker), got)
        choices = np.flatnonzero(want)
        assert choices.size, text
        pick = [i for i in heavy if want[i]]
        t = int(rng.choice(pick) if pick and rng.random() < 0.4 else rng.choice(choices))
        if t in eos:
            break
        assert walker.walk(vocab.tokens[t])
        text += vocab.tokens[t]
        words = walker.words(1234)
        assert SchemaWalker(c.compiled, words).words(1234) == words


def test_depth_cap_and_state_words():
    deep = {"type": "object", "properties": {"x": {}}}
    w = _walker(deep, b'{"x":' + b"[" * SCHEMA_MAX_DEPTH)  # the value of x is at level 1, each array one deeper
    assert w is not None and w.depth == SCHEMA_MAX_DEPTH
    assert not w.copy().walk(b"[") and not w.copy().walk(b"0") and w.copy().walk(b"]")  # an item would sit one level deeper
    assert _walker(deep, b'{"x":' + b"[" * (SCHEMA_MAX_DEPTH + 1)) is None
    assert _walker(deep, b'{"x":' + b"[" * (SCHEMA_MAX_DEPTH - 1) + b"0") is not None
    for text in (b'{"x":' + b"[" * SCHEMA_MAX_DEPTH, b'{"x":' + b"[" * (SCHEMA_MAX_DEPTH - 1) + b"0"):
        assert sref.check(deep, text)[0] and not sref.check(deep, text + b"[")[0] and not sref.check(deep, text + b"{")[0]
    words = w.words(0x7FFF_0000_0000)
    assert len(words) == SCHEMA_STATE_WORDS and SchemaWalker(w.tables, words).words(0x7FFF_0000_0000) == words
    # a required chain deeper than the cap has no complete text
    chain = {"type": "integer"}
    for _ in range(SCHEMA_MAX_DEPTH + 1):
        chain = {"type": "object", "properties": {"c": chain}, "required": ["c"]}
    with pytest.raises(ValueError, match="no complete text fits the depth cap"):
        compile_schema(chain)
    # a tree with a required child array: entering a node needs room for its array
    tree = {"type": "object", "properties": {"t": {"type": "array", "items": {"$ref": "#/$defs/n"}}},
            "$defs": {"n": {"type": "object", "properties": {"k": {"type": "array", "items": {"$ref": "#/$defs/n"}}}, "required": ["k"]}}}
    text = b'{"t":[' + b'{"k":[' * (SCHEMA_MAX_DEPTH // 2 - 1)  # inside an array at level 31: a node there needs level 33
    w = _walker(tree, text)
    assert w is not None and not w.copy().walk(b"{") and w.copy().walk(b"]")
    assert not sref.check(tree, text + b"{")[0] and sref.check(tree, text + b"]")[0]
    assert not w.copy().walk(b" " * 33) and w.copy().walk(b" " * 32)


REFUSALS = [
    ({"type": "object", "properties": {"a": {"type": "string", "minLength": 1}}}, "#/properties/a/minLength", "minLength"),
    ({"type": "object", "properties": {"a": {"type": "number", "minimum": 0}}}, "#/properties/a/minimum", "minimum"),
    ({"type": "object", "properties": {"a": {"type": "string", "format": "date"}}}, "#/properties/a/format", "format"),
    ({"type": "object", "properties": {"a": {"allOf": [{}]}}}, "#/properties/a/allOf", "allOf"),
    ({"type": "object", "properties": {"a": {"oneOf": [{}]}}}, "#/properties/a/oneOf", "oneOf"),
    ({"type": "object", "properties": {"a": {"not": {}}}}, "#/properties/a/not", "not"),
    ({"type": "object", "patternProperties": {"x": {}}}, "#/patternProperties", "patternProperties"),
    ({"type": "object", "properties": {"a": {"type": "array", "prefixItems": []}}}, "#/properties/a/prefixItems", "prefixItems"),
    ({"type": "object", "properties": {"a": {"type": "array", "uniqueItems": True}}}, "#/properties/a/uniqueItems", "uniqueItems"),
    ({"type": "object", "properties": {"a": {"if": {}}}}, "#/properties/a/if", "if"),
    ({"type": "object", "properties": {"a": {"type": "string"}}, "additionalProperties": {"type": "string"}}, "#/additionalProperties",
     "additionalProperties"),
    ({"type": "object", "properties": {"a": {"anyOf": [{"type": "integer"}, {"type": "number"}]}}}, "#/properties/a/anyOf",
     "branches 0 and 1 both start with '-0-9'"),
    ({"type": "object", "properties": {"a": {"anyOf": [{"type": "object"}, {"type": "object", "properties": {}}]}}},
     "#/properties/a/anyOf", "both start with '{'"),
    ({"type": "object", "properties": {"a": {"type": ["integer", "number"]}}}, "#/properties/a/type", "both start"),
    ({"type": "object", "properties": {"a": {"type": "array", "maxItems": SCHEMA_MAX_ITEMS + 1}}}, "#/properties/a/maxItems",
     f"above the limit of {SCHEMA_MAX_ITEMS}"),
    ({"type": "object", "properties": {"a": {"type": "array", "minItems": SCHEMA_MAX_ITEMS + 1}}}, "#/properties/a/minItems", "minItems"),
    ({"type": "object", "properties": {"a": {"type": "string", "pattern": "[a-z]+"}}}, "#/properties/a/pattern", "anchored"),
    ({"type": "object", "properties": {"a": {"$ref": "https://example.com/s.json"}}}, "#/properties/a/\\$ref", "local"),
    ({"type": "array"}, "#", "root must be an object schema"),
    ({"type": "object", "required": ["z"], "properties": {"a": {}}}, "#/required", "not in properties"),
    ({"type": "object", "properties": {"a": {"enum": [[1]]}}}, "#/properties/a/enum", "scalars"),
]


@pytest.mark.parametrize("schema,path,what", REFUSALS, ids=[r[2][:24] for r in REFUSALS])
def test_refusals_name_the_keyword_and_its_path(schema, path, what):
    with pytest.raises(ValueError, match=re.escape(what) if "\\" not in path else what) as err:
        compile_schema(schema)
    assert re.search(f"at {path}", str(err.value)), str(err.value)


def test_table_and_state_caps():
    wide = {"type": "object", "properties": {f"p{i}": {"type": "string", "pattern": "^[a-z]{%d}$" % (40 + i % 7)} for i in range(600)}}
    with pytest.raises(ValueError, match=f"exceeds {SCHEMA_MAX_STATES} states|above the limit of"):
        compile_schema(wide)
    header = (Path(__file__).resolve().parents[1] / "include" / "tiny_llm_b200.h").read_text()
    for name, value in (("TL_SCHEMA_MAX_DEPTH", SCHEMA_MAX_DEPTH), ("TL_SCHEMA_MAX_ITEMS", SCHEMA_MAX_ITEMS),
                        ("TL_SCHEMA_MAX_STATES", SCHEMA_MAX_STATES), ("TL_SCHEMA_STATE_WORDS", SCHEMA_STATE_WORDS)):
        assert f"#define {name} {value}" in header
    assert "#define TL_SCHEMA_SMEM_BYTES (47 * 1024)" in header and SCHEMA_SMEM_BYTES == ext.SCHEMA_SMEM_BYTES == 47 * 1024
    assert SCHEMA_MAX_DEPTH >= 32 and SCHEMA_MAX_ITEMS >= 64


def test_nodes_compile_once_and_tables_are_deterministic():
    shared = {"type": "object", "properties": {"a": {"$ref": "#/$defs/s"}, "b": {"$ref": "#/$defs/s"}},
              "$defs": {"s": {"type": "string", "pattern": "^[a-z]{3}$"}}}
    once = {"type": "object", "properties": {"a": {"$ref": "#/$defs/s"}}, "$defs": shared["$defs"]}
    a, b = compile_schema(shared), compile_schema(once)
    assert a.num_states - b.num_states < 12  # the second reference adds a key and a value position, not a pattern copy
    assert np.array_equal(compile_schema(shared).blob, a.blob)
    assert compile_schema(json.dumps(shared)).blob.tobytes() == a.blob.tobytes()


def test_vocabulary_check_and_constraint_walk():
    schema = SCHEMAS["pattern"][0]
    tables = compile_schema(schema)
    singles = [bytes([b]) for b in range(256)]
    check_vocabulary(tables, TokenVocabulary(singles + [None], [256]))
    check_vocabulary(tables, TokenVocabulary.synthetic(151_936))
    with pytest.raises(ValueError, match="needs a vocabulary with an EOS id"):
        check_vocabulary(tables, TokenVocabulary(singles, []))
    no_upper = [t for t in singles if not 0x41 <= t[0] <= 0x5A] + [b"AB", None]
    with pytest.raises(ValueError, match="one-byte token for .*A"):
        check_vocabulary(tables, TokenVocabulary(no_upper, [len(no_upper) - 1]))
    vocab = jhost.adversarial_vocabulary()
    c = JsonSchemaConstraint({"type": "object"}, vocab, device="cpu")
    ids = {t: i for i, t in enumerate(vocab.tokens) if t is not None}
    eos = vocab.eos_ids[0]
    assert c.walk([ids[b"{"], ids[b"}"]]).complete
    assert c.walk([ids[b"{"], eos]) is None
    w = c.walk([ids[b"{"], ids[b"}"], eos])
    assert w.terminal and np.flatnonzero(c.allowed(w)).tolist() == [eos]
    assert c.walk([ids[b"{"], ids[b"}"], eos, ids[b" "]]) is None


def test_sampling_params_and_refusals_of_other_paths():
    from tiny_llm_b200.generate import _spec_sampling
    from tiny_llm_b200.sampler import sample_tokens

    c = JsonSchemaConstraint({"type": "object"}, TokenVocabulary.synthetic(300), device="cpu")
    assert SamplingParams(0.0, constraint=c).constraint is c
    with pytest.raises(ValueError, match="needs the request's ConstraintRows"):
        sample_tokens(torch.zeros(1, 300), [SamplingParams(0.0, constraint=c)], [1], constraints=torch.zeros(1, 5, dtype=torch.int64))
    with pytest.raises(ValueError, match="speculative decoding is unconstrained"):
        _spec_sampling(SamplingParams(0.0, constraint=c), None)


def test_c_entries_and_shim_refusals_without_a_device():
    lib = ext._lib
    assert lib.tl_schema_token_masks(None, None, -1, 8, 0, None) == -1
    assert b"schema_token_masks: bad shape" in lib.tl_last_error()
    for smem in (-16, 8, 47 * 1024 + 16):
        assert lib.tl_schema_token_masks(None, None, 2, 8, smem, None) == -1
        assert b"schema_token_masks: bad smem_bytes" in lib.tl_last_error()
    assert lib.tl_schema_token_masks(None, None, 2, 8, 0, None) == -1
    assert b"schema_token_masks: null pointer" in lib.tl_last_error()
    assert lib.tl_schema_advance(None, None, None, None, 2, None) == -1
    assert b"schema_advance: null pointer" in lib.tl_last_error()
    assert lib.tl_schema_token_masks(None, None, 0, 8, 0, None) == 0 and lib.tl_schema_advance(None, None, None, None, 0, None) == 0
    i64, i32 = torch.int64, torch.int32
    with pytest.raises(RuntimeError, match=r"schema_states must be int64 \[2, 10\]"):
        ext.schema_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 2, dtype=i64), 64)
    with pytest.raises(RuntimeError, match="vocab must be a positive int"):
        ext.schema_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 10, dtype=i64), 0)
    with pytest.raises(RuntimeError, match=r"smem_bytes must be a multiple of 16 in \[0, 48128\]"):
        ext.schema_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 10, dtype=i64), 64, 100)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.schema_token_masks(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 10, dtype=i64), 64)
    with pytest.raises(RuntimeError, match=r"tokens must be int32 \[2\]"):
        ext.schema_advance(torch.zeros(2, 5, dtype=i64), torch.zeros(2, 10, dtype=i64), torch.zeros(3, dtype=i32), torch.zeros(2, dtype=i32))
    header = (Path(__file__).resolve().parents[1] / "include" / "tiny_llm_b200.h").read_text()
    for name in ("tl_schema_token_masks", "tl_schema_advance"):
        assert f"int {name}(" in header and name in ext.EXPORTED_SYMBOLS


def test_cli_json_schema_argument_errors(tmp_path, capsys):
    from tiny_llm_b200 import cli

    base = ["generate", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2"]
    schema = '{"type": "object"}'
    with pytest.raises(SystemExit, match="give one of --regex, --json-schema, not several"):
        cli.main(base + ["--regex", "a+", "--json-schema", schema])
    with pytest.raises(SystemExit, match="give one of --json, --json-schema, not several"):
        cli.main(base + ["--json", "--json-schema", schema])
    with pytest.raises(SystemExit, match="drop --json-schema"):
        cli.main(base + ["--prompt-lookup", "3", "--json-schema", schema])
    with pytest.raises(SystemExit, match="beam search is deterministic and takes no --json-schema"):
        cli.main(base + ["--num-beams", "2", "--json-schema", schema])
    with pytest.raises(SystemExit, match="--json-schema runs on the CUDA sampling kernel"):
        cli.main(base + ["--json-schema", schema])
    with pytest.raises(SystemExit, match="--json-schema: not a JSON schema file or inline JSON object"):
        cli.main(base + ["--json-schema", str(tmp_path / "missing.json")])
    with pytest.raises(SystemExit, match="--json-schema: not a JSON schema file or inline JSON object"):
        cli.main(base + ["--json-schema", "{not json"])
    (tmp_path / "s.json").write_text(schema)
    with pytest.raises(SystemExit, match="--json-schema runs on the CUDA sampling kernel"):
        cli.main(["batch", "--synthetic", "tiny", "--device", "cpu", "--prompt-ids", "1,2", "--quiet", "--json-schema", str(tmp_path / "s.json")])
    with pytest.raises(SystemExit):
        cli.main(["score", "--synthetic", "tiny", "--json-schema", schema])
    assert "unrecognized arguments: --json-schema" in capsys.readouterr().err
