"""JSON Schema structured outputs (DESIGN.md section 21): generated text restricted to one JSON object that validates
against a schema, with its keys in the order the schema's ``properties`` lists them.

``compile_schema`` turns a schema into a deterministic byte-level pushdown automaton held in tables: one sub-automaton
per distinct schema node (a node reached through several ``$ref``s is compiled once), transition entries that shift to
a state, call a sub-automaton (pushing the return state) or return, a per-state whitespace flag (the whitespace run is
a counter in the row state, as in JSON mode) and a per-state depth need (the stack entries the cheapest completion
from the state still pushes, so that no allowed token leads past the depth cap).  String content, numbers, literals,
enums and patterns are table states too.

A number ends only at the byte after it: its end states hold a *return-and-reprocess* entry on ``,``, ``}``, ``]`` and
whitespace, which pops the return state and looks the same byte up there.  Every other value ends on its last byte.

Each step ``tl_schema_token_masks`` writes every schema row's token mask from its state on the device, the unchanged
``tl_sample_constrained`` draws under it, and ``tl_schema_advance`` walks the drawn token.  ``SchemaWalker`` is the
same automaton on the host, bit for bit: it sets a row's state from its history and checks a vocabulary.  The row
state layout and the caps are in ``include/tiny_llm_b200.h``."""

from __future__ import annotations

import json

import numpy as np
import torch

from .json_mode import JSON_MAX_WS_RUN, _zero_dfa

SCHEMA_MAX_DEPTH = 32  # stack entries: sub-automata open below the root object
SCHEMA_MAX_ITEMS = 64  # the largest minItems / maxItems
SCHEMA_MAX_STATES = 32767  # state ids 1..32767 (0 is the dead state)
SCHEMA_MAX_ACTIONS = 32768  # distinct call / return entries
SCHEMA_MAX_TABLE_BYTES = 1 << 22  # the whole table blob
SCHEMA_STATE_WORDS = 10  # int64 words of one row's state
SCHEMA_SMEM_BYTES = 47 * 1024  # tables up to this size are staged in shared memory

# entry kinds of an action (a transition that is not a plain shift): a shift to a state whose depth need is above the
# source's (checked against the depth cap), a call, a return, a return that reprocesses the byte
CHECKED_SHIFT, CALL, RETURN, REPROCESS = 0, 1, 2, 3
_ACTIVE, _TERMINAL = 1 << 32, 1 << 33
_WS = b" \t\n\r"
_INF = 255
_HEADER_BYTES = 16
_ANNOTATIONS = {"title", "description", "default", "examples", "$schema", "$id", "$comment"}
_TYPE_KEYWORDS = {"object": {"properties", "required", "additionalProperties"}, "array": {"items", "minItems", "maxItems"},
                  "string": {"pattern"}}
_FIRST_CLASSES = {"{": b"{", "[": b"[", '"': b'"', "-0-9": b"-0123456789", "t": b"t", "f": b"f", "n": b"n"}


def _class_of_first(b: int) -> str:
    for name, bs in _FIRST_CLASSES.items():
        if b in bs:
            return name
    return chr(b)


def _ptr(path: str, key) -> str:
    return f"{path}/{str(key).replace('~', '~0').replace('/', '~1')}"


class _Builder:
    """States as dicts byte -> action: ("S", t), ("C", t, r), ("R",) or ("P",) (return and reprocess)."""

    def __init__(self, schema):
        self.schema = schema
        self.edges: list[dict] = [{}]  # state 0: dead
        self.ws: list[bool] = [False]
        self.accept: list[bool] = [False]
        self.starts: dict = {}  # node key -> start state
        self.pending: list = []  # (value state, node key, return state): call entries filled once every node is built
        self.unions: dict = {}  # union start state -> (branch node keys, path), until finish fills it

    def state(self, ws: bool = False) -> int:
        self.edges.append({})
        self.ws.append(ws)
        self.accept.append(False)
        if len(self.edges) - 1 > SCHEMA_MAX_STATES:
            raise ValueError(f"JSON schema: the automaton exceeds {SCHEMA_MAX_STATES} states")
        if ws:
            for b in _WS:
                self.edges[-1][b] = ("S", len(self.edges) - 1)
        return len(self.edges) - 1

    def set(self, s: int, b: int, action, path: str) -> None:
        old = self.edges[s].get(b)
        if old is not None and old != action:
            raise ValueError(f"JSON schema at {path}: the automaton is not deterministic on byte {chr(b)!r}")
        self.edges[s][b] = action

    # ------------------------------------------------------------------------------------------------ nodes --
    def resolve(self, node, path: str, seen=()):
        """(schema dict, its JSON-pointer path) after following local $refs."""
        if not isinstance(node, dict):
            if node is True:
                return {}, path
            raise ValueError(f"JSON schema at {path}: a schema must be an object")
        if "$ref" in node:
            ref = node["$ref"]
            extra = sorted(k for k in node if k not in _ANNOTATIONS and k not in ("$ref", "$defs", "definitions"))
            if extra:
                raise ValueError(f"JSON schema at {_ptr(path, extra[0])}: keyword '{extra[0]}' next to $ref is not supported")
            if not isinstance(ref, str) or not (ref == "#" or ref.startswith("#/$defs/") or ref.startswith("#/definitions/")):
                raise ValueError(f"JSON schema at {_ptr(path, '$ref')}: only local $refs (#, #/$defs/..., #/definitions/...) are supported")
            if ref in seen:
                raise ValueError(f"JSON schema at {_ptr(path, '$ref')}: $ref cycle without a value in between")
            target = self.schema
            for part in ref[2:].split("/") if ref != "#" else []:
                part = part.replace("~1", "/").replace("~0", "~")
                if not isinstance(target, dict) or part not in target:
                    raise ValueError(f"JSON schema at {_ptr(path, '$ref')}: {ref!r} does not resolve")
                target = target[part]
            return self.resolve(target, ref, seen + (ref,))
        return node, path

    def node(self, raw, path: str) -> str:
        """The key of the compiled node for schema ``raw`` at ``path``; built once per distinct node."""
        node, path = self.resolve(raw, path)
        key = json.dumps({k: v for k, v in node.items() if k not in _ANNOTATIONS}, sort_keys=True)
        if key in self.starts:
            return key
        self.starts[key] = None  # in progress: recursion reaches it through a call, filled later
        self.starts[key] = self.build(node, path)
        return key

    def check_keywords(self, node, path, allowed) -> None:
        for k in node:
            if k not in allowed and k not in _ANNOTATIONS and k not in ("$defs", "definitions"):
                raise ValueError(f"JSON schema at {_ptr(path, k)}: keyword '{k}' is not supported")

    def build(self, node, path: str) -> int:
        """The start state of ``node``: its transitions are the value's first bytes (no whitespace)."""
        if "anyOf" in node:
            self.check_keywords(node, path, {"anyOf"})
            branches = node["anyOf"]
            if not isinstance(branches, list) or not branches:
                raise ValueError(f"JSON schema at {_ptr(path, 'anyOf')}: anyOf must be a non-empty list")
            return self.union([(b, _ptr(_ptr(path, "anyOf"), i)) for i, b in enumerate(branches)], _ptr(path, "anyOf"))
        if "enum" in node or "const" in node:
            self.check_keywords(node, path, {"enum", "const", "type"})
            if "enum" in node and "const" in node:
                raise ValueError(f"JSON schema at {_ptr(path, 'const')}: give enum or const, not both")
            values = [node["const"]] if "const" in node else node["enum"]
            kw = "const" if "const" in node else "enum"
            if not isinstance(values, list) or not values:
                raise ValueError(f"JSON schema at {_ptr(path, kw)}: enum must be a non-empty list")
            types = node.get("type")
            if types is not None:
                types = [types] if isinstance(types, str) else types
                values = [v for v in values if _json_type_ok(v, types)]
                if not values:
                    raise ValueError(f"JSON schema at {_ptr(path, kw)}: no value matches the type")
            return self.enum(values, _ptr(path, kw))
        types = node.get("type")
        if types is None:
            self.check_keywords(node, path, set())
            return self.union([({"type": t}, path) for t in ("object", "array", "string", "number", "boolean", "null")], path)
        if isinstance(types, list):
            if not types or not all(isinstance(t, str) for t in types):
                raise ValueError(f"JSON schema at {_ptr(path, 'type')}: type must be a name or a list of names")
            if len(types) > 1:
                self.check_keywords(node, path, {"type"}.union(*(_TYPE_KEYWORDS.get(t, set()) for t in types)))
                return self.union([({"type": t, **{k: v for k, v in node.items() if k in _TYPE_KEYWORDS.get(t, ())}}, path)
                                   for t in types], _ptr(path, "type"))
            types = types[0]
        if types == "object":
            self.check_keywords(node, path, {"type", "properties", "required", "additionalProperties"})
            return self.object(node, path, root=False)
        if types == "array":
            self.check_keywords(node, path, {"type", "items", "minItems", "maxItems"})
            return self.array(node, path)
        if types == "string":
            self.check_keywords(node, path, {"type", "pattern"})
            if "pattern" in node:
                return self.pattern(node["pattern"], _ptr(path, "pattern"))
            return self.string(("R",), path)
        if types in ("number", "integer"):
            self.check_keywords(node, path, {"type"})
            return self.number(types == "integer", path)
        if types == "boolean":
            self.check_keywords(node, path, {"type"})
            return self.enum([True, False], path)
        if types == "null":
            self.check_keywords(node, path, {"type"})
            return self.enum([None], path)
        raise ValueError(f"JSON schema at {_ptr(path, 'type')}: unknown type {types!r}")

    def union(self, branches, path: str) -> int:
        """A start state whose first bytes are those of every branch (filled by ``finish``); branches must differ in
        the value's first-byte class ({, [, ", -0-9, t, f, n)."""
        start = self.state()
        self.unions[start] = ([self.node(raw, bpath) for raw, bpath in branches], path)
        return start

    def fill(self, s: int, visiting=()) -> None:
        """Copy the branches' first bytes into union start ``s`` (unions of unions first)."""
        if s not in self.unions:
            return
        keys, path = self.unions.pop(s)
        owner: dict = {}
        for i, key in enumerate(keys):
            bs = self.starts[key]
            if bs in visiting or bs == s:
                raise ValueError(f"JSON schema at {path}: a schema refers to itself before any value begins")
            self.fill(bs, visiting + (s,))
            for cls in sorted({_class_of_first(b) for b in self.edges[bs]}):
                if cls in owner and owner[cls] != i:
                    raise ValueError(f"JSON schema at {path}: anyOf branches {owner[cls]} and {i} both start with "
                                     f"{cls!r}; branches must differ in their first byte")
                owner[cls] = i
            for b, action in self.edges[bs].items():
                self.set(s, b, action, path)

    # ----------------------------------------------------------------------------------------------- values --
    def chain(self, start: int, data: bytes, end, path: str) -> None:
        """Bytes ``data`` from ``start`` (its first byte already the start's transition), the last byte ``end``."""
        s = start
        for j, b in enumerate(data):
            if j == len(data) - 1:
                self.set(s, b, end, path)
            else:
                nxt = self.edges[s].get(b)
                if nxt is None:
                    t = self.state()
                    self.set(s, b, ("S", t), path)
                    s = t
                elif nxt[0] == "S":
                    s = nxt[1]
                else:
                    raise ValueError(f"JSON schema at {path}: values {data!r} collide")

    def enum(self, values, path: str) -> int:
        start = self.state()
        numbers = []
        for v in values:
            if isinstance(v, (dict, list)):
                raise ValueError(f"JSON schema at {path}: enum and const values must be scalars")
            if isinstance(v, float) and not np.isfinite(v):
                raise ValueError(f"JSON schema at {path}: {v!r} has no JSON form")
            try:
                text = json.dumps(v, ensure_ascii=False).encode()
            except (UnicodeEncodeError, ValueError):
                raise ValueError(f"JSON schema at {path}: {v!r} has no UTF-8 JSON form") from None
            if isinstance(v, (int, float)) and not isinstance(v, bool):
                numbers.append(text)
                continue
            self.chain(start, text, ("R",), path)
        for text in numbers:  # a number ends at the next byte: its last state returns and reprocesses
            s = start
            for b in text:
                nxt = self.edges[s].get(b)
                if nxt is None:
                    t = self.state()
                    self.set(s, b, ("S", t), path)
                    s = t
                elif nxt[0] == "S":
                    s = nxt[1]
                else:
                    raise ValueError(f"JSON schema at {path}: enum values {text!r} collide")
            for b in b",}]" + _WS:
                self.set(s, b, ("P",), path)
        return start

    def string(self, close, path: str) -> int:
        """A JSON string; the closing quote is ``close``.  Content: unescaped bytes 0x20-0x7F but '"' and '\\',
        escapes, \\uXXXX and UTF-8 in shortest form without surrogates."""
        start, body, esc = self.state(), self.state(), self.state()
        hexes = [self.state() for _ in range(4)]
        c1, c2, c3, e0, ed, f0, f4 = (self.state() for _ in range(7))
        self.set(start, 0x22, ("S", body), path)
        for b in range(0x20, 0x80):
            if b not in (0x22, 0x5C):
                self.set(body, b, ("S", body), path)
        self.set(body, 0x22, close, path)
        self.set(body, 0x5C, ("S", esc), path)
        for b in range(0xC2, 0xE0):
            self.set(body, b, ("S", c1), path)
        for b in range(0xE0, 0xF0):
            self.set(body, b, ("S", e0 if b == 0xE0 else ed if b == 0xED else c2), path)
        for b in range(0xF0, 0xF5):
            self.set(body, b, ("S", f0 if b == 0xF0 else f4 if b == 0xF4 else c3), path)
        for s, lo, hi, t in ((c1, 0x80, 0xBF, body), (c2, 0x80, 0xBF, c1), (c3, 0x80, 0xBF, c2), (e0, 0xA0, 0xBF, c1),
                             (ed, 0x80, 0x9F, c1), (f0, 0x90, 0xBF, c2), (f4, 0x80, 0x8F, c2)):
            for b in range(lo, hi + 1):
                self.set(s, b, ("S", t), path)
        for b in b'"\\/bfnrt':
            self.set(esc, b, ("S", body), path)
        self.set(esc, ord("u"), ("S", hexes[0]), path)
        for k in range(4):
            for b in b"0123456789abcdefABCDEF":
                self.set(hexes[k], b, ("S", hexes[k + 1] if k < 3 else body), path)
        return start

    def pattern(self, pattern, path: str) -> int:
        """A string whose raw content bytes (no escapes) fullmatch ``^...$``, compiled with the regex parser of
        ``constrained.py`` and intersected with UTF-8 string content."""
        from .constrained import compile_dfa

        if not isinstance(pattern, str) or not (pattern.startswith("^") and pattern.endswith("$")) or len(pattern) < 2 \
                or pattern.endswith("\\$"):
            raise ValueError(f"JSON schema at {path}: only fully anchored patterns ^...$ are supported")
        try:
            dfa = compile_dfa(pattern[1:-1])
        except ValueError as exc:
            raise ValueError(f"JSON schema at {path}: {exc}") from None
        # the raw content lexer: 0 ready, (k, lo, hi) k continuation bytes to go, the next in [lo, hi]
        def lex(state, b):
            if state == 0:
                if 0x20 <= b < 0x80 and b not in (0x22, 0x5C):
                    return 0
                if 0xC2 <= b <= 0xDF:
                    return (1, 0x80, 0xBF)
                if 0xE0 <= b <= 0xEF:
                    return (2, 0xA0 if b == 0xE0 else 0x80, 0x9F if b == 0xED else 0xBF)
                if 0xF0 <= b <= 0xF4:
                    return (3, 0x90 if b == 0xF0 else 0x80, 0x8F if b == 0xF4 else 0xBF)
                return None
            k, lo, hi = state
            if not lo <= b <= hi:
                return None
            return 0 if k == 1 else (k - 1, 0x80, 0xBF)

        # product states, then trim those from which no match can close
        index = {(0, 0): 0}
        order = [(0, 0)]
        edges: list[dict] = []
        while len(edges) < len(order):
            d, lx = order[len(edges)]
            row = {}
            for b in range(256):
                nd = int(dfa.table[d, b])
                nl = lex(lx, b)
                if nd < 0 or nl is None:
                    continue
                key = (nd, nl)
                if key not in index:
                    index[key] = len(order)
                    order.append(key)
                row[b] = index[key]
            edges.append(row)
        live = [bool(dfa.accept[d]) and lx == 0 for d, lx in order]
        changed = True
        while changed:
            changed = False
            for i, row in enumerate(edges):
                if not live[i] and any(live[t] for t in row.values()):
                    live[i] = changed = True
        if not live[0]:
            raise ValueError(f"JSON schema at {path}: the pattern matches no string content without escapes")
        ids = {i: self.state() for i in range(len(order)) if live[i]}
        start = self.state()
        self.set(start, 0x22, ("S", ids[0]), path)
        for i, s in ids.items():
            for b, t in edges[i].items():
                if live[t]:
                    self.set(s, b, ("S", ids[t]), path)
            if live[i] and dfa.accept[order[i][0]] and order[i][1] == 0:
                self.set(s, 0x22, ("R",), path)
        return start

    def number(self, integer: bool, path: str) -> int:
        start, minus, zero, intg = self.state(), self.state(), self.state(), self.state()
        ends = [zero, intg]
        self.set(start, ord("-"), ("S", minus), path)
        for s in (start, minus):
            self.set(s, ord("0"), ("S", zero), path)
            for b in b"123456789":
                self.set(s, b, ("S", intg), path)
        for b in b"0123456789":
            self.set(intg, b, ("S", intg), path)
        if not integer:
            dot, frac, mark, sign, exp = (self.state() for _ in range(5))
            ends += [frac, exp]
            for s in (zero, intg, frac):
                if s != frac:
                    self.set(s, ord("."), ("S", dot), path)
                for b in b"eE":
                    self.set(s, b, ("S", mark), path)
            for b in b"0123456789":
                for s, t in ((dot, frac), (frac, frac), (mark, exp), (sign, exp), (exp, exp)):
                    self.set(s, b, ("S", t), path)
            for b in b"+-":
                self.set(mark, b, ("S", sign), path)
        for s in ends:
            for b in b",}]" + _WS:
                self.set(s, b, ("P",), path)
        return start

    def value(self, vstate: int, raw, path: str, ret: int) -> None:
        """Value position ``vstate``: the value's first byte calls its node, which returns to ``ret``."""
        self.pending.append((vstate, self.node(raw, path), ret, path))

    def object(self, node, path: str, root: bool) -> int:
        start = self.state(ws=root)
        close = ("S", self.closed()) if root else ("R",)
        props = node.get("properties")
        required = node.get("required", [])
        additional = node.get("additionalProperties")
        if not isinstance(required, list) or not all(isinstance(r, str) for r in required) or len(set(required)) != len(required):
            raise ValueError(f"JSON schema at {_ptr(path, 'required')}: required must be a list of distinct names")
        if props is None and additional is not False and not required:
            if additional not in (None, True):
                raise ValueError(f"JSON schema at {_ptr(path, 'additionalProperties')}: only additionalProperties: false is supported")
            return self.any_object(start, close, path)
        if additional not in (None, False):
            raise ValueError(f"JSON schema at {_ptr(path, 'additionalProperties')}: only additionalProperties: false is supported")
        props = props or {}
        if not isinstance(props, dict):
            raise ValueError(f"JSON schema at {_ptr(path, 'properties')}: properties must be an object")
        names = list(props)
        for r in required:
            if r not in props:
                raise ValueError(f"JSON schema at {_ptr(path, 'required')}: required name {r!r} is not in properties")
        req = [n in required for n in names]
        n = len(names)
        k0 = self.state(ws=True)
        self.set(start, ord("{"), ("S", k0), path)
        colon = [self.state(ws=True) for _ in range(n)]
        vals = [self.state(ws=True) for _ in range(n)]
        after = [self.state(ws=True) for _ in range(n)]
        tries: dict = {}

        def allowed(i):  # keys that may follow member i (-1: none yet): up to and including the next required one
            out = []
            for j in range(i + 1, n):
                out.append(j)
                if req[j]:
                    break
            return tuple(out)

        def trie(keys):
            if keys not in tries:
                t = self.state()
                for j in keys:
                    self.chain(t, json.dumps(names[j], ensure_ascii=False).encode()[1:], ("S", colon[j]), _ptr(path, "properties"))
                tries[keys] = t
            return tries[keys]

        def can_close(i):
            return not any(req[i + 1:])

        if allowed(-1):
            self.set(k0, 0x22, ("S", trie(allowed(-1))), path)
        if can_close(-1):
            self.set(k0, ord("}"), close, path)
        for j, name in enumerate(names):
            self.set(colon[j], ord(":"), ("S", vals[j]), path)
            self.value(vals[j], props[name], _ptr(_ptr(path, "properties"), name), after[j])
            if allowed(j):
                comma = self.state(ws=True)
                self.set(after[j], ord(","), ("S", comma), path)
                self.set(comma, 0x22, ("S", trie(allowed(j))), path)
            if can_close(j):
                self.set(after[j], ord("}"), close, path)
        return start

    def any_object(self, start: int, close, path: str) -> int:
        k0, comma, colon, val, after = (self.state(ws=True) for _ in range(5))
        key = self.string(("S", colon), path)
        self.set(start, ord("{"), ("S", k0), path)
        self.set(k0, ord("}"), close, path)
        for s in (k0, comma):
            self.set(s, 0x22, self.edges[key][0x22], path)
        self.set(colon, ord(":"), ("S", val), path)
        self.value(val, {}, path, after)
        self.set(after, ord(","), ("S", comma), path)
        self.set(after, ord("}"), close, path)
        return start

    def array(self, node, path: str) -> int:
        lo, hi = node.get("minItems", 0), node.get("maxItems")
        for kw, v in (("minItems", lo), ("maxItems", hi)):
            if v is not None and (isinstance(v, bool) or not isinstance(v, int) or v < 0):
                raise ValueError(f"JSON schema at {_ptr(path, kw)}: {kw} must be a non-negative integer")
            if v is not None and v > SCHEMA_MAX_ITEMS:
                raise ValueError(f"JSON schema at {_ptr(path, kw)}: {kw} {v} is above the limit of {SCHEMA_MAX_ITEMS}")
        if hi is not None and hi < lo:
            raise ValueError(f"JSON schema at {_ptr(path, 'maxItems')}: maxItems is below minItems")
        items = node.get("items", {})
        if isinstance(items, list):
            raise ValueError(f"JSON schema at {_ptr(path, 'items')}: items must be one schema")
        ipath = _ptr(path, "items") if "items" in node else path + "/items"
        start, first = self.state(), self.state(ws=True)
        self.set(start, ord("["), ("S", first), path)
        if lo == 0:
            self.set(first, ord("]"), ("R",), path)
        if hi == 0:
            return start
        top = hi if hi is not None else max(lo, 1)
        after = [None] + [self.state(ws=True) for _ in range(top)]  # after[k]: k items so far (top: at least top)
        self.value(first, items, ipath, after[1])
        for k in range(1, top + 1):
            if k >= lo:
                self.set(after[k], ord("]"), ("R",), path)
            if hi is None or k < hi:
                v = self.state(ws=True)
                self.set(after[k], ord(","), ("S", v), path)
                self.value(v, items, ipath, after[min(k + 1, top)])
        return start

    def closed(self) -> int:
        if not hasattr(self, "_closed"):
            self._closed = self.state(ws=True)
            self.accept[self._closed] = True
        return self._closed

    def finish(self) -> None:
        """Fill the value positions' call entries (every node's first bytes are known now)."""
        for s in list(self.unions):
            self.fill(s)
        while self.pending:
            vstate, key, ret, path = self.pending.pop()
            for b, action in self.edges[self.starts[key]].items():
                if action[0] != "S":
                    raise ValueError(f"JSON schema at {path}: a value cannot be empty")
                self.set(vstate, b, ("C", action[1], ret), path)


def _json_type_ok(v, types) -> bool:
    names = {type(None): "null", bool: "boolean", str: "string", int: "integer", float: "number"}
    t = names.get(type(v))
    return t in types or (t == "integer" and "number" in types)


class CompiledSchema:
    """The tables of one schema: ``edges`` (per state, byte -> action), ``ws`` / ``accept`` flags, ``need`` (stack
    entries the cheapest completion pushes), the byte classes, and ``blob``, the device layout (DESIGN.md section 21):

    int32 num_states S, num_classes C, blob bytes, num_actions A; uint8 class_of[256]; uint32 info[S] (bit 0
    whitespace, bit 1 accept, bits 8-15 need); uint32 actions[A] (bits 0-1 kind: 0 checked shift, 1 call, 2 return,
    3 return and reprocess; 2-16 target, 17-31 return state); uint16 trans[S, C] (0 fail, 1-0x7FFF a plain shift to
    that state, whose need is at most the source's, 0x8000 | a action a)."""

    def __init__(self, b: _Builder, start: int):
        self.start = start
        self.edges, self.ws, self.accept = b.edges, b.ws, b.accept
        S = len(self.edges)
        # need: min over completions of the peak extra stack height
        need = [_INF] * S
        for s in range(S):
            if self.accept[s]:
                need[s] = 0
        changed = True
        while changed:
            changed = False
            for s in range(S):
                best = need[s]
                for a in self.edges[s].values():
                    if a[0] in ("R", "P"):
                        n = 0
                    elif a[0] == "S":
                        n = need[a[1]]
                    else:
                        n = max(1 + need[a[1]], need[a[2]])
                    best = min(best, n)
                if best < need[s]:
                    need[s], changed = best, True
        self.need = [min(n, _INF) for n in need]
        if self.need[start] > SCHEMA_MAX_DEPTH:
            raise ValueError(f"JSON schema: no complete text fits the depth cap of {SCHEMA_MAX_DEPTH}")
        # a reprocessed byte is looked up in a return state, where it must not reprocess again
        for s in range(S):
            for a in self.edges[s].values():
                if a[0] == "C":
                    for b, a2 in self.edges[a[2]].items():
                        if a2[0] == "P":
                            raise ValueError("JSON schema: a return state reprocesses")
        # byte classes: bytes every state treats alike
        cols: dict = {}
        class_of = np.zeros(256, dtype=np.uint8)
        for byte in range(256):
            col = tuple(self.edges[s].get(byte) for s in range(S))
            class_of[byte] = cols.setdefault(col, len(cols))
        self.class_of = class_of
        C = len(cols)
        actions: dict = {}
        trans = np.zeros((S, C), dtype=np.uint16)
        for col, c in cols.items():
            for s, a in enumerate(col):
                if a is None:
                    continue
                if a[0] == "S" and self.need[a[1]] <= self.need[s]:
                    trans[s, c] = a[1]  # a plain shift: the need cannot grow, so the depth cap holds without a check
                    continue
                word = {"S": CHECKED_SHIFT, "C": CALL, "R": RETURN, "P": REPROCESS}[a[0]]
                if a[0] in ("S", "C"):
                    word |= a[1] << 2 | (a[2] << 17 if a[0] == "C" else 0)
                if word not in actions:
                    actions[word] = len(actions)
                    if len(actions) > SCHEMA_MAX_ACTIONS:
                        raise ValueError(f"JSON schema: the automaton exceeds {SCHEMA_MAX_ACTIONS} call and return entries")
                trans[s, c] = 0x8000 | actions[word]
        self.trans = trans
        self.actions = np.array(list(actions), dtype=np.uint32)
        info = np.array([(1 if self.ws[s] else 0) | (2 if self.accept[s] else 0) | (self.need[s] << 8) for s in range(S)], dtype=np.uint32)
        A = len(actions)
        nbytes = _HEADER_BYTES + 256 + 4 * S + 4 * A + 2 * S * C
        nbytes = (nbytes + 15) // 16 * 16
        if nbytes > SCHEMA_MAX_TABLE_BYTES:
            raise ValueError(f"JSON schema: the tables take {nbytes} bytes, above the limit of {SCHEMA_MAX_TABLE_BYTES}")
        blob = np.zeros(nbytes, dtype=np.uint8)
        blob[:16] = np.array([S, C, nbytes, A], dtype=np.int32).view(np.uint8)
        at = 16
        blob[at : at + 256] = class_of
        at += 256
        blob[at : at + 4 * S] = info.view(np.uint8)
        at += 4 * S
        blob[at : at + 4 * A] = self.actions.view(np.uint8)
        at += 4 * A
        blob[at : at + 2 * S * C] = trans.reshape(-1).view(np.uint8)
        self.blob = blob
        self._class_list = [int(c) for c in class_of]
        self._dec = [[self._decode(int(e)) for e in row] for row in trans]

    def _decode(self, e: int):
        if e == 0:
            return 0, 0, 0
        if not e & 0x8000:
            return 4, e, 0
        a = int(self.actions[e & 0x7FFF])
        if a & 3 == CHECKED_SHIFT:
            return 4, (a >> 2) & 0x7FFF, 0
        return a & 3, (a >> 2) & 0x7FFF, (a >> 17) & 0x7FFF

    @property
    def num_states(self) -> int:
        return len(self.edges)

    @property
    def num_classes(self) -> int:
        return int(self.trans.shape[1])

    def entry(self, s: int, b: int):
        """(kind, target, return) of the table entry at state ``s`` and byte ``b``: kind 0 fail, 4 shift (plain or
        checked: the walker checks the depth need of every shift, which a plain one always meets)."""
        return self._dec[s][self._class_list[b]]


def compile_schema(schema) -> CompiledSchema:
    """The pushdown automaton of ``schema`` (a dict, or its JSON text).  Raises ``ValueError`` naming the keyword and
    its JSON-pointer path for anything outside the supported subset (DESIGN.md section 21)."""
    if isinstance(schema, (str, bytes)):
        schema = json.loads(schema)
    b = _Builder(schema)
    root, path = b.resolve(schema, "#")
    types = root.get("type")
    if types not in ("object", ["object"]) or "anyOf" in root or "enum" in root or "const" in root:
        raise ValueError("JSON schema at #: the root must be an object schema (type: object)")
    b.check_keywords(root, path, {"type", "properties", "required", "additionalProperties"})
    start = b.object(root, path, root=True)
    b.finish()
    return CompiledSchema(b, start)


# -------------------------------------------------------------------------------------------------- walker --
class SchemaWalker:
    """One row's automaton state, mutable: ``state``, ``depth``, ``ws`` (whitespace run), ``stack`` (return states,
    bottom first) and ``terminal``; ``step`` and ``walk`` return False once the text leaves the language."""

    __slots__ = ("tables", "state", "depth", "ws", "stack", "terminal")

    def __init__(self, tables: CompiledSchema, words=None):
        self.tables = tables
        if words is None:
            self.state, self.depth, self.ws, self.stack, self.terminal = tables.start, 0, 0, [], False
            return
        w1 = int(words[1]) & (1 << 64) - 1
        self.state, self.depth, self.ws = w1 & 0x7FFF, (w1 >> 16) & 63, (w1 >> 24) & 63
        self.terminal = bool(w1 & _TERMINAL)
        self.stack = [(int(words[2 + k // 4]) >> (16 * (k % 4))) & 0xFFFF for k in range(self.depth)]

    def copy(self) -> SchemaWalker:
        w = SchemaWalker.__new__(SchemaWalker)
        w.tables, w.state, w.depth, w.ws, w.stack, w.terminal = self.tables, self.state, self.depth, self.ws, list(self.stack), self.terminal
        return w

    def words(self, tables_ptr: int) -> tuple:
        """The ``SCHEMA_STATE_WORDS`` int64 words of the device state (signed), with ``tables_ptr`` in word 0."""
        w = [tables_ptr, self.state | self.depth << 16 | self.ws << 24 | _ACTIVE | (_TERMINAL if self.terminal else 0)]
        w += [0] * (SCHEMA_STATE_WORDS - 2)
        for k, r in enumerate(self.stack):
            w[2 + k // 4] |= r << (16 * (k % 4))
        return tuple(x - (1 << 64) if x >= 1 << 63 else x for x in w)

    @property
    def complete(self) -> bool:
        return bool(self.tables.accept[self.state]) and self.depth == 0 and not self.terminal

    def step(self, b: int) -> bool:
        t = self.tables
        kind, target, ret = t.entry(self.state, b)
        if kind == REPROCESS:
            if self.depth == 0:
                return False
            self._pop()
            kind, target, ret = t.entry(self.state, b)
            if kind == REPROCESS:
                return False
        if kind == 0:
            return False
        if t.ws[self.state]:
            if b in _WS:
                if self.ws >= JSON_MAX_WS_RUN:
                    return False
                self.ws += 1
            else:
                self.ws = 0
        if kind == 4:
            if self.depth + t.need[target] > SCHEMA_MAX_DEPTH:
                return False
            self.state = target
        elif kind == CALL:
            if self.depth + 1 + t.need[target] > SCHEMA_MAX_DEPTH or self.depth + t.need[ret] > SCHEMA_MAX_DEPTH:
                return False
            self.stack.append(ret)
            self.depth += 1
            self.state = target
        else:  # RETURN
            if self.depth == 0:
                return False
            self._pop()
        return True

    def _pop(self) -> None:
        self.state = self.stack.pop()
        self.depth -= 1

    def walk(self, data: bytes) -> bool:
        if self.terminal or self.state == 0:
            return False
        for b in data:
            if not self.step(b):
                return False
        return True


# ------------------------------------------------------------------------------------------------ vocabulary --
def check_vocabulary(tables: CompiledSchema, vocabulary) -> None:
    """Refuse (``ValueError``) a vocabulary that could leave a reachable state with no allowed token: no EOS id, or no
    one-byte token for a byte the tables demand.  A byte is demanded when, without the bytes that have no one-byte
    token, some state can no longer complete within its depth need: then one-byte tokens alone always complete."""
    if not vocabulary.eos_ids:
        raise ValueError("JSON schema mode needs a vocabulary with an EOS id")
    singles = set()
    for tok in vocabulary.tokens:
        if tok is not None and len(tok) == 1:
            singles.add(tok[0])
    S = tables.num_states
    need = [_INF] * S
    for s in range(S):
        if tables.accept[s]:
            need[s] = 0
    changed = True
    while changed:
        changed = False
        for s in range(S):
            for byte, a in tables.edges[s].items():
                if byte not in singles:
                    continue
                if a[0] in ("R", "P"):
                    n = 0
                elif a[0] == "S":
                    n = need[a[1]]
                else:
                    n = max(1 + need[a[1]], need[a[2]])
                if n < need[s]:
                    need[s], changed = n, True
    missing = set()
    for s in range(S):
        if tables.need[s] < _INF and need[s] > tables.need[s]:
            for byte, a in tables.edges[s].items():
                if byte not in singles:
                    missing.add(byte)
    if missing:
        shown = "".join(chr(x) if 0x20 <= x < 0x7F else f"\\x{x:02x}" for x in sorted(missing))
        raise ValueError(f"JSON schema mode needs a one-byte token for {shown!r}: the schema can demand one of those bytes next")


class JsonSchemaConstraint:
    """A JSON Schema over one vocabulary: ``SamplingParams(constraint=JsonSchemaConstraint(schema, vocabulary))``.
    Compiles the schema once and holds the device tables (``tables``, uint8), the vocabulary's device CSR and its
    EOS-only mask row; the per-row state and mask buffers live with each caller's ``ConstraintRows``."""

    def __init__(self, schema, vocabulary, device="cuda"):
        self.schema = json.loads(schema) if isinstance(schema, (str, bytes)) else schema
        self.compiled = compile_schema(self.schema)
        check_vocabulary(self.compiled, vocabulary)
        self.vocabulary = vocabulary
        self.device = torch.device(device)
        self.tables = torch.from_numpy(self.compiled.blob.copy()).to(self.device)
        self.token_offsets, self.token_bytes = vocabulary.csr(self.device)
        W = (vocabulary.size + 31) // 32
        bits = np.zeros(W * 32, dtype=bool)
        bits[vocabulary.eos_ids] = True
        self.eos_row = torch.from_numpy(np.packbits(bits.reshape(W, 32), axis=1, bitorder="little").view(np.int32).reshape(W).copy()).to(self.device)
        self.dfa = _zero_dfa(self.device)
        self._eos = set(vocabulary.eos_ids)

    @property
    def vocab_size(self) -> int:
        return self.vocabulary.size

    def start(self) -> SchemaWalker:
        return SchemaWalker(self.compiled)

    def words(self, walker: SchemaWalker) -> tuple:
        return walker.words(self.tables.data_ptr())

    def walk(self, token_ids, walker: SchemaWalker | None = None) -> SchemaWalker | None:
        """The state after ``token_ids`` from ``walker`` (default: the start), or None when a token is not allowed."""
        w = self.start() if walker is None else walker.copy()
        for t in token_ids:
            t = int(t)
            if w.terminal:
                if t in self._eos:
                    continue
                return None
            if t in self._eos:
                if not w.complete:
                    return None
                w.terminal = True
                continue
            if not 0 <= t < self.vocab_size or self.vocabulary.tokens[t] is None or not w.walk(self.vocabulary.tokens[t]):
                return None
        return w

    def allowed(self, walker: SchemaWalker) -> np.ndarray:
        """bool ``[V]``: the tokens allowed after ``walker`` (what the device mask holds)."""
        out = np.zeros(self.vocab_size, dtype=bool)
        if walker.terminal:
            out[self.vocabulary.eos_ids] = True
            return out
        for i, t in enumerate(self.vocabulary.tokens):
            if t is None:
                out[i] = i in self._eos and walker.complete
            else:
                out[i] = walker.copy().walk(t)
        return out


def load_schema_arg(text: str):
    """A schema from a CLI argument: inline JSON when it starts with '{', else a file path."""
    if text.lstrip().startswith("{"):
        return json.loads(text)
    with open(text, encoding="utf-8") as f:
        return json.load(f)

