"""An independent reference for the JSON Schema language (DESIGN.md section 21): recursive descent over the schema and
the text, written from the language's definition and sharing no code with ``tiny_llm_b200/json_schema.py``.

A text is complete when it is ``ws object ws`` by RFC 8259 with at most 32 whitespace bytes in a row between grammar
tokens, its value validates against the schema with every object's keys in the order ``properties`` lists them (each
at most once, no others), every ``enum`` / ``const`` value is written the way ``json.dumps(v, ensure_ascii=False)``
writes it, every ``integer`` is ``-?(0|[1-9][0-9]*)``, a ``pattern`` string's raw bytes (no escapes) fullmatch the
pattern, and no value sits more than 32 levels below the root object (the root object's members are at level 1).
A prefix is viable when some completion is complete; ``check`` returns one (the witness), built from the fewest
levels.  Patterns here are sequences of literal characters, ``[...]`` classes and ``\\d``, each with an optional
``{m}``, ``{m,n}``, ``?``, ``*`` or ``+``."""

from __future__ import annotations

import json
import re

MAX_LEVEL = 32
MAX_WS = 32
_WS = b" \t\n\r"
_NUM_CHARS = b"0123456789+-.eE"
_NUMBER = rb"-?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?"
_INTEGER = rb"-?(0|[1-9][0-9]*)"


class Reject(Exception):
    pass


class Incomplete(Exception):
    """The text ended inside a construct that can still complete; ``tail`` completes it and every enclosing one
    unwound so far."""

    def __init__(self, tail: bytes):
        self.tail = tail


def _dumps(v) -> bytes:
    return json.dumps(v, ensure_ascii=False).encode()


class Ref:
    def __init__(self, schema):
        self.root = schema
        self._min: dict = {}

    # ------------------------------------------------------------------------------------------- schema view --
    def deref(self, s):
        while isinstance(s, dict) and "$ref" in s:
            ref = s["$ref"]
            s = self.root
            if ref != "#":
                for part in ref[2:].split("/"):
                    s = s[part]
        return {} if s is True else s

    def branches(self, s):
        """The alternatives of schema ``s`` as (kind, schema) pairs; kind is a JSON type name or 'enum'."""
        s = self.deref(s)
        if "anyOf" in s:
            return [b for x in s["anyOf"] for b in self.branches(x)]
        if "enum" in s or "const" in s:
            values = [s["const"]] if "const" in s else s["enum"]
            types = s.get("type")
            if types is not None:
                types = [types] if isinstance(types, str) else types
                values = [v for v in values if _type_of(v) in types or (_type_of(v) == "integer" and "number" in types)]
            return [("enum", values)]
        t = s.get("type")
        if t is None:
            return [(k, {"type": k}) for k in ("object", "array", "string", "number", "boolean", "null")]
        if isinstance(t, list):
            return [(k, dict(s, type=k)) for k in t]
        return [(t, s)]

    def min_levels(self, s) -> int:
        """The fewest levels below a value of ``s`` that a complete value of it needs (255: no finite value)."""
        key = json.dumps(s, sort_keys=True)
        if key not in self._min:
            self._min[key] = 255
            for _ in range(MAX_LEVEL + 2):  # recursive schemas: iterate to the fixed point
                best = 255
                for kind, b in self.branches(s):
                    if kind == "object":
                        props, req = b.get("properties") or {}, b.get("required", [])
                        best = min(best, max([0] + [1 + self.min_levels(props[r]) for r in req]))
                    elif kind == "array":
                        best = min(best, 0 if b.get("minItems", 0) == 0 else 1 + self.min_levels(b.get("items", {})))
                    else:
                        best = 0
                if min(best, 255) == self._min[key]:
                    break
                self._min[key] = min(best, 255)
        return self._min[key]

    def witness(self, s, level: int) -> bytes:
        """A complete value of ``s`` at ``level`` with the fewest levels below it (Reject: none within the cap)."""
        best = None
        for kind, b in self.branches(s):
            if kind == "object":
                props, req = b.get("properties") or {}, b.get("required", [])
                need = max([0] + [1 + self.min_levels(props[r]) for r in req])
            elif kind == "array":
                need = 0 if b.get("minItems", 0) == 0 else 1 + self.min_levels(b.get("items", {}))
            else:
                need = 0
            if need < 255 and (best is None or need < best[0]):
                best = (need, kind, b)
        if best is None or level + best[0] > MAX_LEVEL:
            raise Reject
        _, kind, b = best
        if kind == "object":
            props, req = b.get("properties") or {}, b.get("required", [])
            return b"{" + b",".join(_dumps(n) + b":" + self.witness(props[n], level + 1) for n in props if n in req) + b"}"
        if kind == "array":
            return b"[" + b",".join(self.witness(b.get("items", {}), level + 1) for _ in range(b.get("minItems", 0))) + b"]"
        if kind == "enum":
            return _dumps(b[0])
        if kind == "string":
            return b'"' + (_pattern_witness(b["pattern"], "") or "").encode() + b'"' if "pattern" in b else b'""'
        return {"number": b"0", "integer": b"0", "boolean": b"true", "null": b"null"}[kind]

    # -------------------------------------------------------------------------------------------------- text --
    def ws(self, t: bytes, i: int) -> int:
        j = i
        while j < len(t) and t[j] in _WS:
            j += 1
        if j - i > MAX_WS:
            raise Reject
        return j

    def value(self, s, t: bytes, i: int, level: int) -> int:
        if level > MAX_LEVEL:
            raise Reject
        if i == len(t):
            raise Incomplete(self.witness(s, level))
        c = t[i]
        for kind, b in self.branches(s):
            if kind == "enum" and any(_dumps(v)[0] == c for v in b):
                return self.enum(b, t, i)
            if kind == "object" and c == 0x7B:
                props, req = b.get("properties") or {}, b.get("required", [])
                if level + max([0] + [1 + self.min_levels(props[r]) for r in req]) > MAX_LEVEL:
                    raise Reject
                return self.obj(b, t, i, level)
            if kind == "array" and c == 0x5B:
                if b.get("minItems", 0) and level + 1 + self.min_levels(b.get("items", {})) > MAX_LEVEL:
                    raise Reject
                return self.arr(b, t, i, level)
            if kind == "string" and c == 0x22:
                return self.string(t, i, b.get("pattern"))
            if kind in ("number", "integer") and c in b"-0123456789":
                return self.number(t, i, kind == "integer")
            if kind == "boolean" and c in b"tf":
                return self.enum([True, False], t, i)
            if kind == "null" and c == 0x6E:
                return self.enum([None], t, i)
        raise Reject

    def enum(self, values, t: bytes, i: int) -> int:
        forms = [_dumps(v) for v in values]
        rest = t[i:]
        full = [f for f in forms if rest.startswith(f)
                and (f[0] not in b"-0123456789" or len(rest) == len(f) or rest[len(f)] not in _NUM_CHARS)]
        if full:
            return i + len(max(full, key=len))
        partial = [f for f in forms if len(f) > len(rest) and f.startswith(rest)]
        if partial:
            raise Incomplete(min(partial, key=len)[len(rest):])
        raise Reject

    def number(self, t: bytes, i: int, integer: bool) -> int:
        pat = _INTEGER if integer else _NUMBER
        j = i
        while j < len(t) and t[j] in _NUM_CHARS:
            j += 1
        if re.fullmatch(pat, t[i:j]):
            return j
        if j == len(t) and re.fullmatch(pat, t[i:j] + b"0"):
            raise Incomplete(b"0")
        raise Reject

    def string(self, t: bytes, i: int, pattern) -> int:
        j = i + 1
        while j < len(t) and t[j] != 0x22:
            if t[j] == 0x5C:
                if pattern is not None:
                    raise Reject
                j += 1
            j += 1
        body = t[i + 1 : min(j, len(t))]
        ok = _valid_content(body)
        if ok is False:
            raise Reject
        if j >= len(t):  # no closing quote yet
            if pattern is None:
                raise Incomplete(_string_tail(body))
            try:
                text = body.decode()
            except UnicodeDecodeError:
                raise Reject from None
            w = _pattern_witness(pattern, text)
            if w is None:
                raise Reject
            return self._incomplete(w[len(text):].encode() + b'"')
        if ok is not True:
            raise Reject
        if pattern is not None and _pattern_witness(pattern, body.decode(), extend=False) is None:
            raise Reject
        return j + 1

    @staticmethod
    def _incomplete(tail: bytes):
        raise Incomplete(tail)

    def obj(self, s, t: bytes, i: int, level: int) -> int:
        props = s.get("properties")
        req = s.get("required", [])
        free = props is None and s.get("additionalProperties") is not False and not req
        names = [] if free else list(props or {})
        done = -1  # index in names of the last member
        count = 0
        i += 1

        def rest(after: int) -> bytes:  # what follows a complete member ``after`` (-1: none yet, after "{")
            out = [n for n in names[after + 1:] if n in req]
            body = b",".join(_dumps(n) + b":" + self.witness(props[n], level + 1) for n in out)
            return (b"," if count and body else b"") + body + b"}"

        while True:
            i = self.ws(t, i)
            if i == len(t):
                raise Incomplete(rest(done))
            can_close = free or not any(n in req for n in names[done + 1:])
            if t[i] == 0x7D and can_close:
                return i + 1
            if count:
                if t[i] != 0x2C:
                    raise Reject
                i = self.ws(t, i + 1)
            allowed = None if free else _allowed(names, req, done)
            if allowed == []:
                raise Reject
            if i == len(t):  # after a comma: a member must follow
                if free:
                    raise Incomplete(b'"":' + self.witness({}, level + 1) + b"}")
                n = self._first_fit(props, allowed, level)
                raise Incomplete(_dumps(n) + b":" + self.witness(props[n], level + 1) + self._after(names, req, props, n, level))
            if t[i] != 0x22:
                raise Reject
            # the key
            if free:
                try:
                    j = self.string(t, i, None)
                except Incomplete as inc:
                    raise Incomplete(inc.tail + b":" + self.witness({}, level + 1) + b"}") from None
                name, child = None, {}
            else:
                name = None
                for n in allowed:
                    f = _dumps(n)
                    if t.startswith(f, i):
                        name = n
                        break
                if name is None:
                    part = t[i:]
                    for n in allowed:
                        f = _dumps(n)
                        if len(f) > len(part) and f.startswith(part):
                            try:
                                tail = f[len(part):] + b":" + self.witness(props[n], level + 1) + self._after(names, req, props, n, level)
                            except Reject:
                                continue
                            raise Incomplete(tail)
                    raise Reject
                j = i + len(_dumps(name))
                child = props[name]
            after = b"}" if free else self._after(names, req, props, name, level)
            i = self.ws(t, j)
            if i == len(t):
                raise Incomplete(b":" + self.witness(child, level + 1) + after)
            if t[i] != 0x3A:
                raise Reject
            i = self.ws(t, i + 1)
            try:
                i = self.value(child, t, i, level + 1)
            except Incomplete as inc:
                raise Incomplete(inc.tail + after) from None
            if not free:
                done = names.index(name)
            count += 1

    def _after(self, names, req, props, name, level) -> bytes:
        k = names.index(name)
        return b"".join(b"," + _dumps(n) + b":" + self.witness(props[n], level + 1) for n in names[k + 1:] if n in req) + b"}"

    def _first_fit(self, props, allowed, level):
        for n in allowed:
            try:
                self.witness(props[n], level + 1)
                return n
            except Reject:
                continue
        raise Reject

    def arr(self, s, t: bytes, i: int, level: int) -> int:
        lo, hi = s.get("minItems", 0), s.get("maxItems")
        items = s.get("items", {})

        def rest(n: int) -> bytes:  # after n complete items
            more = [self.witness(items, level + 1) for _ in range(max(0, lo - n))]
            return b"".join((b"," if n or k else b"") + w for k, w in enumerate(more)) + b"]"

        n = 0
        i += 1
        while True:
            i = self.ws(t, i)
            if i == len(t):
                raise Incomplete(rest(n))
            if t[i] == 0x5D and n >= lo:
                return i + 1
            if n:
                if t[i] != 0x2C or (hi is not None and n >= hi):
                    raise Reject
                i = self.ws(t, i + 1)
            elif hi == 0:
                raise Reject
            try:
                i = self.value(items, t, i, level + 1)
            except Incomplete as inc:
                raise Incomplete(inc.tail + rest(n + 1)) from None
            n += 1

    def document(self, t: bytes) -> int:
        i = self.ws(t, 0)
        if i == len(t):
            raise Incomplete(self.witness(self.root, 0))
        if t[i] != 0x7B:
            raise Reject
        i = self.obj(self.deref(self.root), t, i, 0)
        return self.ws(t, i)


def check(schema, text: bytes):
    """``(viable, complete, witness)``: ``text + witness`` is complete when ``viable`` (witness b"" when complete)."""
    ref = Ref(schema)
    try:
        j = ref.document(text)
    except Reject:
        return False, False, None
    except Incomplete as inc:
        return True, False, inc.tail
    if j != len(text):
        return False, False, None
    return True, True, b""


def _allowed(names, req, done):
    out = []
    for n in names[done + 1:]:
        out.append(n)
        if n in req:
            break
    return out


def _type_of(v) -> str:
    return {type(None): "null", bool: "boolean", str: "string", int: "integer", float: "number"}[type(v)]


def _utf8_len(b: int) -> int:
    return 2 if 0xC2 <= b <= 0xDF else 3 if 0xE0 <= b <= 0xEF else 4 if 0xF0 <= b <= 0xF4 else 0


def _valid_content(raw: bytes):
    """True: a complete string body; None: a viable prefix of one; False: neither."""
    i = 0
    while i < len(raw):
        b = raw[i]
        if b == 0x5C:
            if i + 1 == len(raw):
                return None
            e = raw[i + 1]
            if e == ord("u"):
                h = raw[i + 2 : i + 6]
                if not re.fullmatch(rb"[0-9a-fA-F]*", h):
                    return False
                if len(h) < 4:
                    return None
                i += 6
                continue
            if e not in b'"\\/bfnrt':
                return False
            i += 2
            continue
        if b == 0x22 or b < 0x20:
            return False
        if b < 0x80:
            i += 1
            continue
        n = _utf8_len(b)
        if not n:
            return False
        seq = raw[i : i + n]
        if len(seq) < n:
            return None if _utf8_tail(seq) is not None else False
        try:
            seq.decode("utf-8")
        except UnicodeDecodeError:
            return False
        i += n
    return True


def _utf8_tail(head: bytes):
    """Continuation bytes that complete the UTF-8 character ``head`` starts, or None."""
    need = _utf8_len(head[0]) - len(head)
    for a in range(0x80, 0xC0):
        tail = bytes([a]) + b"\x80" * (need - 1)
        try:
            (head + tail).decode("utf-8")
            return tail
        except UnicodeDecodeError:
            continue
    return None


def _string_tail(body: bytes) -> bytes:
    """Bytes that close a viable string body."""
    m = re.search(rb"(\\+)(u[0-9a-fA-F]{0,3})?$", body)
    if m and len(m.group(1)) % 2:
        return (b"n" if m.group(2) is None else b"0" * (5 - len(m.group(2)))) + b'"'
    for k in range(1, 4):
        if k <= len(body) and _utf8_len(body[-k]) > k and all(0x80 <= c <= 0xBF for c in body[len(body) - k + 1:]):
            return _utf8_tail(body[-k:]) + b'"'
    return b'"'


# ---------------------------------------------------------------------------------------------------- patterns --
def _pattern_atoms(pattern: str):
    """[(set of characters, lo, hi or None)] of ``^...$``."""
    inner = pattern[1:-1]
    atoms, k = [], 0
    while k < len(inner):
        c = inner[k]
        if c == "[":
            end = inner.index("]", k + 1)
            body, chars = inner[k + 1 : end], set()
            j = 0
            while j < len(body):
                if j + 2 < len(body) and body[j + 1] == "-":
                    chars |= {chr(x) for x in range(ord(body[j]), ord(body[j + 2]) + 1)}
                    j += 3
                else:
                    chars.add(body[j])
                    j += 1
            k = end + 1
        elif c == "\\":
            chars = set("0123456789") if inner[k + 1] == "d" else {inner[k + 1]}
            k += 2
        else:
            chars = {c}
            k += 1
        lo, hi = 1, 1
        if k < len(inner) and inner[k] in "?*+{":
            q = inner[k]
            if q == "{":
                end = inner.index("}", k)
                parts = inner[k + 1 : end].split(",")
                lo = int(parts[0])
                hi = lo if len(parts) == 1 else (int(parts[1]) if parts[1] else None)
                k = end + 1
            else:
                lo, hi = {"?": (0, 1), "*": (0, None), "+": (1, None)}[q]
                k += 1
        atoms.append((chars, lo, hi))
    return atoms


def _pattern_witness(pattern: str, text: str, extend: bool = True):
    """The shortest extension of ``text`` that matches ``pattern`` (``extend=False``: ``text`` itself), or None."""
    atoms = _pattern_atoms(pattern)

    def go(a: int, pos: int):
        if pos == len(text):
            if not extend and a < len(atoms) and any(lo for _, lo, _ in atoms[a:]):
                return None
            return "".join(min(ch) * lo for ch, lo, _ in atoms[a:])
        if a == len(atoms):
            return None
        chars, lo, hi = atoms[a]
        n = 0
        while True:  # try every count of this atom that the text allows
            if n >= lo:
                r = go(a + 1, pos + n)
                if r is not None:
                    return r
            if pos + n == len(text):
                if n < lo and extend:
                    return "".join(min(chars) for _ in range(lo - n)) + "".join(min(ch) * l for ch, l, _ in atoms[a + 1:])
                return None
            if (hi is not None and n >= hi) or text[pos + n] not in chars:
                return None
            n += 1

    r = go(0, 0)
    return None if r is None else text + r
