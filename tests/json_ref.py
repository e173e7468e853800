"""An independent reference of JSON mode's language (DESIGN.md section 20): a recursive-descent parser over bytes that
tells a complete text from a viable prefix (one a complete text extends) and from a dead one, and builds a completion
witness for a viable prefix.  It re-parses the whole text on every call: slow, and written apart from the package's
packed-state walker on purpose."""

from __future__ import annotations

import numpy as np

MAX_DEPTH = 64
MAX_WS_RUN = 32
_WS = b" \t\n\r"
_DIGITS = b"0123456789"
_HEX = b"0123456789abcdefABCDEF"


class _Eof(Exception):
    pass


class _Bad(Exception):
    pass


class _Parser:
    def __init__(self, data: bytes):
        self.d, self.i = data, 0
        self.pending: list[bytes] = []  # what closes each open construct, outermost first

    def peek(self) -> int:
        if self.i >= len(self.d):
            raise _Eof
        return self.d[self.i]

    def take(self) -> int:
        b = self.peek()
        self.i += 1
        return b

    def expect(self, b: int) -> None:
        if self.take() != b:
            raise _Bad

    def ws(self) -> None:
        n = 0
        while self.i < len(self.d) and self.d[self.i] in _WS:
            n += 1
            self.i += 1
            if n > MAX_WS_RUN:
                raise _Bad

    def text(self) -> None:
        self.pending.append(b"{}")
        self.ws()
        if self.peek() != ord("{"):
            raise _Bad
        self.pending[-1] = b""
        self.obj(1)
        self.ws()
        if self.i < len(self.d):
            raise _Bad

    def value(self, depth: int, after: bytes) -> None:
        """A value inside a container whose closer, once the value has begun, is ``after``."""
        b = self.peek()
        self.pending[-1] = after
        if b == ord("{"):
            self.obj(depth + 1)
        elif b == ord("["):
            self.arr(depth + 1)
        elif b == ord('"'):
            self.string()
        elif b == ord("-") or b in _DIGITS:
            self.number()
        elif b in b"tfn":
            self.literal({ord("t"): b"true", ord("f"): b"false", ord("n"): b"null"}[b])
        else:
            raise _Bad

    def obj(self, depth: int) -> None:
        if depth > MAX_DEPTH:
            raise _Bad
        self.expect(ord("{"))
        self.pending.append(b"}")
        self.ws()
        if self.peek() == ord("}"):
            self.i += 1
            self.pending.pop()
            return
        while True:
            if self.peek() != ord('"'):
                raise _Bad
            self.pending[-1] = b":0}"
            self.string()
            self.ws()
            self.expect(ord(":"))
            self.pending[-1] = b"0}"
            self.ws()
            self.value(depth, b"}")
            self.ws()
            b = self.take()
            if b == ord("}"):
                self.pending.pop()
                return
            if b != ord(","):
                raise _Bad
            self.pending[-1] = b'"":0}'
            self.ws()

    def arr(self, depth: int) -> None:
        if depth > MAX_DEPTH:
            raise _Bad
        self.expect(ord("["))
        self.pending.append(b"]")
        self.ws()
        if self.peek() == ord("]"):
            self.i += 1
            self.pending.pop()
            return
        while True:
            self.pending[-1] = b"0]"
            self.value(depth, b"]")
            self.ws()
            b = self.take()
            if b == ord("]"):
                self.pending.pop()
                return
            if b != ord(","):
                raise _Bad
            self.pending[-1] = b"0]"
            self.ws()

    def string(self) -> None:
        self.expect(ord('"'))
        self.pending.append(b'"')
        while True:
            b = self.take()
            if b == ord('"'):
                self.pending.pop()
                return
            if b == ord("\\"):
                self.pending.append(b"n")
                e = self.take()
                if e == ord("u"):
                    for k in range(4):
                        self.pending[-1] = b"0" * (4 - k)
                        if self.take() not in _HEX:
                            raise _Bad
                elif e not in b'"\\/bfnrt':
                    raise _Bad
                self.pending.pop()
            elif b < 0x20:
                raise _Bad
            elif b >= 0x80:
                self.utf8(b)

    def utf8(self, lead: int) -> None:
        # the well-formed sequences of the Unicode standard, table 3-7
        if 0xC2 <= lead <= 0xDF:
            ranges = [(0x80, 0xBF)]
        elif lead == 0xE0:
            ranges = [(0xA0, 0xBF), (0x80, 0xBF)]
        elif 0xE1 <= lead <= 0xEC or 0xEE <= lead <= 0xEF:
            ranges = [(0x80, 0xBF)] * 2
        elif lead == 0xED:
            ranges = [(0x80, 0x9F), (0x80, 0xBF)]
        elif lead == 0xF0:
            ranges = [(0x90, 0xBF), (0x80, 0xBF), (0x80, 0xBF)]
        elif 0xF1 <= lead <= 0xF3:
            ranges = [(0x80, 0xBF)] * 3
        elif lead == 0xF4:
            ranges = [(0x80, 0x8F), (0x80, 0xBF), (0x80, 0xBF)]
        else:
            raise _Bad
        self.pending.append(b"")
        for k, (lo, hi) in enumerate(ranges):
            self.pending[-1] = bytes(r[0] for r in ranges[k:])
            if not lo <= self.take() <= hi:
                raise _Bad
        self.pending.pop()

    def digits(self, need: bool) -> None:
        """One or more digits (``need``) or zero or more; at the end of the text a number may stop anywhere it could."""
        if need:
            self.pending.append(b"0")
            if self.take() not in _DIGITS:
                raise _Bad
            self.pending.pop()
        while self.i < len(self.d) and self.d[self.i] in _DIGITS:
            self.i += 1

    def number(self) -> None:
        if self.peek() == ord("-"):
            self.i += 1
        self.pending.append(b"0")
        b = self.take()
        self.pending.pop()
        if b not in _DIGITS:
            raise _Bad
        if b != ord("0"):
            self.digits(False)
        if self.i < len(self.d) and self.d[self.i] == ord("."):
            self.i += 1
            self.digits(True)
        if self.i < len(self.d) and self.d[self.i] in b"eE":
            self.i += 1
            if self.i < len(self.d) and self.d[self.i] in b"+-":
                self.i += 1
            self.digits(True)
        if self.i >= len(self.d):
            raise _Eof  # the number may still go on

    def literal(self, word: bytes) -> None:
        for k, c in enumerate(word):
            self.pending.append(word[k:])
            if self.take() != c:
                raise _Bad
            self.pending.pop()


def classify(data: bytes) -> str:
    """"complete", "prefix" (viable, not complete) or "dead"."""
    p = _Parser(bytes(data))
    try:
        p.text()
    except _Eof:
        return "prefix"
    except _Bad:
        return "dead"
    return "complete"


def viable(data: bytes) -> bool:
    return classify(data) != "dead"


def witness(data: bytes) -> bytes | None:
    """A complete text that extends ``data`` (None when ``data`` is dead)."""
    p = _Parser(bytes(data))
    try:
        p.text()
    except _Eof:
        return bytes(data) + b"".join(reversed(p.pending))
    except _Bad:
        return None
    return bytes(data)


def caps_hold(data: bytes) -> bool:
    """Both caps, checked on a text ``json.loads`` accepts: whitespace runs outside strings and nesting depth."""
    depth = run = 0
    in_str = esc = False
    for b in data:
        if in_str:
            if esc:
                esc = False
            elif b == ord("\\"):
                esc = True
            elif b == ord('"'):
                in_str = False
            continue
        if b in _WS:
            run += 1
            if run > MAX_WS_RUN:
                return False
            continue
        run = 0
        if b == ord('"'):
            in_str = True
        elif b in b"{[":
            depth += 1
            if depth > MAX_DEPTH:
                return False
        elif b in b"}]":
            depth -= 1
    return True


def allowed(text: bytes, tokens, eos_ids, terminal: bool = False) -> np.ndarray:
    """bool ``[V]``: the tokens allowed after ``text`` (``terminal``: after EOS, only EOS)."""
    out = np.zeros(len(tokens), dtype=bool)
    eos = set(eos_ids)
    if terminal:
        out[list(eos)] = True
        return out
    done = classify(text) == "complete"
    for i, t in enumerate(tokens):
        if t is None:
            out[i] = i in eos and done
        else:
            out[i] = viable(text + t)
    return out


def pack(bits: np.ndarray) -> np.ndarray:
    """bool ``[..., V]`` -> int32 ``[..., ceil(V / 32)]`` mask words (bit t of word t // 32)."""
    V = bits.shape[-1]
    W = (V + 31) // 32
    pad = np.zeros(bits.shape[:-1] + (W * 32,), dtype=bool)
    pad[..., :V] = bits
    return np.packbits(pad.reshape(bits.shape[:-1] + (W, 32)), axis=-1, bitorder="little").view(np.int32).reshape(bits.shape[:-1] + (W,))
