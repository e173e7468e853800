"""An independent Earley recognizer over bytes for the GBNF grammars of DESIGN.md section 23.

It shares only the parser's AST with the product (``tiny_llm_b200.grammar.parse_grammar``): the grammar is lowered to
plain BNF here (alternatives and repetitions become fresh nonterminals), and every character class is a terminal that
matches one whole UTF-8 character, decoded with Python's codec and checked against the class's code-point ranges, so
no byte automaton, byte class or call-chain construction of the product is reused.  The recognizer has no depth or
parse cap: it states the grammar's own language.

``Earley(text).check(data)`` -> ``(viable, complete)``: whether ``data`` is a prefix of some text of the language, and
whether it is one.  ``feed`` extends a state by one byte, for enumerations that share prefixes."""

from __future__ import annotations

import codecs

from tiny_llm_b200.grammar import parse_grammar

_LO = {1: 0, 2: 0x80, 3: 0x800, 4: 0x10000}
_HI = {1: 0x7F, 2: 0x7FF, 3: 0xFFFF, 4: 0x10FFFF}


def _char_length(lead: int):
    if lead < 0x80:
        return 1
    if 0xC0 <= lead < 0xE0:
        return 2
    if 0xE0 <= lead < 0xF0:
        return 3
    if 0xF0 <= lead < 0xF8:
        return 4
    return None


def _prefix_interval(buf: bytes):
    """The code points whose UTF-8 encoding starts with ``buf`` (a valid, incomplete prefix) as ``[lo, hi]`` pieces."""
    n = _char_length(buf[0])
    payload = buf[0] & (0x7F >> n if n > 1 else 0x7F)
    for b in buf[1:]:
        payload = payload << 6 | (b & 0x3F)
    rest = 6 * (n - len(buf))
    lo, hi = max(payload << rest, _LO[n]), min(payload << rest | ((1 << rest) - 1), _HI[n])
    pieces = []
    for a, b in ((lo, min(hi, 0xD7FF)), (max(lo, 0xE000), hi)):
        if a <= b:
            pieces.append((a, b))
    return pieces


def _valid_prefix(buf: bytes) -> bool:
    try:
        codecs.getincrementaldecoder("utf-8")().decode(buf, final=False)
    except UnicodeDecodeError:
        return False
    return True


class Earley:
    def __init__(self, text: str):
        rules = parse_grammar(text)
        self.prods: dict = {}  # nonterminal -> list of right-hand sides (tuples of symbols)
        self.fresh = 0
        for name, ast in rules.items():
            self.prods[("rule", name)] = [self.lower(ast)]
        self.start = ("start",)
        self.prods[self.start] = [(("N", ("rule", "root")),)]
        # productive nonterminals; unproductive right-hand sides are never predicted, so every live item can complete
        productive: set = set()
        changed = True
        while changed:
            changed = False
            for nt, rhss in self.prods.items():
                if nt not in productive and any(all(self.symbol_ok(s, productive) for s in rhs) for rhs in rhss):
                    productive.add(nt)
                    changed = True
        self.prods = {nt: [rhs for rhs in rhss if all(self.symbol_ok(s, productive) for s in rhs)] for nt, rhss in self.prods.items()}
        nullable: set = set()
        changed = True
        while changed:
            changed = False
            for nt, rhss in self.prods.items():
                if nt not in nullable and any(all(s[0] == "N" and s[1] in nullable for s in rhs) for rhs in rhss):
                    nullable.add(nt)
                    changed = True
        self.nullable = nullable

    @staticmethod
    def symbol_ok(s, productive) -> bool:
        return bool(s[1]) if s[0] == "T" else s[1] in productive

    def new(self, rhss) -> tuple:
        self.fresh += 1
        nt = ("fresh", self.fresh)
        self.prods[nt] = rhss
        return ("N", nt)

    def lower(self, node) -> tuple:
        kind = node[0]
        if kind == "set":
            return (("T", tuple(node[1])),)
        if kind == "ref":
            return (("N", ("rule", node[1])),)
        if kind == "cat":
            return tuple(s for item in node[1] for s in self.lower(item))
        if kind == "alt":
            return (self.new([self.lower(item) for item in node[1]]),)
        _, sub, lo, hi = node
        body = self.lower(sub)
        out = body * lo
        if hi is None:
            self.fresh += 1
            star = ("fresh", self.fresh)
            self.prods[star] = [body + (("N", star),), ()]
            return out + (("N", star),)
        tail: tuple = ()
        for _ in range(hi - lo):
            tail = (self.new([body + tail, ()]),)
        return out + tail

    # ---------------------------------------------------------------------------------------------- recognizer --
    def close(self, sets: list, items: set) -> frozenset:
        """Predict and complete over ``items`` (the set at position len(sets))."""
        i = len(sets)
        todo = list(items)
        while todo:
            item = todo.pop()
            nt, alt, dot, origin, partial = item
            rhs = self.prods[nt][alt]
            new = []
            if dot < len(rhs):
                sym = rhs[dot]
                if sym[0] == "N" and not partial:
                    for a in range(len(self.prods[sym[1]])):
                        new.append((sym[1], a, 0, i, b""))
                    if sym[1] in self.nullable:
                        new.append((nt, alt, dot + 1, origin, b""))
            else:
                src = items if origin == i else sets[origin]
                for p in list(src):
                    pnt, palt, pdot, porigin, ppartial = p
                    prhs = self.prods[pnt][palt]
                    if not ppartial and pdot < len(prhs) and prhs[pdot] == ("N", nt):
                        new.append((pnt, palt, pdot + 1, porigin, b""))
            for n in new:
                if n not in items:
                    items.add(n)
                    todo.append(n)
        return frozenset(items)

    def initial(self) -> list:
        return [self.close([], {(self.start, 0, 0, 0, b"")})]

    def feed(self, sets: list, byte: int) -> list:
        """The sets after one more byte (the last set empty: not a viable prefix)."""
        nxt = set()
        for nt, alt, dot, origin, partial in sets[-1]:
            rhs = self.prods[nt][alt]
            if dot == len(rhs) or rhs[dot][0] != "T":
                continue
            buf = partial + bytes([byte])
            n = _char_length(buf[0])
            if n is None or not _valid_prefix(buf):
                continue
            ranges = rhs[dot][1]
            if len(buf) == n:
                cp = ord(buf.decode("utf-8"))
                if any(lo <= cp <= hi for lo, hi in ranges):
                    nxt.add((nt, alt, dot + 1, origin, b""))
            elif any(a <= hi and lo <= b for a, b in _prefix_interval(buf) for lo, hi in ranges):
                nxt.add((nt, alt, dot, origin, buf))
        return sets + [self.close(sets, nxt)]

    def viable(self, sets: list) -> bool:
        return bool(sets[-1])

    def complete(self, sets: list) -> bool:
        return (self.start, 0, 1, 0, b"") in sets[-1]

    def check(self, data: bytes) -> tuple[bool, bool]:
        sets = self.initial()
        for b in data:
            sets = self.feed(sets, b)
            if not sets[-1]:
                return False, False
        return True, self.complete(sets)
