"""Regex-constrained generation (DESIGN.md section 8c).

A pattern compiles to a DFA over the UTF-8 bytes of the generated text: parse, Thompson NFA, subset construction, then
trim to the live states (those from which an accepting state is reachable).  The language is that of
``re.fullmatch(pattern, text, re.ASCII)``; anchors, backreferences, lookaround and inline flags are refused.

``TokenConstraint.compile(pattern, vocabulary)`` lifts the DFA to tokens on the GPU (``tl_constraint_token_masks``):
token ``t`` is allowed in state ``s`` iff walking its bytes from ``s`` stays in live states, an EOS id iff ``s``
accepts.  EOS leads to a terminal state ``S`` in which only EOS is allowed.  The sampling kernel
(``tl_sample_constrained``) reads one 40-byte descriptor per row (masks, DFA, vocabulary CSR, current state), draws
an allowed token and advances the state on the device, so decode graphs run constrained without host reads."""

from __future__ import annotations

import numpy as np
import torch

MAX_STATES = 4096  # DFA states a pattern may compile to
MAX_REPEAT = 1000  # bound of a counted repetition {m,n}
_MAX_CP = 0x10FFFF

# ------------------------------------------------------------------------------------------------------ parsing --
# AST: ("set", ranges) | ("cat", [nodes]) | ("alt", [nodes]) | ("rep", node, lo, hi or None).  A set is a sorted list
# of disjoint inclusive code-point ranges.

_DIGIT = [(0x30, 0x39)]
_WORD = [(0x30, 0x39), (0x41, 0x5A), (0x5F, 0x5F), (0x61, 0x7A)]
_SPACE = [(0x09, 0x0D), (0x20, 0x20)]
_CLASS_ESCAPES = {"d": (_DIGIT, False), "w": (_WORD, False), "s": (_SPACE, False),
                  "D": (_DIGIT, True), "W": (_WORD, True), "S": (_SPACE, True)}
_CHAR_ESCAPES = {"n": 0x0A, "t": 0x09, "r": 0x0D, "f": 0x0C, "v": 0x0B, "a": 0x07}


def _normalize(ranges):
    out = []
    for lo, hi in sorted(ranges):
        if out and lo <= out[-1][1] + 1:
            out[-1] = (out[-1][0], max(out[-1][1], hi))
        else:
            out.append((lo, hi))
    return out


def _complement(ranges):
    out, nxt = [], 0
    for lo, hi in _normalize(ranges):
        if lo > nxt:
            out.append((nxt, lo - 1))
        nxt = hi + 1
    if nxt <= _MAX_CP:
        out.append((nxt, _MAX_CP))
    return out


class _Parser:
    def __init__(self, pattern: str):
        self.p, self.i = pattern, 0

    def error(self, what: str):
        return ValueError(f"regex {self.p!r}: {what} at position {self.i}")

    def peek(self, k: int = 0):
        j = self.i + k
        return self.p[j] if j < len(self.p) else None

    def parse(self):
        node = self.alternation()
        if self.i < len(self.p):
            raise self.error("unbalanced parenthesis")
        return node

    def alternation(self):
        branches = [self.sequence()]
        while self.peek() == "|":
            self.i += 1
            branches.append(self.sequence())
        return branches[0] if len(branches) == 1 else ("alt", branches)

    def sequence(self):
        items = []
        while self.peek() is not None and self.peek() not in "|)":
            atom = self.atom()
            items.append(self.quantified(atom))
        return ("cat", items)

    def quantified(self, atom):
        q = self.quantifier()
        if q is None:
            return atom
        if self.peek() == "?":  # lazy: the same language under fullmatch
            self.i += 1
        elif self.peek() == "+":
            raise self.error("possessive quantifiers are not supported")
        if self.quantifier(probe=True):
            raise self.error("multiple repeat")
        return ("rep", atom, *q)

    def quantifier(self, probe: bool = False):
        c, start = self.peek(), self.i
        if c in ("*", "+", "?"):
            if not probe:
                self.i += 1
            return {"*": (0, None), "+": (1, None), "?": (0, 1)}[c]
        if c != "{" or self.peek(1) == "}":
            return None
        j = self.i + 1
        lo = hi = ""
        while j < len(self.p) and self.p[j].isdigit():
            lo += self.p[j]
            j += 1
        comma = j < len(self.p) and self.p[j] == ","
        if comma:
            j += 1
            while j < len(self.p) and self.p[j].isdigit():
                hi += self.p[j]
                j += 1
        if j >= len(self.p) or self.p[j] != "}":
            return None  # not a quantifier: '{' is a literal, as in re
        if probe:
            return True
        self.i = j + 1
        m = int(lo) if lo else 0
        n = (int(hi) if hi else None) if comma else m
        if n is not None and n < m:
            self.i = start
            raise self.error("min repeat greater than max repeat")
        if m > MAX_REPEAT or (n is not None and n > MAX_REPEAT):
            self.i = start
            raise self.error(f"repeat counts above {MAX_REPEAT} are not supported")
        return (m, n)

    def atom(self):
        c = self.peek()
        if c in ("*", "+", "?") or (c == "{" and self.quantifier(probe=True)):
            raise self.error("nothing to repeat")
        if c == "(":
            return self.group()
        if c == "[":
            return ("set", self.char_class())
        if c == ".":
            self.i += 1
            return ("set", _complement([(0x0A, 0x0A)]))
        if c in ("^", "$"):
            raise self.error(f"anchor {c!r} is not supported")
        if c == "\\":
            return ("set", self.escape(in_class=False))
        self.i += 1
        return ("set", [(ord(c), ord(c))])

    def group(self):
        self.i += 1
        if self.peek() == "?":
            nxt = self.peek(1)
            if nxt == ":":
                self.i += 2
            elif nxt == "P" and self.peek(2) == "<":
                end = self.p.find(">", self.i)
                if end < 0:
                    raise self.error("unterminated group name")
                self.i = end + 1
            elif nxt == "P" and self.peek(2) == "=":
                raise self.error("backreference (?P=...) is not supported")
            elif nxt in ("=", "!") or (nxt == "<" and self.peek(2) in ("=", "!")):
                raise self.error("lookaround is not supported")
            elif nxt == ">":
                raise self.error("atomic groups are not supported")
            elif nxt == "#":
                raise self.error("comments are not supported")
            else:
                raise self.error("inline flags are not supported")
        node = self.alternation()
        if self.peek() != ")":
            raise self.error("missing ), unterminated subpattern")
        self.i += 1
        return node

    def escape(self, in_class: bool):
        """The code-point ranges of the escape at ``self.i`` (a backslash)."""
        self.i += 1
        c = self.peek()
        if c is None:
            raise self.error("bad escape (end of pattern)")
        self.i += 1
        if c in _CLASS_ESCAPES:
            ranges, negate = _CLASS_ESCAPES[c]
            return _complement(ranges) if negate else list(ranges)
        if c in _CHAR_ESCAPES:
            return [(_CHAR_ESCAPES[c],) * 2]
        if c in ("x", "u", "U"):
            width = {"x": 2, "u": 4, "U": 8}[c]
            digits = self.p[self.i : self.i + width]
            if len(digits) != width or any(d not in "0123456789abcdefABCDEF" for d in digits):
                raise self.error(f"incomplete escape \\{c}")
            self.i += width
            cp = int(digits, 16)
            if cp > _MAX_CP:
                raise self.error(f"bad escape \\{c}{digits}")
            return [(cp, cp)]
        if c == "0":
            return [(0, 0)]
        if c.isdigit():
            raise self.error(f"backreference \\{c} is not supported")
        if c in "AZbBzG":
            if in_class and c == "b":
                return [(0x08, 0x08)]
            raise self.error(f"anchor \\{c} is not supported")
        if c.isascii() and c.isalnum():
            raise self.error(f"bad escape \\{c}")
        return [(ord(c), ord(c))]

    def char_class(self):
        self.i += 1
        negate = self.peek() == "^"
        if negate:
            self.i += 1
        ranges, first = [], True
        while True:
            c = self.peek()
            if c is None:
                raise self.error("unterminated character set")
            if c == "]" and not first:
                self.i += 1
                break
            first = False
            if c == "\\":
                item = self.escape(in_class=True)
            else:
                self.i += 1
                item = [(ord(c), ord(c))]
            if len(item) == 1 and item[0][0] == item[0][1] and self.peek() == "-" and self.peek(1) not in (None, "]"):
                self.i += 1
                if self.peek() == "\\":
                    hi = self.escape(in_class=True)
                    if len(hi) != 1 or hi[0][0] != hi[0][1]:
                        raise self.error("bad character range")
                    hi = hi[0][0]
                else:
                    hi = ord(self.peek())
                    self.i += 1
                if hi < item[0][0]:
                    raise self.error("bad character range")
                item = [(item[0][0], hi)]
            ranges.extend(item)
        ranges = _normalize(ranges)
        return _complement(ranges) if negate else ranges


# ---------------------------------------------------------------------------------------------- UTF-8 ranges --
def _utf8(cp: int) -> bytes:
    return chr(cp).encode("utf-8", "surrogatepass")


def utf8_sequences(lo: int, hi: int):
    """The code points ``[lo, hi]`` (surrogates excluded) as sequences of byte ranges: each sequence is a list of
    ``(byte_lo, byte_hi)`` and the union of the sequences' byte strings is exactly the UTF-8 encodings of the range."""
    out, stack = [], [(lo, hi)]
    while stack:
        lo, hi = stack.pop()
        if lo > hi:
            continue
        if lo <= 0xDFFF and hi >= 0xD800:  # surrogates have no UTF-8 encoding
            stack += [(lo, 0xD7FF), (0xE000, hi)]
            continue
        split = next((m for m in (0x7F, 0x7FF, 0xFFFF) if lo <= m < hi), None)
        if split is not None:
            stack += [(lo, split), (split + 1, hi)]
            continue
        if hi <= 0x7F:
            out.append([(lo, hi)])
            continue
        done = False
        for k in range(1, 4):
            m = (1 << (6 * k)) - 1
            if (lo & ~m) != (hi & ~m):
                if lo & m:
                    stack += [(lo, lo | m), ((lo | m) + 1, hi)]
                    done = True
                    break
                if (hi & m) != m:
                    stack += [(lo, (hi & ~m) - 1), (hi & ~m, hi)]
                    done = True
                    break
        if not done:
            out.append(list(zip(_utf8(lo), _utf8(hi))))
    return out


# ------------------------------------------------------------------------------------------------------- NFA --
class _Nfa:
    def __init__(self):
        self.eps: list[list[int]] = []
        self.edges: list[list[tuple[int, int, int]]] = []  # (byte lo, byte hi, target)

    def state(self) -> int:
        self.eps.append([])
        self.edges.append([])
        return len(self.eps) - 1

    def build(self, node) -> tuple[int, int]:
        """A fragment (entry, exit) for ``node``."""
        kind = node[0]
        if kind == "set":
            a, b = self.state(), self.state()
            for lo, hi in node[1]:
                for seq in utf8_sequences(lo, hi):
                    cur = a
                    for j, (blo, bhi) in enumerate(seq):
                        nxt = b if j == len(seq) - 1 else self.state()
                        self.edges[cur].append((blo, bhi, nxt))
                        cur = nxt
            return a, b
        if kind == "cat":
            a = cur = self.state()
            for item in node[1]:
                s, e = self.build(item)
                self.eps[cur].append(s)
                cur = e
            return a, cur
        if kind == "alt":
            a, b = self.state(), self.state()
            for item in node[1]:
                s, e = self.build(item)
                self.eps[a].append(s)
                self.eps[e].append(b)
            return a, b
        _, sub, lo, hi = node
        a = cur = self.state()
        for _ in range(lo):
            s, e = self.build(sub)
            self.eps[cur].append(s)
            cur = e
        end = self.state()
        self.eps[cur].append(end)
        if hi is None:  # a loop on one more copy
            s, e = self.build(sub)
            self.eps[cur].append(s)
            self.eps[e].append(cur)
        else:
            for _ in range(hi - lo):
                s, e = self.build(sub)
                self.eps[cur].append(s)
                cur = e
                self.eps[cur].append(end)
        return a, end


def _closure(nfa: _Nfa, states) -> frozenset:
    seen, stack = set(states), list(states)
    while stack:
        for t in nfa.eps[stack.pop()]:
            if t not in seen:
                seen.add(t)
                stack.append(t)
    return frozenset(seen)


# ------------------------------------------------------------------------------------------------------- DFA --
class ByteDfa:
    """A trimmed DFA over bytes: ``table`` int32 ``[S, 256]`` (-1: dead), ``accept`` bool ``[S]``, start state 0.
    Every state is live: an accepting state is reachable from it."""

    def __init__(self, table: np.ndarray, accept: np.ndarray):
        self.table, self.accept = table, accept

    @property
    def num_states(self) -> int:
        return int(self.table.shape[0])

    def walk(self, state: int, data: bytes) -> int:
        """The state after ``data`` from ``state`` (-1 once dead)."""
        for b in data:
            if state < 0:
                return -1
            state = int(self.table[state, b])
        return state

    def matches(self, data: bytes) -> bool:
        s = self.walk(0, data)
        return s >= 0 and bool(self.accept[s])


def compile_dfa(pattern: str, max_states: int = MAX_STATES) -> ByteDfa:
    """``pattern`` -> the trimmed byte DFA of ``re.fullmatch(pattern, ., re.ASCII)`` on UTF-8 text.  Raises
    ``ValueError`` for unsupported syntax, a pattern that matches nothing, or more than ``max_states`` states."""
    if not isinstance(pattern, str):
        raise ValueError("pattern must be a str")
    ast = _Parser(pattern).parse()
    nfa = _Nfa()
    start, final = nfa.build(ast)
    # byte classes: bytes no edge distinguishes move together
    cuts = {0, 256}
    for edges in nfa.edges:
        for lo, hi, _ in edges:
            cuts.update((lo, hi + 1))
    cuts = sorted(cuts)
    classes = list(zip(cuts[:-1], cuts[1:]))
    first = _closure(nfa, [start])
    index = {first: 0}
    order = [first]
    rows: list[list[int]] = []
    while len(rows) < len(order):
        cur = order[len(rows)]
        row = [-1] * len(classes)
        for c, (lo, _) in enumerate(classes):
            targets = [t for s in cur for blo, bhi, t in nfa.edges[s] if blo <= lo <= bhi]
            if not targets:
                continue
            nxt = _closure(nfa, targets)
            if nxt not in index:
                if len(order) >= 4 * max_states:  # untrimmed growth far past the limit: stop early
                    raise ValueError(f"regex {pattern!r}: the automaton exceeds {max_states} states")
                index[nxt] = len(order)
                order.append(nxt)
            row[c] = index[nxt]
        rows.append(row)
    n = len(order)
    accept = np.array([final in s for s in order], dtype=bool)
    by_class = np.array(rows, dtype=np.int64).reshape(n, len(classes))
    widths = [hi - lo for lo, hi in classes]
    table = np.repeat(by_class, widths, axis=1)
    # trim: keep the states from which an accepting state is reachable
    live = accept.copy()
    changed = True
    while changed:
        reach = np.where(table >= 0, live[np.maximum(table, 0)], False).any(axis=1)
        new = live | reach
        changed = bool((new != live).any())
        live = new
    if not live[0]:
        raise ValueError(f"regex {pattern!r} matches nothing")
    keep = np.flatnonzero(live)
    if keep.size > max_states:
        raise ValueError(f"regex {pattern!r}: the automaton has {keep.size} states, above the limit of {max_states}")
    renum = np.full(n + 1, -1, dtype=np.int64)
    renum[keep] = np.arange(keep.size)
    trimmed = renum[np.where(table >= 0, table, n)][keep]
    return ByteDfa(np.ascontiguousarray(trimmed, dtype=np.int32), accept[keep].copy())


# ------------------------------------------------------------------------------------------------ vocabulary --
def gpt2_byte_decoder() -> dict[str, int]:
    """The inverse of GPT-2's byte-to-unicode alphabet (byte-level BPE token strings -> bytes)."""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    chars = list(keep)
    n = 0
    for b in range(256):
        if b not in keep:
            keep.append(b)
            chars.append(256 + n)
            n += 1
    return {chr(c): b for b, c in zip(keep, chars)}


class TokenVocabulary:
    """Each token id's bytes (``None``: the id can never be emitted as text - special tokens, ids past the tokenizer,
    empty strings) and the EOS ids.  ``csr(device)`` is the device form (int32 offsets ``[V + 1]``, uint8 bytes), built
    once per device."""

    def __init__(self, tokens, eos_ids):
        self.tokens = [None if (t is None or len(t) == 0) else bytes(t) for t in tokens]
        self.eos_ids = sorted({int(e) for e in eos_ids})
        if any(not 0 <= e < len(self.tokens) for e in self.eos_ids):
            raise ValueError("EOS ids must be token ids of the vocabulary")
        for e in self.eos_ids:
            self.tokens[e] = None
        self._csr: dict = {}

    @property
    def size(self) -> int:
        return len(self.tokens)

    @classmethod
    def from_tokenizer(cls, tokenizer, vocab_size: int) -> TokenVocabulary:
        """From a Hugging Face byte-level BPE tokenizer (or a wrapper with ``_tokenizer``): regular tokens map back to
        bytes through the GPT-2 alphabet, added non-special tokens are their UTF-8 text, special tokens and ids at or
        past the tokenizer's length are ``None``."""
        tok = getattr(tokenizer, "_tokenizer", tokenizer)
        decoder = gpt2_byte_decoder()
        special = set(getattr(tok, "all_special_ids", ()))
        added = {int(i): t for i, t in getattr(tok, "added_tokens_decoder", {}).items()}
        pieces = tok.convert_ids_to_tokens(list(range(min(len(tok), vocab_size))))
        tokens: list = [None] * vocab_size
        for i, piece in enumerate(pieces):
            if i in special or piece is None:
                continue
            if i in added:
                a = added[i]
                if not getattr(a, "special", False):
                    tokens[i] = str(a).encode()
                continue
            try:
                tokens[i] = bytes(decoder[ch] for ch in piece)
            except KeyError:
                tokens[i] = None
        eos = getattr(tok, "eos_token_id", None)
        eos_ids = set(getattr(tokenizer, "eos_token_ids", ()) or ())
        if eos is not None:
            eos_ids.add(int(eos))
        return cls(tokens, [e for e in eos_ids if e < vocab_size])

    @classmethod
    def synthetic(cls, vocab_size: int, seed: int = 0, max_len: int = 8) -> TokenVocabulary:
        """A deterministic vocabulary for random-weight models: single bytes first (every byte when ``vocab_size`` >
        256 + 1, else printable ASCII, tab and newline), then seeded merges of 2 to ``max_len`` characters (ASCII
        letters, digits, punctuation and space, with some two-byte characters), and EOS = the last id."""
        if vocab_size < 100:
            raise ValueError("the synthetic vocabulary needs at least 100 ids")
        singles = list(range(256)) if vocab_size > 257 else [9, 10] + list(range(0x20, 0x7F))
        tokens: list = [bytes([b]) for b in singles]
        rng = np.random.default_rng(seed)
        alphabet = [chr(c) for c in range(0x20, 0x7F)] + ["é", "ß", "ж", "λ"]
        n_merge = vocab_size - 1 - len(tokens)
        lengths = np.minimum(2 + rng.geometric(0.35, n_merge) - 1, max_len)
        picks = rng.integers(0, len(alphabet), int(lengths.sum()))
        at = 0
        for n in lengths:
            tokens.append("".join(alphabet[j] for j in picks[at : at + n]).encode())
            at += n
        tokens.append(None)
        return cls(tokens, [vocab_size - 1])

    def csr(self, device) -> tuple[torch.Tensor, torch.Tensor]:
        key = str(torch.device(device))
        if key not in self._csr:
            lengths = np.array([0 if t is None else len(t) for t in self.tokens], dtype=np.int64)
            offsets = np.zeros(self.size + 1, dtype=np.int64)
            np.cumsum(lengths, out=offsets[1:])
            if offsets[-1] >= 1 << 31:
                raise ValueError("the vocabulary's bytes exceed 2^31")
            data = np.frombuffer(b"".join(t for t in self.tokens if t is not None) or b"\0", dtype=np.uint8)
            self._csr[key] = (torch.from_numpy(offsets.astype(np.int32)).to(device), torch.from_numpy(data.copy()).to(device))
        return self._csr[key]


# -------------------------------------------------------------------------------------------- token automaton --
DESCRIPTOR_WORDS = 5  # int64 words of one tl_constraint_row: mask, dfa, token_offsets, token_bytes, (num_states, state)


class TokenConstraint:
    """A compiled pattern over one vocabulary.  Owns the device tables (DFA ``[S, 256]``, accept flags ``[S]`` and the
    token masks ``uint32 [S + 1, ceil(V / 32)]``, row ``S`` the terminal state after EOS) and a host mirror of the DFA
    (``dfa``).  ``start_state`` is 0 and ``terminal_state`` is ``S``."""

    def __init__(self, pattern, vocabulary, dfa, masks, dfa_dev, accept_dev, reach):
        self.pattern, self.vocabulary, self.dfa = pattern, vocabulary, dfa
        self.masks, self.dfa_dev, self.accept_dev, self.reach = masks, dfa_dev, accept_dev, reach
        self.start_state = 0
        self.terminal_state = dfa.num_states
        self._eos = set(vocabulary.eos_ids)

    @property
    def vocab_size(self) -> int:
        return self.vocabulary.size

    @classmethod
    def compile(cls, pattern: str, vocabulary: TokenVocabulary, device="cuda", max_states: int = MAX_STATES) -> TokenConstraint:
        from extensions_b200 import tiny_llm_ext_b200 as ext

        dfa = compile_dfa(pattern, max_states)
        offsets, data = vocabulary.csr(device)
        dfa_dev = torch.from_numpy(dfa.table).to(device)
        accept_dev = torch.from_numpy(dfa.accept.astype(np.uint8)).to(device)
        eos = torch.tensor(vocabulary.eos_ids, dtype=torch.int32, device=device)
        masks, reach = ext.constraint_token_masks(dfa_dev, accept_dev, offsets, data, eos)
        check_spellable(pattern, masks.cpu().numpy(), reach.cpu().numpy(), dfa.num_states)
        return cls(pattern, vocabulary, dfa, masks, dfa_dev, accept_dev, reach)

    def walk(self, state: int, token_ids) -> int:
        """The token automaton's state after ``token_ids`` from ``state`` on the host mirror (-1: a token not allowed
        was met)."""
        S = self.terminal_state
        for t in token_ids:
            t = int(t)
            if state < 0:
                return -1
            if t in self._eos:
                state = S if (state == S or self.dfa.accept[state]) else -1
            elif state == S or not 0 <= t < self.vocab_size or self.vocabulary.tokens[t] is None:
                return -1
            else:
                state = self.dfa.walk(state, self.vocabulary.tokens[t])
        return state

    def descriptor(self, state: int | None = None, out: torch.Tensor | None = None) -> torch.Tensor:
        """The ``tl_constraint_row`` of this constraint at ``state`` (default: the start state) as int64
        ``[DESCRIPTOR_WORDS]`` on the constraint's device, written into ``out`` when given."""
        t = torch.tensor(descriptor_values(self, self.start_state if state is None else state), dtype=torch.int64)
        if out is None:
            return t.to(self.masks.device)
        out.copy_(t)
        return out


def descriptor_values(constraint: TokenConstraint | None, state: int = 0) -> list[int]:
    """The five int64 words of one ``tl_constraint_row`` (all zero: unconstrained)."""
    if constraint is None:
        return [0] * DESCRIPTOR_WORDS
    offsets, data = constraint.vocabulary.csr(constraint.masks.device)
    packed = (constraint.terminal_state & 0xFFFFFFFF) | ((state & 0xFFFFFFFF) << 32)
    if packed >= 1 << 63:
        packed -= 1 << 64
    return [constraint.masks.data_ptr(), constraint.dfa_dev.data_ptr(), offsets.data_ptr(), data.data_ptr(), packed]


def descriptor_state(rows: torch.Tensor) -> torch.Tensor:
    """The int32 ``state`` fields of descriptor rows ``[..., DESCRIPTOR_WORDS]`` (a view)."""
    return rows.view(torch.int32)[..., 2 * DESCRIPTOR_WORDS - 1]


def check_spellable(pattern: str, masks: np.ndarray, reach: np.ndarray, num_states: int) -> None:
    """Every state reachable from the start by allowed tokens must allow at least one token; ``masks`` uint32
    ``[S + 1, W]`` and ``reach`` uint32 ``[S, ceil(S / 32)]`` (bit e of row s: an allowed token leads from s to e)."""
    masks = masks.view(np.uint32)
    reach = reach.view(np.uint32)
    seen = np.zeros(num_states, dtype=bool)
    seen[0] = True
    stack = [0]
    while stack:
        s = stack.pop()
        if not masks[s].any():
            raise ValueError(f"regex {pattern!r}: the vocabulary cannot continue the text in DFA state {s} "
                             "(no token is allowed there)")
        bits = np.unpackbits(reach[s].view(np.uint8), bitorder="little")[:num_states]
        for e in np.flatnonzero(bits):
            if not seen[e]:
                seen[e] = True
                stack.append(int(e))


def token_masks_reference(dfa: ByteDfa, vocabulary: TokenVocabulary) -> tuple[np.ndarray, np.ndarray]:
    """What ``tl_constraint_token_masks`` computes, in NumPy: masks uint32 ``[S + 1, ceil(V / 32)]`` and reach uint32
    ``[S, ceil(S / 32)]``.  All tokens step through the table together, one byte position at a time."""
    S, V = dfa.num_states, vocabulary.size
    lengths = np.array([0 if t is None else len(t) for t in vocabulary.tokens], dtype=np.int64)
    L = int(lengths.max()) if V else 0
    padded = np.zeros((V, max(L, 1)), dtype=np.int64)
    for i, t in enumerate(vocabulary.tokens):
        if t is not None:
            padded[i, : len(t)] = np.frombuffer(t, dtype=np.uint8)
    table = np.vstack([dfa.table.astype(np.int64), np.full((1, 256), -1, dtype=np.int64)])  # row S: dead sink
    state = np.repeat(np.arange(S, dtype=np.int64)[:, None], V, axis=1)
    for j in range(L):
        active = lengths > j
        cur = np.where(state < 0, S, state)
        nxt = table[cur, padded[None, :, j]]
        state = np.where(active[None, :], np.where(state < 0, -1, nxt), state)
    allowed = (state >= 0) & (lengths > 0)[None, :]
    eos = np.zeros(V, dtype=bool)
    eos[vocabulary.eos_ids] = True
    allowed = np.vstack([allowed | (eos[None, :] & dfa.accept[:, None]), eos[None, :]])
    W = (V + 31) // 32
    bits = np.zeros((S + 1, W * 32), dtype=bool)
    bits[:, :V] = allowed
    masks = np.packbits(bits.reshape(S + 1, W, 32), axis=2, bitorder="little").view(np.uint32).reshape(S + 1, W)
    RW = (S + 31) // 32
    rbits = np.zeros((S, RW * 32), dtype=bool)
    ss, tt = np.nonzero(allowed[:S] & (lengths > 0)[None, :])
    rbits[ss, state[ss, tt]] = True
    reach = np.packbits(rbits.reshape(S, RW, 32), axis=2, bitorder="little").view(np.uint32).reshape(S, RW)
    return masks, reach
