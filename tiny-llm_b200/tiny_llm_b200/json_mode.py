"""JSON mode (DESIGN.md section 20): generated text restricted to one JSON object.

The language is RFC 8259 ``ws object ws`` over the UTF-8 bytes of the text, with at most ``JSON_MAX_DEPTH`` open
containers (the top-level object counts) and at most ``JSON_MAX_WS_RUN`` consecutive whitespace bytes between tokens
of the grammar (bytes inside strings are content, not whitespace).  Objects nest, so no byte DFA can express it: the
automaton here is a pushdown automaton whose whole state fits two int64 words per row, the container stack as one
bit per level and a lexer word (layout in ``include/tiny_llm_b200.h``).

Each step ``tl_json_token_masks`` writes every JSON row's token mask from its state on the device, the unchanged
``tl_sample_constrained`` draws under it (a JSON row is a one-state ``tl_constraint_row`` whose mask is the row's own
buffer), and ``tl_json_advance`` walks the drawn token.  ``JsonWalker`` is the same automaton on the host, bit for bit:
it sets a row's state from its history and checks a vocabulary."""

from __future__ import annotations

import numpy as np
import torch

JSON_MAX_DEPTH = 64  # open containers, counting the top-level object
JSON_MAX_WS_RUN = 32  # consecutive whitespace bytes
STATE_WORDS = 2

# lexer states (bits 8-12 of word 1), as in csrc/json.cu
START, OBJ_FIRST, OBJ_KEY, COLON, VALUE, ARR_FIRST, AFTER, CLOSED = range(8)
STR, ESC, HEX, UTF8, MINUS, ZERO, INT, DOT, FRAC, EXP_MARK, EXP_SIGN, EXP, LIT = range(8, 21)
DEAD = 31
_ACTIVE, _TERMINAL = 1 << 32, 1 << 33
_WS = frozenset(b" \t\n\r")
_DIGITS = frozenset(b"0123456789")
_HEXDIGITS = frozenset(b"0123456789abcdefABCDEF")
_ESCAPES = frozenset(b'"\\/bfnrt')
_LITERALS = (b"true", b"false", b"null")
# the range of the byte after a UTF-8 lead (index aux2) and of every later continuation byte (0)
_UTF8_RANGE = {0: (0x80, 0xBF), 1: (0xA0, 0xBF), 2: (0x80, 0x9F), 3: (0x90, 0xBF), 4: (0x80, 0x8F)}


def _lead(b: int):
    """(continuation bytes, range index of the next one) of a UTF-8 lead byte, or None."""
    if 0xC2 <= b <= 0xDF:
        return 1, 0
    if 0xE0 <= b <= 0xEF:
        return 2, 1 if b == 0xE0 else 2 if b == 0xED else 0
    if 0xF0 <= b <= 0xF4:
        return 3, 3 if b == 0xF0 else 4 if b == 0xF4 else 0
    return None


class JsonWalker:
    """One row's automaton state, mutable; ``step`` and ``walk`` return False once the text leaves the language."""

    __slots__ = ("stack", "depth", "lex", "ws", "aux", "aux2", "key", "terminal")

    def __init__(self, words=None):
        w0, w1 = (0, _ACTIVE) if words is None else (int(words[0]) & (1 << 64) - 1, int(words[1]) & (1 << 64) - 1)
        self.stack = w0
        self.depth = w1 & 0x7F
        self.lex = (w1 >> 8) & 31
        self.ws = (w1 >> 16) & 63
        self.aux = (w1 >> 24) & 7
        self.aux2 = (w1 >> 27) & 7
        self.key = (w1 >> 30) & 1
        self.terminal = bool(w1 & _TERMINAL)

    def copy(self) -> JsonWalker:
        w = JsonWalker.__new__(JsonWalker)
        for name in self.__slots__:
            setattr(w, name, getattr(self, name))
        return w

    def words(self) -> tuple[int, int]:
        """The two int64 words of the device state (signed)."""
        w1 = (self.depth | self.lex << 8 | self.ws << 16 | self.aux << 24 | self.aux2 << 27 | self.key << 30 | _ACTIVE
              | (_TERMINAL if self.terminal else 0))
        return tuple(w - (1 << 64) if w >= 1 << 63 else w for w in (self.stack, w1))

    @property
    def complete(self) -> bool:
        """The text so far is a complete text of the language (EOS may follow)."""
        return self.lex == CLOSED and not self.terminal

    def _top_array(self) -> bool:
        return bool(self.stack >> (self.depth - 1) & 1)

    def _push(self, array: bool) -> bool:
        if self.depth >= JSON_MAX_DEPTH:
            return False
        bit = 1 << self.depth
        self.stack = self.stack | bit if array else self.stack & ~bit
        self.depth += 1
        self.lex = ARR_FIRST if array else OBJ_FIRST
        return True

    def _pop(self) -> bool:
        self.depth -= 1
        self.lex = CLOSED if self.depth == 0 else AFTER
        return True

    def _value_start(self, b: int) -> bool:
        if b == 0x7B:
            return self._push(False)
        if b == 0x5B:
            return self._push(True)
        if b == 0x22:
            self.lex, self.key = STR, 0
        elif b == 0x2D:
            self.lex = MINUS
        elif b == 0x30:
            self.lex = ZERO
        elif b in _DIGITS:
            self.lex = INT
        elif b in b"tfn":
            self.lex, self.aux, self.aux2 = LIT, b"tfn".index(b), 1
        else:
            return False
        return True

    def _after_value(self, b: int) -> bool:
        self.lex = AFTER
        if b == 0x2C:
            self.lex = VALUE if self._top_array() else OBJ_KEY
            return True
        if b == (0x5D if self._top_array() else 0x7D):
            return self._pop()
        return False

    def step(self, b: int) -> bool:
        lex = self.lex
        number_may_end = lex in (ZERO, INT, FRAC, EXP)
        if lex <= CLOSED or number_may_end:
            if b in _WS:
                if number_may_end:
                    self.lex = AFTER
                if self.ws >= JSON_MAX_WS_RUN:
                    return False
                self.ws += 1
                return True
            self.ws = 0
        if lex == START:
            return b == 0x7B and self._push(False)
        if lex == OBJ_FIRST:
            if b == 0x7D:
                return self._pop()
            if b == 0x22:
                self.lex, self.key = STR, 1
                return True
            return False
        if lex == OBJ_KEY:
            if b == 0x22:
                self.lex, self.key = STR, 1
                return True
            return False
        if lex == COLON:
            if b == 0x3A:
                self.lex = VALUE
                return True
            return False
        if lex == VALUE:
            return self._value_start(b)
        if lex == ARR_FIRST:
            return self._pop() if b == 0x5D else self._value_start(b)
        if lex == AFTER:
            return self._after_value(b)
        if lex == STR:
            if b == 0x22:
                self.lex, self.key = (COLON if self.key else AFTER), 0
            elif b == 0x5C:
                self.lex = ESC
            elif 0x20 <= b < 0x80:
                pass
            else:
                lead = _lead(b)
                if lead is None:
                    return False
                self.lex, (self.aux, self.aux2) = UTF8, lead
            return True
        if lex == ESC:
            if b == 0x75:
                self.lex, self.aux = HEX, 4
                return True
            if b in _ESCAPES:
                self.lex = STR
                return True
            return False
        if lex == HEX:
            if b not in _HEXDIGITS:
                return False
            self.aux -= 1
            if self.aux == 0:
                self.lex = STR
            return True
        if lex == UTF8:
            lo, hi = _UTF8_RANGE[self.aux2]
            if not lo <= b <= hi:
                return False
            self.aux2 = 0
            self.aux -= 1
            if self.aux == 0:
                self.lex = STR
            return True
        if lex == MINUS:
            if b in _DIGITS:
                self.lex = ZERO if b == 0x30 else INT
                return True
            return False
        if lex in (ZERO, INT, FRAC):
            if b in _DIGITS and lex != ZERO:
                return True
            if b == 0x2E and lex != FRAC:
                self.lex = DOT
                return True
            if b in (0x65, 0x45):
                self.lex = EXP_MARK
                return True
            return self._after_value(b)
        if lex == DOT:
            if b in _DIGITS:
                self.lex = FRAC
                return True
            return False
        if lex == EXP_MARK:
            if b in (0x2B, 0x2D):
                self.lex = EXP_SIGN
                return True
            if b in _DIGITS:
                self.lex = EXP
                return True
            return False
        if lex == EXP_SIGN:
            if b in _DIGITS:
                self.lex = EXP
                return True
            return False
        if lex == EXP:
            return True if b in _DIGITS else self._after_value(b)
        if lex == LIT:
            lit = _LITERALS[self.aux]
            if b != lit[self.aux2]:
                return False
            self.aux2 += 1
            if self.aux2 == len(lit):
                self.lex, self.aux, self.aux2 = AFTER, 0, 0
            return True
        return False  # CLOSED, DEAD

    def walk(self, data: bytes) -> bool:
        if self.terminal or self.lex == DEAD:
            return False
        for b in data:
            if not self.step(b):
                return False
        return True


# ------------------------------------------------------------------------------------------------ vocabulary --
_REQUIRED_SINGLES = b'{}]:"0' + b"ruealsn"  # structure, a closing value digit, and every literal's later bytes


def check_vocabulary(vocabulary) -> None:
    """Refuse (``ValueError``) a vocabulary in which some text of the language reachable token by token could not be
    continued.  Sufficient: an EOS id; a one-byte token for each byte that finishes the current construct (``{`` to
    open, ``"`` to close a string or escape, ``0`` for a number, hex digit or value, ``:``, ``}``, ``]``, the literals'
    letters); and for every token that ends inside a UTF-8 character, a one-byte token in the range of each byte that
    character still needs.  From any state those bytes lead, one token at a time, to a complete text."""
    if not vocabulary.eos_ids:
        raise ValueError("JSON mode needs a vocabulary with an EOS id")
    singles = set()
    for t in vocabulary.tokens:
        if t is not None and len(t) == 1:
            singles.add(t[0])
    missing = [chr(b) for b in _REQUIRED_SINGLES if b not in singles]
    if missing:
        raise ValueError(f"JSON mode needs a one-byte token for each of {''.join(missing)!r}: the grammar can demand "
                         "that byte next")
    need = {}  # (lo, hi) -> (lead byte, token id) that needs a one-byte token in [lo, hi]
    for i, t in enumerate(vocabulary.tokens):
        if t is None:
            continue
        for k in range(1, min(3, len(t)) + 1):
            lead = _lead(t[-k])
            if lead is None:
                continue
            n, first = lead
            if k - 1 < n and all(0x80 <= c <= 0xBF for c in t[len(t) - k + 1:]):
                if k == 1:
                    need.setdefault(_UTF8_RANGE[first], (t[-k], i))
                if n - (k - 1) >= (1 if k > 1 else 2):
                    need.setdefault(_UTF8_RANGE[0], (t[-k], i))
            break
    for (lo, hi), (lead, i) in sorted(need.items()):
        if not any(lo <= b <= hi for b in singles):
            raise ValueError(f"JSON mode needs a one-byte token in 0x{lo:02X}-0x{hi:02X}: token {i} ends after the "
                             f"UTF-8 lead byte 0x{lead:02X}, which needs it next")


_ZERO_DFA: dict = {}


def _zero_dfa(device) -> torch.Tensor:
    key = str(torch.device(device))
    if key not in _ZERO_DFA:
        _ZERO_DFA[key] = torch.zeros((1, 256), dtype=torch.int32, device=device)
    return _ZERO_DFA[key]


class JsonConstraint:
    """JSON mode over one vocabulary: ``SamplingParams(constraint=JsonConstraint(vocabulary))``.  Holds the
    vocabulary's device CSR and its EOS-only mask row; the per-row state and mask buffers live with each caller's
    ``ConstraintRows``."""

    def __init__(self, vocabulary, device="cuda"):
        check_vocabulary(vocabulary)
        self.vocabulary = vocabulary
        self.device = torch.device(device)
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

    def walk(self, token_ids, walker: JsonWalker | None = None) -> JsonWalker | None:
        """The state after ``token_ids`` from ``walker`` (default: the start), or None when a token is not allowed."""
        w = JsonWalker() if walker is None else walker.copy()
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

    def allowed(self, walker: JsonWalker) -> np.ndarray:
        """bool ``[V]``: the tokens allowed after ``walker`` (what the device mask holds)."""
        V = self.vocab_size
        out = np.zeros(V, dtype=bool)
        if walker.terminal:
            out[self.vocabulary.eos_ids] = True
            return out
        for i, t in enumerate(self.vocabulary.tokens):
            if t is None:
                out[i] = i in self._eos and walker.complete
            else:
                out[i] = walker.copy().walk(t)
        return out


# -------------------------------------------------------------------------------------------- per-row tables --
class ConstraintRows:
    """The constraint tables of one draw's rows, for any mix of regex, JSON, JSON Schema, grammar and unconstrained
    ``SamplingParams``: ``descriptors`` int64 ``[R, 5]`` ``tl_constraint_row``s and, when a row is in JSON mode,
    ``json_states`` int64 ``[R, 2]`` (zero rows: not JSON), when a row is under a ``JsonSchemaConstraint``,
    ``schema_states`` int64 ``[R, 10]`` (zero rows: not a schema row), when a row is under a ``GrammarConstraint``,
    ``grammar_states`` int64 ``[R, 74]`` (zero rows: not a grammar row), and for any of them ``json_masks`` int32
    ``[R, 2, ceil(V / 32)]`` (row 0 this step's mask, row 1 EOS only).  ``sample`` runs the masks launches,
    ``tl_sample_constrained`` and the advances; regex rows advance inside the draw as before."""

    def __init__(self, rows: int, vocab: int, device, json: bool, schema: bool = False, grammar: bool = False):
        self.rows, self.vocab, self.device = rows, vocab, torch.device(device)
        self.descriptors = torch.zeros((rows, 5), dtype=torch.int64, device=device)
        self.json_states = self.json_masks = self.schema_states = self.grammar_states = None
        self.schema_smem_bytes = 0  # shared memory of the schema masks launch: the largest schema blob that fits
        self.grammar_smem_bytes = 0  # likewise for the grammar masks launch
        self._json_constraints: list = [None] * rows  # the row's JsonConstraint, JsonSchemaConstraint or GrammarConstraint
        if json:
            self.ensure_json()
        if schema:
            self.ensure_schema()
        if grammar:
            self.ensure_grammar()

    @classmethod
    def build(cls, params, vocab: int, device) -> ConstraintRows:
        """Rows at their constraints' start states, one per entry of ``params`` (None: unconstrained)."""
        from .grammar import GrammarConstraint
        from .json_schema import JsonSchemaConstraint

        cons = [None if p is None else p.constraint for p in params]
        out = cls(len(cons), vocab, device, any(isinstance(c, JsonConstraint) for c in cons),
                  any(isinstance(c, JsonSchemaConstraint) for c in cons), any(isinstance(c, GrammarConstraint) for c in cons))
        for r, c in enumerate(cons):
            out.set_row(r, c)
        return out

    @classmethod
    def concat(cls, tables: list) -> ConstraintRows:
        """One table of the rows of ``tables`` in order (device copies of their states)."""
        t0 = tables[0]
        out = cls(sum(t.rows for t in tables), t0.vocab, t0.device, any(t.has_json for t in tables), any(t.has_schema for t in tables),
                  any(t.has_grammar for t in tables))
        r = 0
        for t in tables:
            for s in range(t.rows):
                out.copy_row(r, t, s)
                r += 1
        return out

    @property
    def has_json(self) -> bool:
        return self.json_states is not None

    @property
    def has_schema(self) -> bool:
        return self.schema_states is not None

    @property
    def has_grammar(self) -> bool:
        return self.grammar_states is not None

    def _ensure_masks(self) -> None:
        if self.json_masks is None:
            self.json_masks = torch.zeros((self.rows, 2, (self.vocab + 31) // 32), dtype=torch.int32, device=self.device)

    def ensure_json(self) -> None:
        if self.json_states is None:
            self.json_states = torch.zeros((self.rows, STATE_WORDS), dtype=torch.int64, device=self.device)
            self._ensure_masks()

    def ensure_schema(self) -> None:
        from .json_schema import SCHEMA_STATE_WORDS

        if self.schema_states is None:
            self.schema_states = torch.zeros((self.rows, SCHEMA_STATE_WORDS), dtype=torch.int64, device=self.device)
            self._ensure_masks()

    def ensure_grammar(self) -> None:
        from .grammar import GRAMMAR_STATE_WORDS

        if self.grammar_states is None:
            self.grammar_states = torch.zeros((self.rows, GRAMMAR_STATE_WORDS), dtype=torch.int64, device=self.device)
            self._ensure_masks()

    def _zero_states(self, r: int, keep=None) -> None:
        for states in (self.json_states, self.schema_states, self.grammar_states):
            if states is not None and states is not keep:
                states[r].zero_()

    def set_row(self, r: int, constraint, state=None) -> None:
        """Row ``r`` under ``constraint`` (None: unconstrained) at ``state`` (a regex state, a ``JsonWalker``, a
        ``SchemaWalker`` or a ``GrammarWalker``; default the start)."""
        from .constrained import descriptor_values
        from .grammar import GrammarConstraint
        from .json_schema import JsonSchemaConstraint

        if isinstance(constraint, JsonConstraint):
            self.ensure_json()
            self._zero_states(r, keep=self.json_states)
            w = JsonWalker() if state is None else state
            self.json_masks[r, 1].copy_(constraint.eos_row)
            self.json_states[r].copy_(torch.tensor(w.words(), dtype=torch.int64))
            self.descriptors[r].copy_(torch.tensor(self._json_descriptor(r, constraint, 1 if w.terminal else 0), dtype=torch.int64))
        elif isinstance(constraint, JsonSchemaConstraint):
            self.ensure_schema()
            self._zero_states(r, keep=self.schema_states)
            w = constraint.start() if state is None else state
            self.json_masks[r, 1].copy_(constraint.eos_row)
            self.schema_states[r].copy_(torch.tensor(constraint.words(w), dtype=torch.int64))
            self._fit_schema(constraint)
            self.descriptors[r].copy_(torch.tensor(self._json_descriptor(r, constraint, 1 if w.terminal else 0), dtype=torch.int64))
        elif isinstance(constraint, GrammarConstraint):
            self.ensure_grammar()
            self._zero_states(r, keep=self.grammar_states)
            w = constraint.start() if state is None else state
            self.json_masks[r, 1].copy_(constraint.eos_row)
            self.grammar_states[r].copy_(torch.tensor(constraint.words(w), dtype=torch.int64))
            self._fit_grammar(constraint)
            self.descriptors[r].copy_(torch.tensor(self._json_descriptor(r, constraint, 1 if w.terminal else 0), dtype=torch.int64))
        else:
            self._zero_states(r)
            self.descriptors[r].copy_(torch.tensor(descriptor_values(constraint, 0 if state is None else state), dtype=torch.int64))
        self._json_constraints[r] = constraint if isinstance(constraint, (JsonConstraint, JsonSchemaConstraint, GrammarConstraint)) else None

    def _fit_schema(self, c) -> None:
        from .json_schema import SCHEMA_SMEM_BYTES

        n = int(c.compiled.blob.size)
        if n <= SCHEMA_SMEM_BYTES:
            self.schema_smem_bytes = max(self.schema_smem_bytes, n)

    def _fit_grammar(self, c) -> None:
        from .grammar import GRAMMAR_SMEM_BYTES

        n = int(c.compiled.blob.size)
        if n <= GRAMMAR_SMEM_BYTES:
            self.grammar_smem_bytes = max(self.grammar_smem_bytes, n)

    def _json_descriptor(self, r: int, c, state: int) -> list[int]:
        packed = 1 | (state << 32)  # num_states 1, state 0 (or 1, terminal)
        return [self.json_masks[r].data_ptr(), c.dfa.data_ptr(), c.token_offsets.data_ptr(), c.token_bytes.data_ptr(), packed]

    def copy_row(self, r: int, src: ConstraintRows, s: int = 0) -> None:
        """Row ``r`` takes row ``s`` of ``src`` (a device copy of its state; the descriptor is rebuilt for JSON and
        schema rows, whose mask pointer is per table)."""
        c = src._json_constraints[s]
        if c is None:
            self._zero_states(r)
            self.descriptors[r].copy_(src.descriptors[s])
            self._json_constraints[r] = None
            return
        from .grammar import GrammarConstraint

        if isinstance(c, JsonConstraint):
            self.ensure_json()
            self._zero_states(r, keep=self.json_states)
            self.json_states[r].copy_(src.json_states[s])
        elif isinstance(c, GrammarConstraint):
            self.ensure_grammar()
            self._zero_states(r, keep=self.grammar_states)
            self.grammar_states[r].copy_(src.grammar_states[s])
            self._fit_grammar(c)
        else:
            self.ensure_schema()
            self._zero_states(r, keep=self.schema_states)
            self.schema_states[r].copy_(src.schema_states[s])
            self._fit_schema(c)
        self.json_masks[r].copy_(src.json_masks[s])
        self.descriptors[r, :4].copy_(torch.tensor(self._json_descriptor(r, c, 0)[:4], dtype=torch.int64))
        self.descriptors[r, 4].copy_(src.descriptors[s, 4])  # num_states and the terminal flag
        self._json_constraints[r] = c

    def clear_row(self, r: int) -> None:
        self.descriptors[r].zero_()
        self._zero_states(r)
        self._json_constraints[r] = None

    def before_draw(self, rows: int | None = None) -> None:
        """This step's masks of the JSON, schema and grammar rows among the first ``rows`` (default all)."""
        from extensions_b200 import tiny_llm_ext_b200 as ext

        n = self.rows if rows is None else rows
        if self.json_states is not None:
            ext.json_token_masks(self.descriptors[:n], self.json_states[:n], self.vocab)
        if self.schema_states is not None:
            ext.schema_token_masks(self.descriptors[:n], self.schema_states[:n], self.vocab, self.schema_smem_bytes)
        if self.grammar_states is not None:
            ext.grammar_token_masks(self.descriptors[:n], self.grammar_states[:n], self.vocab, self.grammar_smem_bytes)

    def after_draw(self, tokens: torch.Tensor, positions: torch.Tensor) -> None:
        """Advance the JSON, schema and grammar rows by their drawn ``tokens`` (rows with ``positions > 0``).  A grammar
        row whose drawn token was not allowed raises ``ValueError`` (``check_grammar_rows``)."""
        from extensions_b200 import tiny_llm_ext_b200 as ext

        n = tokens.shape[0]
        if self.json_states is not None:
            ext.json_advance(self.descriptors[:n], self.json_states[:n], tokens, positions)
        if self.schema_states is not None:
            ext.schema_advance(self.descriptors[:n], self.schema_states[:n], tokens, positions)
        if self.grammar_states is not None:
            ext.grammar_advance(self.descriptors[:n], self.grammar_states[:n], tokens, positions, self.vocab)
            self.check_grammar_rows(n)

    def check_grammar_rows(self, rows: int | None = None) -> None:
        """Raise ``ValueError`` when a grammar row among the first ``rows`` (default all) has its failed bit set: its
        parses went past the parse cap, no token was allowed and the draw's fallback token left the grammar."""
        if self.grammar_states is None:
            return
        from .grammar import GRAMMAR_MAX_PARSES, failed_rows

        bad = failed_rows(self.grammar_states[: self.rows if rows is None else rows])
        if bad:
            raise ValueError(f"grammar: row {bad[0]} has no allowed token: every continuation keeps more than "
                             f"GRAMMAR_MAX_PARSES = {GRAMMAR_MAX_PARSES} parses live, so the text cannot stay in the grammar")

    def walkers(self) -> list:
        """The host mirror of each row's JSON or schema state (None for other rows); one device read per kind."""
        from .grammar import GrammarConstraint, GrammarWalker
        from .json_schema import SchemaWalker

        jw = self.json_states.tolist() if self.json_states is not None else None
        sw = self.schema_states.tolist() if self.schema_states is not None else None
        gw = self.grammar_states.tolist() if self.grammar_states is not None else None
        out = []
        for r, c in enumerate(self._json_constraints):
            if c is None:
                out.append(None)
            elif isinstance(c, JsonConstraint):
                out.append(JsonWalker(jw[r]))
            elif isinstance(c, GrammarConstraint):
                out.append(GrammarWalker(c.compiled, gw[r]))
            else:
                out.append(SchemaWalker(c.compiled, sw[r]))
        return out
