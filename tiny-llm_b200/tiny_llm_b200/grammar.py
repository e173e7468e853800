"""Grammar-constrained generation (DESIGN.md section 23): generated text restricted to the language of a user-written
context-free grammar in GBNF (llama.cpp's grammar format; vLLM's ``guided_grammar``).

``compile_grammar`` turns a grammar into a byte-level pushdown automaton held in tables.  Every rule that is not
recursive is inlined where it is used, so the regular parts of the grammar are determinized by subset construction over
byte classes, as ``constrained.compile_dfa`` does; each recursive rule (and ``root``) becomes one sub-automaton, and the
only calls left are calls to recursive rules.  Hand-written grammars are rarely deterministic in the pushdown sense
(``expr ::= term | term "+" expr`` calls ``term`` from two states with different return states), so a state holds, per
byte class, a short *list* of actions: a shift to a state, or a call chain that pushes one or more return states (a call
whose callee starts with another call is precomposed into one action) and lands in a state.  A state whose rule may end
there returns lazily: on the next byte the walker also pops the return state and looks the same byte up there.

A row's state is therefore a *set* of parses, each a (state, return stack) pair, deduplicated after every byte and
capped at ``GRAMMAR_MAX_PARSES``; a parse is kept only while its depth plus its state's *need* (the stack entries its
cheapest completion still pushes) stays within ``GRAMMAR_MAX_DEPTH``, so an allowed token never leads into a state that
cannot complete.

Each step ``tl_grammar_token_masks`` writes every grammar row's token mask from its parse set on the device, the
unchanged ``tl_sample_constrained`` draws under it, and ``tl_grammar_advance`` walks the drawn token.  ``GrammarWalker``
is the same automaton on the host, bit for bit.  The blob layout, the row state and the caps are in
``include/tiny_llm_b200.h``."""

from __future__ import annotations

import numpy as np
import torch

from .constrained import MAX_REPEAT, utf8_sequences
from .json_mode import _zero_dfa

GRAMMAR_MAX_STATES = 32767  # state ids 1..32767 (0 is the dead state)
GRAMMAR_MAX_DEPTH = 32  # return-stack entries of one parse
GRAMMAR_MAX_PARSES = 8  # live parses of one row
GRAMMAR_MAX_TABLE_BYTES = 1 << 22  # the whole table blob
GRAMMAR_STATE_WORDS = 2 + GRAMMAR_MAX_PARSES + GRAMMAR_MAX_PARSES * GRAMMAR_MAX_DEPTH // 4  # int64 words of one row
GRAMMAR_SMEM_BYTES = 46 * 1024  # tables up to this size are staged in shared memory
_MAX_NFA_STATES = 1 << 20  # inlining and counted repetition stop here
_ACTIVE, _TERMINAL, _FAILED = 1 << 32, 1 << 33, 1 << 34
_INF = 255
_HEADER_BYTES = 16
_ANY = [(0, 0x10FFFF)]
_NAME_CHARS = frozenset("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789-")
_ESCAPES = {"n": 0x0A, "t": 0x09, "r": 0x0D, "\\": 0x5C, '"': 0x22, "[": 0x5B, "]": 0x5D, "-": 0x2D, "^": 0x5E}


# ------------------------------------------------------------------------------------------------------ parsing --
# AST: ("set", ranges) | ("cat", [nodes]) | ("alt", [nodes]) | ("rep", node, lo, hi or None) | ("ref", name, position).
class _Parser:
    def __init__(self, text: str):
        self.t, self.i = text, 0
        self.rule = None
        self.rules: dict = {}
        self.where: dict = {}

    def at(self, i: int | None = None) -> str:
        i = self.i if i is None else i
        line = self.t.count("\n", 0, i) + 1
        return f"line {line}, column {i - (self.t.rfind(chr(10), 0, i) + 1) + 1}"

    def error(self, what: str, i: int | None = None) -> ValueError:
        where = f"rule '{self.rule}': " if self.rule is not None else ""
        return ValueError(f"grammar {where}{what} at {self.at(i)}")

    def peek(self, k: int = 0):
        j = self.i + k
        return self.t[j] if j < len(self.t) else None

    def space(self, newlines: bool) -> None:
        while self.i < len(self.t):
            c = self.t[self.i]
            if c in " \t" or (newlines and c in "\r\n"):
                self.i += 1
            elif c == "#":
                while self.i < len(self.t) and self.t[self.i] not in "\r\n":
                    self.i += 1
            else:
                break

    def name(self) -> str:
        j = self.i
        while j < len(self.t) and self.t[j] in _NAME_CHARS:
            j += 1
        name, self.i = self.t[self.i : j], j
        return name

    def parse(self) -> None:
        self.space(True)
        while self.i < len(self.t):
            start = self.i
            self.rule = None
            name = self.name()
            if not name:
                raise self.error(f"expected a rule name, found {self.peek()!r}")
            self.space(False)
            if not self.t.startswith("::=", self.i):
                raise self.error(f"expected '::=' after rule name '{name}'")
            if name in self.rules:
                raise self.error(f"rule '{name}' is defined twice", start)
            self.i += 3
            self.rule = name
            self.space(True)
            self.rules[name] = self.alternatives(nested=False)
            self.where[name] = start
            self.space(False)
            if self.i < len(self.t) and self.t[self.i] not in "\r\n":
                raise self.error(f"unexpected {self.peek()!r}")
            self.space(True)
        self.rule = None

    def alternatives(self, nested: bool):
        branches = [self.sequence(nested)]
        while True:
            save = self.i
            self.space(True)  # an alternative may start on the next line with '|'
            if self.peek() != "|":
                self.i = save
                break
            self.i += 1
            self.space(True)
            branches.append(self.sequence(nested))
        return branches[0] if len(branches) == 1 else ("alt", branches)

    def sequence(self, nested: bool):
        items = []
        while True:
            self.space(nested)
            c = self.peek()
            if c is None or c in "|)" or c in "\r\n":
                break
            atom = self.atom()
            self.space(nested)
            q = self.quantifier()
            if q is not None:
                atom = ("rep", atom, *q)
                self.space(nested)
                if self.peek() in ("*", "+", "?", "{"):
                    raise self.error("multiple repeat")
            items.append(atom)
        return items[0] if len(items) == 1 else ("cat", items)

    def quantifier(self):
        c, start = self.peek(), self.i
        if c in ("*", "+", "?"):
            self.i += 1
            return {"*": (0, None), "+": (1, None), "?": (0, 1)}[c]
        if c != "{":
            return None
        self.i += 1
        self.space(False)
        lo = self.digits()
        if lo is None:
            raise self.error("expected a repeat count", start)
        hi = lo
        self.space(False)
        if self.peek() == ",":
            self.i += 1
            self.space(False)
            hi = self.digits()
            self.space(False)
        if self.peek() != "}":
            raise self.error("expected '}' to close the repeat count", start)
        self.i += 1
        if hi is not None and hi < lo:
            raise self.error("min repeat greater than max repeat", start)
        if lo > MAX_REPEAT or (hi is not None and hi > MAX_REPEAT):
            raise self.error(f"repeat counts above {MAX_REPEAT} are not supported", start)
        return lo, hi

    def digits(self):
        j = self.i
        while j < len(self.t) and self.t[j].isdigit() and self.t[j].isascii():
            j += 1
        if j == self.i:
            return None
        n, self.i = int(self.t[self.i : j]), j
        return n

    def atom(self):
        c, start = self.peek(), self.i
        if c == '"':
            self.i += 1
            chars = []
            while True:
                c = self.peek()
                if c is None or c in "\r\n":
                    raise self.error("unterminated string literal", start)
                if c == '"':
                    self.i += 1
                    break
                chars.append(("set", [(self.char(),) * 2]))
            return chars[0] if len(chars) == 1 else ("cat", chars)
        if c == "[":
            return ("set", self.char_class())
        if c == ".":
            self.i += 1
            return ("set", list(_ANY))
        if c == "(":
            self.i += 1
            self.space(True)
            node = self.alternatives(nested=True)
            self.space(True)
            if self.peek() != ")":
                raise self.error("missing ')'", start)
            self.i += 1
            return node
        if c == "<":
            raise self.error("token references (<...>, <[id]>) are not supported")
        if c in _NAME_CHARS:
            return ("ref", self.name(), start)
        if c in ("*", "+", "?", "{"):
            raise self.error("nothing to repeat")
        raise self.error(f"unexpected {c!r}")

    def char(self) -> int:
        """One code point of a literal or class at ``self.i`` (an escape or a raw character)."""
        c, start = self.peek(), self.i
        self.i += 1
        if c != "\\":
            return ord(c)
        e = self.peek()
        if e is None:
            raise self.error("bad escape (end of grammar)", start)
        self.i += 1
        if e in ("x", "u", "U"):
            width = {"x": 2, "u": 4, "U": 8}[e]
            digits = self.t[self.i : self.i + width]
            if len(digits) != width or any(d not in "0123456789abcdefABCDEF" for d in digits):
                raise self.error(f"incomplete escape \\{e}", start)
            self.i += width
            cp = int(digits, 16)
            if cp > 0x10FFFF:
                raise self.error(f"bad escape \\{e}{digits}", start)
            return cp
        if e in _ESCAPES:
            return _ESCAPES[e]
        raise self.error(f"bad escape \\{e}", start)

    def char_class(self):
        start = self.i
        self.i += 1
        negate = self.peek() == "^"
        if negate:
            self.i += 1
        ranges = []
        while True:
            c = self.peek()
            if c is None or c in "\r\n":
                raise self.error("unterminated character class", start)
            if c == "]":
                self.i += 1
                break
            lo = self.char()
            hi = lo
            if self.peek() == "-" and self.peek(1) not in (None, "]"):
                self.i += 1
                hi = self.char()
                if hi < lo:
                    raise self.error("bad character range", start)
            ranges.append((lo, hi))
        out = []
        for lo, hi in sorted(ranges):
            if out and lo <= out[-1][1] + 1:
                out[-1] = (out[-1][0], max(out[-1][1], hi))
            else:
                out.append((lo, hi))
        if negate:
            comp, nxt = [], 0
            for lo, hi in out:
                if lo > nxt:
                    comp.append((nxt, lo - 1))
                nxt = hi + 1
            if nxt <= 0x10FFFF:
                comp.append((nxt, 0x10FFFF))
            out = comp
        return out


def parse_grammar(text: str) -> dict:
    """The rules of a GBNF grammar: ``{name: AST}``, every reference defined and ``root`` present (``ValueError``
    otherwise, naming the rule and the position)."""
    if not isinstance(text, str):
        raise ValueError("grammar must be a str")
    p = _Parser(text)
    p.parse()
    if "root" not in p.rules:
        raise ValueError("grammar has no 'root' rule")

    def refs(node):
        if node[0] == "ref":
            yield node
        elif node[0] in ("cat", "alt"):
            for n in node[1]:
                yield from refs(n)
        elif node[0] == "rep":
            yield from refs(node[1])

    for name, ast in p.rules.items():
        for _, ref, pos in refs(ast):
            if ref not in p.rules:
                p.rule = name
                raise p.error(f"undefined rule '{ref}'", pos)
    return p.rules


def _refs(node, first: bool, nullable: dict) -> set:
    """Rule names referenced by ``node`` (``first``: only those that can be the first thing it matches)."""
    kind = node[0]
    if kind == "ref":
        return {node[1]}
    if kind == "set":
        return set()
    if kind == "rep":
        return set() if node[3] == 0 else _refs(node[1], first, nullable)
    out = set()
    for n in node[1]:
        out |= _refs(n, first, nullable)
        if first and kind == "cat" and not _nullable(n, nullable):
            break
    return out


def _nullable(node, nullable: dict) -> bool:
    kind = node[0]
    if kind == "set":
        return False
    if kind == "ref":
        return nullable[node[1]]
    if kind == "rep":
        return node[2] == 0 or _nullable(node[1], nullable)
    if kind == "cat":
        return all(_nullable(n, nullable) for n in node[1])
    return any(_nullable(n, nullable) for n in node[1])


# --------------------------------------------------------------------------------------------------- compiling --
class _Nfa:
    """Byte NFA with call edges: ``calls[p]`` holds (callee, return NFA state)."""

    def __init__(self):
        self.eps: list[list[int]] = []
        self.edges: list[list[tuple[int, int, int]]] = []
        self.calls: list[list[tuple[str, int]]] = []

    def state(self) -> int:
        if len(self.eps) >= _MAX_NFA_STATES:
            raise ValueError(f"grammar: inlining the rules exceeds {_MAX_NFA_STATES} automaton states")
        self.eps.append([])
        self.edges.append([])
        self.calls.append([])
        return len(self.eps) - 1


class _Compiler:
    def __init__(self, rules: dict):
        self.rules = rules
        reach, stack = {"root"}, ["root"]
        while stack:
            for r in _refs(rules[stack.pop()], False, {}):
                if r not in reach:
                    reach.add(r)
                    stack.append(r)
        self.names = sorted(reach)
        nullable = {n: False for n in self.names}
        changed = True
        while changed:
            changed = False
            for n in self.names:
                if not nullable[n] and _nullable(rules[n], nullable):
                    nullable[n] = changed = True
        self.nullable = nullable
        self.check_left_recursion()
        graph = {n: _refs(rules[n], False, nullable) for n in self.names}
        self.recursive = set()
        for n in self.names:
            seen, stack = set(), list(graph[n])
            while stack:
                m = stack.pop()
                if m == n:
                    self.recursive.add(n)
                    break
                if m not in seen:
                    seen.add(m)
                    stack.extend(graph[m])
        self.nfa = _Nfa()
        self.autos: dict = {}  # automaton name -> (NFA start, NFA final)
        for name in ["root"] + sorted(self.recursive - {"root"}):
            self.rule = name
            a, b = self.build(rules[name], ())
            self.autos[name] = (a, b)

    def check_left_recursion(self) -> None:
        first = {n: _refs(self.rules[n], True, self.nullable) for n in self.names}
        for n in self.names:
            seen = {n: None}  # rule -> the rule it was reached from
            stack = [(m, n) for m in sorted(first[n])]
            while stack:
                m, parent = stack.pop()
                if m in seen:
                    if m == n:
                        chain = [m]
                        p = parent
                        while p is not None:
                            chain.append(p)
                            p = seen[p]
                        chain.reverse()
                        raise ValueError(f"grammar rule '{n}': left recursion ({' -> '.join(chain)}): "
                                         "a rule may not reach itself before matching a character")
                    continue
                seen[m] = parent
                stack.extend((k, m) for k in sorted(first[m]))

    def build(self, node, inlining: tuple) -> tuple[int, int]:
        nfa = self.nfa
        kind = node[0]
        if kind == "set":
            a, b = nfa.state(), nfa.state()
            for lo, hi in node[1]:
                for seq in utf8_sequences(lo, hi):
                    cur = a
                    for j, (blo, bhi) in enumerate(seq):
                        nxt = b if j == len(seq) - 1 else nfa.state()
                        nfa.edges[cur].append((blo, bhi, nxt))
                        cur = nxt
            return a, b
        if kind == "ref":
            name = node[1]
            if name in self.recursive:
                a, b = nfa.state(), nfa.state()
                nfa.calls[a].append((name, b))
                if self.nullable[name]:
                    nfa.eps[a].append(b)
                return a, b
            return self.build(self.rules[name], inlining + (name,))
        if kind == "cat":
            a = cur = nfa.state()
            for item in node[1]:
                s, e = self.build(item, inlining)
                nfa.eps[cur].append(s)
                cur = e
            return a, cur
        if kind == "alt":
            a, b = nfa.state(), nfa.state()
            for item in node[1]:
                s, e = self.build(item, inlining)
                nfa.eps[a].append(s)
                nfa.eps[e].append(b)
            return a, b
        _, sub, lo, hi = node
        a = cur = nfa.state()
        for _ in range(lo):
            s, e = self.build(sub, inlining)
            nfa.eps[cur].append(s)
            cur = e
        end = nfa.state()
        nfa.eps[cur].append(end)
        if hi is None:
            s, e = self.build(sub, inlining)
            nfa.eps[cur].append(s)
            nfa.eps[e].append(cur)
        else:
            for _ in range(hi - lo):
                s, e = self.build(sub, inlining)
                nfa.eps[cur].append(s)
                cur = e
                nfa.eps[cur].append(end)
        return a, end

    def closure(self, states) -> frozenset:
        eps = self.nfa.eps
        seen, stack = set(states), list(states)
        while stack:
            for t in eps[stack.pop()]:
                if t not in seen:
                    seen.add(t)
                    stack.append(t)
        return frozenset(seen)


class CompiledGrammar:
    """The tables of one grammar: per state ``lists[s][class]`` (a tuple of actions ``(target, pushes, peak)``: go to
    ``target`` after pushing the return states ``pushes``, bottom first; ``peak`` the chain's need, checked against the
    depth cap), ``may_end[s]``, ``need[s]``, the byte classes, ``start`` and ``blob``, the device layout (DESIGN.md
    section 23):

    int32 num_states S (ids 0..S-1, 0 dead), num_classes C, blob bytes, action words A; uint8 class_of[256];
    uint32 info[S] (bit 0 the state's rule may end here, bits 8-15 need); uint32 trans[S, C] (0 no action, else bits
    0-23 the first action word, 24-31 the action count); uint32 acts[A] (per action a word: bits 0-14 target, 16-21
    pushes k, 24-31 peak; then ceil(k / 2) words of 16-bit return states, bottom first)."""

    def __init__(self, c: _Compiler):
        ids: dict = {}
        sets: list = [None]  # state 0: dead
        autos: list = [None]
        final_of = {name: b for name, (a, b) in c.autos.items()}
        nfa = c.nfa
        work: list = []

        def dstate(auto: str, nset: frozenset) -> int:
            sid = ids.get(nset)
            if sid is None:
                sid = ids[nset] = len(sets)
                if sid > GRAMMAR_MAX_STATES:
                    raise ValueError(f"grammar: the automaton exceeds {GRAMMAR_MAX_STATES} states")
                sets.append(nset)
                autos.append(auto)
                work.append(sid)
            return sid

        starts = {name: dstate(name, c.closure([a])) for name, (a, b) in c.autos.items()}
        self.start = starts["root"]
        cuts = {0, 256}
        for edges in nfa.edges:
            for lo, hi, _ in edges:
                cuts.update((lo, hi + 1))
        cuts = sorted(cuts)
        cut_classes = list(zip(cuts[:-1], cuts[1:]))
        memo: dict = {}
        calls_memo: dict = {}

        def calls_of(sid: int):
            if sid not in calls_memo:
                group: dict = {}
                for p in sorted(sets[sid]):
                    for callee, q in nfa.calls[p]:
                        group.setdefault(callee, []).append(q)
                calls_memo[sid] = [(callee, dstate(autos[sid], c.closure(qs))) for callee, qs in sorted(group.items())]
            return calls_memo[sid]

        def actions(sid: int, ci: int) -> tuple:
            key = (sid, ci)
            if key in memo:
                return memo[key]
            memo[key] = ()  # no left recursion: a chain never comes back to its own (state, class)
            byte = cut_classes[ci][0]
            out = []
            targets = [t for p in sets[sid] for lo, hi, t in nfa.edges[p] if lo <= byte <= hi]
            if targets:
                out.append((dstate(autos[sid], c.closure(targets)), ()))
            for callee, ret in calls_of(sid):
                for t, pushes in actions(starts[callee], ci):
                    out.append((t, (ret,) + pushes))
            seen = set()
            out = tuple(a for a in out if not (a in seen or seen.add(a)))
            memo[key] = out
            return out

        while work:
            sid = work.pop()
            for ci in range(len(cut_classes)):
                actions(sid, ci)
        S = len(sets)
        self.may_end = [False] + [final_of[autos[s]] in sets[s] for s in range(1, S)]
        raw = [[memo.get((s, ci), ()) for ci in range(len(cut_classes))] for s in range(S)]
        # need: min over completions of the peak extra stack height
        need = [_INF] * S
        for s in range(1, S):
            if self.may_end[s]:
                need[s] = 0

        def peak(t, pushes):
            k = len(pushes)
            return max([k + need[t]] + [j + need[r] for j, r in enumerate(pushes)])

        changed = True
        while changed:
            changed = False
            for s in range(1, S):
                best = need[s]
                for row in raw[s]:
                    for t, pushes in row:
                        best = min(best, peak(t, pushes))
                if best < need[s]:
                    need[s], changed = best, True
        self.need = [min(n, _INF) for n in need]
        if self.need[self.start] >= _INF:
            raise ValueError("grammar: the language of 'root' is empty")
        if self.need[self.start] > GRAMMAR_MAX_DEPTH:
            raise ValueError(f"grammar: no complete text fits the depth cap of {GRAMMAR_MAX_DEPTH}")
        # drop the actions no parse can take (past the depth cap from depth 0, or into states that never complete)
        lists = [[tuple((t, pushes, peak(t, pushes)) for t, pushes in row if peak(t, pushes) <= GRAMMAR_MAX_DEPTH) for row in rows]
                 for rows in raw]
        # byte classes: cut classes every state treats alike
        cols: dict = {}
        cls_of_cut = []
        for ci in range(len(cut_classes)):
            col = tuple(lists[s][ci] for s in range(S))
            cls_of_cut.append(cols.setdefault(col, len(cols)))
        C = len(cols)
        class_of = np.zeros(256, dtype=np.uint8)
        for ci, (lo, hi) in enumerate(cut_classes):
            class_of[lo:hi] = cls_of_cut[ci]
        self.class_of = class_of
        first_cut = {}
        for ci, k in enumerate(cls_of_cut):
            first_cut.setdefault(k, ci)
        self.lists = [[lists[s][first_cut[k]] for k in range(C)] for s in range(S)]
        # device tables
        acts: list = []
        offsets: dict = {}
        trans = np.zeros((S, C), dtype=np.uint32)
        for s in range(S):
            for k in range(C):
                row = self.lists[s][k]
                if not row:
                    continue
                if row not in offsets:
                    offsets[row] = len(acts)
                    for t, pushes, pk in row:
                        acts.append(t | len(pushes) << 16 | pk << 24)
                        for j in range(0, len(pushes), 2):
                            acts.append(pushes[j] | (pushes[j + 1] << 16 if j + 1 < len(pushes) else 0))
                    if len(acts) >= 1 << 24:
                        raise ValueError(f"grammar: the tables take more than {GRAMMAR_MAX_TABLE_BYTES} bytes")
                trans[s, k] = offsets[row] | len(row) << 24
        A = len(acts)
        info = np.array([(1 if self.may_end[s] else 0) | (self.need[s] << 8) for s in range(S)], dtype=np.uint32)
        nbytes = _HEADER_BYTES + 256 + 4 * S + 4 * S * C + 4 * A
        nbytes = (nbytes + 15) // 16 * 16
        if nbytes > GRAMMAR_MAX_TABLE_BYTES:
            raise ValueError(f"grammar: the tables take {nbytes} bytes, above the limit of {GRAMMAR_MAX_TABLE_BYTES}")
        blob = np.zeros(nbytes, dtype=np.uint8)
        blob[:16] = np.array([S, C, nbytes, A], dtype=np.int32).view(np.uint8)
        at = 16
        blob[at : at + 256] = class_of
        at += 256
        blob[at : at + 4 * S] = info.view(np.uint8)
        at += 4 * S
        blob[at : at + 4 * S * C] = trans.reshape(-1).view(np.uint8)
        at += 4 * S * C
        blob[at : at + 4 * A] = np.array(acts, dtype=np.uint32).view(np.uint8)
        self.blob = blob
        self._class_list = [int(x) for x in class_of]
        self._steps: dict = {}

    @property
    def num_states(self) -> int:
        return len(self.lists)

    @property
    def num_classes(self) -> int:
        return len(self.lists[0])

    def step_set(self, parses: tuple, b: int):
        """The parse set after byte ``b`` from ``parses`` (a tuple of ``(state, stack)``), or None when no parse
        survives or more than ``GRAMMAR_MAX_PARSES`` distinct parses would remain."""
        c = self._class_list[b]
        key = (parses, c)
        hit = self._steps.get(key, False)
        if hit is not False:
            return hit
        out: list = []
        seen = set()
        dead = False
        for s, stack in parses:
            while True:
                for t, pushes, pk in self.lists[s][c]:
                    if len(stack) + pk <= GRAMMAR_MAX_DEPTH:
                        p = (t, stack + pushes)
                        if p not in seen:
                            if len(out) == GRAMMAR_MAX_PARSES:
                                dead = True
                                break
                            seen.add(p)
                            out.append(p)
                if dead or not (self.may_end[s] and stack):
                    break
                s, stack = stack[-1], stack[:-1]
            if dead:
                break
        res = None if dead or not out else tuple(out)
        if len(self._steps) > 1 << 20:
            self._steps.clear()
        self._steps[key] = res
        return res

    def complete(self, parses: tuple) -> bool:
        """Some parse has finished ``root`` at depth 0 (returning through states whose rule may end)."""
        for s, stack in parses:
            while self.may_end[s]:
                if not stack:
                    return True
                s, stack = stack[-1], stack[:-1]
        return False


def compile_grammar(text: str) -> CompiledGrammar:
    """The pushdown automaton of a GBNF grammar.  Raises ``ValueError`` naming the rule (and the position where it has
    one) for syntax outside the supported subset, undefined rules, a missing ``root``, token references, left
    recursion, an empty language and every cap (DESIGN.md section 23)."""
    return CompiledGrammar(_Compiler(parse_grammar(text)))


# -------------------------------------------------------------------------------------------------- walker --
class GrammarWalker:
    """One row's parse set, mutable: ``parses`` (a tuple of ``(state, stack)``, stack a tuple of return states, bottom
    first), ``terminal`` (after EOS) and ``failed`` (a drawn token was not allowed: only past the parse cap); ``step``
    and ``walk`` return False once the text leaves the language or the parse cap."""

    __slots__ = ("tables", "parses", "terminal", "failed")

    def __init__(self, tables: CompiledGrammar, words=None):
        self.tables = tables
        if words is None:
            self.parses, self.terminal, self.failed = ((tables.start, ()),), False, False
            return
        w = [int(x) & (1 << 64) - 1 for x in words]
        n = w[1] & 15
        self.terminal, self.failed = bool(w[1] & _TERMINAL), bool(w[1] & _FAILED)
        parses = []
        for p in range(n):
            s, depth = w[2 + p] & 0x7FFF, (w[2 + p] >> 16) & 63
            stack = tuple((w[2 + GRAMMAR_MAX_PARSES + (p * GRAMMAR_MAX_DEPTH + k) // 4] >> (16 * (k % 4))) & 0xFFFF for k in range(depth))
            parses.append((s, stack))
        self.parses = tuple(parses)

    def copy(self) -> GrammarWalker:
        w = GrammarWalker.__new__(GrammarWalker)
        w.tables, w.parses, w.terminal, w.failed = self.tables, self.parses, self.terminal, self.failed
        return w

    def words(self, tables_ptr: int) -> tuple:
        """The ``GRAMMAR_STATE_WORDS`` int64 words of the device state (signed), with ``tables_ptr`` in word 0."""
        w = [0] * GRAMMAR_STATE_WORDS
        w[0] = tables_ptr
        w[1] = len(self.parses) | _ACTIVE | (_TERMINAL if self.terminal else 0) | (_FAILED if self.failed else 0)
        for p, (s, stack) in enumerate(self.parses):
            w[2 + p] = s | len(stack) << 16
            for k, r in enumerate(stack):
                w[2 + GRAMMAR_MAX_PARSES + (p * GRAMMAR_MAX_DEPTH + k) // 4] |= r << (16 * (k % 4))
        return tuple(x - (1 << 64) if x >= 1 << 63 else x for x in w)

    @property
    def complete(self) -> bool:
        return not self.terminal and self.tables.complete(self.parses)

    @property
    def depth(self) -> int:
        return max((len(stack) for _, stack in self.parses), default=0)

    def step(self, b: int) -> bool:
        nxt = self.tables.step_set(self.parses, b)
        if nxt is None:
            self.parses = ()
            return False
        self.parses = nxt
        return True

    def walk(self, data: bytes) -> bool:
        if self.terminal or self.failed or not self.parses:
            return False
        for b in data:
            if not self.step(b):
                return False
        return True


# ------------------------------------------------------------------------------------------------ vocabulary --
def check_vocabulary(tables: CompiledGrammar, vocabulary) -> None:
    """Refuse (``ValueError``) a vocabulary that could leave a reachable state with no allowed token: no EOS id, or no
    one-byte token for a byte the tables demand.  A byte is demanded when, without the byte classes that have no
    one-byte token, some state can no longer complete within its depth need (DESIGN.md section 21's rule)."""
    if not vocabulary.eos_ids:
        raise ValueError("grammar mode needs a vocabulary with an EOS id")
    singles = set()
    for tok in vocabulary.tokens:
        if tok is not None and len(tok) == 1:
            singles.add(tok[0])
    C = tables.num_classes
    spelled = [False] * C
    for b in singles:
        spelled[tables._class_list[b]] = True
    S = tables.num_states
    need = [_INF] * S
    for s in range(1, S):
        if tables.may_end[s]:
            need[s] = 0
    changed = True
    while changed:
        changed = False
        for s in range(1, S):
            for k in range(C):
                if not spelled[k]:
                    continue
                for t, pushes, _ in tables.lists[s][k]:
                    n = max([len(pushes) + need[t]] + [j + need[r] for j, r in enumerate(pushes)])
                    if n < need[s]:
                        need[s], changed = n, True
    missing = set()
    for s in range(1, S):
        if tables.need[s] < _INF and need[s] > tables.need[s]:
            for k in range(C):
                if tables.lists[s][k] and not spelled[k]:
                    missing.update(b for b in range(256) if tables._class_list[b] == k)
    if missing:
        shown = "".join(chr(x) if 0x20 <= x < 0x7F else f"\\x{x:02x}" for x in sorted(missing))
        raise ValueError(f"grammar mode needs a one-byte token for one of {shown!r}: the grammar can demand one of those bytes next")


class GrammarConstraint:
    """A GBNF grammar over one vocabulary: ``SamplingParams(constraint=GrammarConstraint(grammar, vocabulary))``.
    Compiles the grammar once and holds the device tables (``tables``, uint8), the vocabulary's device CSR and its
    EOS-only mask row; the per-row parse sets and mask buffers live with each caller's ``ConstraintRows``."""

    def __init__(self, grammar: str, vocabulary, device="cuda"):
        self.grammar = grammar
        self.compiled = compile_grammar(grammar)
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
        self._sorted = None

    @property
    def vocab_size(self) -> int:
        return self.vocabulary.size

    def start(self) -> GrammarWalker:
        return GrammarWalker(self.compiled)

    def words(self, walker: GrammarWalker) -> tuple:
        return walker.words(self.tables.data_ptr())

    def walk(self, token_ids, walker: GrammarWalker | None = None) -> GrammarWalker | None:
        """The parse set after ``token_ids`` from ``walker`` (default: the start), or None when a token is not
        allowed."""
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

    def allowed(self, walker: GrammarWalker) -> np.ndarray:
        """bool ``[V]``: the tokens allowed after ``walker`` (what the device mask holds).  Walks the vocabulary in
        byte order, sharing each token's common prefix with the one before."""
        out = np.zeros(self.vocab_size, dtype=bool)
        if walker.terminal:
            out[self.vocabulary.eos_ids] = True
            return out
        if walker.failed or not walker.parses:
            return out
        if walker.complete:
            out[self.vocabulary.eos_ids] = True
        if self._sorted is None:
            self._sorted = sorted((t, i) for i, t in enumerate(self.vocabulary.tokens) if t is not None)
        t = self.compiled
        prev = b""
        states = [walker.parses]  # states[j]: the parse set after j bytes of prev (None: dead)
        for tok, i in self._sorted:
            lcp = 0
            m = min(len(tok), len(prev))
            while lcp < m and tok[lcp] == prev[lcp]:
                lcp += 1
            del states[lcp + 1 :]
            for j in range(lcp, len(tok)):
                cur = states[j]
                states.append(None if cur is None else t.step_set(cur, tok[j]))
            prev = tok
            out[i] = states[len(tok)] is not None
        return out


def failed_rows(states: torch.Tensor) -> list[int]:
    """The rows of grammar states (int64 ``[R, GRAMMAR_STATE_WORDS]``) whose failed bit is set (one device read)."""
    return torch.nonzero((states[:, 1] >> 34) & 1).flatten().tolist()


def load_grammar_arg(text: str) -> str:
    """A grammar from a CLI argument: inline text when it holds '::=', else a file path."""
    if "::=" in text:
        return text
    with open(text, encoding="utf-8") as f:
        return f.read()
