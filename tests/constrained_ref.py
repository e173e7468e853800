"""References for regex-constrained generation: a per-token host walk of the token masks (independent of the NumPy
lifting in ``tiny_llm_b200.constrained.token_masks_reference``), seeded test strings, and the constrained draw as
``oracle/sampling.py`` applied to the row with disallowed entries set to -inf."""

from __future__ import annotations

import numpy as np

PATTERNS = [
    r"abc",
    r"a|b|cd",
    r"[0-9]{4}-[0-9]{2}-[0-9]{2}",
    r"\d+(\.\d{1,3})?",
    r"(ab|cd)*e?",
    r"x{2,4}y{0,2}z{3,}",
    r"[^a-c\n]{1,3}",
    r"(?:yes|no|maybe)",
    r"\w+@\w+\.(com|org)",
    r"\s*\S+\s*",
    r"[a-f\d]{2,}|\D\W",
    r"(a(b(c|d)*)+)?e",
    r".{0,4}!",
    r"é+ж?[α-ω]",
    r"[^é]{2}",
    r"\{\d\}\.\*\[\]",
    r"(?P<x>ab)+?c*?d??",
    r"[-a]+[b-]",
]

ALPHABET_EXTRA = ["é", "ж", "α", "ω", "λ", "中", "😀", "\n", " ", "\t"]


def pattern_alphabet(pattern: str) -> list[str]:
    """The characters a pattern's test strings are drawn from: those it names, near neighbours and some non-ASCII."""
    chars = set(c for c in pattern if c not in "\\")
    chars |= set("abcdexyz0123456789-.@_!{}[]*")
    return sorted(chars) + ALPHABET_EXTRA


def random_strings(pattern: str, n: int, seed: int, max_len: int = 12) -> list[str]:
    rng = np.random.default_rng(seed)
    alphabet = pattern_alphabet(pattern)
    out = []
    for _ in range(n):
        k = int(rng.integers(0, max_len + 1))
        out.append("".join(alphabet[j] for j in rng.integers(0, len(alphabet), k)))
    return out


def token_masks_walk(dfa, vocabulary) -> tuple[np.ndarray, np.ndarray]:
    """Token masks and reach sets by walking every (state, token) on its own: uint32 ``[S + 1, ceil(V / 32)]`` and
    uint32 ``[S, ceil(S / 32)]``."""
    S, V = dfa.num_states, vocabulary.size
    masks = np.zeros((S + 1, (V + 31) // 32), dtype=np.uint32)
    reach = np.zeros((S, (S + 31) // 32), dtype=np.uint32)
    eos = set(vocabulary.eos_ids)

    def put(a, r, c):
        a[r, c >> 5] |= np.uint32(1 << (c & 31))

    for s in range(S):
        for t, data in enumerate(vocabulary.tokens):
            if t in eos:
                if dfa.accept[s]:
                    put(masks, s, t)
            elif data is not None:
                e = dfa.walk(s, data)
                if e >= 0:
                    put(masks, s, t)
                    put(reach, s, e)
    for t in eos:
        put(masks, S, t)
    return masks, reach


def allowed_bits(masks: np.ndarray, state: int, vocab: int) -> np.ndarray:
    """bool ``[vocab]``: the tokens row ``state`` of ``masks`` allows."""
    row = np.asarray(masks).view(np.uint32)[state]
    return np.unpackbits(row.view(np.uint8), bitorder="little")[:vocab].astype(bool)
