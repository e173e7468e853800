"""Restatement of DRY and XTC (DESIGN.md section 24), in numpy, plus an independent brute-force port of
text-generation-webui's DRY loop.

TEST INFRASTRUCTURE.  ``dry_penalize`` is the contract: every token t with l*(t) >= a becomes fl32(x_t - P[l*(t) - a])
(-inf when that P is +inf), one fp32 subtraction each, so the restated row is exact.  ``xtc_sample_row`` is the
penalised draw of ``penalties_ref`` with XTC's exclusion on the exact float64 softmax over the keep set; the kernel
decides p_i >= theta on 2^-40 fixed-point masses, so draws with a p_i within ``XTC_BOUND`` of theta are reported as
near a boundary rather than compared.
"""

from __future__ import annotations

import importlib.util
import sys
from pathlib import Path

import numpy as np

from oracle import sampling as ref


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


penalties_ref = _load("tiny_llm_b200_penalties_ref", "penalties_ref.py")

MAX_MATCH = 64
XTC_BOUND = 2.0**-20
XTC_STREAM = 3


def penalty_table(m: float, b: float, a: int) -> np.ndarray:
    out = np.zeros(MAX_MATCH, dtype=np.float32)
    for k in range(MAX_MATCH - a + 1):
        try:
            v = m * b**k
        except OverflowError:
            v = np.inf
        with np.errstate(over="ignore"):
            out[k] = np.float32(v)
    return out


def match_lengths(hist, breakers, last_n: int = 0, cap: int = MAX_MATCH) -> dict:
    """``{t: l*(t)}`` of the contract over history ``hist`` (``hist[-1]`` the step's input token)."""
    h = [int(t) for t in hist]
    n = len(h)
    B = set(int(t) for t in breakers)
    if n == 0 or h[-1] in B:
        return {}
    lo = 0 if last_n == 0 else max(0, n - last_n)
    best: dict = {}
    for e in range(lo, n - 1):
        t = h[e + 1]
        if t in B:
            continue
        l = 0
        while l < cap and e - l >= lo and h[e - l] == h[n - 1 - l] and h[n - 1 - l] not in B:
            l += 1
        if l > best.get(t, -1):
            best[t] = l
    return best


def dry_penalize(x, hist, m: float, b: float, a: int, last_n: int = 0, breakers=()) -> np.ndarray:
    """The row ``tl_dry_penalty`` leaves: fp32 ``x`` with the contract's penalties."""
    y = np.array(x, dtype=np.float32, copy=True)
    P = penalty_table(m, b, a)
    for t, l in match_lengths(hist, breakers, last_n).items():
        if l >= a and 0 <= t < len(y):
            p = P[l - a]
            y[t] = -np.inf if np.isinf(p) else np.float32(y[t] - p)
    return y


def webui_dry(x, hist, m: float, b: float, a: int, last_n: int = 0, breakers=(), cap: int = MAX_MATCH) -> np.ndarray:
    """Brute-force port of text-generation-webui's ``DRYLogitsProcessor`` loop (window, breakers, a cap on the match
    length), written from its description independently of ``match_lengths``: walk back from the end of the window for
    the breaker-free suffix, then for every earlier occurrence of the last token grow the match backwards and record
    the longest match per following token."""
    y = np.array(x, dtype=np.float32, copy=True)
    seq = [int(t) for t in hist]
    if last_n > 0:
        seq = seq[-last_n:]
    B = set(int(t) for t in breakers)
    if not seq or seq[-1] in B:
        return y
    # the longest suffix free of breakers bounds every match
    free = 0
    for t in reversed(seq):
        if t in B:
            break
        free += 1
    free = min(free, cap)
    longest: dict = {}
    last = seq[-1]
    for idx in range(len(seq) - 1):  # idx: an earlier occurrence of the last token
        if seq[idx] != last:
            continue
        nxt = seq[idx + 1]
        if nxt in B:
            continue
        length = 1
        while length < free and idx - length >= 0 and seq[idx - length] == seq[-1 - length]:
            length += 1
        longest[nxt] = max(longest.get(nxt, 0), length)
    for t, length in longest.items():
        if length >= a and 0 <= t < len(y):
            p = np.float32(m * b ** (length - a)) if length - a < 2000 else np.float32(np.inf)
            y[t] = -np.inf if np.isinf(p) else np.float32(y[t] - p)
    return y


def xtc_uniform(seed: int, pos: int) -> float:
    w = ref.philox4x32_10(np.array([[0, pos & 0xFFFFFFFF, XTC_STREAM, 0]], dtype=np.uint64), (seed & 0xFFFFFFFF, seed >> 32))[0, 0]
    return (2.0 * float(int(w) >> 9) + 1.0) * 2.0**-24


def xtc_keep(x3, keep, temperature: float, threshold: float, probability: float, seed: int, pos: int):
    """``(keep', near)``: the keep set after XTC and whether some kept p_i lies within ``XTC_BOUND`` of the
    threshold (the kernel's fixed-point decision may differ there)."""
    if not probability > 0 or not xtc_uniform(seed, pos) < probability:
        return keep, False
    x = np.asarray(x3, dtype=np.float64)
    m = x[keep].max()
    e = np.where(keep, np.exp((np.where(keep, x, m) - m) / temperature), 0.0)
    p = e / e.sum()
    near = bool(np.any(keep & (np.abs(p - threshold) <= XTC_BOUND)))
    A = keep & (p >= threshold)
    if A.sum() < 2:
        return keep, near
    lowest = x[A].min()
    return keep & ~(A & (x > lowest)), near


def xtc_sample_row(x, state, temperature, top_k, top_p, seed, pos, r=1.0, pres=0.0, freq=0.0, min_p=0.0, threshold=0.1,
                   probability=0.0, allowed=None):
    """``(token, near)`` of the penalised (or, with ``allowed``, constrained) draw with XTC on one fp32 row."""
    x3 = penalties_ref.penalize(x, state, r, pres, freq)
    if allowed is not None:
        x3 = np.where(allowed, x3, np.float32(np.nan)).astype(np.float32)
    x64 = x3.astype(np.float64)
    ok = ~np.isnan(x64)
    if not temperature > 0 or not ok.any() or not np.isfinite(x64[ok].max()):
        return ref.greedy(x64), False
    keep = penalties_ref.keep_set(x3, top_k, top_p, min_p, temperature)
    keep, near = xtc_keep(x3, keep, temperature, threshold, probability, seed, pos)
    score = np.where(keep, ref.perturbed(x64, temperature, seed, pos), -np.inf)
    return int(np.argmax(score)), near
