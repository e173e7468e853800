"""Plain-loop statement of prompt lookup's proposer (``tl_ngram_propose``, DESIGN.md section 14).

For a history ``s[0..L)`` (the prompt and every emitted token; the last entry is the pending token):

1. for each ``e`` in ``[0, L-2]``, ``c(e)`` is the largest ``t <= min(n_max, e+1)`` with ``s[e-t+1..e] == s[L-t..L-1]``
   (0 when ``s[e] != s[L-1]``);
2. no ``e`` with ``c(e) >= n_min``: no match (length 0, no proposals);
3. otherwise ``e*`` maximises ``(c(e), e)``: the longest suffix match, then its latest occurrence;
4. ``p_t = s'[e*+1+t]`` for ``t < k``, ``s'`` being ``s`` followed by ``p`` itself: a continuation that runs past the
   history repeats the matched period, so a match always yields exactly ``k`` proposals.
"""

from __future__ import annotations


def match_length(s, e: int, n_max: int) -> int:
    L = len(s)
    c = 0
    for t in range(1, min(n_max, e + 1) + 1):
        if all(s[e - t + 1 + j] == s[L - t + j] for j in range(t)):
            c = t
    return c


def propose(s, k: int, n_min: int, n_max: int) -> tuple[int, int, list[int]]:
    """``(c(e*), e*, [p_0..p_{k-1}])``; ``(0, -1, [])`` when nothing matches."""
    s = [int(t) for t in s]
    L = len(s)
    best = None
    for e in range(0, L - 1):
        c = match_length(s, e, n_max)
        if c >= n_min and (best is None or (c, e) > best):
            best = (c, e)
    if best is None:
        return 0, -1, []
    c, e = best
    ext = list(s)
    for t in range(k):
        ext.append(ext[e + 1 + t])
    return c, e, ext[L:]


def propose_np(s, k: int, n_min: int, n_max: int) -> tuple[int, int, list[int]]:
    """``propose`` with the match lengths of all ends at once (numpy), for histories of 100K tokens and more."""
    import numpy as np

    s = np.asarray(s, dtype=np.int64)
    L = len(s)
    if L < 2:
        return 0, -1, []
    e = np.arange(L - 1)
    c = np.zeros(L - 1, dtype=np.int64)
    alive = np.ones(L - 1, dtype=bool)
    for t in range(min(n_max, L - 1)):  # c(e) counts the leading run of s[e - t] == s[L - 1 - t] while t < e + 1
        ok = alive & (e - t >= 0)
        ok[ok] = s[e[ok] - t] == s[L - 1 - t]
        c += ok
        alive = ok
    cand = np.flatnonzero(c >= n_min)
    if cand.size == 0:
        return 0, -1, []
    best = cand[np.lexsort((cand, c[cand]))[-1]]
    out = list(s.tolist())
    for t in range(k):
        out.append(out[best + 1 + t])
    return int(c[best]), int(best), out[L:]
