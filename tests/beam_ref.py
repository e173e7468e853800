"""Beam search in plain loops: the rule ``tl_beam_select`` and ``beam_search_ids`` implement (DESIGN.md section 15).

* ``select``: one step's candidates.  Row r's entries ``(top_ids[r, k], top_lp[r, k])`` are ``tl_logprobs``' top-N
  lists, N = W + E; a candidate scores ``s = fl(cum[r] + top_lp[r, k])`` in fp32 and is never taken with id -1 or an
  s of -inf or NaN.  The takeable ones are walked in the order (s descending, r ascending, k ascending), p the
  position: an EOS at p < W finishes a hypothesis, an EOS at p >= W is skipped, any other id becomes a live beam while
  fewer than W are live.
* ``search``: the whole search over a function giving each step's top-N lists, with the scoring, the kept pool of at
  most W finished hypotheses, the stopping rule and the length limit.
* ``beam_select_like_ext``: ``tiny_llm_ext_b200.beam_select``'s surface on CPU tensors (test stand-in).
"""

from __future__ import annotations

import math

import numpy as np

MAX_WIDTH = 8
RESULT_WORDS = 2 + 7 * MAX_WIDTH


def select(top_lp, top_ids, cum, width: int, eos):
    """-> ``(live, finished)``: live ``(parent, token, cum)`` and finished ``(parent, eos id, sum, position)``."""
    top_lp = np.asarray(top_lp, dtype=np.float32)
    top_ids = np.asarray(top_ids)
    cum = np.asarray(cum, dtype=np.float32)
    eos = {int(t) for t in eos}
    candidates = []
    for r in range(top_lp.shape[0]):
        for k in range(top_lp.shape[1]):
            token = int(top_ids[r, k])
            s = np.float32(cum[r] + top_lp[r, k])  # one fp32 rounding
            if token < 0 or math.isnan(s) or s == -math.inf:
                continue
            candidates.append((float(s), r, k, token))
    # s descending, then r, then k: a stable sort on r, k first, then on s alone
    candidates.sort(key=lambda c: (c[1], c[2]))
    candidates.sort(key=lambda c: -c[0])
    live, finished = [], []
    for p, (s, r, _, token) in enumerate(candidates):
        if token in eos:
            if p < width:
                finished.append((r, token, s, p))
            continue
        if len(live) == width:
            break
        live.append((r, token, s))
    return live, finished


def new_cum(live, width: int) -> np.ndarray:
    """``cum`` after a select: the live beams' sums, then -inf."""
    out = np.full(width, -np.inf, dtype=np.float32)
    for j, (_, _, s) in enumerate(live):
        out[j] = s
    return out


def pack(live, finished) -> np.ndarray:
    """The packed result block of ``tl_beam_select``."""
    w = np.zeros(RESULT_WORDS, dtype=np.int32)
    f = w.view(np.float32)
    M = MAX_WIDTH
    w[0], w[1] = len(live), len(finished)
    for j, (parent, token, s) in enumerate(live):
        w[2 + j], w[2 + M + j], f[2 + 2 * M + j] = parent, token, s
    b = 2 + 3 * M
    for j, (parent, token, s, p) in enumerate(finished):
        w[b + j], w[b + M + j], f[b + 2 * M + j], w[b + 3 * M + j] = parent, token, s, p
    return w


def beam_select_like_ext(top_lp, top_ids, cum, num_beams, eos_ids, out, stream=None):
    """``tiny_llm_ext_b200.beam_select`` on CPU tensors: same result block, same in-place ``cum``."""
    import torch

    live, finished = select(top_lp.cpu().numpy(), top_ids.cpu().numpy(), cum.cpu().numpy(), num_beams, eos_ids)
    out.copy_(torch.from_numpy(pack(live, finished)))
    cum.copy_(torch.from_numpy(new_cum(live, num_beams)))
    return out


def score(total: float, length: int, length_penalty: float) -> float:
    return float(total) / (float(length) ** length_penalty)


def search(tops, max_new_tokens: int, width: int, length_penalty: float = 1.0, early_stopping: bool = False,
           num_return_sequences: int = 1, eos=()):
    """The whole search.  ``tops(beams)`` takes the live beams' generated ids (``[[]]`` at step 0) and returns their
    top-N lists ``(top_lp [R, N], top_ids [R, N])``.  Returns ``[(ids, sum, score, finished)]``, best first."""
    if max_new_tokens == 0:
        return []
    eos = list(dict.fromkeys(int(t) for t in eos))
    pool = []  # (ids, sum, score, finished, order)
    beams = [([], 0.0)]
    step = 0
    while True:
        top_lp, top_ids = tops([ids for ids, _ in beams])
        live, finished = select(top_lp, top_ids, [c for _, c in beams], width, eos)
        for parent, _, s, p in finished:
            ids = beams[parent][0]
            pool.append((list(ids), s, score(s, len(ids) + 1, length_penalty), True, (step, p)))
            pool.sort(key=lambda h: (-h[2], h[4]))
            del pool[width:]
        step += 1
        beams_next = [(beams[parent][0] + [token], s) for parent, token, s in live]
        if not beams_next:
            break
        if len(pool) == width:
            best_live = max(score(s, len(ids), length_penalty) for ids, s in beams_next)
            if early_stopping or best_live <= pool[-1][2]:
                break
        if step == max_new_tokens:
            for j, (ids, s) in enumerate(beams_next):
                pool.append((ids, s, score(s, len(ids), length_penalty), False, (max_new_tokens, j)))
            pool.sort(key=lambda h: (-h[2], h[4]))
            del pool[width:]
            break
        beams = beams_next
    return [h[:4] for h in pool[:num_return_sequences]]
