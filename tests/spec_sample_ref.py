"""Float64 restatement of speculative sampling (``tl_speculative_sample``, DESIGN.md section 8d), built on the
float64 sampling oracle (``oracle/sampling.py``).

One verify row j has the target row ``x``, the draft row ``y`` that proposal ``d`` was drawn from, one request's
parameters and ``pos = n_j``, the position of the token the row predicts:

* ``p = row_dist(x)``, ``q = row_dist(y)``: the point mass at ``greedy(row)`` when the temperature is 0 or the row's
  maximum is not finite, else ``exp((x - m) / T)`` normalised over ``keep_set(x, top_k, top_p)``;
* accept iff ``q_d > 0`` and ``u q_d <= p_d``, ``u`` from word 0 of Philox at counter ``(0, pos, 1, 0)``;
* else the residual: argmax over ``{i : p_i > q_i}`` of ``log(p_i - q_i) + g_i``, ``g_i`` from stream 2 (counter
  ``(i >> 2, pos, 2, 0)``); an empty set (which exact arithmetic never leaves after a rejection) gives ``greedy(x)``.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np

from oracle import sampling as S

STREAM_DRAW, STREAM_ACCEPT, STREAM_RESIDUAL = 0, 1, 2


def stream_words(vocab: int, seed: int, pos: int, stream: int) -> np.ndarray:
    """Word ``i % 4`` of Philox4x32-10 at counter ``(i >> 2, pos, stream, 0)`` for ``i < vocab`` (uint64)."""
    groups = (vocab + 3) // 4
    ctr = np.zeros((groups, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(groups, dtype=np.uint64)
    ctr[:, 1] = pos & 0xFFFFFFFF
    ctr[:, 2] = stream
    return S.philox4x32_10(ctr, (seed & 0xFFFFFFFF, seed >> 32)).reshape(-1)[:vocab].astype(np.uint64)


def to_uniform(words) -> np.ndarray:
    return (2.0 * (np.asarray(words, dtype=np.uint64) >> np.uint64(9)).astype(np.float64) + 1.0) * 2.0**-24


def accept_uniform(seed: int, pos: int, stream: int = STREAM_ACCEPT) -> float:
    return float(to_uniform(stream_words(1, seed, pos, stream))[0])


def residual_gumbel(vocab: int, seed: int, pos: int, stream: int = STREAM_RESIDUAL) -> np.ndarray:
    return -np.log(-np.log(to_uniform(stream_words(vocab, seed, pos, stream))))


def is_point(x, temperature: float) -> bool:
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    return not temperature > 0 or not ok.any() or not np.isfinite(x[ok].max())


def row_dist(x, temperature: float, top_k: int | None, top_p: float | None) -> np.ndarray:
    """The distribution ``tl_sample`` draws from on row ``x`` (float64 ``[V]``)."""
    x = np.asarray(x, dtype=np.float64)
    out = np.zeros(len(x))
    if is_point(x, temperature):
        out[S.greedy(x)] = 1.0
        return out
    keep = S.keep_set(x, top_k, top_p)
    m = x[~np.isnan(x)].max()
    e = np.where(keep, np.exp((np.where(keep, x, m) - m) / temperature), 0.0)
    return e / e.sum()


@dataclass
class Decision:
    token: int
    accepted: bool
    margin: float  # |u q_d - p_d|: how far the acceptance test was from flipping
    residual_gap: float  # top-two gap of the residual scores (inf when accepted or a single candidate)


def decide(p, q, d: int, seed: int, pos: int, fallback: int, accept_stream: int = STREAM_ACCEPT,
           residual_stream: int = STREAM_RESIDUAL) -> Decision:
    """The rule on given distributions (the streams are parameters so a test can show why they must differ)."""
    p, q = np.asarray(p, dtype=np.float64), np.asarray(q, dtype=np.float64)
    V = len(p)
    pd = p[d] if 0 <= d < V else 0.0
    qd = q[d] if 0 <= d < V else 0.0
    u = accept_uniform(seed, pos, accept_stream)
    margin = abs(u * qd - pd)
    if qd > 0 and u * qd <= pd:
        return Decision(d, True, margin, np.inf)
    cand = p > q
    if not cand.any():
        return Decision(fallback, False, margin, np.inf)
    score = np.where(cand, np.log(np.where(cand, p - q, 1.0)) + residual_gumbel(V, seed, pos, residual_stream), -np.inf)
    order = np.argsort(-score, kind="stable")
    gap = score[order[0]] - score[order[1]] if cand.sum() > 1 else np.inf
    return Decision(int(order[0]), False, margin, float(gap))


def rule_row(x, y, d: int, temperature: float, top_k: int | None, top_p: float | None, seed: int, pos: int, **streams) -> Decision:
    """One verify row j < k."""
    p = row_dist(x, temperature, top_k, top_p)
    q = row_dist(y, temperature, top_k, top_p)
    return decide(p, q, d, seed, pos, S.greedy(x), **streams)


def rule(target, draft, proposals, temperature, top_k, top_p, seed, positions) -> list[Decision]:
    """All T rows of one launch (per-row parameter arrays as ``ext.speculative_sample`` takes them); the bonus row is
    ``sample_row`` on the last target row and counts as accepted with no margin."""
    target = np.asarray(target, dtype=np.float64)
    draft = np.asarray(draft, dtype=np.float64)
    T = target.shape[0]
    out = []
    for j in range(T):
        args = (float(temperature[j]), int(top_k[j]), float(top_p[j]), int(seed[j]) % 2**64, int(positions[j]))
        if j == T - 1:
            out.append(Decision(S.sample_row(target[j], *args), True, np.inf, np.inf))
        else:
            out.append(rule_row(target[j], draft[j], int(proposals[j]), *args))
    return out


def output_distribution(p, q) -> np.ndarray:
    """The rule's exact output distribution when ``d ~ q``, ``u`` uniform on (0, 1) and the residual a Gumbel-max draw
    (which picks i with probability (p_i - q_i) / sum of the positive differences)."""
    p, q = np.asarray(p, dtype=np.float64), np.asarray(q, dtype=np.float64)
    pos_diff = np.maximum(p - q, 0.0)
    total = pos_diff.sum()
    residual = pos_diff / total if total > 0 else np.zeros_like(p)
    out = np.zeros_like(p)
    for d in np.flatnonzero(q > 0):
        a = min(1.0, p[d] / q[d])
        out[d] += q[d] * a
        out += q[d] * (1.0 - a) * residual
    return out
