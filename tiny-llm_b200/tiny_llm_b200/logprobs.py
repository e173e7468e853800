"""Token log-probabilities and top-N alternatives (``tl_logprobs``, DESIGN.md section 8a).

Every reported value is a log-probability of the raw model distribution, ``logits - logsumexp(logits)`` (the vector
the reference's generation loops build, ``src/tiny_llm_ref/generate.py:25``), whatever temperature, top-k or top-p
chose the token.  ``rank`` is 1 + the number of entries strictly more likely; ``top`` lists the ``N`` most likely
``(id, logprob)`` pairs in descending order, ties to the lower id.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


@dataclass(frozen=True)
class TokenLogprobs:
    """One token's entry: its id, log-probability, rank and the ``top`` ``(id, logprob)`` alternatives."""

    token: int
    logprob: float
    rank: int
    top: tuple[tuple[int, float], ...] = ()


def _check_n(n) -> int:
    if isinstance(n, bool) or not isinstance(n, int) or not 0 <= n <= ext.LOGPROBS_MAX_N:
        raise ValueError(f"logprobs must be an int in [0, {ext.LOGPROBS_MAX_N}], got {n!r}")
    return n


def _host_rows(targets, lp, rank, ids, top) -> list:
    """The five per-row results in one device->host copy (floats travel as their int32 bits): ``[targets, lp, rank,
    ids, top]`` as host lists."""
    R, n = rank.shape[0], ids.shape[1] if ids.dim() == 2 else 0
    packed = torch.cat([targets.reshape(-1).to(torch.int32), lp.view(torch.int32), rank, ids.reshape(-1),
                        top.reshape(-1).view(torch.int32)]).cpu()
    parts = torch.split(packed, [R, R, R, R * n, R * n])
    return [parts[0].tolist(), parts[1].view(torch.float32).tolist(), parts[2].tolist(), parts[3].view(R, n).tolist(),
            parts[4].view(torch.float32).view(R, n).tolist()]


def entries_from_host(targets, lp, rank, ids, top) -> list[TokenLogprobs]:
    """Host lists / arrays of one ``ext.logprobs`` result -> one ``TokenLogprobs`` per row (slots with id -1 dropped)."""
    out = []
    for r, t in enumerate(targets):
        alts = tuple((int(i), float(v)) for i, v in zip(ids[r], top[r]) if int(i) >= 0)
        out.append(TokenLogprobs(int(t), float(lp[r]), int(rank[r]), alts))
    return out


def token_logprobs(logits: torch.Tensor, targets, top_n: int = 0) -> list[TokenLogprobs]:
    """One ``TokenLogprobs`` per row of ``logits [rows, vocab]`` for the token ``targets[r]`` (-1: none; its entry then
    has a NaN logprob and rank 0), with the ``top_n`` most likely alternatives.  One ``ext.logprobs`` launch and one
    device->host read (``targets`` may be a device tensor: the entries then carry its values)."""
    top_n = _check_n(top_n)
    tgt = torch.as_tensor(targets, dtype=torch.int32).reshape(-1).to(logits.device)
    _, lp, rank, ids, top = ext.logprobs(logits.contiguous(), tgt, None, top_n)
    return entries_from_host(*_host_rows(tgt, lp, rank, ids, top))


@dataclass(frozen=True)
class PromptScore:
    """``score_ids``' result: one entry per token of ``ids[1:]`` (conditioned on the tokens before it), the total
    negative log-likelihood in nats, the perplexity ``exp(nll / len(entries))``, and the ``top_n`` alternatives for the
    token after the prompt (the last row's distribution: what generation would draw from first)."""

    entries: list
    nll: float
    perplexity: float
    next_top: tuple[tuple[int, float], ...]


def score_ids(model, ids, chunk: int = 512, top_n: int = 0, device=None) -> PromptScore:
    """Teacher-forced log-probabilities of a prompt.  The prompt goes through ``model(..., logits_to_keep=None)``
    ``chunk`` tokens at a time over one KV cache, so at most ``chunk x vocab`` logits are alive; each chunk's rows are
    scored by ``ext.logprobs`` with the next ids as targets."""
    ids = [int(t) for t in ids]
    if len(ids) < 1:
        raise ValueError("score_ids needs at least one token")
    if isinstance(chunk, bool) or not isinstance(chunk, int) or chunk <= 0:
        raise ValueError("chunk must be a positive int")
    top_n = _check_n(top_n)
    if device is None:
        device = getattr(model, "device", None) or model.embedding.weight.scales.device
    all_ids = torch.as_tensor(ids, dtype=torch.int32, device=device)
    targets = torch.cat([all_ids[1:], torch.full((1,), -1, dtype=torch.int32, device=all_ids.device)])
    parts = []
    cache = model.create_kv_cache()
    try:
        for start in range(0, len(ids), chunk):
            piece = all_ids[start : start + chunk]
            logits = model(piece[None], start, cache, logits_to_keep=None)[0]
            _, lp, rank, alt_ids, alt_lp = ext.logprobs(logits.contiguous(), targets[start : start + piece.numel()], None, top_n)
            parts.append((lp, rank, alt_ids, alt_lp))
    finally:
        for layer_cache in cache:
            layer_cache.release()
    _, lp, rank, alt_ids, alt_lp = _host_rows(targets, *(torch.cat(t) for t in zip(*parts)))
    entries = entries_from_host(ids[1:], lp[:-1], rank[:-1], alt_ids[:-1], alt_lp[:-1])
    nll = -math.fsum(e.logprob for e in entries)
    ppl = math.exp(nll / len(entries)) if entries else float("nan")
    next_top = tuple((int(i), float(v)) for i, v in zip(alt_ids[-1], alt_lp[-1]) if int(i) >= 0)
    return PromptScore(entries, nll, ppl, next_top)
