"""``make_sampler(temp, top_p, top_k)`` (``src/tiny_llm_ref/sampler.py:5-25``) on
torch tensors: greedy at ``temp == 0``; otherwise mask everything outside the ``top_k`` most likely
tokens, then everything outside the smallest prefix of the sorted distribution whose mass reaches
``top_p`` (a token is kept while the mass BEFORE it is < top_p, ``:19``), divide by ``temp`` and draw
from the categorical distribution.  Runs wherever the log-probabilities live (CUDA in the serving
path: one sort + cumsum over the 151,936-wide row, no host round trip); ``generator`` makes the draw
reproducible."""

from __future__ import annotations

import torch


def make_sampler(temp: float, top_p: float | None = None, top_k: int | None = None, generator: torch.Generator | None = None):
    def sample(logprobs: torch.Tensor) -> torch.Tensor:
        if temp == 0:
            return torch.argmax(logprobs, dim=-1)
        lp = logprobs.to(torch.float32).clone()
        if top_k is not None and 0 < top_k < lp.shape[-1]:
            kth = torch.topk(lp, top_k, dim=-1).values[..., -1:]
            lp = torch.where(lp < kth, torch.full_like(lp, float("-inf")), lp)
        if top_p is not None and top_p > 0:
            sorted_lp, sorted_idx = torch.sort(lp, dim=-1, descending=True)
            probs = torch.exp(sorted_lp)
            keep = torch.cumsum(probs, dim=-1) - probs < top_p
            sorted_lp = torch.where(keep, sorted_lp, torch.full_like(sorted_lp, float("-inf")))
            lp = torch.full_like(lp, float("-inf")).scatter(-1, sorted_idx, sorted_lp)
        probs = torch.softmax(lp / temp, dim=-1)
        return torch.multinomial(probs, 1, generator=generator).squeeze(-1)

    return sample
