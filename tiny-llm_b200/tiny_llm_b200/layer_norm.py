"""Readable RMSNorm (``src/tiny_llm_ref/layer_norm.py:4-15``)."""

from __future__ import annotations

import torch


class RMSNorm:
    def __init__(self, dim: int, weight: torch.Tensor, eps: float = 1e-5):
        self.dim = dim
        self.eps = eps
        self.weight = weight

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        # fp32 statistics, storage-dtype product with the weight (two roundings;
        # the fused kernel rounds once - week2_kernels.metal:41-47).
        h = x.to(torch.float32)
        h = h * torch.rsqrt(h.square().mean(dim=-1, keepdim=True) + self.eps)
        return h.to(x.dtype) * self.weight.to(x.dtype)
