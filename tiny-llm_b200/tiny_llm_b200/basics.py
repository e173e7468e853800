"""Readable Week-1 operators on torch tensors.

Signatures of ``src/tiny_llm_ref/basics.py:5-26``.  These are
the un-fused building blocks the early Week-2 checkpoints still use; they run
as ordinary torch ops on whatever device the tensors live on.
"""

from __future__ import annotations

import torch


def softmax(x: torch.Tensor, axis: int) -> torch.Tensor:
    return torch.softmax(x, dim=axis)


def linear(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None) -> torch.Tensor:
    y = torch.matmul(x, w.transpose(-1, -2))
    return y if bias is None else y + bias


def silu(x: torch.Tensor) -> torch.Tensor:
    # sigmoid evaluated through exp(-|x|) so neither branch overflows
    z = torch.exp(-torch.abs(x))
    return x * torch.where(x < 0, z / (1 + z), 1 / (1 + z))
