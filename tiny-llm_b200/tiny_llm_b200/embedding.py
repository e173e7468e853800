"""Embedding tables (``src/tiny_llm_ref/embedding.py``)."""

from __future__ import annotations

import torch

from extensions_b200 import tiny_llm_ext_b200

from .basics import linear
from .quantize import QuantizedWeights, as_packed_i32, dequantize_weights, quantized_linear


class Embedding:
    """Dense table (embedding.py:7-23)."""

    def __init__(self, vocab_size: int, embedding_dim: int, weight: torch.Tensor):
        self.vocab_size = vocab_size
        self.embedding_dim = embedding_dim
        self.weight = weight

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        return self.weight[as_packed_i32(x).long()]

    def as_linear(self, x: torch.Tensor) -> torch.Tensor:
        return linear(x, self.weight)


class QuantizedEmbedding:
    """Packed table (embedding.py:25-57): readable gather+dequantise, or the
    fused gather kernel when ``use_custom_kernel`` and biases are present."""

    def __init__(self, vocab_size: int, embedding_dim: int, weight: QuantizedWeights, use_custom_kernel: bool = False):
        self.vocab_size = vocab_size
        self.embedding_dim = embedding_dim
        self.weight = weight
        self.use_custom_kernel = use_custom_kernel

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        w = self.weight
        if not self.use_custom_kernel or w.biases is None:
            rows = as_packed_i32(x).long()
            return dequantize_weights(
                as_packed_i32(w.weight)[rows],
                w.scales[rows],
                None if w.biases is None else w.biases[rows],
                w.group_size,
                w.bits,
            )
        ids = x if x.dtype in (torch.int32, torch.uint32) else x.to(torch.int32)
        return tiny_llm_ext_b200.quantized_embedding(ids.contiguous(), w.scales, w.biases, w.weight, w.group_size, w.bits)

    def as_linear(self, x: torch.Tensor) -> torch.Tensor:
        return quantized_linear(x, self.weight)
