"""W4A16 operator layer: same callables as
``src/tiny_llm_ref/quantize.py`` over torch tensors and the
CUDA extension.

Packed weights are ``[K, N/8]`` 32-bit words (``torch.uint32`` or ``int32``
with the same bit pattern - torch has no uint32 arithmetic); code ``i`` of a
word is ``(word >> 4*i) & 0xF`` and the value is ``code*scale+bias`` with one
bf16 ``scale``/``bias`` per 128 inputs (quantize.py:103-121).
"""

from __future__ import annotations

from typing import Any

import torch

from extensions_b200 import tiny_llm_ext_b200


def as_packed_i32(t: torch.Tensor) -> torch.Tensor:
    """View packed words as int32 so torch can index / shift them."""
    return t.view(torch.int32) if t.dtype == torch.uint32 else t


class QuantizedWeights:
    """quantize.py:8-27 - a plain bundle; the flags pick the kernel family."""

    def __init__(
        self,
        scales: torch.Tensor,
        biases: torch.Tensor,
        group_size: int,
        bits: int,
        weight: torch.Tensor,
        use_simdgroup_matmul: bool = False,
        use_simdgroup_matvec: bool = True,
        use_split_k_matmul: bool = False,
    ):
        self.scales = scales
        self.biases = biases
        self.group_size = group_size
        self.bits = bits
        self.weight = weight
        self.use_simdgroup_matmul = use_simdgroup_matmul
        self.use_simdgroup_matvec = use_simdgroup_matvec
        self.use_split_k_matmul = use_split_k_matmul

    @staticmethod
    def from_mlx_layer(
        mlx_layer: Any,
        use_simdgroup_matmul: bool = False,
        use_simdgroup_matvec: bool = True,
        use_split_k_matmul: bool = False,
    ) -> "QuantizedWeights":
        """quantize.py:29-46 - scales/biases are carried as bf16."""
        raw_biases = mlx_layer.biases
        return QuantizedWeights(
            scales=mlx_layer.scales.to(torch.bfloat16).contiguous(),
            biases=None if raw_biases is None else raw_biases.to(torch.bfloat16).contiguous(),
            group_size=mlx_layer.group_size,
            bits=mlx_layer.bits,
            weight=mlx_layer.weight.contiguous(),
            use_simdgroup_matmul=use_simdgroup_matmul,
            use_simdgroup_matvec=use_simdgroup_matvec,
            use_split_k_matmul=use_split_k_matmul,
        )


def _flatten_rows(a: torch.Tensor) -> tuple[torch.Tensor, tuple[int, ...]]:
    lead = tuple(a.shape[:-1])
    return a.reshape(-1, a.shape[-1]).contiguous(), lead


def quantized_matmul(
    scales: torch.Tensor,
    biases: torch.Tensor,
    group_size: int,
    bits: int,
    a: torch.Tensor,
    b: torch.Tensor,
    transpose_b: bool = False,
    use_simdgroup: bool = False,
    use_split_k: bool = False,
) -> torch.Tensor:
    """quantize.py:124-148.  NOTE: the Python default ``use_simdgroup=False``
    differs from the extension's ``True`` on purpose (SURVEY 8a' #8)."""
    rows, lead = _flatten_rows(a)
    out = tiny_llm_ext_b200.quantized_matmul(
        scales.contiguous(),
        biases.contiguous(),
        group_size,
        bits,
        rows,
        b.contiguous(),
        transpose_b,
        use_simdgroup,
        use_split_k,
    )
    return out.reshape(*lead, -1)


def quantized_matvec_custom(
    scales: torch.Tensor,
    biases: torch.Tensor,
    group_size: int,
    bits: int,
    a: torch.Tensor,
    b: torch.Tensor,
    transpose_b: bool = False,
) -> torch.Tensor:
    """quantize.py:151-173 - at most 8 rows; relies on the EXTENSION default
    ``use_simdgroup=True`` to reach the weight-streaming kernel."""
    rows, lead = _flatten_rows(a)
    if rows.shape[0] > 8:
        raise ValueError("quantized_matvec_custom supports at most 8 input rows")
    out = tiny_llm_ext_b200.quantized_matmul(
        scales.contiguous(), biases.contiguous(), group_size, bits, rows, b.contiguous(), transpose_b
    )
    return out.reshape(*lead, -1)


def quantized_matmul_vanilla(
    scales: torch.Tensor,
    biases: torch.Tensor,
    group_size: int,
    bits: int,
    a: torch.Tensor,
    b: torch.Tensor,
    transpose_b: bool = False,
) -> torch.Tensor:
    """quantize.py:176-194 - the scalar control kernel."""
    return quantized_matmul(scales, biases, group_size, bits, a, b, transpose_b, use_simdgroup=False)


def quantized_linear(x: torch.Tensor, w: QuantizedWeights, bias: torch.Tensor | None = None) -> torch.Tensor:
    """quantize.py:49-90 - <= 8 rows go to the matvec kernel when the weights
    allow it, everything else to ``quantized_matmul`` with the weight's flags."""
    n_rows = 1
    for extent in x.shape[:-1]:
        n_rows *= extent
    if n_rows <= 8 and w.use_simdgroup_matvec:
        y = quantized_matvec_custom(w.scales, w.biases, w.group_size, w.bits, x, w.weight, True)
    else:
        y = quantized_matmul(
            w.scales,
            w.biases,
            w.group_size,
            w.bits,
            x,
            w.weight,
            True,
            use_simdgroup=w.use_simdgroup_matmul,
            use_split_k=w.use_split_k_matmul,
        )
    return y if bias is None else y + bias


def dequantize_weights(
    weight: torch.Tensor,
    scales: torch.Tensor,
    biases: torch.Tensor | None,
    group_size: int,
    bits: int,
) -> torch.Tensor:
    """quantize.py:103-121 - the layout spec, as plain torch ops (any device)."""
    if bits <= 0 or 32 % bits != 0:
        raise ValueError("bits must divide a 32-bit packed weight")
    per_word = 32 // bits
    words = as_packed_i32(weight)
    shifts = torch.arange(0, 32, bits, dtype=torch.int32, device=words.device)
    codes = (words.unsqueeze(-1) >> shifts) & ((1 << bits) - 1)  # arithmetic shift, then mask: exact
    codes = codes.reshape(*words.shape[:-1], words.shape[-1] * per_word).to(torch.float32)
    wide_scales = scales.to(torch.float32).repeat_interleave(group_size, dim=-1)
    if biases is None:
        return (codes * wide_scales).to(scales.dtype)
    wide_biases = biases.to(torch.float32).repeat_interleave(group_size, dim=-1)
    return (codes * wide_scales + wide_biases).to(scales.dtype)


def dequantize_linear(mx_layer: Any) -> torch.Tensor:
    """quantize.py:93-100 (``mx.dequantize`` then bf16)."""
    return dequantize_weights(
        mx_layer.weight, mx_layer.scales, mx_layer.biases, mx_layer.group_size, mx_layer.bits
    ).to(torch.bfloat16)
