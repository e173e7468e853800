"""Float64 reference of ``tl_moe_router`` (8-bit MLX affine router at group 64) and the error bound its result obeys.

The kernel computes, per group g of 64 inputs, ``D = sum_k code_k a_k`` and ``S = sum_k a_k`` as fp32 sums of exact
products, folds ``acc = fma(bias, S, fma(scale, D, acc))`` over the groups of one of 8 slices, adds the 8 slice partials
and rounds once to the activation dtype.  Every fp32 step adds at most one unit in the last place of a running value
bounded by ``M = sum_g |scale_g| sum_k |code_k a_k| + |bias_g| sum_k |a_k|``, and there are fewer than
``64 + 2 G + 8`` such steps on any path, so

    |out - ref| <= u_T |ref| + (1 + u_T) (64 + 2 G + 8) 2^-23 M        (u_T: 2^-8 for bf16, 2^-11 for fp16)

with ``ref`` the exact value of ``sum_k (scale * code + bias) * a``.
"""

from __future__ import annotations

import torch

GROUP = 64
U_T = {torch.bfloat16: 2.0**-8, torch.float16: 2.0**-11}


def unpack8(weight: torch.Tensor) -> torch.Tensor:
    """Packed 8-bit codes ``[E, H / 4]`` (int32 or uint32 bit patterns) -> int64 codes ``[E, H]``."""
    words = (weight.view(torch.int32) if weight.dtype == torch.uint32 else weight).to(torch.int64) & 0xFFFFFFFF
    shifts = torch.arange(0, 32, 8, dtype=torch.int64, device=words.device)
    return ((words.unsqueeze(-1) >> shifts) & 0xFF).reshape(words.shape[0], -1)


def router_ref(x: torch.Tensor, weight: torch.Tensor, scales: torch.Tensor, biases: torch.Tensor):
    """``(ref [T, E], bound [T, E])`` in float64 for activations ``x [T, H]`` (already normalised)."""
    codes = unpack8(weight).to(torch.float64)
    s = scales.to(torch.float64).repeat_interleave(GROUP, dim=-1)
    b = biases.to(torch.float64).repeat_interleave(GROUP, dim=-1)
    a = x.to(torch.float64)
    ref = a @ (s * codes + b).T
    mag = a.abs() @ (s.abs() * codes + b.abs()).T
    G = x.shape[1] // GROUP
    u = U_T[x.dtype]
    return ref, u * ref.abs() + (1 + u) * (64 + 2 * G + 8) * 2.0**-23 * mag


def probe_value(scale: float, code: int, bias: float, a: float, dtype: torch.dtype) -> float:
    """The kernel's exact result for one input ``a`` times one weight (every other input zero): fp32
    ``fma(bias, a, scale * code * a)`` (the product is exact in fp32), rounded to ``dtype``."""
    dot = torch.tensor(scale * code * a, dtype=torch.float64).to(torch.float32)
    return float((dot.to(torch.float64) + bias * a).to(torch.float32).to(dtype))
