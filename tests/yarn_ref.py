"""Float64 statement of static YaRN RoPE scaling, written from its definition (DESIGN.md "Long context") rather than from
the package: the frequency table, the attention factor, RoPE at any position, and a whole-model float64-table run of the
CPU oracle (``oracle.model.ReferenceCpuModel`` with its RoPE and attention scale replaced)."""

from __future__ import annotations

import math

import numpy as np
import torch


def yarn_table(theta: float, D: int, s: float, L0: int, beta_fast: float = 32.0, beta_slow: float = 1.0):
    """``(inv_freq [D/2] float64 numpy, extrap, low, high)`` by the definition."""
    half = D // 2
    i = np.arange(half, dtype=np.float64)
    extrap = np.power(np.float64(theta), -i / half)
    interp = extrap / s

    def corr(r):
        return D * math.log(L0 / (2 * math.pi * r)) / (2 * math.log(theta))

    low = max(math.floor(corr(beta_fast)), 0)
    high = min(math.ceil(corr(beta_slow)), D - 1)
    if low == high:
        high += 0.001
    ramp = np.clip((i - low) / (high - low), 0.0, 1.0)
    return interp * ramp + extrap * (1.0 - ramp), extrap, low, high


def yarn_mscale(s: float, attention_factor: float | None = None) -> float:
    return float(attention_factor) if attention_factor is not None else 0.1 * math.log(s) + 1.0


def rope_f64(x: torch.Tensor, positions, inv_freq) -> torch.Tensor:
    """Non-traditional RoPE of ``x [..., D]`` (any float dtype) at ``positions`` (broadcast over the leading dims, one per
    row of ``x``'s first dim) in float64."""
    x = x.double()
    inv = torch.as_tensor(np.asarray(inv_freq), dtype=torch.float64, device=x.device)
    pos = torch.as_tensor(positions, dtype=torch.float64, device=x.device)
    angle = pos.reshape(pos.shape + (1,) * (x.dim() - 1 - pos.dim()) + (1,)) * inv
    half = x.shape[-1] // 2
    re, im = x[..., :half], x[..., half:]
    c, s = torch.cos(angle), torch.sin(angle)
    return torch.cat([re * c - im * s, im * c + re * s], dim=-1)


def rope_bound(x: torch.Tensor, positions, inv_freq, dtype) -> torch.Tensor:
    """Elementwise bound on |kernel - rope_f64| for the kernels' arithmetic: the fp32 angle ``float(pos * inv_freq)`` is
    off by up to half an ulp of the angle, ``sincosf`` and the fp32 products and sum add a few ulps of 1, and the
    output is rounded once to ``dtype``."""
    x = x.double()
    inv = torch.as_tensor(np.asarray(inv_freq), dtype=torch.float64, device=x.device)
    pos = torch.as_tensor(positions, dtype=torch.float64, device=x.device)
    angle = (pos.reshape(pos.shape + (1,) * (x.dim() - 1 - pos.dim()) + (1,)) * inv).abs()
    half_ulp_angle = torch.where(angle > 0, torch.exp2(torch.floor(torch.log2(angle.clamp_min(1e-300))) - 24), torch.zeros_like(angle))
    half = x.shape[-1] // 2
    mag = x[..., :half].abs() + x[..., half:].abs()
    pre = mag * (half_ulp_angle + 8 * 2.0**-24)
    pre = torch.cat([pre, pre], dim=-1)
    y = rope_f64(x, positions, inv_freq).abs() + pre
    mant = {torch.float32: 24, torch.float16: 11, torch.bfloat16: 8}[dtype]
    ulp_out = torch.exp2(torch.floor(torch.log2(y.clamp_min(2.0**-126))) - mant + 1)
    return pre + ulp_out


class TableRoPE:
    """The oracle's RoPE (``oracle/readable.py``) with float64 angles from a frequency table; slices of offsets."""

    def __init__(self, inv_freq):
        self.inv_freq = torch.as_tensor(np.asarray(inv_freq), dtype=torch.float64)

    def __call__(self, x, offset=None):
        N, S, H, D = x.shape
        idx = torch.stack([torch.arange(o.start, o.stop) for o in offset]).to(torch.float64)  # [N, S]
        angle = idx[..., None] * self.inv_freq  # [N, S, half]
        c, s = torch.cos(angle).float()[:, :, None, :], torch.sin(angle).float()[:, :, None, :]
        half = D // 2
        x1, x2 = x[..., :half], x[..., half:]
        return torch.cat([x1 * c - x2 * s, x2 * c + x1 * s], dim=-1).to(x.dtype)


def yarn_reference_model(ns_cpu, s: float, L0: int):
    """``ReferenceCpuModel(ns_cpu)`` with YaRN: every attention rotates by the float64 table and scales by ``m^2``."""
    from oracle.model import ReferenceCpuModel

    a = ns_cpu.args
    table, *_ = yarn_table(a.rope_theta, a.head_dim, s, L0)
    m = yarn_mscale(s)
    model = ReferenceCpuModel(ns_cpu)
    for block in model.blocks:
        block.attn.rope = TableRoPE(table)
        block.attn.scale = block.attn.scale * m * m
    return model
