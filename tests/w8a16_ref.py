"""Float64 reference of the 8-bit (W8A16) projection kernels: the W4 reference (w4a16_ref) on 8-bit codes.

Rounding points are those of 4 bits (include/tiny_llm_b200.h): weights exact on the scalar and streaming kernels,
T(code * scale + bias) rounded once on the wgmma kernels, the same prologues and epilogues.  What changes is the
streaming kernel's factorisation: each code is split q = 16 h + l and the group dot product is
scale * (16 d_h + d_l) + bias * asum, where d_h and d_l are the W4 shifted-code sums over nibbles.  ``error_bound``
accounts for it (its docstring has the derivation).  The exact probes are ``w4a16_ref.exact_probes(..., bits=8)``: every
kernel's arithmetic is exact on them, with codes 0, 127, 128 and 255 in every needle column.
"""

from __future__ import annotations

import importlib.util
import sys
from dataclasses import replace
from pathlib import Path

import torch


def _load_w4a16_ref():
    name = "tiny_llm_b200_w4a16_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("w4a16_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


wr = _load_w4a16_ref()
F64 = torch.float64
PROBE_CODES = wr.PROBE_CODES8
# The streaming bound's scale coefficient at 8 bits over the W4 one (see error_bound): 17 nibble sums plus a chain of
# codes up to 255 instead of 15 stay below 18 times the W4 coefficient for every chain length and shift.
STREAM8_SCALE = 18.0


def unpack_codes8(words):
    """[K, N/4] packed words -> [K, N] codes; code i of a word is (w >> 8i) & 255."""
    K, W = words.shape
    w = words.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    shifts = 8 * torch.arange(4, device=words.device, dtype=torch.int64)
    return ((w[..., None] >> shifts) & 255).reshape(K, W * 4)


def pack_codes8(codes):
    """[K, N] codes in [0, 256) -> [K, N/4] uint32 words."""
    K, N = codes.shape
    shifts = 8 * torch.arange(4, dtype=torch.int64, device=codes.device)
    words = (codes.to(torch.int64).reshape(K, N // 4, 4) << shifts).sum(-1)
    return torch.where(words >= 2**31, words - 2**32, words).to(torch.int32).view(torch.uint32)


def weights8(words, scales, biases, rounded):
    """``w4a16_ref.Weights`` of 8-bit packed weights: w [K, N] exact (code * scale + bias has at most 16 + 8
    significant bits and exponents within float64's reach), or rounded once to T."""
    K, G = scales.shape
    s, b = scales.to(F64), biases.to(F64)
    q = unpack_codes8(words).to(F64).view(K, G, 128)
    w = (q * s[:, :, None] + b[:, :, None]).view(K, G * 128)
    if rounded:
        w = wr.round_to(w, scales.dtype)
    return wr.Weights(w, w.abs(), s.abs(), b.abs(), scales.dtype, rounded)


def error_bound(r, W, path, splits=1, gb_per_split=None, norm_chain=None):
    """``w4a16_ref.error_bound`` with the 8-bit streaming kernel's accumulation.

    stream: per group, d_h and d_l are each a W4 shifted-code sum (nibbles 0..15, the shift in the first MMA's
    accumulator): each is off by at most (32 (2 SHIFT + 15) + 8 SHIFT) u sum_g |a|.  16 d_h + d_l is one fma (16 d_h is
    exact): off by 17 times that plus u 255 sum_g |a|.  Then acc += s (16 d_h + d_l) + b asum runs the W4 chain with
    codes up to 255: (2G + 20) u sum_g (255 |s| + |b|) sum_g |a|.  With A = 32 (2 SHIFT + 15) + 8 SHIFT >= 255 the
    scale coefficient chain 255 + 17 A + 255 is at most 18 (chain 15 + A), the W4 coefficient, so the W4 bound on
    18 |s| holds; the bias coefficient is the W4 one.  Every other path keeps the W4 accumulation unchanged: the
    scalar kernel adds (code * s + b) * a terms, and the wgmma kernels multiply the rounded weights."""
    if path == "stream":
        W = replace(W, abs_s=W.abs_s * STREAM8_SCALE)
    return wr.error_bound(r, W, path, splits, gb_per_split, norm_chain)


def embedding_ref(words, scales, biases, ids):
    """Rows ``ids`` of the dequantised table: T(fp32(code * scale + bias)) (the product is exact in fp32, the sum one
    fp32 rounding, then one rounding to T), zero rows for ids outside the vocabulary."""
    q = unpack_codes8(words)
    K, G = scales.shape
    s32 = scales.to(torch.float32).repeat_interleave(128, dim=1)
    b32 = biases.to(torch.float32).repeat_interleave(128, dim=1)
    w32 = q.to(torch.float32) * s32 + b32  # separate ops in float32: the product is exact, so this is the fma
    table = w32.to(scales.dtype)
    ids = ids.to(torch.int64)
    valid = (ids >= 0) & (ids < K)
    out = torch.zeros(ids.numel(), G * 128, dtype=scales.dtype, device=words.device)
    out[valid] = table[ids[valid]]
    return out
