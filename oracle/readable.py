"""Week-1 "readable" operators of tiny_llm_ref, restated on CPU torch.

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).  These are the only
operators of the reference that its own code can run on a CPU
(``main.py:50-61``), so they double as the second, independent
restatement that ``oracle.ops`` is cross-checked against - the same
equalities the reference asserts in ``tests_refsol/test_week_2_day_{4,5}.py``.
"""

from __future__ import annotations

import torch


def softmax(x: torch.Tensor, axis: int) -> torch.Tensor:
    """basics.py:5-7 (mx.softmax)."""
    return torch.softmax(x, dim=axis)


def linear(x, w, bias=None):
    """basics.py:10-18 - x @ w.T (+ bias), in the operand dtype."""
    y = x @ w.T
    return y if bias is None else y + bias


def silu(x):
    """basics.py:21-26 - sign-stable sigmoid."""
    z = torch.exp(-x.abs())
    sig = torch.where(x < 0, z / (1 + z), 1 / (1 + z))
    return x * sig


class RMSNorm:
    """layer_norm.py:4-15 - normalise in fp32, round, THEN scale by the weight."""

    def __init__(self, dim, weight, eps=1e-5):
        self.dim, self.weight, self.eps = dim, weight, eps

    def __call__(self, x):
        dtype = x.dtype
        h = x.to(torch.float32)
        h = h * torch.rsqrt(h.square().mean(-1, keepdim=True) + self.eps)
        return h.to(dtype) * self.weight.to(dtype)


class RoPE:
    """positional_encoding.py:4-66 - cos/sin tables, slice offsets."""

    def __init__(self, dims, seq_len, base=10000, traditional=False):
        assert dims % 2 == 0, "dims must be even"
        self.dims, self.seq_len, self.base, self.traditional = dims, seq_len, base, traditional
        self.half = dims // 2
        inner = torch.arange(self.half, dtype=torch.float32) / self.half
        freqs = torch.outer(torch.arange(seq_len, dtype=torch.float32), torch.pow(torch.tensor(float(base)), -inner))
        self.cos, self.sin = torch.cos(freqs), torch.sin(freqs)

    def __call__(self, x, offset=None):
        N, S, H, D = x.shape
        if offset is None:
            idx = torch.arange(S)[None, :]
        elif isinstance(offset, slice):
            assert offset.stop - offset.start == S
            idx = torch.arange(offset.start, offset.stop)[None, :]
        else:
            assert len(offset) == N
            idx = torch.stack([torch.arange(o.start, o.stop) for o in offset])
        c = self.cos[idx].reshape(-1, S, 1, self.half)
        s = self.sin[idx].reshape(-1, S, 1, self.half)
        if self.traditional:
            pairs = x.reshape(N, S, H, self.half, 2)
            x1, x2 = pairs[..., 0], pairs[..., 1]
        else:
            x1, x2 = x[..., : self.half], x[..., self.half : self.dims]
        real = x1 * c - x2 * s
        imag = x2 * c + x1 * s
        y = torch.stack([real, imag], dim=-1) if self.traditional else torch.cat([real, imag], dim=-1)
        return y.reshape(N, S, H, D).to(x.dtype)


def causal_mask(L: int, S: int, dtype) -> torch.Tensor:
    """attention.py:24-27 - tril(ones(L,S), k=S-L): bottom-right aligned."""
    keep = torch.tril(torch.ones(L, S), diagonal=S - L).bool()
    return torch.where(keep, 0.0, float("-inf")).to(dtype)


def scaled_dot_product_attention_grouped(query, key, value, scale=None, mask=None):
    """attention.py:30-66 - GQA attention in the operand dtype."""
    D = query.shape[-1]
    factor = torch.tensor(D**-0.5 if scale is None else float(scale)).to(query.dtype)
    shape = query.shape
    Hq, L, _ = query.shape[-3:]
    H, S, _ = key.shape[-3:]
    B = query.shape[:-3]
    assert Hq % H == 0
    rep = Hq // H
    q = query.reshape(*B, -1, H, rep, L, D)
    k = key.reshape(*B, -1, H, 1, S, D)
    v = value.reshape(*B, -1, H, 1, S, D)
    scores = (q @ k.transpose(-1, -2)) * factor
    if mask is not None:
        if isinstance(mask, str):
            assert mask == "causal"
            scores = scores + causal_mask(L, S, scores.dtype)
        else:
            m = torch.broadcast_to(mask, (*B, Hq, L, S)).reshape(*B, 1, H, rep, L, S)
            scores = scores + m.to(scores.dtype)
    return (softmax(scores, -1) @ v).reshape(shape)
