"""Readable table-driven RoPE (``src/tiny_llm_ref/positional_encoding.py:4-66``)."""

from __future__ import annotations

import torch


class RoPE:
    def __init__(self, dims: int, seq_len: int, base: int = 10000, traditional: bool = False):
        assert dims % 2 == 0, "dims must be even"
        self.dims = dims
        self.seq_len = seq_len
        self.base = base
        self.half_dims = dims // 2
        self.traditional = traditional
        exponent = torch.arange(self.half_dims, dtype=torch.float32) / self.half_dims
        table = torch.outer(torch.arange(seq_len, dtype=torch.float32), torch.pow(torch.tensor(float(base)), -exponent))
        self.cos_freqs = torch.cos(table)
        self.sin_freqs = torch.sin(table)

    def _tables(self, device):
        if self.cos_freqs.device != device:
            self.cos_freqs = self.cos_freqs.to(device)
            self.sin_freqs = self.sin_freqs.to(device)
        return self.cos_freqs, self.sin_freqs

    def __call__(self, x: torch.Tensor, offset: list[slice] | slice | None = None) -> torch.Tensor:
        N, S, H, D = x.shape
        cos_t, sin_t = self._tables(x.device)
        if offset is None:
            rows = torch.arange(S, device=x.device)[None, :]
        elif isinstance(offset, slice):
            assert offset.stop - offset.start == S, f"offset must be of length {S}"
            rows = torch.arange(offset.start, offset.stop, device=x.device)[None, :]
        else:
            assert len(offset) == N, f"offsets must have the same length as batch size {N}"
            for o in offset:
                assert o.stop - o.start == S, f"offset must be of length {S}"
            rows = torch.stack([torch.arange(o.start, o.stop, device=x.device) for o in offset])
        cos_b = cos_t[rows].reshape(-1, S, 1, self.half_dims)
        sin_b = sin_t[rows].reshape(-1, S, 1, self.half_dims)
        if self.traditional:
            pairs = x.reshape(N, S, H, self.half_dims, 2)
            first, second = pairs[..., 0], pairs[..., 1]
        else:
            first, second = x[..., : self.half_dims], x[..., self.half_dims : self.dims]
        real = first * cos_b - second * sin_b
        imag = second * cos_b + first * sin_b
        if self.traditional:
            y = torch.stack([real, imag], dim=-1)
        else:
            y = torch.cat([real, imag], dim=-1)
        return y.reshape(N, S, H, D).to(x.dtype)
