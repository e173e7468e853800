"""Float64 restatement of seeded sampling (``tl_sample``, DESIGN.md section 8), in numpy.

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).  For one logits row ``x`` and the parameters of
``SamplingParams`` drawing the token at sequence position ``pos``:

1. ``temperature == 0``, or a row whose maximum is not finite: the first maximum, NaN never, 0 for an all-NaN row
   (``tl_argmax``).
2. keep set ``{x_i >= tau}``, ``tau = max(x_(k), v*)``: top-k (on for ``0 < top_k < V``) keeps ``x_i >= x_(k)``, the
   k-th largest value, ties included; top-p (on for ``0 < top_p < 1``) keeps ``i`` when the probability mass strictly
   above ``x_i`` is ``< top_p``.  NaN is never kept.
3. ``argmax`` over the kept ``i`` of ``x_i / temperature + g_i``, ``g_i = -log(-log u_i)``,
   ``u_i = (2 (w >> 9) + 1) 2^-24`` with ``w`` word ``i % 4`` of Philox4x32-10 at counter ``(i >> 2, pos, 0, 0)`` and
   key ``(seed mod 2^32, seed >> 32)``.
"""

from __future__ import annotations

import numpy as np

_M0, _M1 = 0xD2511F53, 0xCD9E8D57
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF


def philox4x32_10(counter, key) -> np.ndarray:
    """Philox4x32-10 of ``counter`` ``[..., 4]`` (uint32) under ``key`` ``(k0, k1)`` -> ``[..., 4]`` uint32."""
    c = np.asarray(counter, dtype=np.uint64) & _MASK
    c0, c1, c2, c3 = (c[..., j].copy() for j in range(4))
    k0, k1 = np.uint64(int(key[0]) & _MASK), np.uint64(int(key[1]) & _MASK)
    for _ in range(10):
        p0 = np.uint64(_M0) * c0
        p1 = np.uint64(_M1) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(_MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(_MASK)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(_W0)) & np.uint64(_MASK)
        k1 = (k1 + np.uint64(_W1)) & np.uint64(_MASK)
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def uniforms(vocab: int, seed: int, pos: int) -> np.ndarray:
    """``u_i`` for ``i < vocab`` (float64, every value exact in fp32 too)."""
    groups = (vocab + 3) // 4
    ctr = np.zeros((groups, 4), dtype=np.uint64)
    ctr[:, 0] = np.arange(groups, dtype=np.uint64)
    ctr[:, 1] = pos & _MASK
    words = philox4x32_10(ctr, (seed & _MASK, seed >> 32)).reshape(-1)[:vocab].astype(np.uint64)
    return (2.0 * (words >> np.uint64(9)).astype(np.float64) + 1.0) * 2.0**-24


def gumbel(vocab: int, seed: int, pos: int) -> np.ndarray:
    return -np.log(-np.log(uniforms(vocab, seed, pos)))


def greedy(x) -> int:
    """``tl_argmax``: the first maximum, NaN never, 0 for an all-NaN row."""
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    if not ok.any():
        return 0
    m = x[ok].max()
    return int(np.flatnonzero(ok & (x == m))[0])


def mass_above(x) -> tuple[np.ndarray, float]:
    """``(M, S)``: ``M_i`` = probability mass strictly above ``x_i`` (NaN entries: inf), ``S = sum exp(x - max)``."""
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    m = x[ok].max()
    e = np.where(ok, np.exp(np.where(ok, x, m) - m), 0.0)
    s = e.sum()
    order = np.argsort(-np.where(ok, x, -np.inf), kind="stable")
    xs, es = x[order], e[order]
    cum = np.cumsum(es) - es  # mass of the entries before each one in descending order
    # equal values share the mass strictly above the first of them
    first = np.concatenate([[True], xs[1:] != xs[:-1]])
    idx = np.maximum.accumulate(np.where(first, np.arange(len(xs)), 0))
    above = np.empty_like(cum)
    above[order] = cum[idx] / s
    above[~ok] = np.inf
    return above, float(s)


def keep_set(x, top_k: int | None, top_p: float | None) -> np.ndarray:
    """Boolean mask of the kept entries of one row."""
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    keep = ok.copy()
    V = len(x)
    if top_k is not None and 0 < top_k < V and top_k <= ok.sum():
        kth = np.sort(x[ok])[::-1][top_k - 1]
        keep &= x >= kth
    if top_p is not None and 0 < top_p < 1:
        keep &= mass_above(x)[0] < top_p
    return keep


def perturbed(x, temperature: float, seed: int, pos: int) -> np.ndarray:
    """``x_i / temperature + g_i`` in float64."""
    x = np.asarray(x, dtype=np.float64)
    return x / temperature + gumbel(len(x), seed, pos)


def sample_row(x, temperature: float, top_k: int | None, top_p: float | None, seed: int, pos: int) -> int:
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    if not temperature > 0 or not ok.any() or not np.isfinite(x[ok].max()):
        return greedy(x)
    keep = keep_set(x, top_k, top_p)
    score = np.where(keep, perturbed(x, temperature, seed, pos), -np.inf)
    return int(np.argmax(score))


def sample(logits, temperature, top_k, top_p, seed, positions) -> np.ndarray:
    """Row-wise ``sample_row`` over ``logits [rows, V]`` and per-row parameter arrays (``top_k <= 0`` and ``top_p``
    outside ``(0, 1)`` are off, as in the kernel) -> int32 ``[rows]``."""
    x = np.asarray(logits, dtype=np.float64)
    out = np.empty(x.shape[0], dtype=np.int32)
    for r in range(x.shape[0]):
        out[r] = sample_row(x[r], float(temperature[r]), int(top_k[r]), float(top_p[r]), int(seed[r]) % 2**64, int(positions[r]))
    return out


def sample_like_ext(logits, temperature, top_k, top_p, seed, positions, stream=None):
    """``tiny_llm_ext_b200.sample``'s signature on CPU tensors (test stand-in) -> int32 ``[rows]`` on ``logits``'
    device."""
    import torch

    cols = [t.detach().cpu().numpy() for t in (logits.float(), temperature, top_k, top_p, seed, positions)]
    return torch.from_numpy(sample(*cols)).to(logits.device)
