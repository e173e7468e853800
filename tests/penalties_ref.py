"""Restatement of the penalised sampler (``tl_sample_penalized``, DESIGN.md section 8b), in numpy.

TEST INFRASTRUCTURE.  The penalties and the min-p threshold are fp32 operations in the kernel, each rounded on its own;
they are restated here with numpy float32, which rounds every operation to nearest, so the penalised row and the
threshold are exact.  The draw on the penalised row is ``oracle.sampling``'s float64 reference.

``state`` holds, per token, bit 30 when the token is in the prompt and in bits 0-29 the number of times it was drawn.
"""

from __future__ import annotations

import numpy as np

from oracle import sampling as ref

PROMPT = 1 << 30
COUNT = PROMPT - 1


def penalize(x, state, r: float, pres: float, freq: float) -> np.ndarray:
    """The penalised row in fp32: ``x1 = seen && r != 1 ? (x > 0 ? x / r : x * r) : x``,
    ``x2 = c > 0 ? x1 - fl(f * c) : x1``, ``x3 = c > 0 ? x2 - pres : x2``."""
    x = np.asarray(x, dtype=np.float32)
    s = np.asarray(state, dtype=np.int64)
    c = s & COUNT
    seen = ((s & PROMPT) != 0) | (c > 0)
    r, pres, f = np.float32(r), np.float32(pres), np.float32(freq)
    with np.errstate(all="ignore"):
        x1 = np.where(seen & (r != np.float32(1)), np.where(x > 0, x / r, x * r), x).astype(np.float32)
        x2 = np.where(c > 0, x1 - f * c.astype(np.float32), x1).astype(np.float32)
        return np.where(c > 0, x2 - pres, x2).astype(np.float32)


def min_p_threshold(m: float, temperature: float, min_p: float) -> np.float32:
    """``fl(m + fl(T * L))``, ``L = log(min_p)`` in double rounded once to fp32 (min_p above 1 acts as 1)."""
    log_p = np.float32(np.log(np.float64(min(np.float32(min_p), np.float32(1)))))
    return np.float32(np.float32(m) + np.float32(np.float32(temperature) * log_p))


def keep_set(x3, top_k, top_p, min_p: float, temperature: float) -> np.ndarray:
    """Keep mask of a penalised fp32 row: top-k and top-p as ``oracle.sampling.keep_set`` and min-p's bound."""
    keep = ref.keep_set(np.asarray(x3, dtype=np.float64), top_k, top_p)
    if min_p > 0:
        ok = ~np.isnan(x3)
        keep &= np.asarray(x3) >= min_p_threshold(np.max(x3[ok]), temperature, min_p)
    return keep


def sample_row(x, state, temperature: float, top_k, top_p, seed: int, pos: int, r=1.0, pres=0.0, freq=0.0, min_p=0.0) -> int:
    """The token ``tl_sample_penalized`` draws from one row (``x`` as the kernel stages it, fp32)."""
    x3 = penalize(x, state, r, pres, freq)
    x64 = x3.astype(np.float64)
    ok = ~np.isnan(x64)
    if not temperature > 0 or not ok.any() or not np.isfinite(x64[ok].max()):
        return ref.greedy(x64)
    keep = keep_set(x3, top_k, top_p, min_p, temperature)
    score = np.where(keep, ref.perturbed(x64, temperature, seed, pos), -np.inf)
    return int(np.argmax(score))


def sample(logits, temperature, top_k, top_p, seed, positions, repetition, presence, frequency, min_p, state) -> np.ndarray:
    """Row-wise ``sample_row``; ``state`` (int32 ``[rows, V]``, numpy) gains 1 at each drawn token of the rows with
    position > 0, as the kernel's does -> int32 ``[rows]``."""
    x = np.asarray(logits, dtype=np.float32)
    out = np.empty(x.shape[0], dtype=np.int32)
    for i in range(x.shape[0]):
        out[i] = sample_row(x[i], state[i], float(temperature[i]), int(top_k[i]), float(top_p[i]), int(seed[i]) % 2**64,
                            int(positions[i]), float(repetition[i]), float(presence[i]), float(frequency[i]), float(min_p[i]))
        if int(positions[i]) > 0:
            state[i, out[i]] += 1
    return out


def sample_penalized_like_ext(logits, temperature, top_k, top_p, seed, positions, repetition, presence, frequency, min_p, state,
                              stream=None):
    """``tiny_llm_ext_b200.sample_penalized``'s signature on CPU tensors (test stand-in): updates ``state`` in place and
    returns int32 ``[rows]`` on ``logits``' device."""
    import torch

    cols = [t.detach().cpu().numpy() for t in (logits.float(), temperature, top_k, top_p, seed, positions, repetition, presence, frequency,
                                               min_p)]
    st = state.detach().cpu().numpy().copy()
    out = sample(*cols, st)
    state.copy_(torch.from_numpy(st))
    return torch.from_numpy(out).to(logits.device)
