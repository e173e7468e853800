"""Float64 references for text embeddings (DESIGN.md section 17): segment-causal attention over packed rows and the
pooling contract of ``tl_embed_pool`` applied to rows that are already RMS-normalised."""

from __future__ import annotations

import numpy as np


def segment_attention_ref(q, k, v, segment_start, scale, num_kv_heads):
    """``q`` [Hq, L, D], ``k`` / ``v`` [Hkv, L, D] (key r = packed row r), ``segment_start`` [L] -> [L, Hq * D]: row l
    attends the keys segment_start[l] <= key <= l; a row with no such key gives zeros."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    seg = np.asarray(segment_start, dtype=np.int64)
    Hq, L, D = q.shape
    G = Hq // num_kv_heads
    idx = np.arange(L)
    mask = (idx[None, :] >= seg[:, None]) & (idx[None, :] <= idx[:, None])
    out = np.zeros((L, Hq, D))
    for h in range(Hq):
        s = np.where(mask, (q[h] @ k[h // G].T) * scale, -np.inf)
        m = s.max(axis=1, keepdims=True)
        live = np.isfinite(m[:, 0])
        p = np.where(mask, np.exp(s - np.where(np.isfinite(m), m, 0.0)), 0.0)
        den = p.sum(axis=1, keepdims=True)
        out[:, h] = np.where(live[:, None], (p @ v[h // G]) / np.where(den > 0, den, 1.0), 0.0)
    return out.reshape(L, Hq * D)


def rms_norm_ref(x, w, eps):
    x = np.asarray(x, dtype=np.float64)
    return x / np.sqrt((x * x).mean(axis=-1, keepdims=True) + eps) * np.asarray(w, dtype=np.float64)


def pool_ref(normed, bounds, pooling="last", dimensions=None, normalize=True):
    """``normed`` [rows, H]: rows already RMS-normalised (and rounded as the kernel rounds them); segment s is rows
    bounds[s] .. bounds[s + 1] - 1.  "last" takes its last row, "mean" the mean of its rows; the first ``dimensions``
    features are kept and, with ``normalize``, divided by their L2 norm (a zero vector stays zero; an empty segment
    gives zeros)."""
    normed = np.asarray(normed, dtype=np.float64)
    H = normed.shape[1]
    d = H if dimensions is None else int(dimensions)
    out = np.zeros((len(bounds) - 1, d))
    for s in range(len(bounds) - 1):
        a, b = int(bounds[s]), int(bounds[s + 1])
        if b <= a:
            continue
        vec = normed[b - 1] if pooling == "last" else normed[a:b].mean(axis=0)
        vec = vec[:d]
        if normalize:
            n = np.sqrt((vec * vec).sum())
            vec = vec / n if n > 0 else vec
        out[s] = vec
    return out
