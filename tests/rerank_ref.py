"""Float64 references for reranking (DESIGN.md section 19): prefixed-segment attention over packed rows, the LM-head
weights ``tl_select_logits`` dequantises, and the selected logits with their log-softmax."""

from __future__ import annotations

import numpy as np
import torch


def prefixed_attention_ref(q, k, v, segment_start, prefix_start, prefix_end, scale, num_kv_heads):
    """``q`` [Hq, L, D], ``k`` / ``v`` [Hkv, L, D] (key r = packed row r) -> [L, Hq * D]: row l attends the keys in
    [prefix_start[l], prefix_end[l]) and [segment_start[l], l]; a row with no such key gives zeros."""
    q, k, v = (np.asarray(t, dtype=np.float64) for t in (q, k, v))
    seg, ps, pe = (np.asarray(a, dtype=np.int64) for a in (segment_start, prefix_start, prefix_end))
    Hq, L, D = q.shape
    G = Hq // num_kv_heads
    idx = np.arange(L)
    own = (idx[None, :] >= seg[:, None]) & (idx[None, :] <= idx[:, None])
    mask = own | ((idx[None, :] >= ps[:, None]) & (idx[None, :] < pe[:, None]) & own.any(axis=1)[:, None])
    out = np.zeros((L, Hq, D))
    for h in range(Hq):
        s = np.where(mask, (q[h] @ k[h // G].T) * scale, -np.inf)
        m = s.max(axis=1, keepdims=True)
        live = np.isfinite(m[:, 0])
        p = np.where(mask, np.exp(s - np.where(np.isfinite(m), m, 0.0)), 0.0)
        den = p.sum(axis=1, keepdims=True)
        out[:, h] = np.where(live[:, None], (p @ v[h // G]) / np.where(den > 0, den, 1.0), 0.0)
    return out.reshape(L, Hq * D)


def unpack_codes(words, bits):
    """[V, H * bits / 32] packed words -> [V, H] int64 codes; code j of a word is (w >> bits * j) & (2**bits - 1)."""
    V, W = words.shape
    w = words.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    per = 32 // bits
    shifts = bits * torch.arange(per, device=words.device, dtype=torch.int64)
    return ((w[..., None] >> shifts) & ((1 << bits) - 1)).reshape(V, W * per)


def head_weights(words, scales, biases, bits):
    """The weights ``tl_select_logits`` multiplies: ``T(code * scale + bias)`` with ``code * scale + bias`` in fp32
    (the product is exact) and T the dtype of ``scales``; returned as float64 [V, H]."""
    codes = unpack_codes(words.cpu(), bits).to(torch.float32)
    s = scales.cpu().to(torch.float32).repeat_interleave(128, dim=1)
    b = biases.cpu().to(torch.float32).repeat_interleave(128, dim=1)
    return (codes * s + b).to(scales.dtype).double().numpy()


def select_logits_ref(normed, weights, row_index, token_ids):
    """``normed`` [rows, H] (the normalised, dtype-rounded rows), ``weights`` [V, H] float64 -> (logits [n, m], log-softmax
    [n, m]) in float64, unrounded."""
    x = np.asarray(normed, dtype=np.float64)[np.asarray(row_index)]
    logits = x @ np.asarray(weights, dtype=np.float64)[np.asarray(token_ids)].T
    return logits, log_softmax(logits)


def log_softmax(logits):
    z = np.asarray(logits, dtype=np.float64)
    m = z.max(axis=1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(axis=1, keepdims=True))
