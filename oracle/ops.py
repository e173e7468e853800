"""Kernel-level CPU restatement of the reference's native primitives.

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).  Every function takes and
returns CPU ``torch`` tensors and follows the arithmetic of one Metal kernel of
``src/extensions_ref/src`` - fp32 math, storage dtype rounded
once at the store - together with the builder-time checks of the matching
``.cpp`` file.  Citations are ``file:line`` relative to the tiny-llm repository.
"""

from __future__ import annotations

import math

import torch

_FLOATS = (torch.float32, torch.float16, torch.bfloat16)
_HALF = (torch.float16, torch.bfloat16)
_PACKED = (torch.int32, torch.uint32)


def as_i32(t: torch.Tensor) -> torch.Tensor:
    """Packed words as int32 (torch's uint32 has no shifts); bit pattern kept."""
    return t.view(torch.int32) if t.dtype == torch.uint32 else t


# --------------------------------------------------------------------------
# W4 layout spec: src/tiny_llm_ref/quantize.py:103-121
# --------------------------------------------------------------------------
def unpack_nibbles(weight: torch.Tensor, bits: int = 4) -> torch.Tensor:
    """[..., W] packed words -> [..., W * 32/bits] integer codes.

    Code ``i`` of a word is ``(word >> (bits*i)) & mask`` (quantize.py:113-115).
    """
    if bits <= 0 or 32 % bits != 0:
        raise ValueError("bits must divide a 32-bit packed weight")
    w = as_i32(weight).to(torch.int64) & 0xFFFFFFFF
    shifts = torch.arange(0, 32, bits, dtype=torch.int64)
    codes = (w.unsqueeze(-1) >> shifts) & ((1 << bits) - 1)
    return codes.reshape(*weight.shape[:-1], weight.shape[-1] * (32 // bits))


def dequantize_fp32(weight, scales, biases, group_size: int = 128, bits: int = 4) -> torch.Tensor:
    """``q*scale+bias`` in fp32, no storage rounding (metal vanilla :41-48)."""
    if bits == 4 and group_size % 8 == 0:
        # same arithmetic as the generic branch, one nibble plane at a time (8x less memory)
        w = as_i32(weight)
        s = scales.to(torch.float32).repeat_interleave(group_size // 8, dim=-1)
        b = None if biases is None else biases.to(torch.float32).repeat_interleave(group_size // 8, dim=-1)
        out = torch.empty(*w.shape, 8, dtype=torch.float32)
        for i in range(8):
            plane = ((w >> (4 * i)) & 0xF).to(torch.float32) * s
            out[..., i] = plane if b is None else plane + b
        return out.reshape(*w.shape[:-1], w.shape[-1] * 8)
    codes = unpack_nibbles(weight, bits).to(torch.float32)
    s = scales.to(torch.float32).repeat_interleave(group_size, dim=-1)
    if biases is None:
        return codes * s
    b = biases.to(torch.float32).repeat_interleave(group_size, dim=-1)
    return codes * s + b


def dequantize_weights(weight, scales, biases, group_size: int, bits: int) -> torch.Tensor:
    """quantize.py:103-121 - fp32 affine map then cast to the scales dtype."""
    return dequantize_fp32(weight, scales, biases, group_size, bits).to(scales.dtype)


# --------------------------------------------------------------------------
# quantized_matmul: quantized_matmul.cpp:14-80 (checks), :111-240 (dispatch)
# --------------------------------------------------------------------------
def _check_qmm(scales, biases, group_size, bits, a, b, transpose_b):
    if scales.dtype not in _HALF:
        raise RuntimeError("quantized_matmul: scales must be float16 or bfloat16")
    if scales.dtype != biases.dtype:
        raise RuntimeError("quantized_matmul: scales and biases must be the same dtype")
    if b.dtype not in _PACKED:
        raise RuntimeError("quantized_matmul: b must be uint32")
    if a.dtype != scales.dtype:
        raise RuntimeError("quantized_matmul: a must be the same dtype as scales")
    if a.dim() != 2:
        raise RuntimeError("quantized_matmul: a must be a 2D array")
    if b.dim() != 2:
        raise RuntimeError("quantized_matmul: b must be a 2D array")
    if bits != 4:
        raise RuntimeError("quantized_matmul: bits must be 4")
    if group_size != 128:
        raise RuntimeError("quantized_matmul: group_size must be 128")
    if not transpose_b:
        raise RuntimeError("quantized_matmul: b must be transposed")
    if scales.shape != biases.shape:
        raise RuntimeError("quantized_matmul: scales and biases must have the same shape")
    if b.shape[0] != scales.shape[0]:
        raise RuntimeError("quantized_matmul: b must have the same number of rows as scales")
    if a.shape[1] % group_size != 0:
        raise RuntimeError("quantized_matmul: a columns must be divisible by group_size")
    if scales.shape[1] != a.shape[1] // group_size:
        raise RuntimeError("quantized_matmul: scales must have one column per input group")
    if b.shape[1] != a.shape[1] // (32 // bits):
        raise RuntimeError("quantized_matmul: a must have the same number of columns as b")


def reference_split_k(M: int, N: int, K: int) -> int:
    """Split policy of the Metal host code (quantized_matmul.cpp:138-150)."""
    block, target, max_split = 32, 320, 16
    tiles = ((M + block - 1) // block) * ((K + block - 1) // block)
    split = min(max_split, max(1, target // max(tiles, 1)), N // 128)
    while split > 1 and N % (split * 128) != 0:
        split -= 1
    return split


def quantized_matmul(
    scales,
    biases,
    group_size,
    bits,
    a,
    b,
    transpose_b=False,
    use_simdgroup=True,
    use_split_k=False,
    stream=None,
):
    """out[i,k] = sum_j a[i,j] * (q[k,j]*s[k,g]+b[k,g]); a:[M,N], b:[K,N/8].

    Rounding points follow the kernel the reference would dispatch
    (quantized_matmul.cpp:137-166):
      * matvec (M<=8, use_simdgroup) and vanilla: weight stays fp32
        (quantized_matmul.metal:41-48, :515-521);
      * tiled: weight rounded to the activation dtype before the MMA (:183-194);
      * split-K: per-partition results stored in the activation dtype, fp32
        reduce (:251-293).
    """
    _check_qmm(scales, biases, group_size, bits, a, b, transpose_b)
    M, N = a.shape
    K = b.shape[0]
    a32 = a.to(torch.float32)
    use_matvec = use_simdgroup and M <= 8
    if use_matvec or not use_simdgroup:
        w = dequantize_fp32(b, scales, biases, group_size, bits)
        return (a32 @ w.T).to(a.dtype)
    w = dequantize_weights(b, scales, biases, group_size, bits).to(torch.float32)
    split = reference_split_k(M, N, K) if use_split_k else 1
    if split <= 1:
        return (a32 @ w.T).to(a.dtype)
    part = N // split
    acc = torch.zeros(M, K, dtype=torch.float32)
    for p in range(split):
        sl = slice(p * part, (p + 1) * part)
        acc += (a32[:, sl] @ w[:, sl].T).to(a.dtype).to(torch.float32)
    return acc.to(a.dtype)


# quantized_matmul.cpp:82-101 (checks); quantized_matmul.metal:58-89 (kernel)
def quantized_embedding(indices, scales, biases, weight, group_size, bits, stream=None):
    if indices.dtype not in _PACKED or weight.dtype not in _PACKED:
        raise RuntimeError("quantized_embedding: indices and weight must use 32-bit integers")
    if scales.dtype != biases.dtype or scales.dtype not in _HALF:
        raise RuntimeError("quantized_embedding: scales and biases must have the same 16-bit dtype")
    if group_size != 128 or bits != 4 or scales.shape != biases.shape:
        raise RuntimeError("quantized_embedding: expected 4-bit weights with group size 128")
    dim = weight.shape[1] * (32 // bits)
    if scales.shape[0] != weight.shape[0] or scales.shape[1] != dim // group_size:
        raise RuntimeError("quantized_embedding: incompatible parameter shapes")
    rows = as_i32(indices).to(torch.int64)
    w = as_i32(weight)[rows]
    return dequantize_weights(w, scales[rows], biases[rows], group_size, bits)


# --------------------------------------------------------------------------
# Week-2 fused kernels: week2_kernels.cpp:36-84, week2_kernels.metal
# --------------------------------------------------------------------------
def _need_float(x, name):
    if x.dtype not in _FLOATS:
        raise RuntimeError(f"{name}: expected float32, float16, or bfloat16")


def rms_norm(x, weight, eps, stream=None):
    """week2_kernels.metal:6-48 - fp32 sum of squares, one rounding at the store."""
    _need_float(x, "rms_norm")
    if x.dtype != weight.dtype or weight.dim() != 1 or weight.shape[0] != x.shape[-1]:
        raise RuntimeError("rms_norm: weight must match the input dtype and final dimension")
    x32 = x.to(torch.float32)
    inv = torch.rsqrt(x32.square().sum(-1, keepdim=True) / x.shape[-1] + eps)
    return (x32 * inv * weight.to(torch.float32)).to(x.dtype)


def rope(x, offsets, dims, base, traditional=False, stream=None):
    """week2_kernels.metal:50-105 - x [B,L,H,D], one int32 offset per batch row."""
    _need_float(x, "rope")
    if x.dim() != 4 or offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.shape[0] != x.shape[0]:
        raise RuntimeError("rope: expected x=[B,L,H,D] and one int32 offset per batch row")
    if dims <= 0 or dims > x.shape[3] or dims % 2 != 0:
        raise RuntimeError("rope: dims must be positive, even, and no larger than the head dimension")
    B, L, H, D = x.shape
    half = dims // 2
    power = -torch.arange(half, dtype=torch.float32) / half
    if x.dtype == torch.float32:
        inv_freq = torch.pow(torch.tensor(float(base), dtype=torch.float32), power)
    else:  # fast::exp2(power * log2(base)), metal :88-92
        inv_freq = torch.exp2(power * math.log2(float(base)))
    pos = (offsets.to(torch.int64)[:, None] + torch.arange(L)[None, :]).to(torch.float32)
    angle = pos[:, :, None] * inv_freq[None, None, :]  # [B,L,half]
    c = torch.cos(angle)[:, :, None, :]
    s = torch.sin(angle)[:, :, None, :]
    x32 = x.to(torch.float32)
    out = x32.clone()
    if traditional:
        re, im = x32[..., 0:dims:2], x32[..., 1:dims:2]
        out[..., 0:dims:2] = re * c - im * s
        out[..., 1:dims:2] = im * c + re * s
    else:
        re, im = x32[..., :half], x32[..., half:dims]
        out[..., :half] = re * c - im * s
        out[..., half:dims] = im * c + re * s
    return out.to(x.dtype)


def swiglu(gate, up, stream=None):
    """week2_kernels.metal:107-117 - g/(1+exp(-g))*u in fp32."""
    _need_float(gate, "swiglu")
    if gate.dtype != up.dtype or gate.shape != up.shape:
        raise RuntimeError("swiglu: gate and up must have the same shape and dtype")
    g = gate.to(torch.float32)
    return ((g / (1.0 + torch.exp(-g))) * up.to(torch.float32)).to(gate.dtype)


def decode_attention(query, key, value, mask, scale, is_causal, has_mask, num_heads, num_kv_heads, stream=None):
    """week2_kernels.metal:119-235 - dense-KV GQA softmax attention.

    q [B*Hq, L, D], k/v [B*Hkv, S, D], mask fp32 [B*Hq, L, S] (or a dummy).
    Causal rule (:165): key ``p`` is skipped when ``p > S - L + l``.
    """
    _need_float(query, "decode_attention")
    if query.dtype != key.dtype or query.dtype != value.dtype or mask.dtype != torch.float32:
        raise RuntimeError("decode_attention: q, k, and v dtypes must match; mask must be float32")
    if (
        query.dim() != 3
        or key.dim() != 3
        or value.dim() != 3
        or query.shape[2] > 256
        or query.shape[2] != key.shape[2]
        or query.shape[2] != value.shape[2]
        or key.shape != value.shape
        or num_heads % num_kv_heads != 0
    ):
        raise RuntimeError("decode_attention: incompatible attention shapes")
    if has_mask and (
        mask.dim() != 3 or mask.shape[0] != query.shape[0] or mask.shape[1] != query.shape[1] or mask.shape[2] != key.shape[1]
    ):
        raise RuntimeError("decode_attention: mask must have shape [B*Hq,L,S]")
    rows, L, D = query.shape
    S = key.shape[1]
    group = num_heads // num_kv_heads
    batch = rows // num_heads
    q = query.to(torch.float32).reshape(batch, num_kv_heads, group, L, D) * scale
    k = key.to(torch.float32).reshape(batch, num_kv_heads, 1, S, D)
    v = value.to(torch.float32).reshape(batch, num_kv_heads, 1, S, D)
    scores = q @ k.transpose(-1, -2)  # [b, hkv, g, L, S]
    if has_mask:
        scores = scores + mask.reshape(batch, num_kv_heads, group, L, S)
    if is_causal:
        pos = torch.arange(S)[None, :]
        lim = (S - L + torch.arange(L))[:, None]
        scores = scores.masked_fill(pos > lim, float("-inf"))
    # The kernel starts from max=-1e30 (finite), so an all-masked row divides
    # 0/0; callers never produce one (context >= L), keep softmax semantics.
    probs = torch.softmax(scores, dim=-1)
    return (probs @ v).reshape(rows, L, D).to(query.dtype)


# --------------------------------------------------------------------------
# Paged KV: paged_attention.cpp:14-31,77-122; paged_attention.metal
# --------------------------------------------------------------------------
def paged_cache_update(pages, values, page_id, start, stream=None):
    """paged_attention.metal:82-106 - in-place slice write, returns ``pages``."""
    if pages.dtype not in (torch.float32, torch.bfloat16) or values.dtype != pages.dtype:
        raise RuntimeError("paged_cache_update: pages and values must have the same float32 or bfloat16 dtype")
    if pages.dim() != 4 or values.dim() != 4 or values.shape[0] != 1:
        raise RuntimeError("paged_cache_update: expected pages [P, H, page_size, D] and values [1, H, length, D]")
    if values.shape[1] != pages.shape[1] or values.shape[3] != pages.shape[3]:
        raise RuntimeError("paged_cache_update: values must match the page head count and head dimension")
    if page_id < 0 or page_id >= pages.shape[0] or start < 0 or start + values.shape[2] > pages.shape[2]:
        raise RuntimeError("paged_cache_update: destination slice is outside page storage")
    pages[page_id, :, start : start + values.shape[2], :] = values[0]
    return pages


def paged_attention(
    query,
    key_pages,
    value_pages,
    block_table,
    context_lens,
    scale=1.0,
    is_causal=False,
    num_kv_heads=None,
    num_heads=None,
    stream=None,
):
    """softmax(q @ paged_k^T * scale) @ paged_v with bottom-right causality.

    q [B*Hq, L, D]; pages [P, Hkv, page, D]; block_table int32 [B, max_pages];
    context_lens int32 [B].  Row ``l`` sees keys ``< clamp(ctx-L+l+1, 0, ctx)``
    (paged_attention.metal:158-160, :411, :610); a row that sees nothing - or a
    page id < 0 - yields exact zeros (:166, :238-240).  Scores, softmax and
    the P@V accumulation are fp32; the L>8 bf16 kernel additionally rounds P to
    bf16 per 32-key tile (:439-444), which this restatement does not model
    (the reference's own tolerance for that path is 2e-2).
    """
    if query.dtype not in (torch.float32, torch.bfloat16) or key_pages.dtype != query.dtype or value_pages.dtype != query.dtype:
        raise RuntimeError("paged_attention: q, key_pages, and value_pages must have the same float32 or bfloat16 dtype")
    if block_table.dtype != torch.int32 or context_lens.dtype != torch.int32:
        raise RuntimeError("paged_attention: block_table and context_lens must be int32")
    if query.dim() != 3:
        raise RuntimeError("paged_attention: q must be 3D [B * H_q, L, D]")
    if key_pages.dim() != 4 or value_pages.dim() != 4:
        raise RuntimeError("paged_attention: page tensors must be 4D [P, H_kv, page_size, D]")
    if block_table.dim() != 2 or context_lens.dim() != 1:
        raise RuntimeError("paged_attention: block_table must be 2D and context_lens must be 1D")
    if num_heads % num_kv_heads != 0:
        raise RuntimeError("paged_attention: num_heads must be divisible by num_kv_heads")
    if query.shape[0] % num_heads != 0:
        raise RuntimeError("paged_attention: q.shape[0] must be divisible by num_heads")
    if key_pages.shape != value_pages.shape:
        raise RuntimeError("paged_attention: key_pages and value_pages must have the same shape")
    if key_pages.shape[1] != num_kv_heads:
        raise RuntimeError("paged_attention: page tensor head count must equal num_kv_heads")
    if query.shape[2] != key_pages.shape[3]:
        raise RuntimeError("paged_attention: q and page tensors must have the same head dimension")
    if block_table.shape[0] != context_lens.shape[0]:
        raise RuntimeError("paged_attention: block_table and context_lens batch sizes must match")
    if query.shape[0] // num_heads != block_table.shape[0]:
        raise RuntimeError("paged_attention: q batch size must match block_table batch size")
    rows, L, D = query.shape
    if D <= 0 or D > 128:
        raise RuntimeError("paged_attention: head dimension must be in the range [1, 128]")
    if L > 8 and query.dtype == torch.bfloat16 and D != 128:
        raise RuntimeError("paged_attention: bfloat16 prefill requires head dimension 128")
    page_size = key_pages.shape[2]
    max_pages = block_table.shape[1]
    group = num_heads // num_kv_heads
    batch = rows // num_heads
    out = torch.zeros(rows, L, D, dtype=torch.float32)
    q32 = query.to(torch.float32).reshape(batch, num_heads, L, D)
    for b in range(batch):
        ctx = int(context_lens[b])
        if ctx <= 0:
            continue
        n_pages = min(max_pages, (ctx + page_size - 1) // page_size)
        ids = block_table[b, :n_pages].to(torch.int64)
        live = ids >= 0
        kb = key_pages[ids.clamp(min=0)].to(torch.float32)  # [n, Hkv, page, D]
        vb = value_pages[ids.clamp(min=0)].to(torch.float32)
        kb = kb.permute(1, 0, 2, 3).reshape(num_kv_heads, n_pages * page_size, D)
        vb = vb.permute(1, 0, 2, 3).reshape(num_kv_heads, n_pages * page_size, D)
        S = n_pages * page_size
        key_pos = torch.arange(S)
        key_ok = (key_pos < ctx) & live.repeat_interleave(page_size)
        for l in range(L):
            visible = max(0, min(ctx, ctx - L + l + 1)) if is_causal else ctx
            ok = key_ok & (key_pos < visible)
            if not bool(ok.any()):
                continue
            qh = q32[b, :, l, :].reshape(num_kv_heads, group, D) * scale
            sc = qh @ kb.transpose(-1, -2)  # [Hkv, g, S]
            sc = sc.masked_fill(~ok[None, None, :], float("-inf"))
            pr = torch.softmax(sc, dim=-1)
            o = pr @ vb  # [Hkv, g, D]
            out.view(batch, num_heads, L, D)[b, :, l, :] = o.reshape(num_heads, D)
    return out.to(query.dtype)
