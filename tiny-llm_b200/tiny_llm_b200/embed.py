"""Text embeddings: pooled, normalised final hidden states of a Qwen3 model (DESIGN.md section 17).

Prompts are packed row after row into passes of a fixed ``max_tokens`` rows and each pass runs the layer stack once:
the same kernels and rounding points as the > 128-row branch of ``engine.PrefillEngine._forward``, except that
attention is segment-causal (``paged_attention_segments``: a row sees only the keys of its own prompt) and the LM
head is replaced by ``embed_pool`` (final RMSNorm, pooling, truncation, L2 normalisation in one launch).

Every pass has the same row count and every prompt starts on a ``SEGMENT_ALIGN``-row boundary, so each projection
runs the same kernel configuration and the attention kernel groups a prompt's keys into the same 64-key tiles
wherever it lands: a prompt's embedding does not depend on which prompts share its pass or on its place in it."""

from __future__ import annotations

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

from .engine import PrefillEngine, _normed, _proj
from .moe import Moe
from .paged_kv_cache import TinyKvPagedCache

SEGMENT_ALIGN = 64  # the attention kernel's key tile: a prompt's first row is a multiple of it
PASS_ALIGN = 128


def _aligned(n: int) -> int:
    return -(-n // SEGMENT_ALIGN) * SEGMENT_ALIGN


def pack_prompts(lengths, max_tokens: int) -> list[list[int]]:
    """Prompt indices per pass, first-fit in input order: each prompt goes to the first pass with room for its
    ``SEGMENT_ALIGN``-rounded length, after the prompts already there; a new pass opens when none has room."""
    if max_tokens <= 0 or max_tokens % PASS_ALIGN != 0:
        raise ValueError(f"max_tokens must be a positive multiple of {PASS_ALIGN}, got {max_tokens}")
    passes, used = [], []
    for i, n in enumerate(lengths):
        if n < 1:
            raise ValueError(f"prompt {i} is empty")
        if n > max_tokens:
            raise ValueError(f"prompt {i} has {n} tokens, more than max_tokens={max_tokens}")
        need = _aligned(n)
        for p, u in enumerate(used):
            if u + need <= max_tokens:
                passes[p].append(i)
                used[p] += need
                break
        else:
            passes.append([i])
            used.append(need)
    return passes


def pass_layout(lengths, max_tokens: int):
    """Per-row arrays of one pass holding prompts of ``lengths`` in order: ``(offsets, context_lens, segment_start,
    bounds)``.  A prompt's rows carry RoPE positions counted from its first row, post-append lengths row + 1 (row r
    writes its K/V to slot r of the pass's page run) and its first row as segment start; padding rows carry offset 0,
    context 0 (nothing appended) and segment start ``max_tokens`` (no visible key).  ``bounds`` [2n]: each prompt's
    first row and its end, as ``embed_pool`` segment starts: segment 2s is prompt s, segment 2s + 1 the alignment gap
    after it (possibly empty, never used)."""
    offsets = np.zeros(max_tokens, dtype=np.int32)
    ctxs = np.zeros(max_tokens, dtype=np.int32)
    seg = np.full(max_tokens, max_tokens, dtype=np.int32)
    starts, r = [], 0
    for n in lengths:
        starts.append(r)
        offsets[r:r + n] = np.arange(n, dtype=np.int32)
        ctxs[r:r + n] = np.arange(r + 1, r + n + 1, dtype=np.int32)
        seg[r:r + n] = r
        r += _aligned(n)
    if r > max_tokens:
        raise ValueError(f"{r} aligned rows do not fit a pass of {max_tokens}")
    # embed_pool reads segment s as rows bounds[s] .. bounds[s + 1] - 1: end each at its prompt's last row
    bounds = np.empty(2 * len(lengths), dtype=np.int32)
    bounds[0::2] = starts
    bounds[1::2] = np.asarray(starts, dtype=np.int32) + np.asarray(lengths, dtype=np.int32)
    return offsets, ctxs, seg, bounds


def _check_model(model, device, op: str = "embed") -> None:
    """Refuse, for the packed passes of ``op``, the models ``run_packed_pass`` does not run."""
    if any(isinstance(block.mlp, Moe) for block in model.layers_inner):
        raise ValueError(f"{op}: Qwen3-MoE models are not supported")
    if model.adapters is not None:
        raise ValueError(f"{op}: models with adapters loaded are not supported")
    if not PrefillEngine.supported(model, device):
        raise ValueError(f"{op}: needs a CUDA device, bf16 weights, head dimension 128 (non-traditional RoPE over the whole head), "
                         "a page size that is a multiple of 64 and a head ratio that divides 128")


def run_packed_pass(model, max_tokens, tokens, offsets, ctxs, arrays, attend, head, device):
    """One packed pass of ``max_tokens`` rows through the layer stack, with pages borrowed from the model's pools for
    the pass and returned in a ``finally``.  ``tokens``, ``offsets`` (RoPE positions) and ``ctxs`` (post-append lengths:
    row r appends its K/V at slot r, 0 appends nothing) are per-row int32 host arrays; ``arrays`` further int32 host
    arrays uploaded with them in one copy.  ``attend(q, attn, pool, table, views)`` is a layer's attention on its
    ``[Hq, T, D]`` queries, ``head(x, views)`` turns the final ``[T, H]`` hidden state into the result; ``views`` are the
    device copies of ``arrays``.  The rest - embedding, norms, projections, K/V append - is the > 128-row branch of
    ``engine.PrefillEngine._forward``."""
    n_pages = -(-max_tokens // model.page_size)
    layers = model.layers_inner
    attn0 = layers[0].self_attn
    Hkv, D = attn0.num_kv_heads, attn0.head_dim
    caches = []
    try:
        for pool in model.page_pools:
            short = n_pages - pool.pages_available()
            if pool._key_pages is None or short > 0:
                pool.reserve(pool.capacity + max(short, 0), Hkv, D, dtype=torch.bfloat16, device=device)
            cache = TinyKvPagedCache(pool)
            caches.append(cache)
            cache.append_slots(max_tokens)
        tables = np.stack([np.asarray(c.page_ids, dtype=np.int32) for c in caches])
        T = max_tokens
        meta = torch.from_numpy(np.concatenate([tokens, offsets, ctxs, *arrays, tables.reshape(-1)]).astype(np.int32, copy=False)).to(device)
        tok, off, ctx = meta[0:T].view(1, T), meta[T:2 * T], meta[2 * T:3 * T]
        views, at_ = [], 3 * T
        for arr in arrays:
            views.append(meta[at_:at_ + len(arr)])
            at_ += len(arr)
        tab = meta[at_:].view(len(caches), n_pages)

        emb = model.embedding.weight
        x = ext.quantized_embedding(tok, emb.scales, emb.biases, emb.weight, emb.group_size, emb.bits).view(T, -1)
        packed = model.packed_layers()
        for i, block in enumerate(layers):
            at, pool, mlp = block.self_attn, model.page_pools[i], block.mlp
            h = _normed(x, block.input_layernorm)
            q = ext.chunk_qk_norm_rope_append(_proj(h, packed[i].qkv), at.q_norm._weight_as(h.dtype, h.device),
                                              at.k_norm._weight_as(h.dtype, h.device), off, tab[i], ctx, pool._key_pages, pool._value_pages,
                                              at.num_heads, at.num_kv_heads, at.rope.base, at.q_norm.eps, inv_freq=at.rope.inv_freq)  # [Hq, T, D]
            a = attend(q, at, pool, tab[i], views)
            x = ext.add(x, _proj(a, at.wo))
            h = _normed(x, block.post_attention_layernorm)
            x = ext.add(x, _proj(ext.swiglu(_proj(h, mlp.w_gate), _proj(h, mlp.w_up)), mlp.w_down))
        return head(x, views)
    finally:
        for cache in caches:
            cache.release()


def _run_pass(model, ids, lengths, max_tokens, pooling, normalize, dimensions, device) -> torch.Tensor:
    """One packed pass: the pooled rows of its prompts, in order."""
    offsets, ctxs, seg, bounds = pass_layout(lengths, max_tokens)
    tokens = np.zeros(max_tokens, dtype=np.int32)
    for p, s in zip(ids, bounds[0::2]):
        tokens[s:s + len(p)] = p

    def attend(q, at, pool, table, views):
        return ext.paged_attention_segments(q, pool._key_pages, pool._value_pages, table, views[0], at.scale, at.num_kv_heads, at.num_heads)

    def head(x, views):
        # segment s of embed_pool = bounds[2s] .. bounds[2s + 1]: pool every other segment (the gaps are padding)
        return ext.embed_pool(x, model.norm._weight_as(x.dtype, x.device), model.norm.eps, views[1], pooling, dimensions, normalize)[0::2]

    return run_packed_pass(model, max_tokens, tokens, offsets, ctxs, [seg, bounds], attend, head, device)


def embed_ids(model, prompts, pooling: str = "last", normalize: bool = True, dimensions: int | None = None, max_tokens: int = 8192,
              device=None) -> torch.Tensor:
    """Embeddings of token-id ``prompts`` (lists of ints), fp32 ``[n, d]`` in input order.

    ``pooling``: "last" (the final row, what Qwen3-Embedding uses: append the EOS id to each prompt) or "mean";
    ``dimensions``: keep the first d features (Matryoshka), all when None; ``normalize``: divide by the L2 norm.
    Prompts are packed first-fit into passes of ``max_tokens`` rows (a multiple of 128); each pass borrows
    ``ceil(max_tokens / page_size)`` pages per layer from the model's pools and returns them, also on an error.
    Qwen3-MoE models and models with adapters raise ``ValueError``."""
    if pooling not in ext.EMBED_POOLING:
        raise ValueError(f"pooling must be one of {sorted(ext.EMBED_POOLING)}, got {pooling!r}")
    H = model.hidden_size
    if dimensions is not None and not 1 <= int(dimensions) <= H:
        raise ValueError(f"dimensions must be in [1, {H}], got {dimensions}")
    device = torch.device(device) if device is not None else model.embedding.weight.scales.device
    _check_model(model, device)
    ids = [[int(t) for t in p] for p in prompts]
    for i, p in enumerate(ids):
        if any(t < 0 or t >= model.vocab_size for t in p):
            raise ValueError(f"prompt {i} holds a token id outside [0, {model.vocab_size})")
    d = H if dimensions is None else int(dimensions)
    out = torch.empty((len(ids), d), dtype=torch.float32, device=device)
    for members in pack_prompts([len(p) for p in ids], max_tokens):
        rows = _run_pass(model, [ids[i] for i in members], [len(ids[i]) for i in members], max_tokens, pooling, normalize, d, device)
        out[torch.tensor(members, device=device)] = rows
    return out
