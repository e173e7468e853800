"""An eager statement of the graph engines' steps, written from the C ABI (include/tiny_llm_b200.h), the model's unpacked
weights and DESIGN section 4: one decode step of ``DecodeEngine`` (B <= 8 on the streaming matvec, B > 8 on the swap-AB
stack) and one chunk of ``PrefillEngine`` (L <= 128 on the swap-AB stack, L > 128 operator by operator), as the library
launches they consist of.  Nothing here reads ``engine.py``'s packing, layer loops or metadata arrays: the fused weights
are packed again with torch indexing and the metadata is built from the request caches.

Every launch is recorded as a ``Stage`` (name, layer, the inputs it received, its output, the route the selection
functions report), so that a test can hold each one in place against a float64 reference.  The kernels are deterministic
(no atomics, split reductions added in split order, split counts from shapes and the SM count), so a captured step and
these launches issued eagerly must give the same bits.

Test helper: no tests in here."""

from __future__ import annotations

from dataclasses import dataclass, field
from types import SimpleNamespace

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

PRO_NONE, PRO_RMSNORM = ext.PRO_NONE, ext.PRO_RMSNORM
EPI_NONE, EPI_RESIDUAL, EPI_SWIGLU_PAIRS = ext.EPI_NONE, ext.EPI_RESIDUAL, ext.EPI_SWIGLU_PAIRS
SWAP_AB_MIN_ROWS = 9  # TL_MATVEC_REF_ROWS + 1: from here every projection of a step is a split-reduction wgmma launch
TOKEN_TILE = 128      # the tensor-core projection's row tile: longer prefill chunks run operator by operator


# ------------------------------------------------------------------- packing --
def _i32(w):
    return w.view(torch.int32) if w.dtype == torch.uint32 else w


def pack_qkv(wq, wk, wv):
    """q|k|v: the rows of wq, then wk, then wv (the header's 'q heads | k heads | v heads')."""
    return SimpleNamespace(weight=torch.cat([_i32(wq.weight), _i32(wk.weight), _i32(wv.weight)]).contiguous(),
                           scales=torch.cat([wq.scales, wk.scales, wv.scales]).contiguous(),
                           biases=torch.cat([wq.biases, wk.biases, wv.biases]).contiguous())


def gate_up_rows(K):
    """Source row of each of the 2K rows of the EPI_SWIGLU_PAIRS layout in cat([gate, up]): rows 16c..16c+7 are gate rows
    8c..8c+7, rows 16c+8..16c+15 are up rows 8c..8c+7."""
    r = torch.arange(2 * K)
    c, j = r // 16, r % 16
    return torch.where(j < 8, 8 * c + j, K + 8 * c + j - 8)


def pack_gate_up(gate, up):
    idx = gate_up_rows(gate.weight.shape[0]).to(gate.scales.device)
    pick = lambda a, b: torch.cat([a, b])[idx].contiguous()  # noqa: E731
    return SimpleNamespace(weight=pick(_i32(gate.weight), _i32(up.weight)), scales=pick(gate.scales, up.scales),
                           biases=pick(gate.biases, up.biases))


# ------------------------------------------------------------------ metadata --
def _slot_caches(entry):
    """Per-slot request caches of one layer: a BatchingKvCache's slots, or one request's cache."""
    return list(entry.kv_caches) if hasattr(entry, "kv_caches") else [entry]


@dataclass
class DecodeMeta:
    tokens: list
    offsets: list       # RoPE position of the appended token (0 for idle slots)
    context_lens: list  # post-append length, offset + 1 (0 for idle slots: nothing appended, no key seen)
    tables: np.ndarray  # int32 [layers, B, max_pages], page ids then -1


def decode_metadata(caches, tokens, max_pages, steps=1):
    """Metadata of the FIRST of ``steps`` one-token appends that the caches already account for (their offsets and page ids
    include every appended token).  ``caches``: per layer, a BatchingKvCache or one request's cache."""
    per_layer = [_slot_caches(entry) for entry in caches]
    B = len(per_layer[0])
    tables = np.full((len(per_layer), B, max_pages), -1, dtype=np.int32)
    offsets, ctx = [0] * B, [0] * B
    for b in range(B):
        c0 = per_layer[0][b]
        if c0 is None:
            continue
        offsets[b] = c0.offset - steps
        ctx[b] = offsets[b] + 1
        for layer, slots in enumerate(per_layer):
            ids = slots[b].page_ids
            assert len(ids) <= max_pages, "request exceeds the table"
            tables[layer, b, : len(ids)] = ids
    toks = [int(t) if per_layer[0][b] is not None else 0 for b, t in enumerate(tokens)]
    return DecodeMeta(toks, offsets, ctx, tables)


@dataclass
class PrefillMeta:
    tokens: list       # [L]: 0 on the padding rows, then the chunk's ids (right-aligned)
    offsets: list      # [L]: offset - pad + l (negative on padding rows in front of position 0)
    context_lens: list  # [L]: offset - pad + l + 1 on real rows, 0 on padding rows
    ctx_after: int     # offset + r
    tables: np.ndarray  # int32 [layers, max_pages]


def prefill_rows(L, r, offset):
    """(pad, offsets, context_lens, ctx_after) of an r-token chunk at ``offset`` right-aligned in L rows."""
    pad = L - r
    pos = [offset - pad + l for l in range(L)]
    return pad, pos, [p + 1 if l >= pad else 0 for l, p in enumerate(pos)], offset + r


def prefill_metadata(cache, token_ids, offset, L, max_pages):
    """Metadata of one chunk whose append the per-layer caches already account for."""
    r = len(token_ids)
    pad, pos, ctx, after = prefill_rows(L, r, offset)
    tables = np.full((len(cache), max_pages), -1, dtype=np.int32)
    for layer, c in enumerate(cache):
        assert c.offset == after
        tables[layer, : len(c.page_ids)] = c.page_ids
    return PrefillMeta([0] * pad + [int(t) for t in token_ids], pos, ctx, after, tables)


# -------------------------------------------------------------------- stages --
@dataclass
class Stage:
    """One launch: ``name``, ``layer`` (None outside the layer stack), the tensors it received (``args``; weights by
    key), what it returned (``out``; a tuple for two outputs) and the route its selection function reports."""

    name: str
    layer: int | None
    args: dict
    out: object
    route: object = None
    attrs: dict = field(default_factory=dict)


def _mm_route(M, N, K, lda, prologue, fused, a, w):
    return ext.quantized_matmul_route(M, N, K, lda, prologue, fused, True, a.dtype, a, w.weight, w.scales, w.biases)


class Plan:
    """The launches of one engine step for ``model`` (a Qwen3ModelWeek3), issued eagerly on the current stream."""

    def __init__(self, model):
        self.model = model
        self.layers = list(model.layers_inner)
        at = self.layers[0].self_attn
        self.Hq, self.Hkv, self.D = at.num_heads, at.num_kv_heads, at.head_dim
        self.base, self.scale = at.rope.base, at.scale
        self.qkv = [pack_qkv(b.self_attn.wq, b.self_attn.wk, b.self_attn.wv) for b in self.layers]
        self.gate_up = [pack_gate_up(b.mlp.w_gate, b.mlp.w_up) for b in self.layers]
        self.head = model.w_lm_head if model.w_lm_head is not None else model.embedding.weight
        dev = model.embedding.weight.scales.device
        self.inv_freq = torch.pow(torch.tensor(float(at.rope.base), dtype=torch.float64),
                                  -torch.arange(self.D // 2, dtype=torch.float64) / (self.D // 2)).to(dev)
        self.stages: list[Stage] = []

    # -- weights and norms by key: what the test takes from the unpacked model for each stage's reference
    def norm(self, key):
        kind, i = key
        if kind == "final":
            return self.model.norm
        b = self.layers[i]
        return {"ln1": b.input_layernorm, "ln2": b.post_attention_layernorm, "q": b.self_attn.q_norm, "k": b.self_attn.k_norm}[kind]

    def weights(self, key):
        kind, i = key
        return {"qkv": lambda: self.qkv[i], "gate_up": lambda: self.gate_up[i], "head": lambda: self.head,
                "o": lambda: self.layers[i].self_attn.wo, "down": lambda: self.layers[i].mlp.w_down,
                "gate": lambda: self.layers[i].mlp.w_gate, "up": lambda: self.layers[i].mlp.w_up}[kind]()

    def _nw(self, key, like):
        return self.norm(key)._weight_as(like.dtype, like.device)

    def _rec(self, *a, **k):
        self.stages.append(Stage(*a, **k))

    # -- launches
    def _embed(self, ids):
        emb = self.model.embedding.weight
        x = ext.quantized_embedding(ids, emb.scales, emb.biases, emb.weight, emb.group_size, emb.bits)
        self._rec("embedding", None, dict(ids=ids), x)
        return x

    def _rms(self, x, key, layer):
        out = ext.rms_norm(x, self._nw(key, x), self.norm(key).eps)
        self._rec("rms_norm", layer, dict(x=x, norm=key), out, ext.rms_norm_route(x.shape[-1], x.dtype, x, self._nw(key, x), out))
        return out

    def _mm(self, name, layer, wkey, a, *, norm=None, residual=None, epilogue=EPI_NONE):
        """quantized_matmul_fused (RMSNorm prologue when ``norm`` is given)."""
        w = self.weights(wkey)
        M, N = a.shape
        K = w.weight.shape[0]
        pro = PRO_RMSNORM if norm is not None else PRO_NONE
        kw = dict(prologue=pro, eps=self.norm(norm).eps) if norm is not None else {}
        out = ext.quantized_matmul_fused(w.scales, w.biases, w.weight, a, self._nw(norm, a) if norm is not None else None, residual=residual,
                                         epilogue=epilogue, **kw)
        self._rec(name, layer, dict(a=a, w=wkey, norm=norm, residual=residual, epilogue=epilogue), out,
                  _mm_route(M, N, K, a.stride(0), pro, True, a, w))
        return out

    def _mm_plain(self, name, layer, wkey, a):
        """quantized_matmul (the per-operator projection)."""
        w = self.weights(wkey)
        out = ext.quantized_matmul(w.scales, w.biases, 128, 4, a, w.weight, True)
        self._rec(name, layer, dict(a=a, w=wkey, norm=None, residual=None, epilogue=EPI_NONE), out,
                  _mm_route(a.shape[0], a.shape[1], w.weight.shape[0], a.shape[1], PRO_NONE, False, a, w))
        return out

    def _mm_norm(self, name, layer, wkey, a, residual, norm):
        """quantized_matmul_residual_norm: (x, rms_norm(x))."""
        w = self.weights(wkey)
        x, h = ext.quantized_matmul_residual_norm(w.scales, w.biases, w.weight, a, residual, self._nw(norm, a), self.norm(norm).eps)
        self._rec(name, layer, dict(a=a, w=wkey, norm=None, residual=residual, epilogue=EPI_RESIDUAL, next_norm=norm), (x, h),
                  _mm_route(a.shape[0], a.shape[1], w.weight.shape[0], a.shape[1], PRO_NONE, True, a, w))
        return x, h

    def _qkn_route(self, dtype):
        return ext.qk_norm_rope_route(self.Hq, self.Hkv, self.D, dtype)

    def _paged(self, name, layer, q, kp, vp, table, ctx, L, token_major=False):
        """paged_attention (decode rows) or paged_attention_token_major (one request's chunk)."""
        if token_major:
            out = ext.paged_attention_token_major(q, kp, vp, table, ctx, self.scale, True, self.Hkv, self.Hq)
        else:
            out = ext.paged_attention(q, kp, vp, table, ctx, self.scale, is_causal=True, num_kv_heads=self.Hkv, num_heads=self.Hq)
        route = ext.paged_attention_route(q, kp, vp, out, q.shape[0], L, self.D, kp.shape[0], kp.shape[2], table.shape[1], self.Hkv, self.Hq, q.dtype)
        self._rec(name, layer, dict(q=q, table=table, ctx=ctx, L=L, token_major=token_major), out, route)
        return out

    # -- steps
    def decode(self, meta: DecodeMeta, pages, attention_fused: bool, rows: int | None = None):
        """One decode step of the first ``rows`` slots (default all).  ``pages``: per layer (key_pages, value_pages), written in
        place.  Returns (logits [R, V], next_tokens int32 [R])."""
        dev = self.model.embedding.weight.scales.device
        B = len(meta.tokens)
        R = B if rows is None else rows
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)  # noqa: E731
        tokens, offsets, ctx = i32(meta.tokens[:R]), i32(meta.offsets[:R]), i32(meta.context_lens[:R])
        tables = torch.from_numpy(np.ascontiguousarray(meta.tables[:, :R])).to(dev)
        max_context = tables.shape[-1] * self.model.page_size  # the table width in tokens: fixes the split count
        self.meta = dict(tokens=tokens, offsets=offsets, ctx=ctx, tables=tables, max_context=max_context)
        Hq, Hkv, D = self.Hq, self.Hkv, self.D
        x = self._embed(tokens)

        def fused_attention(i, qkv):
            kp, vp = pages[i]
            y = ext.decode_attention_fused(qkv, self._nw(("q", i), qkv), self._nw(("k", i), qkv), offsets, tables[i], ctx, self.inv_freq, kp, vp,
                                           Hq, Hkv, self.norm(("q", i)).eps, self.scale, max_context)
            self._rec("attention_fused", i, dict(qkv=qkv, table=tables[i], ctx=ctx, offsets=offsets, max_context=max_context), y)
            return y

        if B <= 8:
            for i in range(len(self.layers)):
                kp, vp = pages[i]
                qkv = self._mm("qkv", i, ("qkv", i), x, norm=("ln1", i))
                if attention_fused:
                    y = fused_attention(i, qkv)
                else:
                    q = ext.decode_qk_norm_rope_append(qkv, self._nw(("q", i), qkv), self._nw(("k", i), qkv), offsets, tables[i], ctx, kp, vp,
                                                       Hq, Hkv, self.base, self.norm(("q", i)).eps)
                    self._rec("qk_norm_rope_append", i, dict(qkv=qkv, table=tables[i], ctx=ctx, offsets=offsets), q, self._qkn_route(qkv.dtype))
                    y = self._paged("attention", i, q.view(R * Hq, 1, D), kp, vp, tables[i], ctx, 1)
                x = self._mm("o", i, ("o", i), y.view(R, Hq * D), residual=x, epilogue=EPI_RESIDUAL)
                act = self._mm("gate_up", i, ("gate_up", i), x, norm=("ln2", i), epilogue=EPI_SWIGLU_PAIRS)
                x = self._mm("down", i, ("down", i), act, residual=x, epilogue=EPI_RESIDUAL)
            logits = self._mm("head", None, ("head", None), x, norm=("final", None))
        else:
            def attention(i, h):
                kp, vp = pages[i]
                if attention_fused:
                    return fused_attention(i, self._mm("qkv", i, ("qkv", i), h))
                q = self._qkv_rope_append(i, h, offsets, tables[i], ctx, kp, vp, chunk=False)
                return self._paged("attention", i, q.view(R * Hq, 1, D), kp, vp, tables[i], ctx, 1).view(R, Hq * D)

            h = self._swap_ab_stack(x, attention)
            logits = self._mm("head", None, ("head", None), h)
        nxt = ext.argmax(logits)
        self._rec("argmax", None, dict(logits=logits), nxt)
        return logits, nxt

    def _qkv_rope_append(self, i, h, offsets, table, ctx, kp, vp, chunk):
        w = self.qkv[i]
        q = ext.qkv_project_rope_append(w.scales, w.biases, w.weight, h, self._nw(("q", i), h), self._nw(("k", i), h), offsets, table, ctx, kp, vp,
                                        self.Hq, self.Hkv, self.base, self.norm(("q", i)).eps, chunk=chunk)
        M, N = h.shape
        self._rec("qkv_rope_append", i, dict(a=h, w=("qkv", i), table=table, ctx=ctx, offsets=offsets, chunk=chunk), q,
                  (_mm_route(M, N, w.weight.shape[0], N, PRO_NONE, True, h, w), self._qkn_route(h.dtype)))
        return q

    def _swap_ab_stack(self, x, attention):
        """rms_norm, then per layer: attention(i, h) -> o + residual + next norm -> gate|up pairs -> down + residual + next norm."""
        n = len(self.layers)
        h = self._rms(x, ("ln1", 0), 0)
        for i in range(n):
            y = attention(i, h)
            x, h = self._mm_norm("o_norm", i, ("o", i), y, x, ("ln2", i))
            act = self._mm("gate_up", i, ("gate_up", i), h, epilogue=EPI_SWIGLU_PAIRS)
            x, h = self._mm_norm("down_norm", i, ("down", i), act, x, ("ln1", i + 1) if i + 1 < n else ("final", None))
        return h

    def prefill(self, meta: PrefillMeta, pages):
        """One chunk of L = len(meta.tokens) rows.  Returns (logits [1, V] of the last row, next token int32 [1])."""
        dev = self.model.embedding.weight.scales.device
        L = len(meta.tokens)
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)  # noqa: E731
        tokens, offsets, ctx, after = i32(meta.tokens), i32(meta.offsets), i32(meta.context_lens), i32([meta.ctx_after])
        tables = torch.from_numpy(np.ascontiguousarray(meta.tables)).to(dev)
        self.meta = dict(tokens=tokens, offsets=offsets, ctx=ctx, ctx_after=after, tables=tables)
        Hq = self.Hq
        x = self._embed(tokens)
        if L <= TOKEN_TILE:
            def attention(i, h):
                kp, vp = pages[i]
                q = self._qkv_rope_append(i, h, offsets, tables[i], ctx, kp, vp, chunk=True)
                return self._paged("attention", i, q, kp, vp, tables[i : i + 1], after, L, token_major=True)

            last = self._swap_ab_stack(x, attention)[L - 1 : L]
        else:
            for i in range(len(self.layers)):
                kp, vp = pages[i]
                h = self._rms(x, ("ln1", i), i)
                qkv = self._mm_plain("qkv", i, ("qkv", i), h)
                q = ext.chunk_qk_norm_rope_append(qkv, self._nw(("q", i), qkv), self._nw(("k", i), qkv), offsets, tables[i], ctx, kp, vp, Hq, self.Hkv,
                                                  self.base, self.norm(("q", i)).eps)
                self._rec("chunk_qk_norm_rope_append", i, dict(qkv=qkv, table=tables[i], ctx=ctx, offsets=offsets), q, self._qkn_route(qkv.dtype))
                y = self._paged("attention", i, q, kp, vp, tables[i : i + 1], after, L, token_major=True)
                o = self._mm_plain("o", i, ("o", i), y)
                x = self._add(i, x, o)
                h = self._rms(x, ("ln2", i), i)
                g = self._mm_plain("gate", i, ("gate", i), h)
                u = self._mm_plain("up", i, ("up", i), h)
                a = ext.swiglu(g, u)
                self._rec("swiglu", i, dict(gate=g, up=u), a)
                x = self._add(i, x, self._mm_plain("down", i, ("down", i), a))
            last = self._rms(x[L - 1 : L], ("final", None), None)
        logits = self._mm_plain("head", None, ("head", None), last)
        nxt = ext.argmax(logits)
        self._rec("argmax", None, dict(logits=logits), nxt)
        return logits, nxt

    def _add(self, i, a, b):
        out = ext.add(a, b)
        self._rec("add", i, dict(a=a, b=b), out)
        return out
