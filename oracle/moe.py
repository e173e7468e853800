"""Qwen3-MoE sparse block on CPU torch: the reference's operator sequence, a float64 referee, and CPU stand-ins for
the extension's ``moe_*`` entry points.

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).

* ``route_ref`` / ``moe_ref``: ``src/tiny_llm_ref/moe.py:36-89`` on dense dequantised weights with the rounding points
  of the project's contract (DESIGN.md, "Qwen3-MoE"): bf16 router logits, probs = bf16(softmax_fp32), top-k with ties
  to the lower id, optional renormalisation, bf16 expert outputs, SwiGLU rounded once, bf16 slot products summed in
  fp32 in slot order.
* ``moe_f64``: the same block with no rounding at all (float64 throughout, routing taken from the caller), the
  referee the bf16 oracle is held to.
* ``ReferenceCpuMoeModel``: ``ReferenceCpuModel`` whose sparse layers run ``moe_ref``.
* ``install(ext, monkeypatch)``: points the extension's ``moe_*`` functions at CPU restatements, beside
  ``oracle.ext_cpu.install``.
"""

from __future__ import annotations

import sys

import torch

from . import ops
from .model import ReferenceCpuModel, _Block, _dense
from .readable import RMSNorm, linear

BF16 = torch.bfloat16


def _r(x: torch.Tensor, dtype=BF16) -> torch.Tensor:
    return x.to(dtype).to(torch.float32)


def topk_from_probs(probs: torch.Tensor, k: int):
    """k largest of each row, descending, ties to the lower index (stable sort of -p)."""
    order = torch.sort(-probs.to(torch.float64), dim=-1, stable=True).indices[..., :k]
    return order, torch.gather(probs, -1, order)


def route_ref(logits: torch.Tensor, k: int, norm: bool):
    """Steps 2-3 of the contract on ``logits [T, E]`` (any float dtype): (probs, ids int64, scores) in logits' dtype."""
    dt = logits.dtype
    probs = torch.softmax(logits.to(torch.float32), dim=-1).to(dt)
    ids, scores = topk_from_probs(probs, k)
    if norm:
        den = _r(scores.to(torch.float32).sum(dim=-1, keepdim=True), dt)
        scores = (scores.to(torch.float32) / den).to(dt)
    return probs, ids, scores


def swiglu_once(g: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
    """The ``swiglu`` kernel's arithmetic on rounded inputs: g / (1 + exp(-g)) * u in fp32, one rounding."""
    g, u = g.to(torch.float32), u.to(torch.float32)
    return (g / (1.0 + torch.exp(-g)) * u).to(BF16)


def experts_ref(h: torch.Tensor, ids: torch.Tensor, scores: torch.Tensor, w_gate, w_up, w_down) -> torch.Tensor:
    """Steps 4-5 without the residual: dense bf16 experts ``w_gate/w_up [E, I, H]``, ``w_down [E, H, I]``."""
    T, k = ids.shape
    out = torch.zeros((T, h.shape[-1]), dtype=torch.float32)
    for j in range(k):
        e = ids[:, j].to(torch.int64)
        g = torch.einsum("th,tih->ti", h.to(torch.float32), w_gate[e].to(torch.float32)).to(BF16)
        u = torch.einsum("th,tih->ti", h.to(torch.float32), w_up[e].to(torch.float32)).to(BF16)
        a = swiglu_once(g, u)
        y = torch.einsum("ti,thi->th", a.to(torch.float32), w_down[e].to(torch.float32)).to(BF16)
        out += _r(y.to(torch.float32) * scores[:, j : j + 1].to(torch.float32))
    return out.to(BF16)


def moe_ref(h: torch.Tensor, w_router, w_gate, w_up, w_down, k: int, norm: bool) -> torch.Tensor:
    """The sparse MLP of one token batch ``h [T, H]`` (bf16) on dense bf16 weights."""
    logits = linear(h, w_router)
    _, ids, scores = route_ref(logits, k, norm)
    return experts_ref(h, ids, scores, w_gate, w_up, w_down)


def moe_f64(h: torch.Tensor, ids: torch.Tensor, scores: torch.Tensor, w_gate, w_up, w_down) -> torch.Tensor:
    """Steps 4-5 in float64 with no rounding (silu(g) * u), for the routing ``ids`` / ``scores``."""
    f = lambda t: t.to(torch.float64)
    out = torch.zeros((h.shape[0], h.shape[-1]), dtype=torch.float64)
    for j in range(ids.shape[1]):
        e = ids[:, j].to(torch.int64)
        g = torch.einsum("th,tih->ti", f(h), f(w_gate[e]))
        u = torch.einsum("th,tih->ti", f(h), f(w_up[e]))
        a = g / (1.0 + torch.exp(-g)) * u
        out += torch.einsum("ti,thi->th", a, f(w_down[e])) * f(scores[:, j : j + 1])
    return out


def dense_experts(layer) -> torch.Tensor:
    """SwitchLinear packed experts ``[E, out, in/8]`` -> dense bf16 ``[E, out, in]``."""
    return ops.dequantize_weights(layer.weight, layer.scales, layer.biases, layer.group_size, layer.bits).to(BF16)


class _MoeBlock(_Block):
    def __init__(self, args, layer):  # noqa: D401 - same wiring as _Block, sparse MLP
        from .model import _Attention

        self.attn = _Attention(args, layer.self_attn)
        self.ln1 = RMSNorm(args.hidden_size, layer.input_layernorm.weight, eps=args.rms_norm_eps)
        self.ln2 = RMSNorm(args.hidden_size, layer.post_attention_layernorm.weight, eps=args.rms_norm_eps)
        sw = layer.mlp.switch_mlp
        self.w_router = _dense(layer.mlp.gate)
        self.w_gate, self.w_up, self.w_down = dense_experts(sw.gate_proj), dense_experts(sw.up_proj), dense_experts(sw.down_proj)
        self.k, self.norm = args.num_experts_per_tok, bool(args.norm_topk_prob)

    def __call__(self, x, offsets, cache, mask):
        h = x + self.attn(self.ln1(x), offsets, cache, mask)
        y = self.ln2(h)
        B, L, H = y.shape
        r = moe_ref(y.reshape(-1, H), self.w_router, self.w_gate, self.w_up, self.w_down, self.k, self.norm)
        return h + r.reshape(B, L, H)


def is_sparse(args, index: int) -> bool:
    return (getattr(args, "num_experts", 0) > 0 and index not in getattr(args, "mlp_only_layers", [])
            and (index + 1) % getattr(args, "decoder_sparse_step", 1) == 0)


class ReferenceCpuMoeModel(ReferenceCpuModel):
    """``ReferenceCpuModel`` with Qwen3-MoE sparse layers (qwen3_week3.py:253-272)."""

    def __init__(self, mlx_model):
        super().__init__(SimpleDense(mlx_model))
        a = mlx_model.args
        self.blocks = [(_MoeBlock if is_sparse(a, i) else _Block)(a, layer) for i, layer in enumerate(mlx_model.model.layers)]


def SimpleDense(mlx_model):
    """The model with every sparse layer hidden, so that ``ReferenceCpuModel.__init__`` builds only what it can."""
    from types import SimpleNamespace

    a = mlx_model.args
    dense_layers = [layer for i, layer in enumerate(mlx_model.model.layers) if not is_sparse(a, i)]
    model = SimpleNamespace(embed_tokens=mlx_model.model.embed_tokens, layers=dense_layers, norm=mlx_model.model.norm)
    out = SimpleNamespace(args=a, model=model)
    if hasattr(mlx_model, "lm_head"):
        out.lm_head = mlx_model.lm_head
    return out


# ---------------------------------------------------------------- CPU stand-ins of the extension's moe_* functions --
MOE_CONTROL, MOE_WGMMA = 0, 1


def moe_topk(logits, top_k, norm_topk_prob=False, stream=None):
    probs, ids, scores = route_ref(logits, int(top_k), bool(norm_topk_prob))
    return probs, ids.to(torch.int32), scores


def moe_group(ids, num_experts, nt=0, stream=None):
    flat = ids.reshape(-1).to(torch.int64)
    perm = torch.sort(flat, stable=True).indices.to(torch.int32)
    counts = torch.bincount(flat, minlength=int(num_experts))
    offsets = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(counts, 0)]).to(torch.int32)
    return offsets, perm, None


def moe_gather(x, perm, rows_per_source, norm_weight=None, eps=0.0, stream=None):
    rows = x[perm.to(torch.int64) // int(rows_per_source)]
    return rows if norm_weight is None else ops.rms_norm(rows, norm_weight, eps)


def moe_grouped_matmul_route(T, k, E, N, K, epilogue, dtype, a, b):
    return MOE_CONTROL, 0, 0


def moe_grouped_matmul(scales, biases, b, a, offsets, tiles, top_k, out_index=None, epilogue=0, stream=None):
    w = ops.dequantize_fp32(b.reshape(-1, b.shape[-1]), scales.reshape(-1, scales.shape[-1]), biases.reshape(-1, biases.shape[-1]))
    E, K = b.shape[0], b.shape[1]
    w = w.reshape(E, K, -1).to(a.dtype).to(torch.float32)  # the wgmma kernel's weights are rounded to the activation dtype
    R = a.shape[0]
    seg = torch.bucketize(torch.arange(R), offsets[1:].to(torch.int64), right=True)
    acc = torch.einsum("rn,rkn->rk", a.to(torch.float32), w[seg])
    if epilogue == 2:  # EPI_SWIGLU_PAIRS
        acc = acc.reshape(R, K // 16, 2, 8)
        out = swiglu_once(_r(acc[:, :, 0, :], a.dtype), _r(acc[:, :, 1, :], a.dtype)).reshape(R, K // 2).to(a.dtype)
    else:
        out = acc.to(a.dtype)
    if out_index is None:
        return out
    res = torch.empty_like(out)
    res[out_index.to(torch.int64)] = out
    return res


def moe_combine(y, scores, residual=None, norm_weight=None, eps=0.0, stream=None):
    T, k = scores.shape
    yy = y.reshape(T, k, -1).to(torch.float32)
    r = _r(yy * scores.to(torch.float32)[:, :, None], y.dtype).sum(dim=1).to(y.dtype)
    out = r if residual is None else (residual.to(torch.float32) + r.to(torch.float32)).to(y.dtype)
    return out if norm_weight is None else (out, ops.rms_norm(out, norm_weight, eps))


OPS = ("moe_topk", "moe_group", "moe_gather", "moe_grouped_matmul_route", "moe_grouped_matmul", "moe_combine")


def install(ext_module, monkeypatch) -> None:
    me = sys.modules[__name__]
    for name in OPS:
        monkeypatch.setattr(ext_module, name, getattr(me, name))
