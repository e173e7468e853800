"""Qwen3-MoE sparse block (``src/tiny_llm_ref/moe.py``) on the CUDA extension.

Same names and signatures as the reference.  The expert weights are ``QuantizedWeights`` whose tensors carry a
leading expert axis (``weight [E, out, in/8]``, ``scales``/``biases [E, out, in/128]``, the ``mlx_lm`` SwitchLinear
layout).  A layer is one fixed launch sequence that never reads a count back to the host, so it can be captured in
a CUDA graph:

    router projection (router_logits) -> moe_topk -> moe_group -> moe_gather -> grouped gate|up (SwiGLU epilogue, sorted rows)
    -> grouped down (scattered back to token order) -> moe_combine

Rounding follows the reference's operator sequence, except that SwiGLU is the project's ``swiglu`` arithmetic on the
rounded gate and up outputs (one rounding) instead of ``silu(gate) * up`` (DESIGN.md, "Qwen3-MoE").
"""

from __future__ import annotations

import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

from .quantize import QuantizedWeights, as_packed_i32, quantized_linear


def _experts(w: QuantizedWeights, op: str) -> tuple[int, int, int]:
    if w.bits == 8:
        raise ValueError(f"{op}: Qwen3-MoE with 8-bit weights is not supported (there is no 8-bit grouped expert GEMM); use a 4-bit checkpoint")
    if w.weight.dim() != 3 or w.scales.dim() != 3 or w.group_size != 128 or w.bits != 4 or w.biases is None:
        raise ValueError(f"{op}: expert weights must be 4-bit / group 128 [E, out, in/8] with scales and biases [E, out, in/128]")
    E, out_dim, words = w.weight.shape
    return E, out_dim, words * 8


def _grouped(rows: torch.Tensor, w: QuantizedWeights, offsets, tiles_by_nt: dict, top_k: int, out_index, epilogue) -> torch.Tensor:
    E, K, N = _experts(w, "grouped_expert_linear")
    R = rows.shape[0]
    route, nt, _ = ext.moe_grouped_matmul_route(R // top_k, top_k, E, N, K, epilogue, rows.dtype, rows, w.weight)
    return ext.moe_grouped_matmul(w.scales, w.biases, w.weight, rows, offsets, tiles_by_nt.get(nt) if route == ext.MOE_WGMMA else None, top_k,
                                  out_index=out_index, epilogue=epilogue)


def _group(ids: torch.Tensor, E: int, nt: int):
    offsets, perm, tiles = ext.moe_group(ids, E, nt)
    return offsets, perm, {nt: tiles} if tiles is not None else {}


def grouped_expert_linear(x: torch.Tensor, w_experts: QuantizedWeights, expert_ids: torch.Tensor) -> torch.Tensor:
    """moe.py:7-33 - row r of ``x [..., D]`` through expert ``expert_ids[r]`` -> ``[..., out]``."""
    *lead, D = x.shape
    E, K, N = _experts(w_experts, "grouped_expert_linear")
    if N != D:
        raise ValueError(f"grouped_expert_linear: x has {D} features, the experts take {N}")
    flat = x.reshape(-1, D).contiguous()
    ids = expert_ids.reshape(-1).to(torch.int32).contiguous()
    if ids.numel() != flat.shape[0]:
        raise ValueError("grouped_expert_linear: one expert id per row")
    R = flat.shape[0]
    route, nt, _ = ext.moe_grouped_matmul_route(R, 1, E, N, K, ext.EPI_NONE, flat.dtype, flat, w_experts.weight)
    offsets, perm, tiles = _group(ids, E, nt)
    xs = ext.moe_gather(flat, perm, 1)
    out = _grouped(xs, w_experts, offsets, tiles, 1, perm, ext.EPI_NONE)
    return out.reshape(*lead, K)


ROUTER_G64 = (8, ext.MOE_ROUTER_GROUP)  # (bits, group_size) of the routers mlx_lm stores apart from the model's setting


def _check_router(w: QuantizedWeights) -> None:
    if w.group_size == ext.MOE_ROUTER_GROUP and (w.bits, w.group_size) != ROUTER_G64:
        raise ValueError(f"Moe: a group-{w.group_size} router must have 8-bit codes (got {w.bits} bits)")


def router_logits(h: torch.Tensor, w: QuantizedWeights, norm=None, projection=quantized_linear) -> torch.Tensor:
    """Router logits ``[..., E]`` of the rows ``h [..., H]``: the one place that picks the router's kernel.  An 8-bit
    group-64 router (``ROUTER_G64``) runs ``ext.moe_router``; any other runs ``projection(h, w)`` (the caller's
    projection launch), or with ``norm = (weight, eps)`` the streaming projection with the RMSNorm prologue.  With
    ``norm``, ``h`` is not yet normalised; both forms give the bits of ``rms_norm`` followed by the projection."""
    if (w.bits, w.group_size) == ROUTER_G64:
        rows = h.reshape(-1, h.shape[-1]).contiguous()
        return ext.moe_router(rows, w.weight, w.scales, w.biases, *(norm or ())).reshape(*h.shape[:-1], -1)
    if norm is not None:
        return ext.quantized_matmul_fused(w.scales, w.biases, w.weight, h, norm[0], prologue=ext.PRO_RMSNORM, eps=norm[1])
    return projection(h, w)


def route_topk(x: torch.Tensor, w_router: QuantizedWeights, top_k: int, norm_topk_prob: bool = False):
    """moe.py:36-49 - ``(probs [..., E], ids [..., k], scores [..., k])``; ids in descending order of probability."""
    logits = router_logits(x, w_router)
    *lead, E = logits.shape
    probs, ids, scores = ext.moe_topk(logits.reshape(-1, E).contiguous(), int(top_k), norm_topk_prob)
    return probs.reshape(*lead, E), ids.reshape(*lead, top_k), scores.reshape(*lead, top_k)


class Moe:
    """moe.py:52-89 - the sparse MLP of a Qwen3-MoE layer; ``__call__(x [..., H])`` returns the expert mixture (the
    block adds the residual).  Keeps one extra copy of the gate and up experts, interleaved per expert in blocks of 8
    rows, for the grouped GEMM's SwiGLU epilogue."""

    def __init__(
        self,
        w_router: QuantizedWeights,
        w_gate: QuantizedWeights,
        w_up: QuantizedWeights,
        w_down: QuantizedWeights,
        num_experts_per_tok: int,
        norm_topk_prob: bool = False,
    ):
        self.w_router = w_router
        self.w_gate = w_gate
        self.w_up = w_up
        self.w_down = w_down
        self.num_experts_per_tok = num_experts_per_tok
        self.norm_topk_prob = norm_topk_prob
        _check_router(w_router)
        E, inter, hidden = _experts(w_gate, "Moe")
        if _experts(w_up, "Moe") != (E, inter, hidden) or _experts(w_down, "Moe") != (E, hidden, inter):
            raise ValueError("Moe: gate / up must be [E, I, H] and down [E, H, I] experts")
        if inter % 128 or hidden % 128:
            # each is the reduction width of one grouped projection, which takes whole 128-wide quantisation groups
            raise ValueError(f"Moe: the hidden size ({hidden}) and the experts' intermediate size ({inter}) must be multiples of 128")
        self.num_experts, self.intermediate_size, self.hidden_size = E, inter, hidden

        def pairs(g: torch.Tensor, u: torch.Tensor) -> torch.Tensor:
            # flattened [E I] rows: blocks of 8 never straddle two experts, so expert e owns rows [2 I e, 2 I (e + 1))
            return ext.interleave_gate_up(g.reshape(E * inter, -1), u.reshape(E * inter, -1)).reshape(E, 2 * inter, -1)

        self.w_gate_up = QuantizedWeights(
            scales=pairs(w_gate.scales, w_up.scales),
            biases=pairs(w_gate.biases, w_up.biases),
            group_size=w_gate.group_size,
            bits=w_gate.bits,
            weight=pairs(as_packed_i32(w_gate.weight), as_packed_i32(w_up.weight)),
        )

    def __call__(self, x: torch.Tensor) -> torch.Tensor:
        *lead, H = x.shape
        h = x.reshape(-1, H).contiguous()
        k = self.num_experts_per_tok
        _, ids, scores = route_topk(h, self.w_router, k, self.norm_topk_prob)
        return self.experts(h, ids, scores).reshape(*lead, H)

    def experts(self, h: torch.Tensor, ids: torch.Tensor, scores: torch.Tensor, residual: torch.Tensor | None = None, gather_norm=None,
                next_norm=None):
        """Steps after routing, for ``h [T, H]``, ``ids`` / ``scores [T, k]``: the expert mixture, plus ``residual``.
        ``gather_norm = (weight, eps)``: ``h`` is not yet normalised and the gather applies that RMSNorm to each row it
        copies.  ``next_norm = (weight, eps)``: also return the RMSNorm of the result, as ``(out, normed)``."""
        T, H = h.shape
        k = self.num_experts_per_tok
        E, inter = self.num_experts, self.intermediate_size
        # the tile width follows (T, k, E) alone, so both projections share one table when either runs on the wgmma kernel
        nt = max(ext.moe_grouped_matmul_route(T, k, E, H, 2 * inter, ext.EPI_SWIGLU_PAIRS, h.dtype, h, self.w_gate_up.weight)[1],
                 ext.moe_grouped_matmul_route(T, k, E, inter, H, ext.EPI_NONE, h.dtype, h, self.w_down.weight)[1])
        offsets, perm, tiles = _group(ids.reshape(-1).contiguous(), E, nt)
        xs = ext.moe_gather(h, perm, k) if gather_norm is None else ext.moe_gather(h, perm, k, gather_norm[0], gather_norm[1])
        act = _grouped(xs, self.w_gate_up, offsets, tiles, k, None, ext.EPI_SWIGLU_PAIRS)
        y = _grouped(act, self.w_down, offsets, tiles, k, perm, ext.EPI_NONE)
        if next_norm is None:
            return ext.moe_combine(y, scores.contiguous(), residual)
        return ext.moe_combine(y, scores.contiguous(), residual, next_norm[0], next_norm[1])
