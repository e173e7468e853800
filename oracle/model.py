"""tiny_llm_ref's CPU-capable model path, restated on CPU torch.

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).  This is
``Qwen3ModelWeek2(mlx_model, checkpoint="kv-cache")``
(``src/tiny_llm_ref/qwen3_week2.py:251-392``): packed weights
dequantised to dense bf16 at load (``:286``), readable RMSNorm / RoPE / SiLU,
attention promoted to fp32 (``:138-144``), concat-growth KV cache
(``kv_cache.py:246-276``), driven by the greedy loop of
``simple_generate_with_kv_cache`` (``generate.py:49-81``).  It is the only
end-to-end path of the reference that runs without a GPU, hence "the
reference's CPU path" for parity of whole-model logits and for the reported
``cpu_baseline``.
"""

from __future__ import annotations

import time

import torch

from . import ops
from .readable import RMSNorm, RoPE, linear, scaled_dot_product_attention_grouped, silu


class DenseCache:
    """TinyKvFullCache (kv_cache.py:246-287)."""

    def __init__(self):
        self.key_values = None
        self.offset = 0

    def update_and_fetch(self, key, value, mask_length=None, mask=None):
        if self.key_values is None:
            self.key_values = (key, value)
            self.offset = key.shape[2]
        else:
            k, v = self.key_values
            self.key_values = (torch.cat([k, key], dim=2), torch.cat([v, value], dim=2))
            self.offset += key.shape[2]
        return (*self.key_values, self.offset, mask)


def _dense(layer) -> torch.Tensor:
    """dequantize_linear (quantize.py:93-100): MLX dequantise then bf16."""
    return ops.dequantize_weights(layer.weight, layer.scales, layer.biases, layer.group_size, layer.bits).to(torch.bfloat16)


class _Attention:
    def __init__(self, args, attn):
        self.hq, self.hkv, self.d = args.num_attention_heads, args.num_key_value_heads, args.head_dim
        self.scale = self.d**-0.5
        self.wq, self.wk, self.wv, self.wo = (_dense(attn.q_proj), _dense(attn.k_proj), _dense(attn.v_proj), _dense(attn.o_proj))
        self.rope = RoPE(self.d, args.max_position_embeddings, args.rope_theta)
        self.q_norm = RMSNorm(self.d, attn.q_norm.weight, eps=args.rms_norm_eps)
        self.k_norm = RMSNorm(self.d, attn.k_norm.weight, eps=args.rms_norm_eps)

    def __call__(self, x, offsets, cache, mask):
        B, L, _ = x.shape
        q = self.q_norm(linear(x, self.wq).reshape(B, L, self.hq, self.d))
        k = self.k_norm(linear(x, self.wk).reshape(B, L, self.hkv, self.d))
        v = linear(x, self.wv).reshape(B, L, self.hkv, self.d)
        sl = [slice(o, o + L) for o in offsets]
        q, k = self.rope(q, offset=sl), self.rope(k, offset=sl)
        q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)
        k, v, _, mask = cache.update_and_fetch(k, v, mask_length=L, mask=mask)
        o = scaled_dot_product_attention_grouped(
            q.to(torch.float32), k.to(torch.float32), v.to(torch.float32), scale=self.scale, mask=mask
        ).to(x.dtype)
        o = o.transpose(1, 2).reshape(B, L, self.hq * self.d)
        return linear(o, self.wo)


class _Block:
    def __init__(self, args, layer):
        self.attn = _Attention(args, layer.self_attn)
        self.w_gate, self.w_up, self.w_down = (_dense(layer.mlp.gate_proj), _dense(layer.mlp.up_proj), _dense(layer.mlp.down_proj))
        self.ln1 = RMSNorm(args.hidden_size, layer.input_layernorm.weight, eps=args.rms_norm_eps)
        self.ln2 = RMSNorm(args.hidden_size, layer.post_attention_layernorm.weight, eps=args.rms_norm_eps)

    def __call__(self, x, offsets, cache, mask):
        h = x + self.attn(self.ln1(x), offsets, cache, mask)
        y = self.ln2(h)
        return h + linear(silu(linear(y, self.w_gate)) * linear(y, self.w_up), self.w_down)


class ReferenceCpuModel:
    """Qwen3ModelWeek2(checkpoint="kv-cache") on CPU torch."""

    def __init__(self, mlx_model):
        a = mlx_model.args
        self.args = a
        self.num_hidden_layers = a.num_hidden_layers
        self.embed = _dense(mlx_model.model.embed_tokens)
        self.blocks = [_Block(a, layer) for layer in mlx_model.model.layers]
        self.norm = RMSNorm(a.hidden_size, mlx_model.model.norm.weight, eps=a.rms_norm_eps)
        self.lm_head = None if a.tie_word_embeddings else _dense(mlx_model.lm_head)

    def create_kv_cache(self):
        return [DenseCache() for _ in range(self.num_hidden_layers)]

    def __call__(self, inputs, offset, cache, logits_to_keep=None):
        B, L = inputs.shape
        offsets = [int(offset)] * B if isinstance(offset, int) else [int(o) for o in offset]
        h = self.embed[inputs.to(torch.int64)]
        mask = None if L == 1 else "causal"  # qwen3_week2.py:371
        for block, layer_cache in zip(self.blocks, cache):
            h = block(h, offsets, layer_cache, mask)
        if logits_to_keep is not None:
            if logits_to_keep <= 0:
                raise ValueError("logits_to_keep must be positive")
            h = h[:, -logits_to_keep:, :]
        h = self.norm(h)
        return linear(h, self.embed if self.lm_head is None else self.lm_head)


def greedy_decode(model, prompt_ids, max_new_tokens, return_logprobs=False, timings=None):
    """generate.py:49-81 without the tokenizer: prefill, then one token a step.

    Returns the generated ids (first one comes from the prefill).  ``timings``
    (a dict) receives ``prefill_s`` and the list ``decode_s``.
    """
    cache = model.create_kv_cache()
    tokens = torch.tensor(prompt_ids, dtype=torch.int64)[None]
    offset, out, logprobs, decode_s = 0, [], [], []
    for step in range(max_new_tokens):
        t0 = time.perf_counter()
        logits = model(tokens, offset, cache, logits_to_keep=1)[:, -1, :].to(torch.float32)
        lp = logits - torch.logsumexp(logits, dim=-1, keepdim=True)
        nxt = int(torch.argmax(lp, dim=-1)[0])
        dt = time.perf_counter() - t0
        if timings is not None:
            if step == 0:
                timings["prefill_s"] = dt
            else:
                decode_s.append(dt)
        out.append(nxt)
        if return_logprobs:
            logprobs.append(lp[0])
        offset += tokens.shape[1]
        tokens = torch.tensor([[nxt]], dtype=torch.int64)
    if timings is not None:
        timings["decode_s"] = decode_s
    return (out, logprobs) if return_logprobs else out
