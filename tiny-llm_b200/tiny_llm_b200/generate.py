"""Single-request greedy generation with a KV cache
(``src/tiny_llm_ref/generate.py:49-81``)."""

from __future__ import annotations

import torch

from .batch import greedy_tokens


def _release_kv_cache(kv_cache) -> None:
    if kv_cache is not None:
        for layer_cache in kv_cache:
            layer_cache.release()


def greedy_generate_ids(model, prompt_ids, max_new_tokens: int, eos_token_id: int | None = None, device=None, on_token=None, sampler=None):
    """The loop of ``simple_generate_with_kv_cache`` on token ids: the whole
    prompt is prefilled at offset 0 (its last-row logits give the first token),
    then one token per step at a growing offset.  Returns the generated ids.
    ``sampler`` (``make_sampler``; CUDA extension - the reference's cached loop is greedy only) draws
    from ``logits - logsumexp`` instead of taking the arg-max."""
    kv_cache = model.create_kv_cache()
    produced: list[int] = []
    try:
        tokens = torch.as_tensor(list(prompt_ids), dtype=torch.int32, device=device)
        offset = 0
        while len(produced) < max_new_tokens:
            logits = model(tokens[None], offset, kv_cache, logits_to_keep=1)
            if sampler is None:
                token = greedy_tokens(logits[:, -1, :])
            else:
                row = logits[:, -1, :].to(torch.float32)
                token = sampler(row - torch.logsumexp(row, dim=-1, keepdim=True))
            value = int(token.reshape(-1)[0])  # device->host read, one per step (mx.eval + .item())
            if eos_token_id is not None and value == eos_token_id:
                break
            produced.append(value)
            if on_token is not None:
                on_token(value)
            offset += tokens.numel()
            tokens = token.reshape(1).to(torch.int32)
    finally:
        _release_kv_cache(kv_cache)
    return produced


def simple_generate_with_kv_cache(model, tokenizer, prompt: str, max_new_tokens: int = 1 << 30) -> str:
    """generate.py:49-81 - streams the text to stdout and returns it."""
    detokenizer = tokenizer.detokenizer
    detokenizer.reset()

    def emit(token: int) -> None:
        detokenizer.add_token(token)
        print(detokenizer.last_segment, end="", flush=True)

    device = getattr(model, "device", None)
    greedy_generate_ids(
        model,
        tokenizer.encode(prompt, add_special_tokens=False),
        max_new_tokens,
        eos_token_id=tokenizer.eos_token_id,
        device=device,
        on_token=emit,
    )
    return detokenizer.text
