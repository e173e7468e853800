"""CPU stand-in for the native extension module, for tests only.

TEST INFRASTRUCTURE (see ``oracle/__init__.py``).  Exposes the function surface
of ``_ext`` (``src/extensions_ref/bindings.cpp:14-46``) over
``oracle.ops`` so that ``tests/`` can exercise the product's *host* logic
(page pools, block tables, scheduler, model wiring) on CPU tensors by
monkeypatching ``tiny_llm_ext_b200``'s entry points.  The product never does
this itself.
"""

from __future__ import annotations

from .ops import (  # noqa: F401
    decode_attention,
    paged_attention,
    paged_cache_update,
    quantized_embedding,
    quantized_matmul,
    rms_norm,
    rope,
    swiglu,
)

import torch


def add(a, b, stream=None):
    return a + b


def argmax(logits, stream=None):
    return torch.argmax(logits.to(torch.float32), dim=-1).to(torch.int32)


def paged_cache_append_decode(key_pages, value_pages, keys, values, block_table, context_lens, stream=None):
    """Row b writes its single token at position context_lens[b]-1 (idle rows skipped)."""
    page_size = key_pages.shape[2]
    for b in range(keys.shape[0]):
        ctx = int(context_lens[b])
        if ctx <= 0:
            continue
        tok = ctx - 1
        pid = int(block_table[b, tok // page_size])
        if pid < 0 or pid >= key_pages.shape[0]:
            continue
        key_pages[pid, :, tok % page_size, :] = keys[b, :, 0, :]
        value_pages[pid, :, tok % page_size, :] = values[b, :, 0, :]


OPS = (
    "quantized_matmul",
    "quantized_embedding",
    "rms_norm",
    "rope",
    "swiglu",
    "decode_attention",
    "paged_cache_update",
    "paged_attention",
    "add",
    "argmax",
    "paged_cache_append_decode",
)


def load_library(path: str) -> None:  # utils.cpp:9-14 registers a metallib; nothing to do
    return None


def install(ext_module, monkeypatch=None) -> None:
    """Point ``ext_module``'s eight ops at the CPU restatement."""
    import sys

    me = sys.modules[__name__]
    for name in OPS:
        if monkeypatch is not None:
            monkeypatch.setattr(ext_module, name, getattr(me, name))
        else:
            setattr(ext_module, name, getattr(me, name))
