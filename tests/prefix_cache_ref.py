"""CPU stand-in of ``paged_cache_copy_prefix`` for the host tests of prefix caching: the same argument checks as the
shim (``check_prefix_copies``), then the copy as torch slicing.  Also the expected result of a copy list, which the GPU
tests compare the kernel against."""

import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


def copy_prefix_like_ext(key_slabs, value_slabs, copies, stream=None):
    for layer, src, dst, slots in ext.check_prefix_copies(key_slabs, value_slabs, copies):
        for slab in (key_slabs[layer], value_slabs[layer]):
            slab[dst, :, :slots] = slab[src, :, :slots]


def expected_after(key_slabs, value_slabs, copies):
    """Clones of the slabs with ``copies`` applied, from the slabs as they are now."""
    keys, values = [k.clone() for k in key_slabs], [v.clone() for v in value_slabs]
    copy_prefix_like_ext(keys, values, copies)
    return keys, values


def install(ext_module, monkeypatch) -> None:
    monkeypatch.setattr(ext_module, "paged_cache_copy_prefix", copy_prefix_like_ext)
