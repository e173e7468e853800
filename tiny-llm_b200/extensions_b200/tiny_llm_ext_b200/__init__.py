"""H100 (sm_90a) replacement for tiny-llm's native extension module.

Same function names, positional order, keyword names and defaults as the
nanobind module ``tiny_llm_ext_ref._ext``
(``src/extensions_ref/bindings.cpp:14-46``), but the arrays are
contiguous CUDA ``torch.Tensor`` s instead of ``mx.array`` s and ``stream`` is
an optional ``torch.cuda.Stream``.  Every function is a thin ctypes call into
``libtiny_llm_b200.so`` (C ABI: ``include/tiny_llm_b200.h``); torch only owns
the device memory and the stream.

There is no CPU path: like the reference primitives' ``eval_cpu``
(``quantized_matmul.cpp:103-109``) a CPU tensor raises
``"<op>: the course extension is GPU-only"``, and a missing shared library
raises at import.  Builder-time shape/dtype checks raise ``RuntimeError`` with
the reference's messages (``quantized_matmul.cpp:24-72``,
``week2_kernels.cpp:36-84``, ``paged_attention.cpp:14-31,77-122``).
"""

from __future__ import annotations

import ctypes
import os
from pathlib import Path

import torch

__all__ = [
    "load_library",
    "quantized_matmul",
    "quantized_embedding",
    "rms_norm",
    "rope",
    "rope_table",
    "rope_default_inv_freq",
    "rms_norm_route",
    "rope_route",
    "qk_norm_rope_route",
    "swiglu",
    "decode_attention",
    "paged_cache_update",
    "paged_attention",
    # CUDA extension
    "paged_attention_route",
    "paged_cache_append_decode",
    "paged_cache_copy_prefix",
    "add",
    "argmax",
    "sample",
    "sample_penalized",
    "sample_constrained",
    "speculative_sample",
    "SPECULATIVE_SAMPLE_MAX_VOCAB",
    "log_rows",
    "ngram_propose",
    "beam_select",
    "NGRAM_MAX_K",
    "NGRAM_MAX_N",
    "NGRAM_MAX_APPEND",
    "NGRAM_TILE",
    "NGRAM_STATE_WORDS",
    "constraint_token_masks",
    "json_token_masks",
    "json_advance",
    "JSON_STATE_WORDS",
    "schema_token_masks",
    "schema_advance",
    "SCHEMA_STATE_WORDS",
    "logprobs",
    "LOGPROBS_MAX_N",
    "decode_advance",
    "quantized_matmul_fused",
    "quantized_matmul_route",
    "decode_qk_norm_rope_append",
    "chunk_qk_norm_rope_append",
    "set_pdl",
    "launch_count",
    "device_info",
    "current_library_path",
    "quantized_matmul_residual_norm",
    "paged_attention_token_major",
    "qkv_project_rope_append",
    "moe_topk",
    "moe_group",
    "moe_gather",
    "moe_grouped_matmul",
    "moe_grouped_matmul_route",
    "moe_combine",
    "moe_router",
    "MOE_ROUTER_GROUP",
    "LoraSite",
    "lora_apply",
    "lora_apply_route",
    "shared_prefix_attention",
    "shared_prefix_attention_workspace",
    "paged_attention_segments",
    "embed_pool",
    "paged_attention_prefixed_segments",
    "select_logits",
    "SELECT_MAX_IDS",
]

_HERE = Path(__file__).resolve().parent
_LIB_NAME = "libtiny_llm_b200.so"
_lib = None
_lib_path = None

_VP = ctypes.c_void_p
_I = ctypes.c_int
_F = ctypes.c_float
_LL = ctypes.c_longlong
_SZ = ctypes.c_size_t

_SIGNATURES = {
    "tl_abi_version": (_I, []),
    "tl_last_error": (ctypes.c_char_p, []),
    "tl_launch_count": (_LL, []),
    "tl_device_info": (_I, [ctypes.POINTER(_I)] * 3),
    "tl_quantized_matmul_workspace": (_SZ, [_I] * 6),
    "tl_quantized_matmul": (_I, [_VP] * 5 + [_I] * 6 + [_VP, _SZ, _VP]),
    "tl_quantized_embedding": (_I, [_VP] * 5 + [_I] * 4 + [_VP]),
    "tl_quantized_matmul_workspace_bits": (_SZ, [_I] * 7),
    "tl_quantized_matmul_bits": (_I, [_VP] * 5 + [_I] * 7 + [_VP, _SZ, _VP]),
    "tl_quantized_embedding_bits": (_I, [_VP] * 5 + [_I] * 5 + [_VP]),
    "tl_rms_norm": (_I, [_VP] * 3 + [_I, _I, _F, _I, _VP]),
    "tl_rope": (_I, [_VP] * 3 + [_I] * 5 + [_F, _I, _I, _VP]),
    "tl_rope_table": (_I, [_VP] * 3 + [_I] * 5 + [_F, _I, _I, _VP, _VP]),
    "tl_rope_inv_freq": (_I, [_VP, _I, _F, _VP]),
    "tl_rms_norm_route": (_I, [_I, _I] + [_VP] * 3 + [ctypes.POINTER(_I)]),
    "tl_rope_route": (_I, [_I] * 6),
    "tl_qk_norm_rope_route": (_I, [_I] * 4),
    "tl_swiglu": (_I, [_VP] * 3 + [_LL, _I, _VP]),
    "tl_add": (_I, [_VP] * 3 + [_LL, _I, _VP]),
    "tl_decode_attention": (_I, [_VP] * 5 + [_I] * 6 + [_F, _I, _I, _I, _VP]),
    "tl_paged_cache_update": (_I, [_VP, _VP] + [_I] * 8 + [_VP]),
    "tl_paged_cache_append_decode": (_I, [_VP] * 6 + [_I] * 7 + [_VP]),
    "tl_paged_attention_workspace": (_SZ, [_I] * 6),
    "tl_paged_attention": (_I, [_VP] * 6 + [_I] * 6 + [_F] + [_I] * 4 + [_VP, _SZ, _VP]),
    "tl_paged_attention_route": (_I, [_VP] * 4 + [_I] * 9),
    "tl_argmax_workspace": (_SZ, [_I, _I]),
    "tl_argmax": (_I, [_VP, _VP, _I, _I, _I, _VP, _SZ, _VP]),
    "tl_decode_advance": (_I, [_VP] * 6 + [_I, _I, _VP]),
    "tl_sample": (_I, [_VP] * 7 + [_I] * 3 + [_VP]),
    "tl_speculative_sample": (_I, [_VP] * 9 + [_I] * 3 + [_VP]),
    "tl_log_rows": (_I, [_VP] * 3 + [_I, _LL, _VP]),
    "tl_ngram_propose": (_I, [_VP, _I, _I, _VP] + [_I] * 4 + [_VP] * 3 + [_I] * 3 + [_VP]),
    "tl_beam_select": (_I, [_VP] * 3 + [_I] * 3 + [_VP, _I, _VP, _VP]),
    "tl_sample_penalized": (_I, [_VP] * 12 + [_I] * 3 + [_VP]),
    "tl_sample_constrained": (_I, [_VP] * 13 + [_I] * 3 + [_VP]),
    "tl_constraint_token_masks": (_I, [_VP, _VP, _I, _VP, _VP, _I, _VP, _I, _VP, _VP, _VP]),
    "tl_json_token_masks": (_I, [_VP, _VP, _I, _I, _VP]),
    "tl_json_advance": (_I, [_VP] * 4 + [_I, _VP]),
    "tl_schema_token_masks": (_I, [_VP, _VP, _I, _I, _I, _VP]),
    "tl_schema_advance": (_I, [_VP] * 4 + [_I, _VP]),
    "tl_logprobs": (_I, [_VP] * 9 + [_I] * 5 + [_VP]),
    "tl_qkv_project_rope_append": (_I, [_VP] * 13 + [_I] * 5 + [_F, _F] + [_I] * 5 + [_VP, _SZ, _VP]),
    "tl_qkv_project_rope_append_table": (_I, [_VP] * 13 + [_I] * 5 + [_F, _F] + [_I] * 5 + [_VP, _SZ, _VP, _VP]),
    "tl_qkv_project_rope_append_bits": (_I, [_VP] * 13 + [_I] * 5 + [_F, _F] + [_I] * 6 + [_VP, _SZ, _VP]),
    "tl_qkv_project_rope_append_table_bits": (_I, [_VP] * 13 + [_I] * 5 + [_F, _F] + [_I] * 6 + [_VP, _SZ, _VP, _VP]),
    "tl_paged_attention_token_major": (_I, [_VP] * 6 + [_I] * 5 + [_F] + [_I] * 3 + [_VP]),
    "tl_paged_attention_token_major_workspace": (_SZ, [_I] * 4),
    "tl_paged_attention_token_major_split": (_I, [_VP] * 6 + [_I] * 5 + [_F] + [_I] * 3 + [_VP, _SZ, _VP]),
    "tl_quantized_matmul_fused_workspace": (_SZ, [_I] * 6),
    "tl_quantized_matmul_route": (_I, [_I] * 8 + [_VP] * 4 + [ctypes.POINTER(_I)] * 4),
    "tl_quantized_matmul_fused": (_I, [_VP] * 7 + [_I] * 6 + [_F, _I, _VP, _SZ, _VP]),
    "tl_quantized_matmul_residual_norm": (_I, [_VP] * 8 + [_I] * 3 + [_F, _I, _VP, _SZ, _VP]),
    "tl_quantized_matmul_fused_workspace_bits": (_SZ, [_I] * 7),
    "tl_quantized_matmul_route_bits": (_I, [_I] * 9 + [_VP] * 4 + [ctypes.POINTER(_I)] * 4),
    "tl_quantized_matmul_fused_bits": (_I, [_VP] * 7 + [_I] * 6 + [_F, _I, _I, _VP, _SZ, _VP]),
    "tl_quantized_matmul_residual_norm_bits": (_I, [_VP] * 8 + [_I] * 3 + [_F, _I, _I, _VP, _SZ, _VP]),
    "tl_decode_qk_norm_rope_append": (_I, [_VP] * 9 + [_I] * 4 + [_F, _F] + [_I] * 4 + [_VP]),
    "tl_decode_qk_norm_rope_append_table": (_I, [_VP] * 9 + [_I] * 4 + [_F, _F] + [_I] * 4 + [_VP, _VP]),
    "tl_chunk_qk_norm_rope_append": (_I, [_VP] * 9 + [_I] * 4 + [_F, _F] + [_I] * 4 + [_VP]),
    "tl_chunk_qk_norm_rope_append_table": (_I, [_VP] * 9 + [_I] * 4 + [_F, _F] + [_I] * 4 + [_VP, _VP]),
    "tl_decode_attention_fused_workspace": (_SZ, [_I, _I, _I]),
    "tl_decode_attention_fused": (_I, [_VP] * 11 + [_I] * 4 + [_F, _F] + [_I] * 5 + [_VP]),
    "tl_decode_attention_fused_rows_workspace": (_SZ, [_I, _I, _I, _I]),
    "tl_decode_attention_fused_rows": (_I, [_VP] * 11 + [_I] * 5 + [_F, _F] + [_I] * 5 + [_VP]),
    "tl_paged_cache_append_chunk": (_I, [_VP] * 5 + [_I] * 4 + [ctypes.c_longlong, ctypes.c_longlong, _I, _VP]),
    "tl_paged_cache_copy_prefix": (_I, [_VP, _VP] + [_I] * 4 + [_VP]),
    "tl_set_pdl": (_I, [_I]),
    "tl_moe_topk": (_I, [_VP] * 4 + [_I] * 5 + [_VP]),
    "tl_moe_tile_table_size": (_I, [_I] * 3),
    "tl_moe_group": (_I, [_VP, _I, _I, _I] + [_VP] * 4),
    "tl_moe_gather": (_I, [_VP] * 3 + [_F, _VP] + [_I] * 4 + [_VP]),
    "tl_moe_grouped_matmul_route": (_I, [_I] * 7 + [_VP] * 2 + [ctypes.POINTER(_I)] * 2),
    "tl_moe_grouped_matmul": (_I, [_VP] * 8 + [_I] * 7 + [_VP]),
    "tl_moe_combine": (_I, [_VP] * 4 + [_F, _VP, _VP] + [_I] * 4 + [_VP]),
    "tl_moe_router": (_I, [_VP, _VP, _F] + [_VP] * 4 + [_I] * 4 + [_VP]),
    "tl_lora_apply_route": (_I, [_I, _I, _VP]),
    "tl_lora_apply": (_I, [_VP] * 6 + [_I, _I, _VP]),
    "tl_shared_prefix_attention_workspace": (_SZ, [_I] * 5),
    "tl_shared_prefix_attention": (_I, [_VP] * 7 + [_I, _VP] + [_I] * 5 + [_F] + [_I] * 3 + [_VP, _SZ, _VP]),
    "tl_paged_attention_segments": (_I, [_VP] * 6 + [_I] * 5 + [_F] + [_I] * 3 + [_VP]),
    "tl_embed_pool": (_I, [_VP, _VP, _F, _VP] + [_I] * 6 + [_VP, _I, _VP]),
    "tl_paged_attention_prefixed_segments": (_I, [_VP] * 8 + [_I] * 5 + [_F] + [_I] * 3 + [_VP]),
    "tl_select_logits": (_I, [_VP, _VP, _F, _VP] + [_I] * 3 + [_VP] * 3 + [_I, _I, _VP, _I, _VP, _VP, _I, _VP]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def load_library(path: str | os.PathLike | None = None) -> None:
    """Load ``libtiny_llm_b200.so`` (reference: ``load_library(path)`` registers
    the metallib, ``utils.cpp:9-14``).  Called once at import with the in-tree
    library; raises ``ImportError`` when it has not been built."""
    global _lib, _lib_path
    candidate = Path(path) if path is not None else _HERE / _LIB_NAME
    if candidate.is_dir():
        candidate = candidate / _LIB_NAME
    if not candidate.exists():
        raise ImportError(
            f"{candidate} not found: build it with `python tiny-llm_b200/csrc/build.py` "
            "(there is no CPU fallback for the CUDA backend)"
        )
    lib = ctypes.CDLL(str(candidate))
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here == ABI mismatch, fail loudly
        fn.restype = restype
        fn.argtypes = argtypes
    _lib, _lib_path = lib, candidate


def current_library_path() -> Path:
    return _lib_path


_DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
_FLOATS = (torch.float32, torch.float16, torch.bfloat16)
_HALF = (torch.float16, torch.bfloat16)
_PACKED = (torch.int32, torch.uint32)


def _gpu(op: str, *tensors: torch.Tensor) -> None:
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError(f"{op}: the course extension is GPU-only")


def _contig(op: str, **named: torch.Tensor) -> None:
    for name, t in named.items():
        if not t.is_contiguous():
            raise RuntimeError(f"{op}: {name} must be contiguous")


def _inv_freq(op: str, inv_freq, half: int) -> None:
    """A RoPE frequency table (``rope_table`` and the ``inv_freq=`` forms): float64 [half], contiguous."""
    if inv_freq is None:
        return
    if inv_freq.dtype != torch.float64 or tuple(inv_freq.shape) != (half,) or not inv_freq.is_contiguous():
        raise RuntimeError(f"{op}: inv_freq must be a contiguous float64 [{half}] table")
    _gpu(op, inv_freq)


def _norm_weights(op: str, dtype: torch.dtype, head_dim: int, **named: torch.Tensor) -> None:
    """Per-head RMSNorm weights: the kernels read head_dim contiguous elements of the activation dtype."""
    for name, w in named.items():
        if w.dtype != dtype:
            raise RuntimeError(f"{op}: {name} must have the dtype of qkv ({dtype})")
        if tuple(w.shape) != (head_dim,) or not w.is_contiguous():
            raise RuntimeError(f"{op}: {name} must be contiguous [head_dim = {head_dim}]")


def _int32(op: str, rows: int | None = None, **named: torch.Tensor) -> None:
    """int32 index tensors; with ``rows``, one entry per row ([rows])."""
    for name, t in named.items():
        if t.dtype != torch.int32:
            raise RuntimeError(f"{op}: {name} must be int32")
        if rows is not None and (t.dim() != 1 or t.shape[0] != rows):
            raise RuntimeError(f"{op}: {name} must hold one entry per row ([{rows}])")


def _block_table(op: str, block_table: torch.Tensor, rows: int | None) -> None:
    """int32 [rows, max_pages], or (rows None: a prefill chunk) the request's int32 [max_pages] row."""
    _int32(op, block_table=block_table)
    if block_table.dim() != (1 if rows is None else 2) or (rows is not None and block_table.shape[0] != rows):
        raise RuntimeError(f"{op}: block_table must be int32 " + ("[max_pages]" if rows is None else f"[{rows}, max_pages]"))


def _stream_ptr(stream, ref: torch.Tensor) -> int:
    if stream is None:
        return torch.cuda.current_stream(ref.device).cuda_stream
    return stream.cuda_stream


def _check(code: int) -> None:
    if code != 0:
        raise RuntimeError(_lib.tl_last_error().decode() or f"tiny_llm_b200 error {code}")


def _workspace(nbytes: int, device) -> torch.Tensor | None:
    if nbytes == 0:
        return None
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


_ZERO_WS: dict = {}
_ZERO_WS_KEEP: list = []  # outgrown buffers may still be referenced by captured CUDA graphs


def _zero_workspace(nbytes: int, device) -> torch.Tensor | None:
    """Persistent workspace per device for the split-reduction GEMM (fp32 partial planes): one buffer serves
    every launch issued in stream order and captured graphs keep a stable pointer."""
    if nbytes == 0:
        return None
    key = torch.device(device)
    buf = _ZERO_WS.get(key)
    if buf is None or buf.numel() < nbytes:
        if buf is not None:
            _ZERO_WS_KEEP.append(buf)
        buf = torch.zeros(max(nbytes, 16 << 20), dtype=torch.uint8, device=device)
        _ZERO_WS[key] = buf
    return buf


# --------------------------------------------------------------------------
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
    """``a [M,N] @ dequant(b [K,N*bits/32]).T -> [M,K]`` (bindings.cpp:16-33); ``bits`` is 4 or 8."""
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
    if bits not in (4, 8):
        raise RuntimeError("quantized_matmul: bits must be 4 or 8")
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
    if b.shape[1] != a.shape[1] * bits // 32:
        raise RuntimeError("quantized_matmul: a must have the same number of columns as b")
    _gpu("quantized_matmul", scales, biases, a, b)
    _contig("quantized_matmul", a=a, b=b, scales=scales, biases=biases)
    M, N = a.shape
    K = b.shape[0]
    out = torch.empty((M, K), dtype=a.dtype, device=a.device)
    code = _DTYPE_CODE[a.dtype]
    ws_bytes = _lib.tl_quantized_matmul_workspace_bits(M, N, K, code, int(bits), int(use_simdgroup), int(use_split_k))
    ws = _zero_workspace(ws_bytes, a.device)
    _check(
        _lib.tl_quantized_matmul_bits(
            scales.data_ptr(), biases.data_ptr(), a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, code, int(bits),
            int(use_simdgroup), int(use_split_k), None if ws is None else ws.data_ptr(), ws_bytes,
            _stream_ptr(stream, a),
        )
    )
    return out


def quantized_embedding(indices, scales, biases, weight, group_size, bits, stream=None):
    """Row gather + dequantise (bindings.cpp:34-35); ``bits`` is 4 or 8."""
    if indices.dtype not in _PACKED or weight.dtype not in _PACKED:
        raise RuntimeError("quantized_embedding: indices and weight must use 32-bit integers")
    if scales.dtype != biases.dtype or scales.dtype not in _HALF:
        raise RuntimeError("quantized_embedding: scales and biases must have the same 16-bit dtype")
    if group_size != 128 or bits not in (4, 8) or scales.shape != biases.shape:
        raise RuntimeError("quantized_embedding: expected 4-bit weights with group size 128" if bits == 4 else
                           "quantized_embedding: expected 4- or 8-bit weights with group size 128")
    dim = weight.shape[1] * 32 // bits
    if scales.shape[0] != weight.shape[0] or scales.shape[1] != dim // group_size:
        raise RuntimeError("quantized_embedding: incompatible parameter shapes")
    _gpu("quantized_embedding", indices, scales, biases, weight)
    _contig("quantized_embedding", indices=indices, scales=scales, biases=biases, weight=weight)
    out = torch.empty((*indices.shape, dim), dtype=scales.dtype, device=scales.device)
    _check(
        _lib.tl_quantized_embedding_bits(
            indices.data_ptr(), scales.data_ptr(), biases.data_ptr(), weight.data_ptr(), out.data_ptr(),
            indices.numel(), weight.shape[0], dim, _DTYPE_CODE[scales.dtype], int(bits), _stream_ptr(stream, scales),
        )
    )
    return out


def rms_norm(x, weight, eps, stream=None):
    """bindings.cpp:36; week2_kernels.cpp:36-42."""
    if x.dtype not in _FLOATS:
        raise RuntimeError("rms_norm: expected float32, float16, or bfloat16")
    if x.dtype != weight.dtype or weight.dim() != 1 or x.dim() < 1 or weight.shape[0] != x.shape[-1]:
        raise RuntimeError("rms_norm: weight must match the input dtype and final dimension")
    _gpu("rms_norm", x, weight)
    _contig("rms_norm", x=x, weight=weight)
    out = torch.empty_like(x)
    dim = x.shape[-1]
    rows = x.numel() // dim if dim else 0
    _check(_lib.tl_rms_norm(x.data_ptr(), weight.data_ptr(), out.data_ptr(), rows, dim, float(eps), _DTYPE_CODE[x.dtype], _stream_ptr(stream, x)))
    return out


def rope(x, offsets, dims, base, traditional=False, stream=None):
    """bindings.cpp:37-38; week2_kernels.cpp:44-55."""
    return _rope("rope", x, offsets, dims, base, None, traditional, stream)


def rope_table(x, offsets, dims, inv_freq, traditional=False, stream=None):
    """``rope`` with the frequencies of a float64 ``[dims / 2]`` device table (a scaled RoPE such as YaRN,
    ``rope_scaling.py``) instead of ``base^(-i / (dims / 2))``."""
    if inv_freq is None:
        raise RuntimeError("rope_table: inv_freq is required")
    return _rope("rope_table", x, offsets, dims, 0.0, inv_freq, traditional, stream)


def _rope(op, x, offsets, dims, base, inv_freq, traditional, stream):
    if x.dtype not in _FLOATS:
        raise RuntimeError(f"{op}: expected float32, float16, or bfloat16")
    if x.dim() != 4 or offsets.dtype != torch.int32 or offsets.dim() != 1 or offsets.shape[0] != x.shape[0]:
        raise RuntimeError(f"{op}: expected x=[B,L,H,D] and one int32 offset per batch row")
    if dims <= 0 or dims > x.shape[3] or dims % 2 != 0:
        raise RuntimeError(f"{op}: dims must be positive, even, and no larger than the head dimension")
    _inv_freq(op, inv_freq, int(dims) // 2)
    _gpu(op, x, offsets)
    _contig(op, x=x, offsets=offsets)
    out = torch.empty_like(x)
    B, L, H, D = x.shape
    args = (x.data_ptr(), offsets.data_ptr(), out.data_ptr(), B, L, H, D, int(dims), float(base), int(bool(traditional)),
            _DTYPE_CODE[x.dtype], _stream_ptr(stream, x))
    _check(_lib.tl_rope(*args) if inv_freq is None else _lib.tl_rope_table(*args, inv_freq.data_ptr()))
    return out


def rope_default_inv_freq(head_dim: int, base: float, device, stream=None) -> torch.Tensor:
    """float64 ``[head_dim / 2]`` unscaled RoPE frequencies formed on the device with the RoPE kernels' own expression
    (``exp2(-i / half * log2(base))`` in double): a site given this table computes the bits of its ``base`` path."""
    if head_dim <= 0 or head_dim % 2:
        raise RuntimeError("rope_inv_freq: head_dim must be positive and even")
    out = torch.empty(head_dim // 2, dtype=torch.float64, device=device)
    _gpu("rope_inv_freq", out)
    _check(_lib.tl_rope_inv_freq(out.data_ptr(), int(head_dim), float(base), _stream_ptr(stream, out)))
    return out


ROPE_ELEMENT, ROPE_HEADS = 0, 1
QKN_HEAD, QKN_ROW = 0, 1


def rms_norm_route(dim, dtype, x, weight, out):
    """The kernel ``rms_norm`` runs, decided without launching or reading anything: ``(threads_per_row, vec)`` with
    32 or 256 threads per row and ``vec`` True for 16-byte accesses.  ``x``, ``weight`` and ``out`` are tensors or plain
    addresses: only their 16-byte alignment counts.  ``dtype`` is a torch dtype."""

    def addr(t):
        return t.data_ptr() if isinstance(t, torch.Tensor) else int(t)

    vec = _I()
    code = _lib.tl_rms_norm_route(int(dim), _DTYPE_CODE[dtype], addr(x), addr(weight), addr(out), ctypes.byref(vec))
    _check(min(code, 0))
    return code, bool(vec.value)


def rope_route(B, L, H, D, dims, dtype):
    """``ROPE_HEADS`` (one thread per (token, pair) walking the heads) or ``ROPE_ELEMENT``: the kernel ``rope`` runs."""
    code = _lib.tl_rope_route(int(B), int(L), int(H), int(D), int(dims), _DTYPE_CODE[dtype])
    _check(min(code, 0))
    return code


def qk_norm_rope_route(num_heads, num_kv_heads, head_dim, dtype):
    """``QKN_ROW`` (one CTA per row) or ``QKN_HEAD`` (one CTA per head and row): the kernel the fused q/k norm + RoPE +
    K/V append runs in ``decode_qk_norm_rope_append``, ``chunk_qk_norm_rope_append`` and ``qkv_project_rope_append``."""
    code = _lib.tl_qk_norm_rope_route(int(num_heads), int(num_kv_heads), int(head_dim), _DTYPE_CODE[dtype])
    _check(min(code, 0))
    return code


def swiglu(gate, up, stream=None):
    """bindings.cpp:39; week2_kernels.cpp:57-63."""
    if gate.dtype not in _FLOATS:
        raise RuntimeError("swiglu: expected float32, float16, or bfloat16")
    if gate.dtype != up.dtype or gate.shape != up.shape:
        raise RuntimeError("swiglu: gate and up must have the same shape and dtype")
    _gpu("swiglu", gate, up)
    _contig("swiglu", gate=gate, up=up)
    out = torch.empty_like(gate)
    _check(_lib.tl_swiglu(gate.data_ptr(), up.data_ptr(), out.data_ptr(), gate.numel(), _DTYPE_CODE[gate.dtype], _stream_ptr(stream, gate)))
    return out


def decode_attention(query, key, value, mask, scale, is_causal, has_mask, num_heads, num_kv_heads, stream=None):
    """bindings.cpp:40-41; week2_kernels.cpp:65-84."""
    if query.dtype not in _FLOATS:
        raise RuntimeError("decode_attention: expected float32, float16, or bfloat16")
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
    _gpu("decode_attention", query, key, value, mask)
    _contig("decode_attention", query=query, key=key, value=value, mask=mask)
    out = torch.empty_like(query)
    rows, L, D = query.shape
    _check(
        _lib.tl_decode_attention(
            query.data_ptr(), key.data_ptr(), value.data_ptr(), mask.data_ptr(), out.data_ptr(), rows, L, key.shape[1], D,
            int(num_heads), int(num_kv_heads), float(scale), int(bool(is_causal)), int(bool(has_mask)),
            _DTYPE_CODE[query.dtype], _stream_ptr(stream, query),
        )
    )
    return out


def paged_cache_update(pages, values, page_id, start, stream=None):
    """In-place slice write; returns ``pages`` itself, as the reference output
    aliases its input buffer (bindings.cpp:43-44; paged_attention.cpp:14-31,46-49)."""
    if pages.dtype not in (torch.float32, torch.bfloat16) or values.dtype != pages.dtype:
        raise RuntimeError("paged_cache_update: pages and values must have the same float32 or bfloat16 dtype")
    if pages.dim() != 4 or values.dim() != 4 or values.shape[0] != 1:
        raise RuntimeError("paged_cache_update: expected pages [P, H, page_size, D] and values [1, H, length, D]")
    if values.shape[1] != pages.shape[1] or values.shape[3] != pages.shape[3]:
        raise RuntimeError("paged_cache_update: values must match the page head count and head dimension")
    if page_id < 0 or page_id >= pages.shape[0] or start < 0 or start + values.shape[2] > pages.shape[2]:
        raise RuntimeError("paged_cache_update: destination slice is outside page storage")
    _gpu("paged_cache_update", pages, values)
    if not pages.is_contiguous() or not values.is_contiguous():
        raise RuntimeError("paged_cache_update: pages and values must be contiguous")
    P, H, page_size, D = pages.shape
    _check(
        _lib.tl_paged_cache_update(pages.data_ptr(), values.data_ptr(), P, H, page_size, D, values.shape[2], int(page_id), int(start),
                                   _DTYPE_CODE[pages.dtype], _stream_ptr(stream, pages))
    )
    return pages


PAGE_SPANS = 64


class PageSpanList(ctypes.Structure):
    """``tl_page_span_list``: (page id, first row, rows, first source token) of up to 64 page slices."""

    _fields_ = [("page_id", ctypes.c_int32 * PAGE_SPANS), ("start", ctypes.c_int32 * PAGE_SPANS), ("count", ctypes.c_int32 * PAGE_SPANS),
                ("src", ctypes.c_int32 * PAGE_SPANS), ("n", ctypes.c_int32)]


def paged_cache_append_chunk(key_pages, value_pages, keys, values, spans, stream=None):
    """Write one request's chunk ``keys/values [1, H, L, D]`` (any head/token strides, unit inner
    stride) into the page slices ``spans = [(page_id, start, count, src_token), ...]`` - K and V,
    every page, one launch per 64 spans."""
    if key_pages.dtype not in (torch.float32, torch.bfloat16) or value_pages.dtype != key_pages.dtype or keys.dtype != key_pages.dtype or values.dtype != key_pages.dtype:
        raise RuntimeError("paged_cache_append_chunk: pages and values must have the same float32 or bfloat16 dtype")
    if key_pages.dim() != 4 or keys.dim() != 4 or keys.shape[0] != 1 or keys.shape != values.shape or key_pages.shape != value_pages.shape:
        raise RuntimeError("paged_cache_append_chunk: expected pages [P, H, page_size, D] and chunks [1, H, L, D]")
    if keys.shape[1] != key_pages.shape[1] or keys.shape[3] != key_pages.shape[3]:
        raise RuntimeError("paged_cache_append_chunk: chunks must match the page head count and head dimension")
    if keys.stride(3) != 1 or values.stride() != keys.stride():
        raise RuntimeError("paged_cache_append_chunk: chunks need a unit inner stride and identical K/V strides")
    _gpu("paged_cache_append_chunk", key_pages, value_pages, keys, values)
    if not key_pages.is_contiguous() or not value_pages.is_contiguous():
        raise RuntimeError("paged_cache_append_chunk: pages must be contiguous")
    P, H, page_size, D = key_pages.shape
    L = keys.shape[2]
    for pid, start, count, src in spans:
        if src < 0 or src + count > L:
            raise RuntimeError("paged_cache_append_chunk: source rows are outside the chunk")
    for first in range(0, len(spans), PAGE_SPANS):
        part = spans[first : first + PAGE_SPANS]
        rec = PageSpanList()
        rec.n = len(part)
        for i, (pid, start, count, src) in enumerate(part):
            rec.page_id[i], rec.start[i], rec.count[i], rec.src[i] = int(pid), int(start), int(count), int(src)
        _check(
            _lib.tl_paged_cache_append_chunk(key_pages.data_ptr(), value_pages.data_ptr(), keys.data_ptr(), values.data_ptr(), ctypes.byref(rec),
                                             P, H, page_size, D, keys.stride(1), keys.stride(2), _DTYPE_CODE[key_pages.dtype],
                                             _stream_ptr(stream, key_pages))
        )


PREFIX_COPY_LAYERS = 64
PREFIX_COPIES = 128


class KvSlabTable(ctypes.Structure):
    """``tl_kv_slab_table``: per layer, the K and V slab base pointers and the slab's page count (up to 64 layers)."""

    _fields_ = [("key", ctypes.c_void_p * PREFIX_COPY_LAYERS), ("value", ctypes.c_void_p * PREFIX_COPY_LAYERS),
                ("num_pages", ctypes.c_int32 * PREFIX_COPY_LAYERS), ("n", ctypes.c_int32)]


class PrefixCopyList(ctypes.Structure):
    """``tl_prefix_copy_list``: (layer, source page, destination page, slots) of up to 128 copies."""

    _fields_ = [("layer", ctypes.c_int32 * PREFIX_COPIES), ("src", ctypes.c_int32 * PREFIX_COPIES), ("dst", ctypes.c_int32 * PREFIX_COPIES),
                ("slots", ctypes.c_int32 * PREFIX_COPIES), ("n", ctypes.c_int32)]


def check_prefix_copies(key_slabs, value_slabs, copies) -> list[tuple[int, int, int, int]]:
    """Every check of ``paged_cache_copy_prefix`` that needs no device: the slabs (one ``[P, H, page_size, D]`` K and V
    per layer, one dtype, shared H / page_size / D, P per layer) and the records.  Returns the records as int tuples."""
    if len(key_slabs) != len(value_slabs) or not key_slabs:
        raise RuntimeError("paged_cache_copy_prefix: one key and one value slab per layer required")
    dtype, shape = key_slabs[0].dtype, tuple(key_slabs[0].shape[1:])
    if dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("paged_cache_copy_prefix: float32 or bfloat16 pages required")
    for k, v in zip(key_slabs, value_slabs):
        if k.dtype != dtype or v.dtype != dtype:
            raise RuntimeError("paged_cache_copy_prefix: every slab must have the same float32 or bfloat16 dtype")
        if k.dim() != 4 or k.shape != v.shape or tuple(k.shape[1:]) != shape:
            raise RuntimeError("paged_cache_copy_prefix: expected K/V slabs [P, H, page_size, D] with one H, page_size and D")
    page_size = shape[1]
    out, dsts, srcs = [], set(), set()
    for rec in copies:
        layer, src, dst, slots = (int(x) for x in rec)
        if not 0 <= layer < len(key_slabs):
            raise RuntimeError(f"paged_cache_copy_prefix: layer {layer} outside the {len(key_slabs)} slabs")
        pages = key_slabs[layer].shape[0]
        if not (0 <= src < pages and 0 <= dst < pages):
            raise RuntimeError(f"paged_cache_copy_prefix: page outside the {pages} pages of layer {layer}")
        if not 1 <= slots <= page_size:
            raise RuntimeError(f"paged_cache_copy_prefix: slots {slots} outside [1, {page_size}]")
        if src == dst:
            raise RuntimeError(f"paged_cache_copy_prefix: page {src} copied onto itself")
        if (layer, dst) in dsts:
            raise RuntimeError(f"paged_cache_copy_prefix: destination page {dst} named twice in layer {layer}")
        if (layer, dst) in srcs or (layer, src) in dsts:
            raise RuntimeError(f"paged_cache_copy_prefix: a page is both a source and a destination in layer {layer}")
        dsts.add((layer, dst))
        srcs.add((layer, src))
        out.append((layer, src, dst, slots))
    return out


def paged_cache_copy_prefix(key_slabs, value_slabs, copies, stream=None):
    """Copy on write of shared KV pages: for each ``(layer, src_page, dst_page, slots)`` of ``copies``,
    ``key_slabs[layer][dst, :, :slots] = key_slabs[layer][src, :, :slots]`` and the same for values.  Rows at or beyond
    ``slots`` of the destination and the source are not written.  One launch per 64 layers and 128 records."""
    recs = check_prefix_copies(key_slabs, value_slabs, copies)
    _gpu("paged_cache_copy_prefix", *key_slabs, *value_slabs)
    for t in (*key_slabs, *value_slabs):
        if not t.is_contiguous():
            raise RuntimeError("paged_cache_copy_prefix: slabs must be contiguous")
    if not recs:
        return
    _, H, page_size, D = key_slabs[0].shape
    for base in range(0, len(key_slabs), PREFIX_COPY_LAYERS):
        group = [r for r in recs if base <= r[0] < base + PREFIX_COPY_LAYERS]
        if not group:
            continue
        table = KvSlabTable()
        layers = range(base, min(base + PREFIX_COPY_LAYERS, len(key_slabs)))
        table.n = len(layers)
        for i, layer in enumerate(layers):
            table.key[i], table.value[i] = key_slabs[layer].data_ptr(), value_slabs[layer].data_ptr()
            table.num_pages[i] = key_slabs[layer].shape[0]
        for first in range(0, len(group), PREFIX_COPIES):
            part = group[first : first + PREFIX_COPIES]
            rec = PrefixCopyList()
            rec.n = len(part)
            for i, (layer, src, dst, slots) in enumerate(part):
                rec.layer[i], rec.src[i], rec.dst[i], rec.slots[i] = layer - base, src, dst, slots
            _check(
                _lib.tl_paged_cache_copy_prefix(ctypes.byref(table), ctypes.byref(rec), H, page_size, D, _DTYPE_CODE[key_slabs[0].dtype],
                                                _stream_ptr(stream, key_slabs[0]))
            )


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
    """bindings.cpp:45-46; paged_attention.cpp:77-122 (checks), :129-225 (dispatch)."""
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
    _gpu("paged_attention", query, key_pages, value_pages, block_table, context_lens)
    if not all(t.is_contiguous() for t in (query, key_pages, value_pages, block_table, context_lens)):
        raise RuntimeError("paged_attention: all inputs must be contiguous")
    rows, L, D = query.shape
    P, _, page_size, _ = key_pages.shape
    out = torch.empty_like(query)
    code = _DTYPE_CODE[query.dtype]
    ws_bytes = _lib.tl_paged_attention_workspace(rows, L, D, int(num_kv_heads), int(num_heads), code)
    ws = _workspace(ws_bytes, query.device)
    _check(
        _lib.tl_paged_attention(
            query.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), block_table.data_ptr(), context_lens.data_ptr(),
            out.data_ptr(), rows, L, D, P, page_size, block_table.shape[1], float(scale), int(bool(is_causal)),
            int(num_kv_heads), int(num_heads), code, None if ws is None else ws.data_ptr(), ws_bytes,
            _stream_ptr(stream, query),
        )
    )
    return out


PAGED_ROWWISE, PAGED_GQA, PAGED_FLASH, PAGED_WGMMA = 0, 1, 2, 3


def paged_attention_route(q, key_pages, value_pages, out, rows, L, D, num_pages, page_size, max_pages, num_kv_heads, num_heads, dtype):
    """The kernel ``paged_attention`` runs for these arguments (``PAGED_ROWWISE`` / ``PAGED_GQA`` / ``PAGED_FLASH`` /
    ``PAGED_WGMMA``), decided without launching or reading anything.  ``q``, ``key_pages``, ``value_pages`` and
    ``out`` are tensors or plain addresses: only their 16-byte alignment counts.  ``dtype`` is a torch dtype."""

    def addr(x):
        return x.data_ptr() if isinstance(x, torch.Tensor) else int(x)

    code = _lib.tl_paged_attention_route(addr(q), addr(key_pages), addr(value_pages), addr(out), int(rows), int(L), int(D), int(num_pages),
                                         int(page_size), int(max_pages), int(num_kv_heads), int(num_heads), _DTYPE_CODE[dtype])
    _check(min(code, 0))
    return code


# ---- CUDA extension (not in the reference module) -------------------------
def paged_cache_append_decode(key_pages, value_pages, keys, values, block_table, context_lens, stream=None):
    """Batched, device-driven form of the per-request K/V append
    (kv_cache.py:191-199 -> paged_kv_cache.py:196-234): row ``b`` of
    ``keys/values [B,H,1,D]`` lands at token ``context_lens[b]-1``."""
    if key_pages.shape != value_pages.shape or keys.shape != values.shape or keys.dim() != 4 or keys.shape[2] != 1:
        raise RuntimeError("paged_cache_append_decode: expected keys/values [B, H, 1, D]")
    if key_pages.dtype != keys.dtype or value_pages.dtype != values.dtype or key_pages.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("paged_cache_append_decode: dtype mismatch")
    if block_table.dtype != torch.int32 or context_lens.dtype != torch.int32:
        raise RuntimeError("paged_cache_append_decode: block_table and context_lens must be int32")
    _gpu("paged_cache_append_decode", key_pages, value_pages, keys, values, block_table, context_lens)
    _contig("paged_cache_append_decode", key_pages=key_pages, value_pages=value_pages, keys=keys, values=values,
            block_table=block_table, context_lens=context_lens)
    P, H, page_size, D = key_pages.shape
    B = keys.shape[0]
    _check(
        _lib.tl_paged_cache_append_decode(
            key_pages.data_ptr(), value_pages.data_ptr(), keys.data_ptr(), values.data_ptr(), block_table.data_ptr(),
            context_lens.data_ptr(), B, P, H, page_size, D, block_table.shape[1], _DTYPE_CODE[keys.dtype],
            _stream_ptr(stream, keys),
        )
    )


def add(a, b, stream=None):
    if a.dtype not in _FLOATS or a.dtype != b.dtype or a.shape != b.shape:
        raise RuntimeError("add: operands must have the same shape and float dtype")
    _gpu("add", a, b)
    _contig("add", a=a, b=b)
    out = torch.empty_like(a)
    _check(_lib.tl_add(a.data_ptr(), b.data_ptr(), out.data_ptr(), a.numel(), _DTYPE_CODE[a.dtype], _stream_ptr(stream, a)))
    return out


def argmax(logits, stream=None):
    """Greedy token per row of ``logits [rows, vocab]`` -> int32 ``[rows]``."""
    if logits.dtype not in _FLOATS or logits.dim() != 2:
        raise RuntimeError("argmax: expected 2D float logits")
    _gpu("argmax", logits)
    _contig("argmax", logits=logits)
    rows, vocab = logits.shape
    out = torch.empty((rows,), dtype=torch.int32, device=logits.device)
    ws_bytes = _lib.tl_argmax_workspace(rows, vocab)
    ws = _workspace(ws_bytes, logits.device)
    _check(_lib.tl_argmax(logits.data_ptr(), out.data_ptr(), rows, vocab, _DTYPE_CODE[logits.dtype],
                          None if ws is None else ws.data_ptr(), ws_bytes, _stream_ptr(stream, logits)))
    return out


def sample(logits, temperature, top_k, top_p, seed, positions, stream=None):
    """Seeded token per row of ``logits [rows, vocab]`` -> int32 ``[rows]`` (``tl_sample``).  Per-row device arrays:
    ``temperature`` float32 (0: greedy, ``argmax``'s token), ``top_k`` int32 (on for 0 < k < vocab), ``top_p`` float32
    (on for 0 < p < 1), ``seed`` int64 and ``positions`` int32, the index of the token being drawn."""
    if logits.dtype not in _FLOATS or logits.dim() != 2:
        raise RuntimeError("sample: expected 2D float logits")
    rows = logits.shape[0]
    for name, t, dtype in (("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32), ("top_p", top_p, torch.float32),
                           ("seed", seed, torch.int64), ("positions", positions, torch.int32)):
        if t.dtype != dtype or t.dim() != 1 or t.shape[0] != rows:
            raise RuntimeError(f"sample: {name} must be {str(dtype).replace('torch.', '')} [{rows}]")
    _contig("sample", logits=logits, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed, positions=positions)
    _gpu("sample", logits, temperature, top_k, top_p, seed, positions)
    out = torch.empty((rows,), dtype=torch.int32, device=logits.device)
    _check(_lib.tl_sample(logits.data_ptr(), temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), seed.data_ptr(), positions.data_ptr(),
                          out.data_ptr(), rows, logits.shape[1], _DTYPE_CODE[logits.dtype], _stream_ptr(stream, logits)))
    return out


SPECULATIVE_SAMPLE_MAX_VOCAB = 204800


def speculative_sample(target, draft, proposals, temperature, top_k, top_p, seed, positions, out=None, stream=None):
    """The speculative rejection rule over one verify pass (``tl_speculative_sample``, DESIGN.md section 8d) -> int32
    ``[T]``.  ``target [T, vocab]`` and ``draft [T - 1, vocab]`` logits of one float dtype, ``proposals`` int32
    ``[T - 1]`` (each drawn by ``sample`` from its draft row with the same parameters), per-row device arrays as
    ``sample`` takes them and ``positions`` the index n_j of the token row j predicts.  Row j < T - 1 is d_j when
    accepted, else the residual draw; row T - 1 is ``sample``'s draw on the last target row.  ``out`` (int32 ``[T]``)
    receives the tokens when given.  vocab is at most ``SPECULATIVE_SAMPLE_MAX_VOCAB``."""
    if target.dtype not in _FLOATS or target.dim() != 2:
        raise RuntimeError("speculative_sample: expected 2D float target logits")
    rows, vocab = target.shape
    if vocab > SPECULATIVE_SAMPLE_MAX_VOCAB:
        raise RuntimeError(f"speculative_sample: vocab {vocab} exceeds {SPECULATIVE_SAMPLE_MAX_VOCAB}")
    k = rows - 1
    if draft.dtype != target.dtype or tuple(draft.shape) != (k, vocab):
        raise RuntimeError(f"speculative_sample: draft must be {str(target.dtype).replace('torch.', '')} [{k}, {vocab}]")
    if proposals.dtype != torch.int32 or tuple(proposals.shape) != (k,):
        raise RuntimeError(f"speculative_sample: proposals must be int32 [{k}]")
    for name, t, dtype in (("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32), ("top_p", top_p, torch.float32),
                           ("seed", seed, torch.int64), ("positions", positions, torch.int32)):
        if t.dtype != dtype or t.dim() != 1 or t.shape[0] != rows:
            raise RuntimeError(f"speculative_sample: {name} must be {str(dtype).replace('torch.', '')} [{rows}]")
    if out is None:
        out = torch.empty((rows,), dtype=torch.int32, device=target.device)
    elif out.dtype != torch.int32 or tuple(out.shape) != (rows,):
        raise RuntimeError(f"speculative_sample: out must be int32 [{rows}]")
    named = dict(target=target, draft=draft, proposals=proposals, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed,
                 positions=positions, out=out)
    _contig("speculative_sample", **named)
    _gpu("speculative_sample", *named.values())
    _check(_lib.tl_speculative_sample(target.data_ptr(), draft.data_ptr(), proposals.data_ptr(), temperature.data_ptr(), top_k.data_ptr(),
                                      top_p.data_ptr(), seed.data_ptr(), positions.data_ptr(), out.data_ptr(), rows, vocab,
                                      _DTYPE_CODE[target.dtype], _stream_ptr(stream, target)))
    return out


def log_rows(src, dst, out_index, stream=None):
    """``dst[out_index[0]] = src`` when ``0 <= out_index[0] < dst.shape[0]`` (``tl_log_rows``; ``out_index`` int32 ``[1]``
    on the device): a captured step logs its rows at the step counter."""
    if src.dtype != dst.dtype or dst.dim() < 1 or tuple(dst.shape[1:]) != tuple(src.shape):
        raise RuntimeError("log_rows: dst must be [capacity, *src.shape] of src's dtype")
    if out_index.dtype != torch.int32 or out_index.numel() != 1:
        raise RuntimeError("log_rows: out_index must be int32 [1]")
    _contig("log_rows", src=src, dst=dst, out_index=out_index)
    _gpu("log_rows", src, dst, out_index)
    _check(_lib.tl_log_rows(src.data_ptr(), dst.data_ptr(), out_index.data_ptr(), dst.shape[0], src.numel() * src.element_size(),
                            _stream_ptr(stream, src)))


NGRAM_MAX_K = 7
NGRAM_MAX_N = 8
NGRAM_MAX_APPEND = 8
NGRAM_TILE = 1024
NGRAM_STATE_WORDS = 12


def ngram_propose(history, length, appended, k, n_min, n_max, out, state, onehot=None, grid=0, stream=None):
    """Prompt-lookup proposals (``tl_ngram_propose``, DESIGN.md section 14): append the host ids ``appended`` (at most
    ``NGRAM_MAX_APPEND``, passed by value) to ``history`` (int32 ``[capacity]``, holding ``length`` tokens), then
    write into ``out`` (int32 ``[2 + k]``) the longest-then-latest match length c (0: no match), its end e (-1) and the
    k tokens that followed it (-1s).  ``state`` (int32 ``[NGRAM_STATE_WORDS]``, zeroed once) belongs to one history
    and one ``onehot`` (``[k, vocab]`` float, filled with -inf once), whose rows then hold exactly 0 at each current
    proposal and -inf elsewhere.  ``grid`` > 0 fixes the number of CTAs (the result does not depend on it).  No host
    synchronisation: the call captures into a CUDA graph.  Returns ``out``."""
    appended = [int(t) for t in appended]
    if not isinstance(k, int) or not 1 <= k <= NGRAM_MAX_K:
        raise RuntimeError(f"ngram_propose: k must be in [1, {NGRAM_MAX_K}]")
    if not (isinstance(n_min, int) and isinstance(n_max, int) and 1 <= n_min <= n_max <= NGRAM_MAX_N):
        raise RuntimeError(f"ngram_propose: need 1 <= n_min <= n_max <= {NGRAM_MAX_N}")
    if len(appended) > NGRAM_MAX_APPEND:
        raise RuntimeError(f"ngram_propose: at most {NGRAM_MAX_APPEND} appended tokens")
    if history.dtype != torch.int32 or history.dim() != 1:
        raise RuntimeError("ngram_propose: history must be int32 [capacity]")
    if not (isinstance(length, int) and 0 <= length and length + len(appended) <= history.shape[0]):
        raise RuntimeError(f"ngram_propose: {length} + {len(appended)} tokens exceed the history's capacity {history.shape[0]}")
    if out.dtype != torch.int32 or tuple(out.shape) != (2 + k,):
        raise RuntimeError(f"ngram_propose: out must be int32 [{2 + k}]")
    if state.dtype != torch.int32 or tuple(state.shape) != (NGRAM_STATE_WORDS,):
        raise RuntimeError(f"ngram_propose: state must be int32 [{NGRAM_STATE_WORDS}]")
    named = dict(history=history, out=out, state=state)
    vocab, dtype = 0, 0
    if onehot is not None:
        if onehot.dtype not in _FLOATS or onehot.dim() != 2 or onehot.shape[0] != k:
            raise RuntimeError(f"ngram_propose: onehot must be float [{k}, vocab]")
        vocab, dtype = onehot.shape[1], _DTYPE_CODE[onehot.dtype]
        named["onehot"] = onehot
    _contig("ngram_propose", **named)
    _gpu("ngram_propose", *named.values())
    ids = (ctypes.c_int32 * NGRAM_MAX_APPEND)(*appended)
    _check(_lib.tl_ngram_propose(history.data_ptr(), history.shape[0], length, ids, len(appended), k, n_min, n_max, out.data_ptr(),
                                 state.data_ptr(), None if onehot is None else onehot.data_ptr(), vocab, dtype, grid,
                                 _stream_ptr(stream, history)))
    return out


BEAM_MAX_WIDTH = 8
BEAM_MAX_EOS = 4
BEAM_RESULT_WORDS = 2 + 7 * BEAM_MAX_WIDTH


def beam_select(top_lp, top_ids, cum, num_beams, eos_ids, out, stream=None):
    """Beam search's cross-beam selection (``tl_beam_select``, DESIGN.md section 15) over ``tl_logprobs``' top-N lists
    ``top_lp`` float32 / ``top_ids`` int32 ``[rows, N]`` of ``rows <= num_beams`` rows, ``N = num_beams + len(eos_ids)``,
    and the rows' cumulative log-probabilities ``cum`` (float32 ``[num_beams]``, device), which the launch rewrites in
    place with the live beams' sums (-inf past them).  The EOS ids travel as kernel arguments.  Writes the packed result
    into ``out`` (int32 ``[BEAM_RESULT_WORDS]``): live and finished counts, the live beams' (parent, token, cum bits) and
    the finished records' (parent, EOS id, sum bits, walk position).  No host synchronisation: the call captures into a
    CUDA graph.  Returns ``out``."""
    eos = [int(t) for t in eos_ids]
    if not isinstance(num_beams, int) or isinstance(num_beams, bool) or not 1 <= num_beams <= BEAM_MAX_WIDTH:
        raise RuntimeError(f"beam_select: num_beams must be in [1, {BEAM_MAX_WIDTH}]")
    if len(eos) > BEAM_MAX_EOS:
        raise RuntimeError(f"beam_select: at most {BEAM_MAX_EOS} EOS ids")
    n = num_beams + len(eos)
    if top_lp.dtype != torch.float32 or top_lp.dim() != 2 or top_lp.shape[1] != n:
        raise RuntimeError(f"beam_select: top_lp must be float32 [rows, {n}]")
    rows = top_lp.shape[0]
    if not 1 <= rows <= num_beams:
        raise RuntimeError(f"beam_select: rows must be in [1, {num_beams}]")
    if top_ids.dtype != torch.int32 or tuple(top_ids.shape) != (rows, n):
        raise RuntimeError(f"beam_select: top_ids must be int32 [{rows}, {n}]")
    if cum.dtype != torch.float32 or tuple(cum.shape) != (num_beams,):
        raise RuntimeError(f"beam_select: cum must be float32 [{num_beams}]")
    if out.dtype != torch.int32 or tuple(out.shape) != (BEAM_RESULT_WORDS,):
        raise RuntimeError(f"beam_select: out must be int32 [{BEAM_RESULT_WORDS}]")
    named = dict(top_lp=top_lp, top_ids=top_ids, cum=cum, out=out)
    _contig("beam_select", **named)
    _gpu("beam_select", *named.values())
    ids = (ctypes.c_int32 * BEAM_MAX_EOS)(*eos)
    _check(_lib.tl_beam_select(top_lp.data_ptr(), top_ids.data_ptr(), cum.data_ptr(), rows, n, num_beams, ids, len(eos), out.data_ptr(),
                               _stream_ptr(stream, top_lp)))
    return out


def sample_penalized(logits, temperature, top_k, top_p, seed, positions, repetition, presence, frequency, min_p, state, stream=None):
    """``sample`` with token-history penalties and min-p (``tl_sample_penalized``) -> int32 ``[rows]``.  Further
    per-row device arrays: ``repetition``, ``presence``, ``frequency`` and ``min_p`` float32 ``[rows]``, and ``state``
    int32 ``[rows, vocab]`` (bit 30: token in the prompt, bits 0-29: times drawn), read, and for rows with
    ``positions > 0`` incremented at the drawn token."""
    if logits.dtype not in _FLOATS or logits.dim() != 2:
        raise RuntimeError("sample_penalized: expected 2D float logits")
    rows, vocab = logits.shape
    for name, t, dtype in (("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32), ("top_p", top_p, torch.float32),
                           ("seed", seed, torch.int64), ("positions", positions, torch.int32), ("repetition", repetition, torch.float32),
                           ("presence", presence, torch.float32), ("frequency", frequency, torch.float32), ("min_p", min_p, torch.float32)):
        if t.dtype != dtype or t.dim() != 1 or t.shape[0] != rows:
            raise RuntimeError(f"sample_penalized: {name} must be {str(dtype).replace('torch.', '')} [{rows}]")
    if state.dtype != torch.int32 or tuple(state.shape) != (rows, vocab):
        raise RuntimeError(f"sample_penalized: state must be int32 [{rows}, {vocab}]")
    named = dict(logits=logits, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed, positions=positions, repetition=repetition,
                 presence=presence, frequency=frequency, min_p=min_p, state=state)
    _contig("sample_penalized", **named)
    _gpu("sample_penalized", *named.values())
    out = torch.empty((rows,), dtype=torch.int32, device=logits.device)
    _check(_lib.tl_sample_penalized(logits.data_ptr(), temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), seed.data_ptr(),
                                    positions.data_ptr(), repetition.data_ptr(), presence.data_ptr(), frequency.data_ptr(), min_p.data_ptr(),
                                    state.data_ptr(), out.data_ptr(), rows, vocab, _DTYPE_CODE[logits.dtype], _stream_ptr(stream, logits)))
    return out


CONSTRAINT_ROW_WORDS = 5  # int64 words of one tl_constraint_row (40 bytes)


def sample_constrained(logits, temperature, top_k, top_p, seed, positions, constraints, repetition=None, presence=None, frequency=None,
                       min_p=None, state=None, stream=None):
    """``sample`` (no penalty arrays) or ``sample_penalized`` (all of them) restricted per row to the tokens of its
    constraint (``tl_sample_constrained``) -> int32 ``[rows]``.  ``constraints`` int64 ``[rows, 5]``: one
    ``tl_constraint_row`` per row (all zero: unconstrained), whose state the launch advances for rows with
    ``positions > 0``."""
    if logits.dtype not in _FLOATS or logits.dim() != 2:
        raise RuntimeError("sample_constrained: expected 2D float logits")
    rows, vocab = logits.shape
    pen = (repetition, presence, frequency, min_p, state)
    if any(t is None for t in pen) and any(t is not None for t in pen):
        raise RuntimeError("sample_constrained: give every penalty array and the state, or none")
    checks = [("temperature", temperature, torch.float32), ("top_k", top_k, torch.int32), ("top_p", top_p, torch.float32),
              ("seed", seed, torch.int64), ("positions", positions, torch.int32)]
    if state is not None:
        checks += [("repetition", repetition, torch.float32), ("presence", presence, torch.float32), ("frequency", frequency, torch.float32),
                   ("min_p", min_p, torch.float32)]
        if state.dtype != torch.int32 or tuple(state.shape) != (rows, vocab):
            raise RuntimeError(f"sample_constrained: state must be int32 [{rows}, {vocab}]")
    for name, t, dtype in checks:
        if t.dtype != dtype or t.dim() != 1 or t.shape[0] != rows:
            raise RuntimeError(f"sample_constrained: {name} must be {str(dtype).replace('torch.', '')} [{rows}]")
    if constraints.dtype != torch.int64 or tuple(constraints.shape) != (rows, CONSTRAINT_ROW_WORDS):
        raise RuntimeError(f"sample_constrained: constraints must be int64 [{rows}, {CONSTRAINT_ROW_WORDS}]")
    named = dict(logits=logits, temperature=temperature, top_k=top_k, top_p=top_p, seed=seed, positions=positions, constraints=constraints)
    if state is not None:
        named.update(repetition=repetition, presence=presence, frequency=frequency, min_p=min_p, state=state)
    _contig("sample_constrained", **named)
    _gpu("sample_constrained", *named.values())
    out = torch.empty((rows,), dtype=torch.int32, device=logits.device)
    ptr = [None if t is None else t.data_ptr() for t in pen]
    _check(_lib.tl_sample_constrained(logits.data_ptr(), temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), seed.data_ptr(),
                                      positions.data_ptr(), *ptr, constraints.data_ptr(), out.data_ptr(), rows, vocab,
                                      _DTYPE_CODE[logits.dtype], _stream_ptr(stream, logits)))
    return out


JSON_STATE_WORDS = 2  # int64 words of one JSON row's automaton state (include/tiny_llm_b200.h)


def _json_rows(op, constraints, json_states):
    if constraints.dtype != torch.int64 or constraints.dim() != 2 or constraints.shape[1] != CONSTRAINT_ROW_WORDS:
        raise RuntimeError(f"{op}: constraints must be int64 [rows, {CONSTRAINT_ROW_WORDS}]")
    rows = constraints.shape[0]
    if json_states.dtype != torch.int64 or tuple(json_states.shape) != (rows, JSON_STATE_WORDS):
        raise RuntimeError(f"{op}: json_states must be int64 [{rows}, {JSON_STATE_WORDS}]")
    return rows


def json_token_masks(constraints, json_states, vocab, stream=None):
    """Row 0 of each JSON row's mask buffer (``tl_json_token_masks``): ``constraints`` int64 ``[rows, 5]``
    descriptors, ``json_states`` int64 ``[rows, 2]`` automaton states; rows not in JSON mode, or terminal, are not
    touched.  Writes through the descriptors' mask pointers; returns nothing."""
    rows = _json_rows("json_token_masks", constraints, json_states)
    if isinstance(vocab, bool) or not isinstance(vocab, int) or vocab <= 0:
        raise RuntimeError("json_token_masks: vocab must be a positive int")
    _contig("json_token_masks", constraints=constraints, json_states=json_states)
    _gpu("json_token_masks", constraints, json_states)
    _check(_lib.tl_json_token_masks(constraints.data_ptr(), json_states.data_ptr(), rows, vocab, _stream_ptr(stream, constraints)))


def json_advance(constraints, json_states, tokens, positions, stream=None):
    """Advance each JSON row's automaton state by its drawn token (``tl_json_advance``), for rows with
    ``positions > 0``; ``tokens`` and ``positions`` int32 ``[rows]``."""
    rows = _json_rows("json_advance", constraints, json_states)
    for name, t in (("tokens", tokens), ("positions", positions)):
        if t.dtype != torch.int32 or tuple(t.shape) != (rows,):
            raise RuntimeError(f"json_advance: {name} must be int32 [{rows}]")
    named = dict(constraints=constraints, json_states=json_states, tokens=tokens, positions=positions)
    _contig("json_advance", **named)
    _gpu("json_advance", *named.values())
    _check(_lib.tl_json_advance(constraints.data_ptr(), json_states.data_ptr(), tokens.data_ptr(), positions.data_ptr(), rows,
                                _stream_ptr(stream, constraints)))


SCHEMA_STATE_WORDS = 10  # int64 words of one JSON Schema row's automaton state (include/tiny_llm_b200.h)
SCHEMA_SMEM_BYTES = 47 * 1024  # TL_SCHEMA_SMEM_BYTES: the largest table blob a masks launch stages in shared memory


def _schema_rows(op, constraints, schema_states):
    if constraints.dtype != torch.int64 or constraints.dim() != 2 or constraints.shape[1] != CONSTRAINT_ROW_WORDS:
        raise RuntimeError(f"{op}: constraints must be int64 [rows, {CONSTRAINT_ROW_WORDS}]")
    rows = constraints.shape[0]
    if schema_states.dtype != torch.int64 or tuple(schema_states.shape) != (rows, SCHEMA_STATE_WORDS):
        raise RuntimeError(f"{op}: schema_states must be int64 [{rows}, {SCHEMA_STATE_WORDS}]")
    return rows


def schema_token_masks(constraints, schema_states, vocab, smem_bytes=0, stream=None):
    """Row 0 of each JSON Schema row's mask buffer (``tl_schema_token_masks``): ``constraints`` int64 ``[rows, 5]``
    descriptors, ``schema_states`` int64 ``[rows, 10]`` automaton states (word 0 the row's table blob); rows not in
    schema mode, or terminal, are not touched.  ``smem_bytes``: the shared memory that stages blobs up to that size
    (``ConstraintRows.schema_smem_bytes``).  Writes through the descriptors' mask pointers; returns nothing."""
    rows = _schema_rows("schema_token_masks", constraints, schema_states)
    if isinstance(vocab, bool) or not isinstance(vocab, int) or vocab <= 0:
        raise RuntimeError("schema_token_masks: vocab must be a positive int")
    if isinstance(smem_bytes, bool) or not isinstance(smem_bytes, int) or not 0 <= smem_bytes <= SCHEMA_SMEM_BYTES or smem_bytes % 16:
        raise RuntimeError(f"schema_token_masks: smem_bytes must be a multiple of 16 in [0, {SCHEMA_SMEM_BYTES}]")
    _contig("schema_token_masks", constraints=constraints, schema_states=schema_states)
    _gpu("schema_token_masks", constraints, schema_states)
    _check(_lib.tl_schema_token_masks(constraints.data_ptr(), schema_states.data_ptr(), rows, vocab, smem_bytes,
                                      _stream_ptr(stream, constraints)))


def schema_advance(constraints, schema_states, tokens, positions, stream=None):
    """Advance each JSON Schema row's automaton state by its drawn token (``tl_schema_advance``), for rows with
    ``positions > 0``; ``tokens`` and ``positions`` int32 ``[rows]``."""
    rows = _schema_rows("schema_advance", constraints, schema_states)
    for name, t in (("tokens", tokens), ("positions", positions)):
        if t.dtype != torch.int32 or tuple(t.shape) != (rows,):
            raise RuntimeError(f"schema_advance: {name} must be int32 [{rows}]")
    named = dict(constraints=constraints, schema_states=schema_states, tokens=tokens, positions=positions)
    _contig("schema_advance", **named)
    _gpu("schema_advance", *named.values())
    _check(_lib.tl_schema_advance(constraints.data_ptr(), schema_states.data_ptr(), tokens.data_ptr(), positions.data_ptr(), rows,
                                  _stream_ptr(stream, constraints)))


def constraint_token_masks(dfa, accept, token_offsets, token_bytes, eos_ids, stream=None):
    """Token masks of a byte DFA over a vocabulary (``tl_constraint_token_masks``).  ``dfa`` int32 ``[S, 256]``,
    ``accept`` uint8 ``[S]``, ``token_offsets`` int32 ``[V + 1]``, ``token_bytes`` uint8, ``eos_ids`` int32 ``[E]``.
    Returns ``(masks, reach)``: int32 ``[S + 1, ceil(V / 32)]`` (bit t of row s: token t allowed in state s; row S the
    terminal state) and int32 ``[S, ceil(S / 32)]`` (bit e of row s: an allowed token leads from s to e)."""
    if dfa.dtype != torch.int32 or dfa.dim() != 2 or dfa.shape[1] != 256 or dfa.shape[0] == 0:
        raise RuntimeError("constraint_token_masks: dfa must be int32 [S, 256]")
    S = dfa.shape[0]
    if accept.dtype != torch.uint8 or tuple(accept.shape) != (S,):
        raise RuntimeError(f"constraint_token_masks: accept must be uint8 [{S}]")
    if token_offsets.dtype != torch.int32 or token_offsets.dim() != 1 or token_offsets.shape[0] < 2:
        raise RuntimeError("constraint_token_masks: token_offsets must be int32 [V + 1]")
    if token_bytes.dtype != torch.uint8 or token_bytes.dim() != 1:
        raise RuntimeError("constraint_token_masks: token_bytes must be uint8")
    if eos_ids.dtype != torch.int32 or eos_ids.dim() != 1:
        raise RuntimeError("constraint_token_masks: eos_ids must be int32 [E]")
    named = dict(dfa=dfa, accept=accept, token_offsets=token_offsets, token_bytes=token_bytes, eos_ids=eos_ids)
    _contig("constraint_token_masks", **named)
    _gpu("constraint_token_masks", *named.values())
    V = token_offsets.shape[0] - 1
    masks = torch.empty((S + 1, (V + 31) // 32), dtype=torch.int32, device=dfa.device)
    reach = torch.zeros((S, (S + 31) // 32), dtype=torch.int32, device=dfa.device)
    _check(_lib.tl_constraint_token_masks(dfa.data_ptr(), accept.data_ptr(), S, token_offsets.data_ptr(), token_bytes.data_ptr(), V,
                                          eos_ids.data_ptr() if eos_ids.numel() else None, eos_ids.numel(), masks.data_ptr(),
                                          reach.data_ptr(), _stream_ptr(stream, dfa)))
    return masks, reach


LOGPROBS_MAX_N = 20


def logprobs(logits, targets=None, top_n=None, max_n=0, out=None, out_index=None, stream=None):
    """Log-probabilities of the raw distribution of each row of ``logits [rows, vocab]`` (``tl_logprobs``).
    ``targets`` int32 ``[rows]`` (device; -1: none), ``top_n`` int32 ``[rows]`` (device; None: ``max_n`` for every row),
    ``0 <= max_n <= 20``.  Returns ``(lse, target_lp, target_rank, top_ids, top_lp)``: float32 / float32 / int32
    ``[rows]`` and int32 / float32 ``[rows, max_n]`` (ids -1 and -inf past each row's list).  ``out`` (those five
    tensors with a leading ``[capacity, ...]`` dimension) and ``out_index`` (int32 ``[1]``, device) write row r at
    ``out[...][out_index, r]`` instead: a captured graph logs step after step into one buffer.  An ``out_index`` outside
    ``[0, capacity)`` writes nothing."""
    if logits.dtype not in _FLOATS or logits.dim() != 2:
        raise RuntimeError("logprobs: expected 2D float logits")
    if not isinstance(max_n, int) or isinstance(max_n, bool) or not 0 <= max_n <= LOGPROBS_MAX_N:
        raise RuntimeError(f"logprobs: max_n must be an integer in [0, {LOGPROBS_MAX_N}]")
    rows, vocab = logits.shape
    named = {"logits": logits}
    for name, t in (("targets", targets), ("top_n", top_n)):
        if t is not None:
            if t.dtype != torch.int32 or t.dim() != 1 or t.shape[0] != rows:
                raise RuntimeError(f"logprobs: {name} must be int32 [{rows}]")
            named[name] = t
    if out is None:
        if out_index is not None:
            raise RuntimeError("logprobs: out_index needs out")
        dev = logits.device
        out = (torch.empty(rows, dtype=torch.float32, device=dev), torch.empty(rows, dtype=torch.float32, device=dev),
               torch.empty(rows, dtype=torch.int32, device=dev), torch.empty((rows, max_n), dtype=torch.int32, device=dev),
               torch.empty((rows, max_n), dtype=torch.float32, device=dev))
        lead = ()
    else:
        if out_index is None or out_index.dtype != torch.int32 or out_index.numel() != 1:
            raise RuntimeError("logprobs: out needs out_index, int32 [1]")
        named["out_index"] = out_index
        lead = (out[0].shape[0],)
    shapes = (lead + (rows,),) * 3 + (lead + (rows, max_n),) * 2
    for t, shape, dtype in zip(out, shapes, (torch.float32, torch.float32, torch.int32, torch.int32, torch.float32)):
        if t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous():
            raise RuntimeError("logprobs: out must be float32 lse, float32 lp, int32 rank [..., rows], int32 ids and float32 lp [..., rows, max_n]")
    _contig("logprobs", **named)
    _gpu("logprobs", *named.values(), *out)
    lse, lp, rank, ids, top = out
    _check(_lib.tl_logprobs(logits.data_ptr(), None if targets is None else targets.data_ptr(), None if top_n is None else top_n.data_ptr(),
                            None if out_index is None else out_index.data_ptr(), lse.data_ptr(), lp.data_ptr(), rank.data_ptr(),
                            ids.data_ptr() if max_n else None, top.data_ptr() if max_n else None, rows, vocab, max_n,
                            lead[0] if lead else 1, _DTYPE_CODE[logits.dtype], _stream_ptr(stream, logits)))
    return lse, lp, rank, ids, top


def decode_advance(tokens, next_tokens, offsets, context_lens, out_log, step_counter, stream=None):
    """Feed the sampled tokens back and advance positions on the device (one tiny
    launch between two graph-captured decode steps)."""
    for t in (tokens, next_tokens, offsets, context_lens, out_log, step_counter):
        if t.dtype != torch.int32 or not t.is_contiguous():
            raise RuntimeError("decode_advance: expected contiguous int32 tensors")
    _gpu("decode_advance", tokens, next_tokens, offsets, context_lens, out_log, step_counter)
    batch = tokens.numel()
    _check(_lib.tl_decode_advance(tokens.data_ptr(), next_tokens.data_ptr(), offsets.data_ptr(), context_lens.data_ptr(),
                                  out_log.data_ptr(), step_counter.data_ptr(), batch, out_log.numel() // max(batch, 1),
                                  _stream_ptr(stream, tokens)))


PRO_NONE, PRO_RMSNORM, PRO_SWIGLU = 0, 1, 2
EPI_NONE, EPI_RESIDUAL, EPI_SWIGLU_PAIRS = 0, 1, 2


def packed_bits(b, N: int):
    """Code width of packed weights ``b [K, N * bits / 32]`` over ``N`` inputs, ``32 * b.shape[1] / N``: 4 or 8, else
    None (the fused functions refuse it)."""
    bits, rem = divmod(32 * b.shape[1], N) if N > 0 else (0, 1)
    return bits if rem == 0 and bits in (4, 8) else None


def quantized_matmul_fused(scales, biases, b, p0, p1=None, residual=None, prologue=PRO_NONE, epilogue=EPI_NONE, eps=0.0,
                           out=None, stream=None):
    """Decode projection with the neighbouring element-wise operator folded in
    (``include/tiny_llm_b200.h``): ``p0`` is ``[M, N]`` (row stride ``p0.stride(0)``),
    ``b`` ``[K, N/8]`` (4-bit codes) or ``[K, N/4]`` (8-bit); bit-identical to the unfused operator sequence."""
    if p0.dim() != 2 or b.dim() != 2 or p0.stride(1) != 1:
        raise RuntimeError("quantized_matmul_fused: p0 must be 2D with unit inner stride")
    M, N = p0.shape
    K = b.shape[0]
    bits = packed_bits(b, N)
    if bits is None or tuple(scales.shape) != (K, N // 128) or scales.shape != biases.shape:
        raise RuntimeError("quantized_matmul_fused: incompatible parameter shapes (b must hold 4- or 8-bit codes: [K, N/8] or [K, N/4])")
    if scales.dtype not in _HALF or p0.dtype != scales.dtype or biases.dtype != scales.dtype:
        raise RuntimeError("quantized_matmul: a must be the same dtype as scales")
    _gpu("quantized_matmul_fused", scales, biases, b, p0)
    _contig("quantized_matmul_fused", b=b, scales=scales, biases=biases)
    lda = p0.stride(0)
    if prologue == PRO_SWIGLU and (p1 is None or p1.shape != p0.shape or p1.stride(0) != lda or p1.stride(1) != 1):
        raise RuntimeError("quantized_matmul_fused: gate and up must share shape and strides")
    if prologue == PRO_RMSNORM and (p1 is None or tuple(p1.shape) != (N,) or not p1.is_contiguous()):
        raise RuntimeError("quantized_matmul_fused: norm weight must be [N]")
    if epilogue == EPI_RESIDUAL and (residual is None or tuple(residual.shape) != (M, K) or not residual.is_contiguous()):
        raise RuntimeError("quantized_matmul_fused: residual must be contiguous [M, K]")
    if epilogue == EPI_SWIGLU_PAIRS and K % 16:
        raise RuntimeError("quantized_matmul_fused: interleaved gate|up rows need K % 16 == 0")
    if out is None:
        out = torch.empty((M, K // 2 if epilogue == EPI_SWIGLU_PAIRS else K), dtype=p0.dtype, device=p0.device)
    code = _DTYPE_CODE[p0.dtype]
    ws_bytes = _lib.tl_quantized_matmul_fused_workspace_bits(M, N, K, lda, int(prologue), code, bits)
    ws = _zero_workspace(ws_bytes, p0.device)
    _check(
        _lib.tl_quantized_matmul_fused_bits(
            scales.data_ptr(), biases.data_ptr(), b.data_ptr(), out.data_ptr(), p0.data_ptr(),
            None if p1 is None else p1.data_ptr(), None if residual is None else residual.data_ptr(), M, N, K, lda,
            int(prologue), int(epilogue), float(eps), code, bits, None if ws is None else ws.data_ptr(), ws_bytes,
            _stream_ptr(stream, p0),
        )
    )
    return out


W4_VANILLA, W4_STREAM, W4_SKINNY, W4_TILES = 0, 1, 2, 3


def quantized_matmul_route(M, N, K, lda, prologue, fused, use_simdgroup, dtype, a, b, scales, biases, bits=4):
    """The kernel a W4A16 projection runs, decided without launching or reading anything: ``(route, splits,
    gb_per_split, rows_per_pass, units)`` with ``route`` one of ``W4_VANILLA`` / ``W4_STREAM`` / ``W4_SKINNY`` /
    ``W4_TILES`` (``include/tiny_llm_b200.h`` documents the other fields).  ``fused`` selects the rule of
    ``quantized_matmul_fused`` / ``quantized_matmul_residual_norm``.  ``a``, ``b``, ``scales`` and ``biases`` are tensors
    or plain addresses: only their alignment counts.  ``dtype`` is a torch dtype; ``bits`` (4 or 8) the code width."""

    def addr(x):
        return x.data_ptr() if isinstance(x, torch.Tensor) else int(x)

    facts = [_I() for _ in range(4)]
    code = _lib.tl_quantized_matmul_route_bits(int(M), int(N), int(K), int(lda), int(prologue), int(bool(fused)), int(bool(use_simdgroup)),
                                               _DTYPE_CODE[dtype], int(bits), addr(a), addr(b), addr(scales), addr(biases),
                                               *map(ctypes.byref, facts))
    _check(min(code, 0))
    return (code, *(f.value for f in facts))


def shared_prefix_attention_workspace(batch: int, num_heads: int, num_kv_heads: int, page_size: int, max_pages: int) -> int:
    """Bytes of workspace ``shared_prefix_attention`` takes for these shapes (its split partials)."""
    return int(_lib.tl_shared_prefix_attention_workspace(int(batch), int(num_heads), int(num_kv_heads), int(page_size), int(max_pages)))


def shared_prefix_attention(query, key_pages, value_pages, block_table, context_lens, groups, groups_host, scale, num_kv_heads, num_heads,
                            workspace=None, stream=None):
    """Decode attention (L = 1, causal) of ``batch`` slots where groups of consecutive slots share their leading pages
    (``tl_shared_prefix_attention``, DESIGN.md section 16): each group's shared pages are streamed once for all its
    query rows, every row then attends its own keys after them, and the partials are merged.  The result is
    ``paged_attention(..., is_causal=True)``'s up to the order of the sums.  ``groups``: int32 ``[num_groups, 3]``
    ``(first_slot, count, shared_pages)`` on the device (rows with count 0 unused); ``groups_host``: the same on the
    host, checked by the C entry.  ``workspace``: a byte buffer of ``shared_prefix_attention_workspace`` bytes (a
    fresh one when None)."""
    op = "shared_prefix_attention"
    if query.dtype != torch.bfloat16 or key_pages.dtype != torch.bfloat16 or value_pages.dtype != torch.bfloat16:
        raise RuntimeError(f"{op}: q, key_pages and value_pages must be bfloat16")
    if query.dim() != 3 or query.shape[1] != 1 or key_pages.dim() != 4 or key_pages.shape != value_pages.shape:
        raise RuntimeError(f"{op}: q must be [B * H_q, 1, D] and the page tensors [P, H_kv, page_size, D]")
    if groups.dtype != torch.int32 or groups.dim() != 2 or groups.shape[1] != 3 or tuple(groups_host.shape) != tuple(groups.shape):
        raise RuntimeError(f"{op}: groups must be int32 [num_groups, 3] with a host copy of the same shape")
    if groups_host.dtype != torch.int32 or groups_host.is_cuda or not groups_host.is_contiguous():
        raise RuntimeError(f"{op}: groups_host must be a contiguous int32 CPU tensor")
    batch = query.shape[0] // int(num_heads)
    _int32(op, batch, context_lens=context_lens)
    _block_table(op, block_table, batch)
    _gpu(op, query, key_pages, value_pages, block_table, context_lens, groups)
    _contig(op, query=query, key_pages=key_pages, value_pages=value_pages, block_table=block_table, context_lens=context_lens, groups=groups)
    P, _, page_size, D = key_pages.shape
    max_pages = block_table.shape[1]
    need = shared_prefix_attention_workspace(batch, num_heads, num_kv_heads, page_size, max_pages)
    if workspace is None:
        workspace = _workspace(max(need, 1), query.device)
    out = torch.empty_like(query)
    _check(_lib.tl_shared_prefix_attention(query.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), block_table.data_ptr(),
                                           context_lens.data_ptr(), groups.data_ptr(), groups_host.data_ptr(), groups.shape[0], out.data_ptr(),
                                           batch, D, P, page_size, max_pages, float(scale), int(num_kv_heads), int(num_heads),
                                           _DTYPE_CODE[query.dtype], workspace.data_ptr(), workspace.numel() * workspace.element_size(),
                                           _stream_ptr(stream, query)))
    return out


def paged_attention_token_major_workspace(rows: int, L: int, page_size: int, max_pages: int) -> int:
    """Bytes of the split workspace ``paged_attention_token_major(..., workspace=)`` takes for ``rows = B * Hq`` query heads of
    ``L`` rows over a block table of ``max_pages`` pages: 0 when the table spans at most 8,192 keys (no split there)."""
    return int(_lib.tl_paged_attention_token_major_workspace(int(rows), int(L), int(page_size), int(max_pages)))


def paged_attention_token_major(query, key_pages, value_pages, block_table, context_lens, scale, is_causal, num_kv_heads, num_heads, stream=None,
                                workspace=None):
    """Prefill attention (L > 8) with the output already in the o-projection's layout: ``query`` [B * Hq, L, D] ->
    ``[B * L, Hq * D]``.  Only on the wgmma kernel (bf16, D = 128, page size a multiple of 64); otherwise - and for
    L <= 8 - ``paged_attention`` + a transpose copy.  ``workspace`` (uint8, ``paged_attention_token_major_workspace``
    bytes): a block table spanning more than 8,192 keys splits the key range over more CTAs and merges the partials;
    None never splits."""
    rows, L, D = query.shape
    B = rows // num_heads
    P, Hkv, page_size, _ = key_pages.shape
    fast = (L > 8 and query.dtype == torch.bfloat16 and D == 128 and page_size % 64 == 0 and 128 % (num_heads // num_kv_heads) == 0
            and query.is_contiguous() and block_table.shape[0] == B and Hkv == num_kv_heads)
    if fast:
        _gpu("paged_attention", query, key_pages, value_pages, block_table, context_lens)
        out = torch.empty((B * L, num_heads * D), dtype=query.dtype, device=query.device)
        args = (query.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), block_table.data_ptr(), context_lens.data_ptr(), out.data_ptr(),
                rows, L, P, page_size, block_table.shape[1], float(scale), int(bool(is_causal)), int(num_kv_heads), int(num_heads))
        if workspace is None:
            rc = _lib.tl_paged_attention_token_major(*args, _stream_ptr(stream, query))
        else:
            if not workspace.is_cuda or not workspace.is_contiguous():
                raise RuntimeError("paged_attention_token_major: workspace must be a contiguous CUDA tensor")
            rc = _lib.tl_paged_attention_token_major_split(*args, workspace.data_ptr(), workspace.numel() * workspace.element_size(),
                                                           _stream_ptr(stream, query))
        if rc == 0:
            return out
    y = paged_attention(query, key_pages, value_pages, block_table, context_lens, scale, is_causal=is_causal, num_kv_heads=num_kv_heads,
                        num_heads=num_heads, stream=stream)
    return y.view(B, num_heads, L, D).transpose(1, 2).reshape(B * L, num_heads * D)


def paged_attention_segments(query, key_pages, value_pages, block_table, segment_start, scale, num_kv_heads, num_heads, stream=None):
    """Segment-causal prefill attention of one packed request (``tl_paged_attention_segments``, DESIGN.md section 17):
    ``query`` [Hq, L, 128] (``chunk_qk_norm_rope_append``'s output) -> ``[L, Hq * 128]`` token-major, row ``l`` seeing
    the keys ``segment_start[l] <= key <= l`` through the one block-table row ``block_table`` [max_pages]; a row with
    ``segment_start[l] > l`` gives zeros.  bf16 or fp16; page size a multiple of 64, Hq / Hkv dividing 128."""
    op = "paged_attention_segments"
    if query.dim() != 3 or key_pages.dim() != 4 or key_pages.shape != value_pages.shape:
        raise RuntimeError(f"{op}: q must be [H_q, L, D] and the page tensors [P, H_kv, page_size, D]")
    if query.dtype not in _HALF or key_pages.dtype != query.dtype or value_pages.dtype != query.dtype:
        raise RuntimeError(f"{op}: q, key_pages and value_pages must share one dtype, float16 or bfloat16")
    Hq, L, D = query.shape
    if Hq != num_heads or key_pages.shape[1] != num_kv_heads:
        raise RuntimeError(f"{op}: q must hold num_heads heads and the pages num_kv_heads")
    _int32(op, L, segment_start=segment_start)
    _block_table(op, block_table, None)
    _gpu(op, query, key_pages, value_pages, block_table, segment_start)
    _contig(op, query=query, key_pages=key_pages, value_pages=value_pages, block_table=block_table, segment_start=segment_start)
    P, _, page_size, _ = key_pages.shape
    out = torch.empty((L, Hq * D), dtype=query.dtype, device=query.device)
    _check(_lib.tl_paged_attention_segments(query.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), block_table.data_ptr(),
                                            segment_start.data_ptr(), out.data_ptr(), L, D, P, page_size, block_table.shape[0], float(scale),
                                            int(num_kv_heads), int(num_heads), _DTYPE_CODE[query.dtype], _stream_ptr(stream, query)))
    return out


EMBED_POOLING = {"last": 0, "mean": 1}


def embed_pool(hidden, norm_weight, eps, segment_start, pooling="last", dimensions=None, normalize=True, stream=None):
    """Pooled embeddings of packed hidden states (``tl_embed_pool``, DESIGN.md section 17): ``hidden`` [rows, H] bf16 or
    fp16, segments ``segment_start[s] .. segment_start[s + 1] - 1`` (int32 ``[n + 1]``).  Each pooled row is
    ``rms_norm(row, norm_weight, eps)`` bit for bit; ``pooling`` "last" takes the segment's last row, "mean" the fp32
    mean of its normalised rows; the first ``dimensions`` features (all when None) are kept and, with ``normalize``,
    divided by their L2 norm.  Returns fp32 ``[n, dimensions]``."""
    op = "embed_pool"
    if pooling not in EMBED_POOLING:
        raise ValueError(f"{op}: pooling must be one of {sorted(EMBED_POOLING)}, got {pooling!r}")
    if hidden.dim() != 2 or hidden.dtype not in _HALF or norm_weight.dtype != hidden.dtype or tuple(norm_weight.shape) != (hidden.shape[1],):
        raise RuntimeError(f"{op}: hidden must be float16 or bfloat16 [rows, H] with a norm weight [H] of its dtype")
    rows, H = hidden.shape
    d = H if dimensions is None else int(dimensions)
    if not 1 <= d <= H:
        raise ValueError(f"{op}: dimensions must be in [1, {H}], got {d}")
    if segment_start.dtype != torch.int32 or segment_start.dim() != 1 or segment_start.shape[0] < 1:
        raise RuntimeError(f"{op}: segment_start must be int32 [n + 1]")
    _gpu(op, hidden, norm_weight, segment_start)
    _contig(op, hidden=hidden, norm_weight=norm_weight, segment_start=segment_start)
    n = segment_start.shape[0] - 1
    out = torch.empty((n, d), dtype=torch.float32, device=hidden.device)
    _check(_lib.tl_embed_pool(hidden.data_ptr(), norm_weight.data_ptr(), float(eps), segment_start.data_ptr(), n, rows, H, d,
                              EMBED_POOLING[pooling], int(bool(normalize)), out.data_ptr(), _DTYPE_CODE[hidden.dtype], _stream_ptr(stream, hidden)))
    return out


def paged_attention_prefixed_segments(query, key_pages, value_pages, block_table, segment_start, prefix_start, prefix_end, scale,
                                      num_kv_heads, num_heads, stream=None):
    """Prefixed-segment prefill attention of one packed request (``tl_paged_attention_prefixed_segments``, DESIGN.md
    section 19): ``paged_attention_segments`` where row ``l`` also sees the keys ``prefix_start[l] <= key <
    prefix_end[l]`` (int32 ``[L]`` each, ``prefix_end[l] <= segment_start[l]``; equal bounds: no prefix)."""
    op = "paged_attention_prefixed_segments"
    if query.dim() != 3 or key_pages.dim() != 4 or key_pages.shape != value_pages.shape:
        raise RuntimeError(f"{op}: q must be [H_q, L, D] and the page tensors [P, H_kv, page_size, D]")
    if query.dtype not in _HALF or key_pages.dtype != query.dtype or value_pages.dtype != query.dtype:
        raise RuntimeError(f"{op}: q, key_pages and value_pages must share one dtype, float16 or bfloat16")
    Hq, L, D = query.shape
    if Hq != num_heads or key_pages.shape[1] != num_kv_heads:
        raise RuntimeError(f"{op}: q must hold num_heads heads and the pages num_kv_heads")
    _int32(op, L, segment_start=segment_start, prefix_start=prefix_start, prefix_end=prefix_end)
    _block_table(op, block_table, None)
    _gpu(op, query, key_pages, value_pages, block_table, segment_start, prefix_start, prefix_end)
    _contig(op, query=query, key_pages=key_pages, value_pages=value_pages, block_table=block_table, segment_start=segment_start,
            prefix_start=prefix_start, prefix_end=prefix_end)
    P, _, page_size, _ = key_pages.shape
    out = torch.empty((L, Hq * D), dtype=query.dtype, device=query.device)
    _check(_lib.tl_paged_attention_prefixed_segments(query.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), block_table.data_ptr(),
                                                     segment_start.data_ptr(), prefix_start.data_ptr(), prefix_end.data_ptr(), out.data_ptr(), L,
                                                     D, P, page_size, block_table.shape[0], float(scale), int(num_kv_heads), int(num_heads),
                                                     _DTYPE_CODE[query.dtype], _stream_ptr(stream, query)))
    return out


SELECT_MAX_IDS = 32


def select_logits(hidden, norm_weight, eps, row_index, weight, scales, biases, token_ids, stream=None):
    """Selected-token logits (``tl_select_logits``, DESIGN.md section 19): rows ``row_index`` (int32 ``[n]``) of
    ``hidden`` [rows, H] (bf16 or fp16) RMS-normalised with ``norm_weight`` bit for bit as ``rms_norm``, then the
    logits of ``token_ids`` (int32 ``[m]``, 1 <= m <= 32) under the packed MLX affine head ``weight`` [V, H * bits / 32]
    u32 with ``scales`` / ``biases`` [V, H / 128] (group 128; the width, 4 or 8 bits, follows from ``weight``'s shape).
    Returns fp32 ``(logits [n, m], logprobs [n, m])``: the logits rounded to the hidden dtype, and their log-softmax
    over the m ids."""
    op = "select_logits"
    if hidden.dim() != 2 or hidden.dtype not in _HALF or norm_weight.dtype != hidden.dtype or tuple(norm_weight.shape) != (hidden.shape[1],):
        raise RuntimeError(f"{op}: hidden must be float16 or bfloat16 [rows, H] with a norm weight [H] of its dtype")
    rows, H = hidden.shape
    if H % 128 != 0:
        raise RuntimeError(f"{op}: the hidden size must be a multiple of 128 (group 128), got {H}")
    if weight.dim() != 2 or weight.dtype not in _PACKED or weight.shape[1] * 32 % H != 0 or weight.shape[1] * 32 // H not in (4, 8):
        raise RuntimeError(f"{op}: weight must be packed 4- or 8-bit codes [V, H * bits / 32] (int32 or uint32)")
    bits = weight.shape[1] * 32 // H
    V = weight.shape[0]
    if scales.dtype != hidden.dtype or biases.dtype != hidden.dtype or tuple(scales.shape) != (V, H // 128) or scales.shape != biases.shape:
        raise RuntimeError(f"{op}: scales and biases must be [V, H / 128] of the hidden dtype")
    _int32(op, row_index=row_index, token_ids=token_ids)
    if row_index.dim() != 1 or token_ids.dim() != 1:
        raise RuntimeError(f"{op}: row_index and token_ids must be 1-D")
    m = token_ids.shape[0]
    if not 1 <= m <= SELECT_MAX_IDS:
        raise RuntimeError(f"{op}: 1 to {SELECT_MAX_IDS} token ids, got {m}")
    _gpu(op, hidden, norm_weight, row_index, weight, scales, biases, token_ids)
    _contig(op, hidden=hidden, norm_weight=norm_weight, row_index=row_index, weight=weight, scales=scales, biases=biases, token_ids=token_ids)
    n = row_index.shape[0]
    logits = torch.empty((n, m), dtype=torch.float32, device=hidden.device)
    logprobs = torch.empty((n, m), dtype=torch.float32, device=hidden.device)
    _check(_lib.tl_select_logits(hidden.data_ptr(), norm_weight.data_ptr(), float(eps), row_index.data_ptr(), n, rows, H, weight.data_ptr(),
                                 scales.data_ptr(), biases.data_ptr(), V, bits, token_ids.data_ptr(), m, logits.data_ptr(), logprobs.data_ptr(),
                                 _DTYPE_CODE[hidden.dtype], _stream_ptr(stream, hidden)))
    return logits, logprobs


def quantized_matmul_residual_norm(scales, biases, b, p0, residual, norm_weight, norm_eps, stream=None):
    """``x = residual + p0 @ W^T`` and ``h = rms_norm(x, norm_weight, norm_eps)`` in one call (the o / down projection
    of a block followed by the RMSNorm that opens the next one); returns ``(x, h)``.  Same rounding points as
    ``quantized_matmul_fused(epilogue=EPI_RESIDUAL)`` followed by ``rms_norm``."""
    if p0.dim() != 2 or b.dim() != 2 or not p0.is_contiguous():
        raise RuntimeError("quantized_matmul_residual_norm: p0 must be contiguous [M, N]")
    M, N = p0.shape
    K = b.shape[0]
    bits = packed_bits(b, N)
    if bits is None or tuple(scales.shape) != (K, N // 128) or scales.shape != biases.shape:
        raise RuntimeError("quantized_matmul_fused: incompatible parameter shapes (b must hold 4- or 8-bit codes: [K, N/8] or [K, N/4])")
    if scales.dtype not in _HALF or p0.dtype != scales.dtype or biases.dtype != scales.dtype or norm_weight.dtype != scales.dtype:
        raise RuntimeError("quantized_matmul: a must be the same dtype as scales")
    if tuple(residual.shape) != (M, K) or not residual.is_contiguous() or residual.dtype != p0.dtype:
        raise RuntimeError("quantized_matmul_fused: residual must be contiguous [M, K]")
    if tuple(norm_weight.shape) != (K,) or not norm_weight.is_contiguous():
        raise RuntimeError("quantized_matmul_residual_norm: norm weight must be [K]")
    _gpu("quantized_matmul_residual_norm", scales, biases, b, p0, residual, norm_weight)
    _contig("quantized_matmul_residual_norm", b=b, scales=scales, biases=biases)
    out = torch.empty((M, K), dtype=p0.dtype, device=p0.device)
    normed = torch.empty_like(out)
    code = _DTYPE_CODE[p0.dtype]
    ws_bytes = _lib.tl_quantized_matmul_fused_workspace_bits(M, N, K, N, int(PRO_NONE), code, bits)
    ws = _zero_workspace(ws_bytes, p0.device)
    _check(
        _lib.tl_quantized_matmul_residual_norm_bits(
            scales.data_ptr(), biases.data_ptr(), b.data_ptr(), out.data_ptr(), p0.data_ptr(), residual.data_ptr(), norm_weight.data_ptr(),
            normed.data_ptr(), M, N, K, float(norm_eps), code, bits, None if ws is None else ws.data_ptr(), ws_bytes, _stream_ptr(stream, p0),
        )
    )
    return out, normed


def chunk_qk_norm_rope_append(qkv, q_norm_weight, k_norm_weight, offsets, block_table_row, context_lens, key_pages, value_pages,
                              num_heads, num_kv_heads, base, eps, stream=None, inv_freq=None):
    """Prefill-chunk form of ``decode_qk_norm_rope_append``: the rows of ``qkv`` are consecutive tokens of one
    request; returns the rotated queries ``[Hq, tokens, D]`` (the layout ``paged_attention`` takes).  ``inv_freq``: a
    float64 ``[D / 2]`` frequency table replacing ``base`` (``rope_table``)."""
    T = qkv.shape[0]
    P, Hkv, page_size, D = key_pages.shape
    if qkv.dim() != 2 or qkv.shape[1] != (num_heads + 2 * num_kv_heads) * D or Hkv != num_kv_heads:
        raise RuntimeError("chunk_qk_norm_rope_append: qkv must be [tokens, (Hq + 2*Hkv) * D]")
    if qkv.dtype != key_pages.dtype or value_pages.dtype != key_pages.dtype or q_norm_weight.dtype != qkv.dtype:
        raise RuntimeError("chunk_qk_norm_rope_append: dtype mismatch")
    if block_table_row.dim() != 1 or offsets.numel() != T or context_lens.numel() != T:
        raise RuntimeError("chunk_qk_norm_rope_append: one block-table row, one offset and one context length per token")
    _int32("chunk_qk_norm_rope_append", T, offsets=offsets, context_lens=context_lens)
    _int32("chunk_qk_norm_rope_append", block_table_row=block_table_row)
    _norm_weights("chunk_qk_norm_rope_append", qkv.dtype, D, q_norm_weight=q_norm_weight, k_norm_weight=k_norm_weight)
    _inv_freq("chunk_qk_norm_rope_append", inv_freq, D // 2)
    _gpu("chunk_qk_norm_rope_append", qkv, q_norm_weight, k_norm_weight, offsets, block_table_row, context_lens, key_pages, value_pages)
    _contig("chunk_qk_norm_rope_append", qkv=qkv, offsets=offsets, block_table_row=block_table_row, context_lens=context_lens,
            key_pages=key_pages, value_pages=value_pages)
    q_out = torch.empty((num_heads, T, D), dtype=qkv.dtype, device=qkv.device)
    args = (qkv.data_ptr(), q_norm_weight.data_ptr(), k_norm_weight.data_ptr(), offsets.data_ptr(), block_table_row.data_ptr(),
            context_lens.data_ptr(), q_out.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), T, int(num_heads),
            int(num_kv_heads), D, float(base), float(eps), P, page_size, block_table_row.shape[0], _DTYPE_CODE[qkv.dtype],
            _stream_ptr(stream, qkv))
    _check(_lib.tl_chunk_qk_norm_rope_append(*args) if inv_freq is None else _lib.tl_chunk_qk_norm_rope_append_table(*args, inv_freq.data_ptr()))
    return q_out


def interleave_gate_up(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    """Row layout EPI_SWIGLU_PAIRS expects: blocks of 8 gate rows followed by the matching 8 up rows."""
    K = gate.shape[0]
    if gate.shape != up.shape or K % 8:
        raise RuntimeError("interleave_gate_up: gate and up must share a shape with rows % 8 == 0")
    tail = gate.shape[1:]
    return torch.stack((gate.reshape(K // 8, 8, *tail), up.reshape(K // 8, 8, *tail)), dim=1).reshape(2 * K, *tail).contiguous()


def decode_qk_norm_rope_append(qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, key_pages, value_pages,
                               num_heads, num_kv_heads, base, eps, stream=None, inv_freq=None):
    """Fused per-head q/k RMSNorm + RoPE + K/V append of one decode step; returns
    the rotated queries ``[B, Hq, D]``.  ``inv_freq``: a float64 ``[D / 2]`` frequency table replacing ``base``."""
    B = qkv.shape[0]
    P, Hkv, page_size, D = key_pages.shape
    if qkv.dim() != 2 or qkv.shape[1] != (num_heads + 2 * num_kv_heads) * D or Hkv != num_kv_heads:
        raise RuntimeError("decode_qk_norm_rope_append: qkv must be [B, (Hq + 2*Hkv) * D]")
    if qkv.dtype != key_pages.dtype or value_pages.dtype != key_pages.dtype or q_norm_weight.dtype != qkv.dtype:
        raise RuntimeError("decode_qk_norm_rope_append: dtype mismatch")
    _norm_weights("decode_qk_norm_rope_append", qkv.dtype, D, q_norm_weight=q_norm_weight, k_norm_weight=k_norm_weight)
    _int32("decode_qk_norm_rope_append", B, offsets=offsets, context_lens=context_lens)
    _block_table("decode_qk_norm_rope_append", block_table, B)
    _inv_freq("decode_qk_norm_rope_append", inv_freq, D // 2)
    _gpu("decode_qk_norm_rope_append", qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, key_pages, value_pages)
    _contig("decode_qk_norm_rope_append", qkv=qkv, offsets=offsets, block_table=block_table, context_lens=context_lens,
            key_pages=key_pages, value_pages=value_pages)
    q_out = torch.empty((B, num_heads, D), dtype=qkv.dtype, device=qkv.device)
    args = (qkv.data_ptr(), q_norm_weight.data_ptr(), k_norm_weight.data_ptr(), offsets.data_ptr(), block_table.data_ptr(),
            context_lens.data_ptr(), q_out.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), B, int(num_heads),
            int(num_kv_heads), D, float(base), float(eps), P, page_size, block_table.shape[1], _DTYPE_CODE[qkv.dtype],
            _stream_ptr(stream, qkv))
    _check(_lib.tl_decode_qk_norm_rope_append(*args) if inv_freq is None else _lib.tl_decode_qk_norm_rope_append_table(*args, inv_freq.data_ptr()))
    return q_out


def qkv_project_rope_append(scales, biases, b, p0, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, key_pages, value_pages,
                            num_heads, num_kv_heads, base, eps, chunk=False, stream=None, inv_freq=None):
    """``qkv = p0 @ W_qkv^T`` then per-head q/k RMSNorm + RoPE + K/V append (``decode_qk_norm_rope_append``; ``chunk``: the
    rows are consecutive tokens of one request and ``block_table`` is its row).  Returns the rotated queries
    (``[rows, Hq, D]``, or ``[Hq, rows, D]`` for a chunk).  With 9..128 rows the projection's split-reduction planes
    feed the second kernel directly; results are those of the two separate calls.  ``inv_freq``: a float64 ``[D / 2]``
    frequency table replacing ``base``."""
    rows, N = p0.shape
    P, Hkv, page_size, D = key_pages.shape
    K = b.shape[0]
    bits = packed_bits(b, N)
    if K != (num_heads + 2 * num_kv_heads) * D or Hkv != num_kv_heads or bits is None:
        raise RuntimeError("qkv_project_rope_append: weight rows must be (Hq + 2*Hkv) * D")
    if (p0.dtype != torch.bfloat16 or key_pages.dtype != p0.dtype or value_pages.dtype != p0.dtype or scales.dtype != p0.dtype
            or biases.dtype != p0.dtype or not p0.is_contiguous()):
        raise RuntimeError("qkv_project_rope_append: contiguous bfloat16 inputs required")
    op = "qkv_project_rope_append"
    _norm_weights(op, p0.dtype, D, q_norm_weight=q_norm_weight, k_norm_weight=k_norm_weight)
    _int32(op, rows, offsets=offsets, context_lens=context_lens)
    _block_table(op, block_table, None if chunk else rows)
    _inv_freq(op, inv_freq, D // 2)
    _gpu(op, scales, biases, b, p0, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, key_pages, value_pages)
    _contig(op, b=b, scales=scales, biases=biases, offsets=offsets, block_table=block_table, context_lens=context_lens, key_pages=key_pages,
            value_pages=value_pages)
    scratch = torch.empty((rows, K), dtype=p0.dtype, device=p0.device)
    q_out = torch.empty((num_heads, rows, D) if chunk else (rows, num_heads, D), dtype=p0.dtype, device=p0.device)
    code = _DTYPE_CODE[p0.dtype]
    ws_bytes = _lib.tl_quantized_matmul_fused_workspace_bits(rows, N, K, N, int(PRO_NONE), code, bits)
    ws = _zero_workspace(ws_bytes, p0.device)
    max_pages = block_table.shape[-1]
    args = (scales.data_ptr(), biases.data_ptr(), b.data_ptr(), p0.data_ptr(), scratch.data_ptr(), q_norm_weight.data_ptr(), k_norm_weight.data_ptr(),
            offsets.data_ptr(), block_table.data_ptr(), context_lens.data_ptr(), q_out.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(),
            rows, N, int(num_heads), int(num_kv_heads), D, float(base), float(eps), P, page_size, max_pages, int(bool(chunk)), code, bits,
            None if ws is None else ws.data_ptr(), ws_bytes, _stream_ptr(stream, p0))
    _check(_lib.tl_qkv_project_rope_append_bits(*args) if inv_freq is None else _lib.tl_qkv_project_rope_append_table_bits(*args, inv_freq.data_ptr()))
    return q_out


def rope_inv_freq_table(head_dim: int, base: float, device) -> torch.Tensor:
    """float64 [head_dim / 2] frequencies base^(-i / (head_dim / 2)) (rope.py:13-15 forms them the same way).  The
    unscaled ``decode_attention_fused`` path keeps reading this table so that its bits do not change; it can differ in
    the last bits from ``rope_default_inv_freq``, the kernels' inline expression that every other site (and YaRN) uses."""
    half = head_dim // 2
    return torch.pow(torch.tensor(float(base), dtype=torch.float64), -torch.arange(half, dtype=torch.float64) / half).to(device)


def decode_attention_fused_workspace(batch: int, num_heads: int, num_kv_heads: int, rows_per_request: int = 1) -> int:
    """float32 values of the split workspace for ``batch`` requests of ``rows_per_request`` query rows each."""
    R = _rows_per_request("decode_attention_fused_workspace", rows_per_request)
    if R == 1:
        return int(_lib.tl_decode_attention_fused_workspace(int(batch), int(num_heads), int(num_kv_heads)))
    return int(_lib.tl_decode_attention_fused_rows_workspace(int(batch), R, int(num_heads), int(num_kv_heads)))


def _rows_per_request(op: str, rows_per_request) -> int:
    if isinstance(rows_per_request, bool) or not isinstance(rows_per_request, int) or not 1 <= rows_per_request <= 8:
        raise RuntimeError(f"{op}: rows_per_request must be an int in [1, 8]")
    return rows_per_request


def decode_attention_fused(qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, rope_inv_freq, key_pages,
                           value_pages, num_heads, num_kv_heads, eps, scale, max_context, out=None, workspace=None, stream=None,
                           rows_per_request=1):
    """One decode step of attention for ``qkv [B, (Hq + 2 Hkv) * 128]`` (bf16): per-head q/k RMSNorm +
    RoPE, append of the newest K/V row, paged GQA attention (context_lens are post-append) ->
    ``[B, Hq * 128]``.  ``max_context`` bounds every context length (it fixes the split count).

    ``rows_per_request = R`` (1..8): the ``B`` rows are ``B / R`` requests of R consecutive query rows each (row j of
    a request at context ``context_lens[row 0] + j``), sharing one block-table row (``[B / R, max_pages]``).  Every
    row equals, bit for bit, the single-row call on it alone with the rows before it already appended."""
    R = _rows_per_request("decode_attention_fused", rows_per_request)
    B = qkv.shape[0]
    P, Hkv, page_size, D = key_pages.shape
    if qkv.dim() != 2 or qkv.shape[1] != (num_heads + 2 * num_kv_heads) * D or Hkv != num_kv_heads:
        raise RuntimeError("decode_attention_fused: qkv must be [B, (Hq + 2*Hkv) * D]")
    if R > 1 and B % R != 0:
        raise RuntimeError(f"decode_attention_fused: qkv rows must be a multiple of rows_per_request ({R})")
    requests = B // R
    if qkv.dtype != key_pages.dtype or value_pages.dtype != key_pages.dtype or q_norm_weight.dtype != qkv.dtype or k_norm_weight.dtype != qkv.dtype:
        raise RuntimeError("decode_attention_fused: dtype mismatch")
    if rope_inv_freq.dtype != torch.float64 or rope_inv_freq.numel() != D // 2:
        raise RuntimeError("decode_attention_fused: rope_inv_freq must be float64 [head_dim / 2]")
    if R == 1:
        if block_table.dim() != 2 or block_table.shape[0] != B or block_table.dtype != torch.int32 or context_lens.dtype != torch.int32:
            raise RuntimeError("decode_attention_fused: block_table must be int32 [B, max_pages] and context_lens int32 [B]")
    elif block_table.dim() != 2 or block_table.shape[0] != requests or block_table.dtype != torch.int32 or context_lens.dtype != torch.int32:
        raise RuntimeError("decode_attention_fused: block_table must be int32 [B / rows_per_request, max_pages] and context_lens int32 [B]")
    _norm_weights("decode_attention_fused", qkv.dtype, D, q_norm_weight=q_norm_weight, k_norm_weight=k_norm_weight)
    _int32("decode_attention_fused", B, offsets=offsets, context_lens=context_lens)
    _gpu("decode_attention_fused", qkv, q_norm_weight, k_norm_weight, offsets, block_table, context_lens, rope_inv_freq, key_pages, value_pages)
    _contig("decode_attention_fused", qkv=qkv, offsets=offsets, block_table=block_table, context_lens=context_lens,
            key_pages=key_pages, value_pages=value_pages, rope_inv_freq=rope_inv_freq)
    if out is None:
        out = torch.empty((B, num_heads * D), dtype=qkv.dtype, device=qkv.device)
    need = decode_attention_fused_workspace(requests, num_heads, num_kv_heads, rows_per_request=R)
    if workspace is None:
        workspace = torch.empty(need, dtype=torch.float32, device=qkv.device)
    elif workspace.dtype != torch.float32 or workspace.numel() < need or not workspace.is_cuda:
        raise RuntimeError("decode_attention_fused: workspace must hold decode_attention_fused_workspace() float32 values")
    args = (qkv.data_ptr(), q_norm_weight.data_ptr(), k_norm_weight.data_ptr(), offsets.data_ptr(), block_table.data_ptr(),
            context_lens.data_ptr(), rope_inv_freq.data_ptr(), key_pages.data_ptr(), value_pages.data_ptr(), out.data_ptr(),
            workspace.data_ptr())
    tail = (int(num_heads), int(num_kv_heads), D, float(eps), float(scale), P, page_size, block_table.shape[1], int(max_context),
            _DTYPE_CODE[qkv.dtype], _stream_ptr(stream, qkv))
    if R == 1:
        _check(_lib.tl_decode_attention_fused(*args, B, *tail))
    else:
        _check(_lib.tl_decode_attention_fused_rows(*args, requests, R, *tail))
    return out


# ---- Qwen3-MoE sparse block (include/tiny_llm_b200.h, "Qwen3-MoE") -------------
MOE_CONTROL, MOE_WGMMA = 0, 1
MOE_MAX_EXPERTS, MOE_MAX_TOPK = 256, 8


def _moe_shape(op: str, E: int, k: int) -> None:
    if E <= 0 or E > MOE_MAX_EXPERTS:
        raise RuntimeError(f"{op}: at most {MOE_MAX_EXPERTS} experts (got {E})")
    if k <= 0 or k > MOE_MAX_TOPK or k > E:
        raise RuntimeError(f"{op}: top-k must be in [1, min({MOE_MAX_TOPK}, experts)] (got k = {k}, E = {E})")


def moe_topk(logits, top_k, norm_topk_prob=False, stream=None):
    """Router top-k of ``logits [T, E]``: ``(probs [T, E], ids int32 [T, k], scores [T, k])`` with probs the rounded
    fp32 softmax, ids the k largest probs in descending order (ties to the lower expert id) and scores optionally
    renormalised over the k (``include/tiny_llm_b200.h`` gives the rounding points)."""
    if logits.dtype not in _FLOATS or logits.dim() != 2:
        raise RuntimeError("moe_topk: expected 2D float logits [T, E]")
    T, E = logits.shape
    _moe_shape("moe_topk", E, int(top_k))
    _gpu("moe_topk", logits)
    _contig("moe_topk", logits=logits)
    probs = torch.empty_like(logits)
    ids = torch.empty((T, top_k), dtype=torch.int32, device=logits.device)
    scores = torch.empty((T, top_k), dtype=logits.dtype, device=logits.device)
    _check(_lib.tl_moe_topk(logits.data_ptr(), probs.data_ptr(), ids.data_ptr(), scores.data_ptr(), T, E, int(top_k), int(bool(norm_topk_prob)),
                            _DTYPE_CODE[logits.dtype], _stream_ptr(stream, logits)))
    return probs, ids, scores


def moe_group(ids, num_experts, nt=0, stream=None):
    """Expert grouping of ``ids`` (int32, R entries): ``(offsets int32 [E + 1], perm int32 [R], tiles)`` with perm the
    stable sort of the rows by expert and, for ``nt > 0``, the grouped GEMM's tile table (else None)."""
    if ids.dtype != torch.int32:
        raise RuntimeError("moe_group: ids must be int32")
    E = int(num_experts)
    if E <= 0 or E > MOE_MAX_EXPERTS:
        raise RuntimeError(f"moe_group: at most {MOE_MAX_EXPERTS} experts (got {E})")
    if nt < 0:
        raise RuntimeError("moe_group: nt must be >= 0")
    _gpu("moe_group", ids)
    _contig("moe_group", ids=ids)
    R = ids.numel()
    offsets = torch.empty((E + 1,), dtype=torch.int32, device=ids.device)
    perm = torch.empty((R,), dtype=torch.int32, device=ids.device)
    size = int(_lib.tl_moe_tile_table_size(R, E, int(nt)))
    _check(min(size, 0))
    tiles = torch.empty((size,), dtype=torch.int32, device=ids.device) if size > 0 else None
    _check(_lib.tl_moe_group(ids.data_ptr(), R, E, int(nt), offsets.data_ptr(), perm.data_ptr(), None if tiles is None else tiles.data_ptr(),
                             _stream_ptr(stream, ids)))
    return offsets, perm, tiles


def moe_gather(x, perm, rows_per_source, norm_weight=None, eps=0.0, stream=None):
    """``xs[j] = x[perm[j] // rows_per_source]`` (optionally RMSNorm-ed with ``norm_weight``) -> ``[R, H]``."""
    if x.dtype not in _FLOATS or x.dim() != 2:
        raise RuntimeError("moe_gather: expected 2D float x [rows, H]")
    if perm.dtype != torch.int32 or perm.dim() != 1:
        raise RuntimeError("moe_gather: perm must be int32 [R]")
    if int(rows_per_source) <= 0:
        raise RuntimeError("moe_gather: rows_per_source must be positive")
    H = x.shape[1]
    if norm_weight is not None and (norm_weight.dtype != x.dtype or tuple(norm_weight.shape) != (H,)):
        raise RuntimeError("moe_gather: norm weight must be [H] in the dtype of x")
    _gpu("moe_gather", x, perm, *([] if norm_weight is None else [norm_weight]))
    _contig("moe_gather", x=x, perm=perm, **({} if norm_weight is None else {"norm_weight": norm_weight}))
    R = perm.numel()
    xs = torch.empty((R, H), dtype=x.dtype, device=x.device)
    _check(_lib.tl_moe_gather(x.data_ptr(), perm.data_ptr(), None if norm_weight is None else norm_weight.data_ptr(), float(eps), xs.data_ptr(), R,
                              int(rows_per_source), H, _DTYPE_CODE[x.dtype], _stream_ptr(stream, x)))
    return xs


def moe_grouped_matmul_route(T, k, E, N, K, epilogue, dtype, a, b):
    """The kernel ``moe_grouped_matmul`` runs: ``(route, nt, max_tiles)`` with route ``MOE_WGMMA`` or ``MOE_CONTROL``.
    ``a`` and ``b`` are tensors or plain addresses (only their alignment counts); ``dtype`` is a torch dtype."""

    def addr(t):
        return t.data_ptr() if isinstance(t, torch.Tensor) else int(t)

    nt, tiles = _I(), _I()
    code = _lib.tl_moe_grouped_matmul_route(int(T), int(k), int(E), int(N), int(K), int(epilogue), _DTYPE_CODE[dtype], addr(a), addr(b),
                                            ctypes.byref(nt), ctypes.byref(tiles))
    _check(min(code, 0))
    return code, nt.value, tiles.value


def moe_grouped_matmul(scales, biases, b, a, offsets, tiles, top_k, out_index=None, epilogue=EPI_NONE, stream=None):
    """Grouped W4A16 projection of the expert-sorted rows ``a [R, N]`` (R = T * top_k) by the experts ``b [E, K, N/8]``
    (scales / biases ``[E, K, N/128]``), segments ``offsets [E + 1]`` and tile table ``tiles`` from ``moe_group`` (with
    the ``nt`` of ``moe_grouped_matmul_route``).  Returns ``[R, K]`` (``EPI_SWIGLU_PAIRS``: ``[R, K/2]`` over each
    expert's interleaved gate|up rows); row j lands at ``out_index[j]`` when given."""
    if b.dim() != 3 or scales.dim() != 3 or a.dim() != 2:
        raise RuntimeError("moe_grouped_matmul: expected b [E, K, N/8], scales [E, K, N/128] and a [R, N]")
    E, K, words = b.shape
    R, N = a.shape
    if words * 8 != N or N % 128 or tuple(scales.shape) != (E, K, N // 128) or scales.shape != biases.shape:
        raise RuntimeError("moe_grouped_matmul: incompatible parameter shapes")
    if scales.dtype not in _HALF or a.dtype != scales.dtype or biases.dtype != scales.dtype or b.dtype not in _PACKED:
        raise RuntimeError("moe_grouped_matmul: a, scales and biases must share a 16-bit dtype and b must be 32-bit words")
    _moe_shape("moe_grouped_matmul", E, int(top_k))
    if R % top_k:
        raise RuntimeError("moe_grouped_matmul: rows must be a multiple of top_k")
    if epilogue not in (EPI_NONE, EPI_SWIGLU_PAIRS) or (epilogue == EPI_SWIGLU_PAIRS and K % 16):
        raise RuntimeError("moe_grouped_matmul: epilogue must be EPI_NONE or EPI_SWIGLU_PAIRS (K % 16 == 0)")
    _int32("moe_grouped_matmul", offsets=offsets)
    if offsets.numel() != E + 1:
        raise RuntimeError("moe_grouped_matmul: offsets must be int32 [E + 1]")
    if out_index is not None:
        _int32("moe_grouped_matmul", R, out_index=out_index)
    extra = [t for t in (tiles, out_index) if t is not None]
    _gpu("moe_grouped_matmul", scales, biases, b, a, offsets, *extra)
    _contig("moe_grouped_matmul", scales=scales, biases=biases, b=b, a=a, offsets=offsets)
    T = R // top_k
    route, nt, _ = moe_grouped_matmul_route(T, top_k, E, N, K, epilogue, a.dtype, a, b)
    if route == MOE_WGMMA and (tiles is None or tiles.numel() != int(_lib.tl_moe_tile_table_size(R, E, nt))):
        raise RuntimeError(f"moe_grouped_matmul: the wgmma route needs moe_group's tile table for nt = {nt}")
    out = torch.empty((R, K // 2 if epilogue == EPI_SWIGLU_PAIRS else K), dtype=a.dtype, device=a.device)
    _check(_lib.tl_moe_grouped_matmul(scales.data_ptr(), biases.data_ptr(), b.data_ptr(), a.data_ptr(), out.data_ptr(), offsets.data_ptr(),
                                      None if tiles is None else tiles.data_ptr(), None if out_index is None else out_index.data_ptr(), T,
                                      int(top_k), E, N, K, int(epilogue), _DTYPE_CODE[a.dtype], _stream_ptr(stream, a)))
    return out


def moe_combine(y, scores, residual=None, norm_weight=None, eps=0.0, stream=None):
    """``out[t] = T(residual[t] + T(sum_j T(y[t k + j] * scores[t, j])))`` (without residual: the rounded sum) for
    ``y [T k, H]`` and ``scores [T, k]``; with ``norm_weight`` returns ``(out, rms_norm(out))``."""
    if y.dtype not in _FLOATS or y.dim() != 2 or scores.dim() != 2 or scores.dtype != y.dtype:
        raise RuntimeError("moe_combine: expected y [T k, H] and scores [T, k] of one float dtype")
    T, k = scores.shape
    H = y.shape[1]
    if k <= 0 or k > MOE_MAX_TOPK or y.shape[0] != T * k:
        raise RuntimeError(f"moe_combine: y must be [T * k, H] with 1 <= k <= {MOE_MAX_TOPK}")
    if residual is not None and (residual.dtype != y.dtype or tuple(residual.shape) != (T, H)):
        raise RuntimeError("moe_combine: residual must be [T, H] in the dtype of y")
    if norm_weight is not None and (norm_weight.dtype != y.dtype or tuple(norm_weight.shape) != (H,) or H > 4096):
        raise RuntimeError("moe_combine: norm weight must be [H] (H <= 4096) in the dtype of y")
    extra = {n: t for n, t in (("residual", residual), ("norm_weight", norm_weight)) if t is not None}
    _gpu("moe_combine", y, scores, *extra.values())
    _contig("moe_combine", y=y, scores=scores, **extra)
    out = torch.empty((T, H), dtype=y.dtype, device=y.device)
    normed = None if norm_weight is None else torch.empty_like(out)
    _check(_lib.tl_moe_combine(y.data_ptr(), scores.data_ptr(), None if residual is None else residual.data_ptr(),
                               None if norm_weight is None else norm_weight.data_ptr(), float(eps), out.data_ptr(),
                               None if normed is None else normed.data_ptr(), T, k, H, _DTYPE_CODE[y.dtype], _stream_ptr(stream, y)))
    return out if normed is None else (out, normed)


LORA_MAX_SEGMENTS, LORA_MAX_RANK, LORA_MAX_ADAPTERS = 3, 64, 32
MOE_ROUTER_GROUP = 64  # group size of the 8-bit routers moe_router takes


def moe_router(x, weight, scales, biases, norm_weight=None, eps=0.0, stream=None):
    """Router logits ``[T, E]`` of an MLX affine 8-bit router at group 64 (``tl_moe_router``): ``x [T, H]`` (bf16 or
    fp16), ``weight`` packed codes ``[E, H / 4]`` (int32 or uint32), ``scales`` / ``biases [E, H / 64]`` of x's dtype;
    ``sum_k (scale * code + bias) * a`` in fp32, rounded once.  With ``norm_weight [H]``, ``a`` is the row's RMSNorm,
    bit for bit ``rms_norm(x, norm_weight, eps)``; else ``a = x``."""
    op = "moe_router"
    if x.dim() != 2 or x.dtype not in _HALF:
        raise RuntimeError(f"{op}: x must be float16 or bfloat16 [T, H]")
    T, H = x.shape
    if H <= 0 or H % MOE_ROUTER_GROUP:
        raise RuntimeError(f"{op}: the hidden size must be a positive multiple of {MOE_ROUTER_GROUP}, got {H}")
    if weight.dim() != 2 or weight.dtype not in _PACKED or weight.shape[1] * 4 != H:
        raise RuntimeError(f"{op}: weight must be packed 8-bit codes [E, H / 4] = [E, {H // 4}] (int32 or uint32), got {tuple(weight.shape)}")
    E = weight.shape[0]
    if E <= 0 or E > MOE_MAX_EXPERTS:
        raise RuntimeError(f"{op}: 1 to {MOE_MAX_EXPERTS} experts (got {E})")
    G = H // MOE_ROUTER_GROUP
    if scales.dtype != x.dtype or biases.dtype != x.dtype or tuple(scales.shape) != (E, G) or scales.shape != biases.shape:
        raise RuntimeError(f"{op}: scales and biases must be [E, H / 64] = [{E}, {G}] of x's dtype")
    if norm_weight is not None and (norm_weight.dtype != x.dtype or tuple(norm_weight.shape) != (H,)):
        raise RuntimeError(f"{op}: norm weight must be [H] in the dtype of x")
    extra = {} if norm_weight is None else {"norm_weight": norm_weight}
    _gpu(op, x, weight, scales, biases, *extra.values())
    _contig(op, x=x, weight=weight, scales=scales, biases=biases, **extra)
    out = torch.empty((T, E), dtype=x.dtype, device=x.device)
    _check(_lib.tl_moe_router(x.data_ptr(), None if norm_weight is None else norm_weight.data_ptr(), float(eps), weight.data_ptr(),
                              scales.data_ptr(), biases.data_ptr(), out.data_ptr(), T, E, H, _DTYPE_CODE[x.dtype], _stream_ptr(stream, x)))
    return out


LORA_RANKS = (8, 16, 32, 64)
LORA_ROWS, LORA_TILES = 0, 1


class _LoraSiteC(ctypes.Structure):
    """``tl_lora_site``."""

    _fields_ = [("a", _VP), ("b", _VP * 3), ("scales", _VP), ("ranks", _VP), ("seg_mask", _VP),
                ("n_adapters", ctypes.c_int32), ("nseg", ctypes.c_int32), ("r_max", ctypes.c_int32), ("N", ctypes.c_int32),
                ("K", ctypes.c_int32 * 3)]


class LoraSite:
    """The packed adapters of one site (``tl_lora_site``): ``a`` bf16 ``[n_adapters, nseg * r_max, N]``, ``b`` one bf16
    ``[n_adapters, K_s, r_max]`` per segment, ``scales`` f32, ``ranks`` and ``seg_mask`` int32 ``[n_adapters]``.  It keeps
    the tensors alive for the launches (and captured graphs) that read them."""

    def __init__(self, a, b, scales, ranks, seg_mask):
        b = list(b)
        if a.dtype != torch.bfloat16 or a.dim() != 3 or any(t.dtype != torch.bfloat16 or t.dim() != 3 for t in b):
            raise RuntimeError("lora_apply: A and B must be bfloat16 [n_adapters, rows, cols]")
        n, J, N = a.shape
        if not 1 <= len(b) <= LORA_MAX_SEGMENTS or J % len(b) != 0:
            raise RuntimeError(f"lora_apply: a site has 1 to {LORA_MAX_SEGMENTS} segments, A [n_adapters, nseg * r_max, N]")
        r_max = J // len(b)
        if not 1 <= n <= LORA_MAX_ADAPTERS:
            raise RuntimeError(f"lora_apply: a set holds 1 to {LORA_MAX_ADAPTERS} adapters")
        if r_max not in LORA_RANKS:
            raise RuntimeError(f"lora_apply: r_max must be one of {LORA_RANKS}")
        if N % 8 != 0:
            raise RuntimeError("lora_apply: the input width must be a multiple of 8")
        if any(t.shape[0] != n or t.shape[2] != r_max for t in b):
            raise RuntimeError("lora_apply: every B must be [n_adapters, K_s, r_max]")
        if scales.dtype != torch.float32 or ranks.dtype != torch.int32 or seg_mask.dtype != torch.int32 \
                or any(tuple(t.shape) != (n,) for t in (scales, ranks, seg_mask)):
            raise RuntimeError("lora_apply: scales f32, ranks and seg_mask int32, one entry per adapter")
        _contig("lora_apply", a=a, scales=scales, ranks=ranks, seg_mask=seg_mask, **{f"b{s}": t for s, t in enumerate(b)})
        self.a, self.b, self.scales, self.ranks, self.seg_mask = a, b, scales, ranks, seg_mask
        self.n_adapters, self.nseg, self.r_max, self.N = n, len(b), r_max, N
        self.K = [t.shape[1] for t in b]
        ptrs = [t.data_ptr() for t in b] + [None] * (3 - len(b))
        self.c = _LoraSiteC(a.data_ptr(), (_VP * 3)(*ptrs), scales.data_ptr(), ranks.data_ptr(), seg_mask.data_ptr(), n, len(b), r_max, N,
                            (ctypes.c_int32 * 3)(*(self.K + [0] * (3 - len(b)))))


def _lora_segments(y, site, name):
    """``y`` (one ``[M, sum K_s]`` tensor holding the segments side by side, or one ``[M, K_s]`` tensor per segment) as
    per-segment views."""
    if not all(t.is_contiguous() for t in ([y] if isinstance(y, torch.Tensor) else y)):
        raise RuntimeError(f"lora_apply: {name} must be contiguous (it is updated in place)")
    if isinstance(y, torch.Tensor):
        y2 = y.reshape(-1, y.shape[-1])
        if y2.shape[1] != sum(site.K):
            raise RuntimeError(f"lora_apply: {name} must be [M, {sum(site.K)}] (the site's segments side by side)")
        return list(torch.split(y2, site.K, dim=1))
    segs = [t.reshape(-1, t.shape[-1]) for t in y]
    if [t.shape[1] for t in segs] != site.K:
        raise RuntimeError(f"lora_apply: {name} must hold one [M, K_s] tensor per segment, K = {site.K}")
    return segs


def _lora_args(x, y, adapter_ids, site, residual):
    if not isinstance(site, LoraSite):
        raise RuntimeError("lora_apply: site must be a LoraSite")
    M = adapter_ids.numel()
    ys = _lora_segments(y, site, "y")
    rs = None if residual is None else _lora_segments(residual, site, "residual")
    if x.dtype != torch.bfloat16 or any(t.dtype != torch.bfloat16 for t in ys + (rs or [])):
        raise RuntimeError("lora_apply: activations must be bfloat16")
    if x.shape[-1] != site.N or x.numel() != M * site.N:
        raise RuntimeError(f"lora_apply: x must be [{M}, {site.N}] (one row per adapter id)")
    for s, t in enumerate(ys):
        if t.shape[0] != M or t.stride(1) != 1:
            raise RuntimeError(f"lora_apply: segment {s} of y must be [{M}, {site.K[s]}] with unit column stride")
        if rs is not None and (rs[s].shape != t.shape or rs[s].stride() != t.stride()):
            raise RuntimeError("lora_apply: residual must have the layout of y")
    _int32("lora_apply", M, adapter_ids=adapter_ids)
    return M, ys, rs


def lora_apply_route(M: int, site: LoraSite) -> int:
    """``LORA_ROWS`` (a cluster per row, M <= 64) or ``LORA_TILES`` (a cluster per 8 rows) for ``M`` rows of ``site``."""
    route = _lib.tl_lora_apply_route(int(M), _DTYPE_CODE[torch.bfloat16], ctypes.byref(site.c))
    if route < 0:
        _check(route)
    return route


def lora_apply(x, y, adapter_ids, site: LoraSite, residual=None, stream=None):
    """Add each row's adapter to the projection output ``y`` in place and return it (``tl_lora_apply``): row m with
    ``adapter_ids[m] = a >= 0`` becomes ``T(y + sc_a * B_a T(A_a x))`` per targeted segment, then ``T(residual + y)`` with
    a residual; rows with a negative id keep their bits (or take the residual add alone).  ``y`` (and ``residual``): one
    tensor with the site's segments side by side, or a list of one tensor per segment."""
    M, ys, rs = _lora_args(x, y, adapter_ids, site, residual)
    _gpu("lora_apply", x, adapter_ids, site.a, *ys, *(rs or []))
    _contig("lora_apply", x=x, adapter_ids=adapter_ids)
    n = site.nseg
    y_ptrs = (_VP * n)(*[t.data_ptr() for t in ys])
    r_ptrs = None if rs is None else (_VP * n)(*[t.data_ptr() for t in rs])
    ld = (_LL * n)(*[t.stride(0) if t.shape[0] > 1 else t.shape[1] for t in ys])
    _check(_lib.tl_lora_apply(x.data_ptr(), y_ptrs, r_ptrs, ld, adapter_ids.data_ptr(), ctypes.byref(site.c), M, _DTYPE_CODE[x.dtype],
                              _stream_ptr(stream, x)))
    return y


def set_pdl(enabled: bool) -> None:
    """Programmatic dependent launch for the weight-streaming kernels."""
    _check(_lib.tl_set_pdl(int(bool(enabled))))


def launch_count() -> int:
    return int(_lib.tl_launch_count())


def device_info() -> tuple[int, int, int]:
    sms, major, minor = _I(), _I(), _I()
    _check(_lib.tl_device_info(ctypes.byref(sms), ctypes.byref(major), ctypes.byref(minor)))
    return sms.value, major.value, minor.value


# TL_LIB selects an experiment build (tiny-llm_b200/csrc/build.py with TL_LIB_SUFFIX); default: the in-tree product library.
load_library(os.environ.get("TL_LIB") or None)
