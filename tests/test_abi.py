"""The C-ABI shared library: it loads on a machine without a GPU, exports every
symbol include/tiny_llm_b200.h declares, and the Python shim refuses CPU
tensors (no CPU fallback).  No kernel is launched here."""

import ctypes
import re
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

ROOT = Path(__file__).resolve().parent.parent
HEADER = (ROOT / "include" / "tiny_llm_b200.h").read_text()


def declared_functions():
    body = re.sub(r"/\*.*?\*/", "", HEADER, flags=re.S)
    return sorted(set(re.findall(r"\b(tl_[a-z0-9_]+)\s*\(", body)))


def test_library_is_in_tree_and_loaded():
    path = ext.current_library_path()
    assert path is not None and path.exists()
    assert ROOT in path.parents, "the extension must be built in-tree (not in a JIT cache)"


def test_every_declared_symbol_is_exported_and_bound():
    lib = ctypes.CDLL(str(ext.current_library_path()))
    names = declared_functions()
    assert len(names) >= 18
    for name in names:
        assert hasattr(lib, name), f"{name} declared in the header but not exported"
    assert set(names) == set(ext.EXPORTED_SYMBOLS), "shim bindings and header disagree"
    assert lib.tl_abi_version() == 1


def test_reference_entry_points_keep_names_and_defaults():
    # src/extensions_ref/bindings.cpp:14-46
    import inspect

    expected = {
        "quantized_matmul": ["scales", "biases", "group_size", "bits", "a", "b", "transpose_b", "use_simdgroup", "use_split_k", "stream"],
        "quantized_embedding": ["indices", "scales", "biases", "weight", "group_size", "bits", "stream"],
        "rms_norm": ["x", "weight", "eps", "stream"],
        "rope": ["x", "offsets", "dims", "base", "traditional", "stream"],
        "swiglu": ["gate", "up", "stream"],
        "decode_attention": ["query", "key", "value", "mask", "scale", "is_causal", "has_mask", "num_heads", "num_kv_heads", "stream"],
        "paged_cache_update": ["pages", "values", "page_id", "start", "stream"],
        "paged_attention": ["query", "key_pages", "value_pages", "block_table", "context_lens", "scale", "is_causal", "num_kv_heads", "num_heads", "stream"],
    }
    for name, params in expected.items():
        sig = inspect.signature(getattr(ext, name))
        assert list(sig.parameters) == params, name
        assert sig.parameters["stream"].default is None
    qm = inspect.signature(ext.quantized_matmul).parameters
    assert (qm["transpose_b"].default, qm["use_simdgroup"].default, qm["use_split_k"].default) == (False, True, False)
    pa = inspect.signature(ext.paged_attention).parameters
    assert (pa["scale"].default, pa["is_causal"].default) == (1.0, False)
    assert inspect.signature(ext.rope).parameters["traditional"].default is False
    assert callable(ext.load_library)


def test_cpu_tensors_are_refused_gpu_only():
    bf = torch.bfloat16
    with pytest.raises(RuntimeError, match="rms_norm: the course extension is GPU-only"):
        ext.rms_norm(torch.zeros(2, 8, dtype=bf), torch.ones(8, dtype=bf), 1e-5)
    with pytest.raises(RuntimeError, match="swiglu: the course extension is GPU-only"):
        ext.swiglu(torch.zeros(4), torch.zeros(4))
    with pytest.raises(RuntimeError, match="quantized_matmul: the course extension is GPU-only"):
        ext.quantized_matmul(torch.zeros(4, 1, dtype=bf), torch.zeros(4, 1, dtype=bf), 128, 4, torch.zeros(1, 128, dtype=bf),
                             torch.zeros(4, 16, dtype=torch.int32), True)
    with pytest.raises(RuntimeError, match="paged_cache_update: the course extension is GPU-only"):
        ext.paged_cache_update(torch.zeros(2, 1, 4, 2), torch.zeros(1, 1, 1, 2), 0, 0)


def test_builder_checks_run_before_the_device_check():
    bf = torch.bfloat16
    with pytest.raises(RuntimeError, match="b must be transposed"):
        ext.quantized_matmul(torch.zeros(4, 1, dtype=bf), torch.zeros(4, 1, dtype=bf), 128, 4, torch.zeros(1, 128, dtype=bf),
                             torch.zeros(4, 16, dtype=torch.int32), False)
    with pytest.raises(RuntimeError, match="dims must be positive, even"):
        ext.rope(torch.zeros(1, 1, 1, 4), torch.zeros(1, dtype=torch.int32), 3, 10000.0)
    with pytest.raises(RuntimeError, match="destination slice is outside page storage"):
        ext.paged_cache_update(torch.zeros(2, 1, 4, 2), torch.zeros(1, 1, 2, 2), 0, 3)
    with pytest.raises(RuntimeError, match="mask must be float32"):
        ext.decode_attention(torch.zeros(1, 1, 4), torch.zeros(1, 1, 4), torch.zeros(1, 1, 4), torch.zeros(1, dtype=bf), 1.0, False, False, 1, 1)


def test_c_abi_reports_argument_errors_without_a_device():
    lib = ctypes.CDLL(str(ext.current_library_path()))
    lib.tl_last_error.restype = ctypes.c_char_p
    lib.tl_rms_norm.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_void_p]
    assert lib.tl_rms_norm(None, None, None, 4, 8, 1e-5, 7, None) == -2  # TL_EDTYPE
    assert b"expected float32, float16, or bfloat16" in lib.tl_last_error()
    assert lib.tl_rms_norm(None, None, None, 4, 8, 1e-5, 2, None) == -1  # TL_EINVAL: null pointers
    assert lib.tl_rms_norm(None, None, None, 0, 8, 1e-5, 2, None) == 0  # empty input is a no-op


def test_gate_up_interleave_layout_and_span_record():
    """Host-side helpers of the CUDA extension: the row layout the SWIGLU_PAIRS epilogue expects,
    and the by-value span record of tl_paged_cache_append_chunk (4 x 64 int32 + count)."""
    import ctypes

    import torch

    from extensions_b200 import tiny_llm_ext_b200 as ext

    gate = torch.arange(32 * 3, dtype=torch.int32).reshape(32, 3)
    up = -gate - 1
    both = ext.interleave_gate_up(gate, up)
    assert both.shape == (64, 3)
    for c in range(4):
        assert torch.equal(both[16 * c : 16 * c + 8], gate[8 * c : 8 * c + 8])
        assert torch.equal(both[16 * c + 8 : 16 * c + 16], up[8 * c : 8 * c + 8])
    try:
        ext.interleave_gate_up(gate[:30], up[:30])
    except RuntimeError as exc:
        assert "rows % 8" in str(exc)
    else:
        raise AssertionError("rows not divisible by 8 must be rejected")
    assert ctypes.sizeof(ext.PageSpanList) == 4 * 64 * 4 + 4
    assert ext.EPI_SWIGLU_PAIRS == 2 and ext.PAGE_SPANS == 64


# ------------------------------------------------------- paged attention routing --
# tl_paged_attention_route answers from sizes and pointer alignment alone, so the selection rules of
# paged_attention_path() (c_abi.cu) are checked here with made-up addresses: nothing is read or launched.
A16, A2 = 0x7F0000010000, 0x7F0000010002  # 16-byte aligned, and 2 bytes past that (a bf16 element offset)
BF, F32 = torch.bfloat16, torch.float32


def route(L=1, D=128, page=64, max_pages=16, Hq=32, Hkv=8, B=1, dtype=BF, q=A16, k=A16, v=A16, out=A16, num_pages=64):
    return ext.paged_attention_route(q, k, v, out, B * Hq, L, D, num_pages, page, max_pages, Hkv, Hq, dtype)


def test_route_rowwise_for_f32_other_head_sizes_and_unaligned_operands():
    assert route(dtype=F32) == ext.PAGED_ROWWISE
    assert route(dtype=F32, L=300) == ext.PAGED_ROWWISE
    for D in (64, 80, 127):
        assert route(D=D) == ext.PAGED_ROWWISE
    for where in ("q", "k", "v"):
        assert route(**{where: A2}) == ext.PAGED_ROWWISE, where
        assert route(L=100, **{where: A2}) == ext.PAGED_ROWWISE, where
    assert route(q=A16 + 8) == ext.PAGED_ROWWISE  # 8-byte alignment is not enough for the 16-byte vector loads


def test_route_decode_key_range_boundary():
    # PAGED_WGMMA_MIN_KEYS = 1024: the block table's capacity, not the context, decides
    assert route(page=64, max_pages=15) == ext.PAGED_GQA
    assert route(page=64, max_pages=16) == ext.PAGED_WGMMA
    assert route(page=128, max_pages=7) == ext.PAGED_GQA
    assert route(page=128, max_pages=8) == ext.PAGED_WGMMA
    assert route(page=1024, max_pages=1) == ext.PAGED_WGMMA
    # pages that are not a multiple of 64 slots never reach the wgmma kernel
    assert route(page=16, max_pages=4096) == ext.PAGED_GQA
    assert route(page=96, max_pages=100) == ext.PAGED_GQA
    assert route(page=192, max_pages=100) == ext.PAGED_WGMMA
    # the wgmma kernel writes out with 16-byte stores
    assert route(page=64, max_pages=16, out=A2) == ext.PAGED_GQA


def test_route_decode_rows_and_one_tile_rule():
    # PAGED_DECODE_ROWS = 8: L <= 8 is a decode step, L = 9 a prefill whatever the key range
    assert route(L=8, page=64, max_pages=1, Hq=8, Hkv=8) == ext.PAGED_GQA
    assert route(L=9, page=64, max_pages=1, Hq=8, Hkv=8) == ext.PAGED_WGMMA
    assert route(L=9, page=16, max_pages=1, Hq=8, Hkv=8) == ext.PAGED_FLASH
    # decode reaches the wgmma kernel only while the G x L query rows of a KV head fit one 128-row tile
    assert route(L=8, Hq=32, Hkv=2) == ext.PAGED_WGMMA  # G = 16: 128 rows
    assert route(L=8, Hq=32, Hkv=1) == ext.PAGED_GQA    # G = 32: 256 rows
    assert route(L=4, Hq=32, Hkv=1) == ext.PAGED_WGMMA  # 128 rows
    assert route(L=5, Hq=32, Hkv=1) == ext.PAGED_GQA    # 160 rows
    assert route(L=1, Hq=128, Hkv=1) == ext.PAGED_WGMMA
    assert route(L=2, Hq=128, Hkv=1) == ext.PAGED_GQA


def test_route_prefill_head_ratio_page_size_and_grid_limit():
    assert route(L=100) == ext.PAGED_WGMMA
    assert route(L=100, page=16) == ext.PAGED_FLASH
    assert route(L=100, page=32) == ext.PAGED_FLASH
    assert route(L=100, Hq=6, Hkv=2) == ext.PAGED_FLASH     # G = 3 does not divide 128
    assert route(L=100, Hq=256, Hkv=1) == ext.PAGED_FLASH   # G = 256 > 128
    assert route(L=100, Hq=128, Hkv=1) == ext.PAGED_WGMMA
    assert route(L=100, out=A2) == ext.PAGED_FLASH
    # the mma.sync kernel puts the B * Hq query rows on grid.y (at most 65535)
    assert route(L=100, page=16, Hq=1, Hkv=1, B=65535) == ext.PAGED_FLASH
    assert route(L=100, page=16, Hq=1, Hkv=1, B=65536) == ext.PAGED_GQA
    assert route(L=100, page=64, Hq=1, Hkv=1, B=65536) == ext.PAGED_WGMMA


def test_route_rejects_what_paged_attention_rejects():
    with pytest.raises(RuntimeError, match="num_heads must be divisible"):
        route(Hq=6, Hkv=4)
    with pytest.raises(RuntimeError, match="float32 or bfloat16"):
        route(dtype=torch.float16)
    with pytest.raises(RuntimeError, match="bfloat16 prefill requires head dimension 128"):
        route(L=9, D=64)
    with pytest.raises(RuntimeError, match=r"range \[1, 128\]"):
        route(D=256, dtype=F32)


# ---------------------------------------------------------------- W4A16 routing --
# tl_quantized_matmul_route runs the selection of the W4A16 launches (w4a16_path(), w4a16_skinny_splits() and the
# streaming kernel's plan) without a device.  Without a GPU the split count assumes 132 SMs (an H100 SXM).
F16 = torch.float16


def w4_route(M, N, K, lda=None, prologue=0, fused=False, simd=True, dtype=BF, a=A16, b=A16, scales=A16, biases=A16):
    return ext.quantized_matmul_route(M, N, K, N if lda is None else lda, prologue, fused, simd, dtype, a, b, scales, biases)


def test_w4_route_row_boundaries():
    for dtype in (BF, F16):
        assert w4_route(8, 2560, 1024, dtype=dtype)[0] == ext.W4_STREAM
        assert w4_route(9, 2560, 1024, dtype=dtype)[0] == ext.W4_SKINNY
        assert w4_route(128, 2560, 1024, dtype=dtype)[0] == ext.W4_SKINNY
        assert w4_route(129, 2560, 1024, dtype=dtype) == (ext.W4_TILES, 1, 20, 0, 0)
        assert w4_route(1, 2560, 1024, dtype=dtype, simd=False) == (ext.W4_VANILLA, 0, 0, 0, 0)
        assert w4_route(300, 2560, 1024, dtype=dtype, simd=False)[0] == ext.W4_VANILLA
    # the fused forms carry their epilogues only on the split-reduction launch: M > 128 stays on the streaming kernel
    assert w4_route(128, 2560, 1024, fused=True)[0] == ext.W4_SKINNY
    assert w4_route(129, 2560, 1024, fused=True) == (ext.W4_STREAM, 0, 0, 32, 1)
    assert w4_route(1000, 2560, 1024, fused=True)[0] == ext.W4_STREAM


def test_w4_route_prologue_or_row_stride_forces_the_streaming_kernel():
    for prologue in (1, 2):
        for M in (9, 64, 128):
            assert w4_route(M, 2560, 1024, prologue=prologue, fused=True)[0] == ext.W4_STREAM
    assert w4_route(64, 2560, 1024, lda=2568, fused=True)[0] == ext.W4_STREAM
    assert w4_route(64, 2560, 1024, lda=2560, fused=True)[0] == ext.W4_SKINNY
    with pytest.raises(RuntimeError, match="needs a fused form"):
        w4_route(1, 2560, 1024, prologue=1)
    with pytest.raises(RuntimeError, match="needs a fused form"):
        w4_route(1, 2560, 1024, lda=2568)


def test_w4_route_rejects_misaligned_operands_of_the_wgmma_kernels():
    for M in (9, 129):
        for where in ("a", "b"):
            with pytest.raises(RuntimeError, match="16-byte aligned"):
                w4_route(M, 2560, 1024, **{where: A2})
    # the streaming kernel reads a and b with 16-byte loads too; scales and biases only need 2 bytes
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        w4_route(1, 2560, 1024, a=A2)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        w4_route(4, 2560, 1024, lda=2564, fused=True)
    assert w4_route(9, 2560, 1024, scales=A2)[0] == ext.W4_SKINNY
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        w4_route(1, 2560, 1024, dtype=torch.float32)


def test_w4_route_streaming_units():
    # two 128-column groups per unit need an even group count, 4-byte aligned scale/bias rows and at most 16 rows
    assert w4_route(1, 2560, 1024)[4] == 2
    assert w4_route(16, 2560, 1024, lda=2568, fused=True)[4] == 2
    assert w4_route(17, 2560, 1024, lda=2568, fused=True)[4] == 1
    for N in (128, 384, 1152):
        assert w4_route(1, N, 100)[4] == 1, N
    assert w4_route(1, 2560, 1024, scales=A2)[4] == 1
    assert w4_route(1, 2560, 1024, biases=A2)[4] == 1


def test_w4_route_streaming_rows_per_pass():
    for M, rpp in ((1, 1), (2, 2), (3, 4), (5, 8), (8, 8)):
        assert w4_route(M, 2560, 1024)[3] == rpp, M
    for M in (32, 33, 200):
        assert w4_route(M, 2560, 2560, lda=2568, fused=True)[3] == 32, M
    # a 9728-wide reduction leaves shared memory for 8 activation rows per pass: 16 rows run in two passes, 17 in three
    for M in (8, 16, 17):
        assert w4_route(M, 9728, 2560, prologue=2, fused=True)[3] == 8, M
    assert w4_route(4, 9728, 2560)[3] == 4


def test_w4_route_skinny_splits():
    # 76 group blocks over 20 feature tiles: 6 splits of 13 on 132 SMs (an odd split length starts every second split
    # in the second half of a two-group TMA box)
    if not torch.cuda.is_available():
        assert w4_route(16, 9728, 2560)[:3] == (ext.W4_SKINNY, 6, 13)
    route, splits, gbps, rpp, units = w4_route(33, 2560, 1000)
    assert route == ext.W4_SKINNY and splits > 1 and (splits - 1) * gbps < 20 <= splits * gbps and (rpp, units) == (0, 0)
    # the split count is a function of (N, K) alone: every row count of one token tile gets the same split
    assert len({w4_route(M, 2560, 9728)[1:3] for M in (9, 16, 17, 64, 65, 128)}) == 1


# ------------------------------------------------------------ element-wise routing --
# tl_rms_norm_route, tl_rope_route and tl_qk_norm_rope_route call the selection functions the launches use
# (rms_norm_path, rope_heads_path, qkv_planes_rope_supported in elementwise.cu).
def test_rms_norm_route_threads_per_row_and_vector_accesses():
    for dtype, epv in ((BF, 8), (F16, 8), (F32, 4)):
        assert ext.rms_norm_route(512, dtype, A16, A16, A16) == (32, True)
        assert ext.rms_norm_route(513, dtype, A16, A16, A16) == (256, False)
        assert ext.rms_norm_route(4096, dtype, A16, A16, A16) == (256, True)
        assert ext.rms_norm_route(16, dtype, A16, A16, A16) == (32, True)
        assert ext.rms_norm_route(4096 + epv, dtype, A16, A16, A16) == (256, True)
        assert ext.rms_norm_route(4096 + epv // 2, dtype, A16, A16, A16) == (256, False)
        for where in range(3):  # a 2-byte offset of x, weight or out takes the scalar path
            ptrs = [A16, A16, A16]
            ptrs[where] = A2
            assert ext.rms_norm_route(2560, dtype, *ptrs) == (256, False)
    assert ext._lib.tl_rms_norm_route(128, 7, A16, A16, A16, None) == -2  # TL_EDTYPE
    assert ext._lib.tl_rms_norm_route(0, 2, A16, A16, A16, None) == -1    # TL_EINVAL


def test_rope_route_per_pair_kernel_needs_heads_tokens_and_full_rotation():
    for dtype in (BF, F16, F32):
        assert ext.rope_route(1, 64, 2, 128, 128, dtype) == ext.ROPE_HEADS
        assert ext.rope_route(8, 8, 32, 128, 128, dtype) == ext.ROPE_HEADS
        assert ext.rope_route(7, 9, 32, 128, 128, dtype) == ext.ROPE_ELEMENT   # B * L = 63
        assert ext.rope_route(8, 8, 1, 128, 128, dtype) == ext.ROPE_ELEMENT    # H = 1
        assert ext.rope_route(8, 8, 4, 128, 64, dtype) == ext.ROPE_ELEMENT     # dims < D: the tail is copied
    with pytest.raises(RuntimeError, match="dims must be positive, even"):
        ext.rope_route(1, 1, 1, 64, 66, BF)


def test_qk_norm_rope_route_row_kernel_up_to_64_bf16_heads_of_128():
    assert ext.qk_norm_rope_route(32, 8, 128, BF) == ext.QKN_ROW
    assert ext.qk_norm_rope_route(48, 8, 128, BF) == ext.QKN_ROW   # 64 heads: every warp holds QKN_MAXH = 4
    assert ext.qk_norm_rope_route(50, 7, 128, BF) == ext.QKN_ROW
    assert ext.qk_norm_rope_route(64, 8, 128, BF) == ext.QKN_HEAD  # 80 heads (Qwen3-32B)
    assert ext.qk_norm_rope_route(49, 8, 128, BF) == ext.QKN_HEAD  # 65 heads
    assert ext.qk_norm_rope_route(32, 8, 128, F32) == ext.QKN_HEAD
    assert ext.qk_norm_rope_route(8, 2, 64, BF) == ext.QKN_HEAD
    assert ext.qk_norm_rope_route(8, 2, 256, BF) == ext.QKN_HEAD
    with pytest.raises(RuntimeError, match="bfloat16 or float32 required"):
        ext.qk_norm_rope_route(8, 2, 128, F16)
    with pytest.raises(RuntimeError, match="bad shape"):
        ext.qk_norm_rope_route(8, 2, 514, BF)


# ------------------------------------------------------------- fused-form input checks --
def _qk_args(B=2, Hq=4, Hkv=2, D=8, dtype=BF, **over):
    """CPU arguments of decode_qk_norm_rope_append / decode_attention_fused that pass every builder check."""
    a = dict(qkv=torch.zeros(B, (Hq + 2 * Hkv) * D, dtype=dtype), q_norm_weight=torch.ones(D, dtype=dtype),
             k_norm_weight=torch.ones(D, dtype=dtype), offsets=torch.zeros(B, dtype=torch.int32),
             block_table=torch.zeros(B, 3, dtype=torch.int32), context_lens=torch.ones(B, dtype=torch.int32),
             key_pages=torch.zeros(4, Hkv, 16, D, dtype=dtype), value_pages=torch.zeros(4, Hkv, 16, D, dtype=dtype))
    a.update(over)
    return a


QK_OPS = ("decode_qk_norm_rope_append", "chunk_qk_norm_rope_append", "decode_attention_fused")
QK_BAD = {  # name: (argument, bad value for head size D and 2 rows, message)
    "k_norm-dtype": ("k_norm_weight", lambda D: torch.ones(D, dtype=F32), r"k_norm_weight must have the dtype of qkv"),
    "q_norm-length": ("q_norm_weight", lambda D: torch.ones(D - 1, dtype=BF), r"q_norm_weight must be contiguous \[head_dim = {D}\]"),
    "k_norm-strided": ("k_norm_weight", lambda D: torch.ones(2 * D, dtype=BF)[::2], r"k_norm_weight must be contiguous \[head_dim = {D}\]"),
    "offsets-dtype": ("offsets", lambda D: torch.zeros(2, dtype=torch.int64), "offsets must be int32"),
    "offsets-short": ("offsets", lambda D: torch.zeros(1, dtype=torch.int32), r"offsets must hold one entry per row \(\[2\]\)"),
    "context_lens-dtype": ("context_lens", lambda D: torch.ones(2, dtype=torch.int64), "context_lens must be int32"),
    "context_lens-rank": ("context_lens", lambda D: torch.ones(2, 1, dtype=torch.int32), r"context_lens must hold one entry per row \(\[2\]\)"),
}
# inputs an older check of the same operator refuses first, with its own message
QK_EARLIER = {
    ("chunk_qk_norm_rope_append", "offsets-short"): "one block-table row, one offset and one context length per token",
    ("decode_attention_fused", "k_norm-dtype"): "dtype mismatch",
    ("decode_attention_fused", "context_lens-dtype"): r"block_table must be int32 \[B, max_pages\] and context_lens int32 \[B\]",
}


def _call_qk(op, **over):
    """One call of op on CPU tensors: D = 8 for the standalone forms, 128 for decode_attention_fused."""
    D = 128 if op == "decode_attention_fused" else 8
    a = _qk_args(D=D, **over)
    if op == "chunk_qk_norm_rope_append" and "block_table" not in over:
        a["block_table"] = a["block_table"][0]
    if op == "decode_attention_fused":
        return ext.decode_attention_fused(a["qkv"], a["q_norm_weight"], a["k_norm_weight"], a["offsets"], a["block_table"], a["context_lens"],
                                          torch.zeros(D // 2, dtype=torch.float64), a["key_pages"], a["value_pages"], 4, 2, 1e-6, 1.0, 16)
    return getattr(ext, op)(*a.values(), 4, 2, 1e6, 1e-6)


@pytest.mark.parametrize("op", QK_OPS)
def test_fused_q_k_norm_forms_accept_good_inputs_up_to_the_device_check(op):
    with pytest.raises(RuntimeError, match=f"^{op}: the course extension is GPU-only$"):
        _call_qk(op)


@pytest.mark.parametrize("op", QK_OPS)
@pytest.mark.parametrize("case", sorted(QK_BAD))
def test_fused_q_k_norm_forms_check_their_inputs_before_the_device(op, case):
    arg, bad, msg = QK_BAD[case]
    D = 128 if op == "decode_attention_fused" else 8
    msg = QK_EARLIER.get((op, case), msg.replace("{D}", str(D)))
    with pytest.raises(RuntimeError, match=f"^{op}: {msg}"):
        _call_qk(op, **{arg: bad(D)})


def test_decode_q_k_norm_checks_the_block_table():
    for bt, msg in ((torch.zeros(2, 3, dtype=torch.int64), "block_table must be int32"),
                    (torch.zeros(3, 3, dtype=torch.int32), r"block_table must be int32 \[2, max_pages\]"),
                    (torch.zeros(6, dtype=torch.int32), r"block_table must be int32 \[2, max_pages\]")):
        with pytest.raises(RuntimeError, match=f"decode_qk_norm_rope_append: {msg}"):
            ext.decode_qk_norm_rope_append(*_qk_args(block_table=bt).values(), 4, 2, 1e6, 1e-6)
    a = _qk_args()
    a["block_table"] = torch.zeros(3, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="chunk_qk_norm_rope_append: block_table_row must be int32"):
        ext.chunk_qk_norm_rope_append(*a.values(), 4, 2, 1e6, 1e-6)


def test_qkv_project_rope_append_checks_its_inputs_before_the_device():
    D, Hq, Hkv, N, rows = 128, 2, 1, 256, 3
    K = (Hq + 2 * Hkv) * D

    def call(chunk=False, **over):
        a = dict(scales=torch.zeros(K, N // 128, dtype=BF), biases=torch.zeros(K, N // 128, dtype=BF), b=torch.zeros(K, N // 8, dtype=torch.int32),
                 p0=torch.zeros(rows, N, dtype=BF), q_norm_weight=torch.ones(D, dtype=BF), k_norm_weight=torch.ones(D, dtype=BF),
                 offsets=torch.zeros(rows, dtype=torch.int32), block_table=torch.zeros(3, dtype=torch.int32) if chunk else torch.zeros(rows, 3, dtype=torch.int32),
                 context_lens=torch.ones(rows, dtype=torch.int32), key_pages=torch.zeros(4, Hkv, 16, D, dtype=BF),
                 value_pages=torch.zeros(4, Hkv, 16, D, dtype=BF))
        a.update(over)
        return ext.qkv_project_rope_append(*a.values(), Hq, Hkv, 1e6, 1e-6, chunk=chunk)

    with pytest.raises(RuntimeError, match="GPU-only"):
        call()
    with pytest.raises(RuntimeError, match="GPU-only"):
        call(chunk=True)
    bad = [
        (dict(q_norm_weight=torch.ones(D, dtype=torch.float32)), "q_norm_weight must have the dtype of qkv"),
        (dict(k_norm_weight=torch.ones(64, dtype=BF)), r"k_norm_weight must be contiguous \[head_dim = 128\]"),
        (dict(offsets=torch.zeros(rows, dtype=torch.int64)), "offsets must be int32"),
        (dict(offsets=torch.zeros(rows - 1, dtype=torch.int32)), "offsets must hold one entry per row"),
        (dict(context_lens=torch.ones(rows + 1, dtype=torch.int32)), "context_lens must hold one entry per row"),
        (dict(block_table=torch.zeros(rows, 3, dtype=torch.int64)), "block_table must be int32"),
        (dict(block_table=torch.zeros(rows + 1, 3, dtype=torch.int32)), r"block_table must be int32 \[3, max_pages\]"),
        (dict(biases=torch.zeros(K, N // 128, dtype=F16)), "contiguous bfloat16 inputs required"),
        (dict(value_pages=torch.zeros(4, Hkv, 16, D, dtype=F32)), "contiguous bfloat16 inputs required"),
    ]
    for over, msg in bad:
        with pytest.raises(RuntimeError, match=f"qkv_project_rope_append: {msg}"):
            call(**over)
    with pytest.raises(RuntimeError, match=r"qkv_project_rope_append: block_table must be int32 \[max_pages\]"):
        call(chunk=True, block_table=torch.zeros(rows, 3, dtype=torch.int32))


def test_qkv_project_rope_append_bounds_the_head_size_like_the_other_q_k_forms():
    """The per-head kernel holds at most 8 warp partials (head_dim <= 512), as tl_decode_qk_norm_rope_append checks."""
    lib = ext._lib

    def call(D):
        return lib.tl_qkv_project_rope_append(*([None] * 13), 1, 128, 1, 1, D, 1e6, 1e-6, 1, 16, 1, 0, 2, None, 0, None)

    assert call(514) == -1 and b"qkv_project_rope_append: bad shape" in lib.tl_last_error()
    assert call(512) == -1 and b"qkv_project_rope_append: null pointer" in lib.tl_last_error()  # the shape is accepted
    assert ext.qk_norm_rope_route(1, 1, 512, BF) == ext.QKN_HEAD
