"""Every norm, RoPE, K/V-append and element-wise kernel, standalone and fused, against a float64 reference
(tests/elementwise_ref.py).

Each case states the kernel it must reach (tl_rms_norm_route, tl_rope_route, tl_qk_norm_rope_route,
tl_quantized_matmul_route, the argmax part count of tl_argmax_workspace, or the documented 16/4/2-byte rule of the
paged append) and asserts it.  Exact probes come first: rows whose inverse norm is exactly 1 at position 0, and
needles whose every other output must be exactly 0.  Then random rows, rows with a large dynamic range, tiny rows where
eps dominates and rows at the dtype's extremes, within the bound, which has no absolute term.  add,
quantized_embedding and argmax are bit-exact on any input; V rows, and K rows on exact probes, land bit for bit; every
page element outside the target slots keeps its bits.  The coverage test at the end requires every cell and prints
the largest error/bound ratio and the largest error in output ulps per cell and dtype."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import ops as oracle


def _load(name, file):
    """A helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


er = _load("tiny_llm_b200_elementwise_ref", "elementwise_ref.py")

pytestmark = pytest.mark.gpu
F64, F32, BF16, F16 = torch.float64, torch.float32, torch.bfloat16, torch.float16
DT = {F32: "f32", F16: "f16", BF16: "bf16"}
STATS = {}     # (cell, dtype) -> [max error / bound, max error in output ulps]
REACHED = {}   # cell -> first case that reached it
RSQRT_EXACT = {}  # dtype -> whether the f32 unit-norm probes were bit-exact (bf16 / f16 must be)
A16 = 0x7F0000010000


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def reach(cell, case):
    REACHED.setdefault(cell, case)


def within(got, b, cell, dtype, what):
    """Asserts the bound and records (error / bound, error in output ulps over outputs >= 1/8 of the largest)."""
    got = got.to(F64).reshape(b.pre.shape)
    ratio = er.assert_within(got, b.pre, b.tol, what)
    big = b.pre.abs() >= b.pre.abs().amax() / 8
    ul = float(torch.where(big, er.ulps(got, b.pre, dtype), torch.zeros_like(got)).max()) if bool(big.any()) else 0.0
    old = STATS.get((cell, DT[dtype]), [0.0, 0.0])
    STATS[(cell, DT[dtype])] = [max(old[0], ratio), max(old[1], ul)]
    zero = b.pre == 0
    er.assert_exact(got[zero], b.pre[zero], f"{what}: outputs that must be exactly 0")


def rows_for(mode, shape, g, dtype, lo_exp=-80):
    """Random rows: gauss, dynamic (2^-e..2^e in one row), tiny (eps dominates), extreme (f16: its largest power of two
    and its smallest subnormal; bf16 / f32: 2^40 and 2^lo_exp, the range over which sums of squares stay finite and
    normalised values normal in fp32)."""
    x = torch.randn(*shape, generator=g, dtype=F64)
    if mode == "dynamic":
        e = 12 if dtype == F16 else 40
        x = x * torch.pow(2.0, torch.randint(-e, e + 1, shape, generator=g).to(F64))
    elif mode == "tiny":
        x = x * 1e-4
    elif mode == "extreme":
        hi, lo = {F16: (2.0**15, 2.0**-24), BF16: (2.0**40, 2.0**lo_exp), F32: (2.0**40, 2.0**lo_exp)}[dtype]
        pick = torch.randint(0, 3, shape, generator=g)
        x = torch.where(pick == 0, x.sign() * hi, torch.where(pick == 1, x.sign() * lo, x))
    return x.to(dtype)


def aligned_view(t, off_elems, dev):
    """A contiguous copy of t that starts off_elems elements past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 16, dtype=t.dtype, device=dev)
    v = buf[off_elems : off_elems + t.numel()].view(t.shape)
    v.copy_(t)
    return v


# ------------------------------------------------------------------- rms_norm --
RMS_DIMS = [16, 128, 129, 256, 260, 512, 513, 1000, 2048, 2056, 2560, 4096, 4104, 8192]


@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("dim", RMS_DIMS)
def test_rms_norm(dev, dtype, dim):
    """The vector path keeps KEEP = 2 16-byte chunks per thread in registers between its two passes, so dim <= 2 * TPR *
    16 bytes reads x once and larger rows read it again: the boundary is bf16 / f16 4096 / 4104 and f32 2048 / 2056 at
    TPR 256, f32 256 / 260 at TPR 32 (bf16 / f16 reach it at 512, the last dim before TPR switches from 32 to 256
    between 512 and 513).  Dims that are no multiple of 16 bytes (129; 260 in bf16 / f16) and 2-byte offset views take
    the scalar path."""
    g = torch.Generator().manual_seed(dim + 7 * len(DT[dtype]))
    epv = 16 // torch.tensor([], dtype=dtype).element_size()
    offs = [0, 1] if dim % epv == 0 else [0]
    for off in offs:
        w = aligned_view((1 + 0.2 * torch.randn(dim, generator=g)).to(dtype), 0, dev)
        for mode in ("unit", "gauss", "dynamic", "tiny", "extreme"):
            for eps in ((0.0,) if mode == "unit" else (1e-6, 1e-5)):
                if mode == "unit":
                    x = er.unit_norm_rows(3, 1, dim, g).view(3, dim).to(dtype)
                    wu = aligned_view(er.pow2_norm_weight(dim, 0).to(dtype), 0, dev)
                else:
                    x, wu = rows_for(mode, (5, dim), g, dtype), w
                xd = aligned_view(x, off, dev)
                tpr, vec = ext.rms_norm_route(dim, dtype, xd, wu, A16)
                assert vec == (dim % epv == 0 and off == 0)
                assert tpr == (32 if dim <= 512 else 256)
                cell = f"rms_norm TPR{tpr} {'vec' if vec else 'scalar'}"
                got = ext.rms_norm(xd, wu, eps)
                b = er.rms_norm_ref(xd, wu, eps, dtype)
                what = f"rms_norm {DT[dtype]} dim {dim} +{off} {mode} eps {eps}"
                if mode == "unit":
                    exact = bool((got.to(F64) == b.out).all())
                    if dtype == F32:  # rsqrtf(1) may be off by its 2 ulp: f32 outputs show it, 16-bit ones round it away
                        RSQRT_EXACT["rms_norm"] = RSQRT_EXACT.get("rms_norm", True) and exact
                        within(got, b, cell, dtype, what)
                    else:
                        er.assert_exact(got, b.out, what)
                else:
                    within(got, b, cell, dtype, what)
                reach(cell, what)
        if dtype != F16:  # a sum of squares that overflows fp32: inv = 0, as the fp32 oracle has it
            x = torch.full((2, dim), 2.0**100).to(dtype)
            got = ext.rms_norm(aligned_view(x, off, dev), w, 1e-6).cpu()
            want = oracle.rms_norm(x, w.cpu(), 1e-6)
            assert torch.equal(got, want) and bool((got == 0).all())
            reach("rms_norm fp32 overflow", f"{DT[dtype]} {dim}")


# ----------------------------------------------------------------------- rope --
ROPE_CASES = [  # (name, B, L, H, D, dims, traditional, base)
    ("d128", 7, 9, 4, 128, 128, False, 1e6),
    ("d128-bl64", 8, 8, 4, 128, 128, False, 1e6),
    ("d64-trad", 8, 8, 3, 64, 64, True, 1e4),
    ("d64-trad-bl63", 7, 9, 3, 64, 64, True, 1e4),
    ("d16", 1, 64, 2, 16, 16, False, 1e4),
    ("dims<D", 8, 8, 4, 128, 64, False, 1e4),
    ("dims<D-trad", 7, 9, 2, 64, 32, True, 1e6),
    ("h1-bl64", 8, 8, 1, 128, 128, False, 1e6),
]
POSITIONS = [0, 1, 4095, 32767, 40959, 131071 - 8]


@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("c", ROPE_CASES, ids=[c[0] for c in ROPE_CASES])
def test_rope(dev, dtype, c):
    """Positions 0, 1, 4095 / 4096 (the first two of a row starting at 4095), 32767, 40959, 131071 and, in f32,
    1,000,000: the f32 cases past 4096 are the ones an fp32-formed frequency fails."""
    name, B, L, H, D, dims, trad, base = c
    g = torch.Generator().manual_seed(len(name) * 31 + D)
    route = ext.rope_route(B, L, H, D, dims, dtype)
    heads = dims == D and H > 1 and B * L >= 64
    assert route == (ext.ROPE_HEADS if heads else ext.ROPE_ELEMENT)
    cell = "rope heads" if heads else "rope element"
    pos = (POSITIONS + ([1000000] if dtype == F32 else [65536]) + [12345, 7])[:B]
    offsets = torch.tensor(pos, dtype=torch.int32, device=dev)
    for mode in ("needle", "gauss", "dynamic", "extreme"):
        if mode == "needle":  # one entry per (token, head) row, walking the elements: every other output must be 0
            r = torch.arange(B * L * H)
            x = torch.zeros(B * L * H, D)
            x[r, r % D] = torch.where(r % 2 == 0, 1.0, -1.0)
            x = x.view(B, L, H, D).to(dtype).to(dev)
        else:
            x = rows_for(mode, (B, L, H, D), g, dtype).to(dev)
        got = ext.rope(x, offsets, dims, base, trad)
        b = er.rope_ref(x, offsets, dims, base, trad, dtype)
        what = f"rope {name} {DT[dtype]} {mode}"
        er.assert_exact(got[0, 0], b.out[0, 0], f"{what}: position 0")  # sincosf(0) = (0, 1)
        within(got, b, cell, dtype, what)
        reach(cell, what)


# --------------------------------------------------------- q/k norm + RoPE + append --
def batch(R, H, D, g, dev, chunk, probe):
    """Rows, pages and slots of one call: offsets differ from ctx - 1 everywhere; an idle row, a row whose token is past
    the block table, and rows whose page id is -1 or >= num_pages (decode: whole table rows; chunk: table entries)."""
    page, maxp = 16, 8
    P = R // 4 + 8
    if chunk:
        start = 5
        ctx = torch.arange(start + 1, start + R + 1, dtype=torch.int32)
        ctx[min(3, R - 1)] = 0  # a padding row
        bt = P - 1 - torch.arange(maxp, dtype=torch.int32)
        bt[1], bt[2] = -1, P  # tokens 16..47 are dropped
        if R > 6:
            ctx[-1] = page * maxp + 9  # past the table
    else:
        ctx = torch.zeros(R, dtype=torch.int32)
        bt = torch.full((R, maxp), -1, dtype=torch.int32)
        for b in range(R):
            lp = int(torch.randint(0, maxp, (1,), generator=g))
            bt[b, lp] = b % P
            ctx[b] = lp * page + (b // P) % page + 1
        if R > 4:
            ctx[1] = 0                  # idle
            ctx[2] = page * maxp + 3    # past the table
            bt[3] = -1
            bt[4] = P
    offsets = torch.zeros(R, dtype=torch.int32) if probe == "unit" else (ctx - 1).clamp(min=0) + 3000 + torch.arange(R, dtype=torch.int32)
    return offsets.to(dev), ctx.to(dev), bt.to(dev), page, P


def qk_inputs(R, Hq, Hkv, D, g, probe, dtype):
    H = Hq + 2 * Hkv
    if probe == "unit":
        x = er.unit_norm_rows(R, H, D, g)
    elif probe == "needle":
        x, _ = er.needle_rows(R, H, D)
    else:  # the normalised value of a 2^-60 entry next to 2^40 ones is 2^-100: its rotated products stay normal in fp32
        x = rows_for(probe, (R, H, D), g, dtype, lo_exp=-60).to(F64)
    if probe in ("unit", "needle"):
        qw, kw = er.pow2_norm_weight(D, 0), er.pow2_norm_weight(D, 1)
    else:
        qw, kw = 1 + 0.2 * torch.randn(D, generator=g), 1 + 0.2 * torch.randn(D, generator=g)
    return x.reshape(R, H * D).to(dtype), qw.to(dtype), kw.to(dtype)


def check_fused(ref, q, before_k, before_v, kp, vp, slots, cell, dtype, what, exact):
    if exact:
        er.assert_exact(q, ref.q.out, f"{what} q")
        er.check_pages(before_k, kp, slots, ref.k.out, f"{what} K")
    else:
        within(q, ref.q, cell, dtype, f"{what} q")
        er.check_pages(before_k, kp, slots, None, f"{what} K", tol=ref.k.tol, pre=ref.k.pre)
        if slots:
            b_idx = [b for b, _, _ in slots]
            k_rows = torch.stack([kp[pid, :, t] for _, pid, t in slots])
            within(k_rows, er.Bound(ref.k.out[b_idx], ref.k.pre[b_idx], ref.k.tol[b_idx]), cell, dtype, f"{what} K")
    er.check_pages(before_v, vp, slots, ref.v, f"{what} V")


QK_CASES = [  # (name, form, dtype, Hq, Hkv, D, rows, route)
    ("row-48", "decode", BF16, 32, 8, 128, 12, "row"),
    ("row-64", "decode", BF16, 48, 8, 128, 12, "row"),
    ("row-48-chunk", "chunk", BF16, 32, 8, 128, 40, "row"),
    ("row-64-chunk", "chunk", BF16, 48, 8, 128, 40, "row"),
    ("head-f32", "decode", F32, 8, 2, 128, 12, "head"),
    ("head-f32-chunk", "chunk", F32, 8, 2, 128, 40, "head"),
    ("head-d64", "decode", BF16, 8, 2, 64, 12, "head"),
    ("head-d64-chunk", "chunk", BF16, 8, 2, 64, 40, "head"),
    ("head-80", "decode", BF16, 64, 8, 128, 12, "head"),
    ("head-80-chunk", "chunk", BF16, 64, 8, 128, 40, "head"),
]


def sentinel(P, Hkv, page, D, dtype, dev):
    return (((torch.arange(P * Hkv * page * D) % 2039) - 1019) / 64.0).view(P, Hkv, page, D).to(dtype).to(dev)


@pytest.mark.parametrize("c", QK_CASES, ids=[c[0] for c in QK_CASES])
def test_qk_norm_rope_append(dev, c):
    name, form, dtype, Hq, Hkv, D, R0, route = c
    chunk = form == "chunk"
    assert ext.qk_norm_rope_route(Hq, Hkv, D, dtype) == (ext.QKN_ROW if route == "row" else ext.QKN_HEAD)
    cell = f"qk {route} {form}"
    g = torch.Generator().manual_seed(len(name) * 13 + R0)
    fn = ext.chunk_qk_norm_rope_append if chunk else ext.decode_qk_norm_rope_append
    for probe in ("unit", "needle", "gauss", "dynamic", "tiny", "extreme"):
        R = D if probe == "needle" else R0
        eps = 0.0 if probe == "unit" else (1e-5 if probe == "tiny" else 1e-6)
        offsets, ctx, bt, page, P = batch(R, Hq + 2 * Hkv, D, g, dev, chunk, probe)
        qkv, qw, kw = (t.to(dev) for t in qk_inputs(R, Hq, Hkv, D, g, probe, dtype))
        kp, vp = sentinel(P, Hkv, page, D, dtype, dev), sentinel(P, Hkv, page, D, dtype, dev) * -1
        k0, v0 = kp.clone(), vp.clone()
        q = fn(qkv, qw, kw, offsets, bt, ctx, kp, vp, Hq, Hkv, 1e6, eps)
        if chunk:
            q = q.transpose(0, 1)
        ref = er.qk_norm_rope_ref(qkv, qw, kw, offsets, Hq, Hkv, 1e6, eps)
        slots = er.append_slots(ctx, bt, page, P, chunk=chunk)
        assert len(slots) >= R - 4 if not chunk else len(slots) >= 3
        what = f"{name} {probe}"
        exact = probe == "unit" and dtype != F32
        check_fused(ref, q, k0, v0, kp, vp, slots, cell, dtype, what, exact)
        if probe == "unit" and dtype == F32:
            RSQRT_EXACT["qk " + route] = RSQRT_EXACT.get("qk " + route, True) and bool((q.to(F64) == ref.q.out).all())
        reach(cell, what)
    if Hq + 2 * Hkv == 64 and route == "row":
        reach("qk row 64 heads " + form, name)


# ------------------------------------------------------- q|k|v projection + append --
PLANES = [  # (name, rows, chunk, Hq, Hkv, planes expected)
    ("planes-decode-16", 16, False, 16, 8, True),
    ("planes-decode-64", 64, False, 16, 8, True),
    ("planes-chunk-40", 40, True, 16, 4, True),
    ("planes-chunk-128", 128, True, 16, 4, True),
    ("fallback-decode-4", 4, False, 16, 8, False),
    ("fallback-chunk-8", 8, True, 16, 4, False),
]


@pytest.mark.parametrize("c", PLANES, ids=[c[0] for c in PLANES])
def test_qkv_project_rope_append(dev, c):
    """The reference is applied to the q|k|v that quantized_matmul_fused returns for the same rows: the planes kernel
    adds the split-reduction planes in the order that launch does and rounds once."""
    name, R, chunk, Hq, Hkv, planes = c
    D, N = 128, 2560
    K = (Hq + 2 * Hkv) * D
    route, splits, *_ = ext.quantized_matmul_route(R, N, K, N, 0, True, True, BF16, A16, A16, A16, A16)
    assert (route == ext.W4_SKINNY and splits > 1) == planes, (route, splits)
    assert ext.qk_norm_rope_route(Hq, Hkv, D, BF16) == ext.QKN_ROW
    cell = f"qkv {'planes' if planes else 'fallback'} {'chunk' if chunk else 'decode'}"
    g = torch.Generator().manual_seed(R + 3 * chunk)
    sigma = 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32).to(dev)
    scales = (torch.randn(K, N // 128, generator=g) * sigma).to(BF16)
    biases = (-7.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma).to(BF16).to(dev)
    scales = scales.to(dev)
    for mode in ("gauss", "dynamic"):
        p0 = (torch.randn(R, N, generator=g) * (1.0 if mode == "gauss" else 30.0)).to(BF16).to(dev)
        qw = (1 + 0.2 * torch.randn(D, generator=g)).to(BF16).to(dev)
        kw = (1 + 0.2 * torch.randn(D, generator=g)).to(BF16).to(dev)
        offsets, ctx, bt, page, P = batch(R, Hq + 2 * Hkv, D, g, dev, chunk, mode)
        kp, vp = sentinel(P, Hkv, page, D, BF16, dev), -sentinel(P, Hkv, page, D, BF16, dev)
        k0, v0 = kp.clone(), vp.clone()
        q = ext.qkv_project_rope_append(scales, biases, words, p0, qw, kw, offsets, bt, ctx, kp, vp, Hq, Hkv, 1e6, 1e-6, chunk=chunk)
        if chunk:
            q = q.transpose(0, 1)
        qkv = ext.quantized_matmul_fused(scales, biases, words, p0)
        ref = er.qk_norm_rope_ref(qkv, qw, kw, offsets, Hq, Hkv, 1e6, 1e-6)
        slots = er.append_slots(ctx, bt, page, P, chunk=chunk)
        check_fused(ref, q, k0, v0, kp, vp, slots, cell, BF16, f"{name} {mode}", False)
        reach(cell, name)


def test_qkv_project_rope_append_refuses_strided_operands(dev):
    """A strided view would be read or written as if it were row-major; the check follows the device check."""
    D, Hq, Hkv, N, R = 128, 2, 1, 256, 3
    K = (Hq + 2 * Hkv) * D
    args = dict(scales=torch.zeros(K, N // 128, dtype=BF16), biases=torch.zeros(K, N // 128, dtype=BF16), b=torch.zeros(K, N // 8, dtype=torch.int32),
                p0=torch.zeros(R, N, dtype=BF16), q_norm_weight=torch.ones(D, dtype=BF16), k_norm_weight=torch.ones(D, dtype=BF16),
                offsets=torch.zeros(R, dtype=torch.int32), block_table=torch.zeros(R, 3, dtype=torch.int32),
                context_lens=torch.ones(R, dtype=torch.int32), key_pages=torch.zeros(4, Hkv, 16, D, dtype=BF16),
                value_pages=torch.zeros(4, Hkv, 16, D, dtype=BF16))
    args = {k: v.to(dev) for k, v in args.items()}
    strided = dict(key_pages=torch.zeros(4, Hkv, 32, D, dtype=BF16, device=dev)[:, :, ::2], value_pages=torch.zeros(4, Hkv, 16, 2 * D, dtype=BF16, device=dev)[..., :D],
                   b=torch.zeros(K, N // 4, dtype=torch.int32, device=dev)[:, ::2], scales=torch.zeros(K, N // 64, dtype=BF16, device=dev)[:, ::2])
    for name, t in strided.items():
        assert tuple(t.shape) == tuple(args[name].shape) and not t.is_contiguous()
        with pytest.raises(RuntimeError, match=f"qkv_project_rope_append: {name} must be contiguous"):
            ext.qkv_project_rope_append(*{**args, name: t}.values(), Hq, Hkv, 1e6, 1e-6)


def test_decode_attention_fused_appends_the_reference_rows(dev):
    """The K/V rows decode_attention_fused appends (its attention output is tests/test_gpu_attention_numerics.py's)."""
    Hq, Hkv, D, R = 16, 4, 128, 10
    g = torch.Generator().manual_seed(11)
    freq = ext.rope_inv_freq_table(D, 1e6, dev)
    for probe in ("unit", "gauss", "tiny"):
        eps = 0.0 if probe == "unit" else 1e-6
        offsets, ctx, bt, page, P = batch(R, Hq + 2 * Hkv, D, g, dev, False, probe)
        # row 2's context runs past its table: this kernel clamps it to the table (as the attention's key range is) and
        # appends the row at the table's last slot, where the standalone q/k forms skip the row
        maxp = bt.shape[1]
        assert int(ctx[2]) > maxp * page
        bt[2, maxp - 1] = 2
        qkv, qw, kw = (t.to(dev) for t in qk_inputs(R, Hq, Hkv, D, g, probe, BF16))
        kp, vp = sentinel(P, Hkv, page, D, BF16, dev), -sentinel(P, Hkv, page, D, BF16, dev)
        k0, v0 = kp.clone(), vp.clone()
        ext.decode_attention_fused(qkv, qw, kw, offsets, bt, ctx, freq, kp, vp, Hq, Hkv, eps, D**-0.5, int(ctx.max()))
        torch.cuda.synchronize()
        ref = er.qk_norm_rope_ref(qkv, qw, kw, offsets, Hq, Hkv, 1e6, eps, inv_freq=freq)
        slots = er.append_slots(ctx.clamp(max=maxp * page), bt, page, P)
        assert (2, 2, page - 1) in slots
        what = f"decode_attention_fused {probe}"
        if probe == "unit":
            er.check_pages(k0, kp, slots, ref.k.out, f"{what} K")
        else:
            er.check_pages(k0, kp, slots, None, f"{what} K", tol=ref.k.tol, pre=ref.k.pre)
        er.check_pages(v0, vp, slots, ref.v, f"{what} V")
        reach("qk decode_attention_fused", what)


# ------------------------------------------------------------- swiglu / add --
@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
def test_swiglu_and_add(dev, dtype):
    g = torch.Generator().manual_seed(len(DT[dtype]))
    epv = 16 // torch.tensor([], dtype=dtype).element_size()
    for n, off in ((4096 * 3, 0), (4097, 0), (4096, 1)):
        vec = n % epv == 0 and off == 0
        cell = "vec" if vec else "scalar"
        gate = aligned_view((torch.rand(n, generator=g) * 200 - 100).to(dtype), off, dev)
        up = aligned_view(torch.randn(n, generator=g).to(dtype), off, dev)
        within(ext.swiglu(gate, up), er.swiglu_ref(gate, up, dtype), f"swiglu {cell}", dtype, f"swiglu {DT[dtype]} {n} +{off}")
        e = 6 if dtype == F16 else 40  # exponent gaps beyond fp32's 24 bits: T(fp32(a + b)) rounds twice
        a = aligned_view((torch.randn(n, generator=g) * torch.pow(2.0, torch.randint(-e, e, (n,), generator=g))).to(dtype), off, dev)
        b = aligned_view(torch.randn(n, generator=g).to(dtype), off, dev)
        er.assert_exact(ext.add(a, b), er.add_ref(a, b, dtype), f"add {DT[dtype]} {n} +{off}")
        reach(f"swiglu {cell}", DT[dtype])
        reach(f"add {cell}", DT[dtype])


# -------------------------------------------------------- quantized_embedding --
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("dim", [128, 2560])
def test_quantized_embedding(dev, dtype, dim):
    vocab = 1000
    g = torch.Generator().manual_seed(dim)
    weight = torch.randint(-(2**31), 2**31, (vocab, dim // 8), dtype=torch.int64, generator=g).to(torch.int32).to(dev)
    scales = (torch.randn(vocab, dim // 128, generator=g) * 0.02).to(dtype)
    biases = (-7.5 * scales.float() + torch.randn(vocab, dim // 128, generator=g) * 0.01).to(dtype).to(dev)
    scales = scales.to(dev)
    ids = torch.tensor([0, vocab - 1, -1, -(2**31), vocab, vocab + 7, 2**31 - 1, *torch.randint(0, vocab, (9,), generator=g).tolist()],
                       dtype=torch.int32, device=dev)
    got = ext.quantized_embedding(ids, scales, biases, weight, 128, 4)
    want = er.embedding_ref(ids, scales, biases, weight, dtype)
    er.assert_exact(got, want, f"quantized_embedding {DT[dtype]} {dim}")
    assert bool((got[2:7] == 0).all())
    reach("quantized_embedding", DT[dtype])


# ---------------------------------------------------------------------- argmax --
@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("vocab", [1, 4096, 4097, 151936, 262144, 262145])
def test_argmax(dev, dtype, vocab):
    """Ties inside a part and across parts, maxima at the first and last index, all -inf rows.  NaN rows: the kernel
    never picks a NaN and an all-NaN row gives 0 (the fp32 oracle follows torch.argmax, which picks it: unpinned)."""
    g = torch.Generator().manual_seed(vocab)
    parts = ext._lib.tl_argmax_workspace(1, vocab) // 8
    assert parts == (1 if vocab <= 4096 else min(-(-vocab // 4096), 64))
    chunk = -(-(-(-vocab // parts)) // 8) * 8
    x = torch.randn(10, vocab, generator=g).to(dtype).to(F64)
    top = float(x.amax()) + 1
    x[0, 0] = top                                  # first index
    x[1, -1] = top                                 # last index
    if vocab > 8:
        x[2, 3], x[2, 5] = top, top                # a tie inside a part
    if parts > 1:
        x[3, chunk - 1], x[3, chunk], x[3, vocab - 1] = top, top, top  # a tie across parts
    x[4] = float("-inf")                           # all -inf
    x[5] = float("nan")                            # all NaN
    x[6, ::3] = float("nan")                       # NaN among numbers
    x[6, -1] = float("nan")
    x[7, :] = float("-inf")
    x[7, vocab // 2] = float("nan")
    x = x.to(dtype)
    want = er.argmax_ref(x)
    assert want[5] == 0 and want[7] == 0
    for off in (0, 1):
        xd = aligned_view(x, off, dev)
        vec = dtype != F32 and vocab % 8 == 0 and off == 0
        got = ext.argmax(xd)
        assert torch.equal(got.cpu().long(), want), f"argmax {DT[dtype]} {vocab} +{off}: {got.tolist()} != {want.tolist()}"
        reach(f"argmax {'vec' if vec else 'scalar'} parts {'1' if parts == 1 else ('64' if parts == 64 else '>1')}", f"{DT[dtype]} {vocab}")
        reach(f"argmax {DT[dtype]}", str(vocab))


# ---------------------------------------------------------- paged append decode --
@pytest.mark.parametrize("dtype", [BF16, F32], ids=["bf16", "f32"])
@pytest.mark.parametrize("D,off", [(128, 0), (128, 1), (6, 0), (12, 0)])
def test_paged_cache_append_decode(dev, dtype, D, off):
    """16-byte vectors when D * element size is a multiple of 16 and every buffer is 16-byte aligned; otherwise 4-byte
    (f32) or 2-byte (bf16) elements."""
    es = torch.tensor([], dtype=dtype).element_size()
    path = "16-byte" if (D * es) % 16 == 0 and off == 0 else f"{es}-byte"
    g = torch.Generator().manual_seed(D + off)
    R, Hkv = 12, 3
    offsets, ctx, bt, page, P = batch(R, Hkv, D, g, dev, False, "gauss")
    keys = aligned_view(torch.randn(R, Hkv, 1, D, generator=g).to(dtype), off, dev)
    vals = aligned_view(torch.randn(R, Hkv, 1, D, generator=g).to(dtype), off, dev)
    kp = aligned_view(sentinel(P, Hkv, page, D, dtype, "cpu"), off, dev)
    vp = aligned_view(-sentinel(P, Hkv, page, D, dtype, "cpu"), off, dev)
    k0, v0 = kp.clone(), vp.clone()
    ext.paged_cache_append_decode(kp, vp, keys, vals, bt, ctx)
    torch.cuda.synchronize()
    slots = er.append_slots(ctx, bt, page, P)
    assert len(slots) == R - 4
    er.check_pages(k0, kp, slots, keys[:, :, 0], f"append {DT[dtype]} D {D} +{off} K")
    er.check_pages(v0, vp, slots, vals[:, :, 0], f"append {DT[dtype]} D {D} +{off} V")
    reach(f"append {path} {DT[dtype]}", f"D {D} +{off}")


# ------------------------------------------------------------------- coverage --
REQUIRED = {
    *(f"rms_norm TPR{t} {v}" for t in (32, 256) for v in ("vec", "scalar")), "rms_norm fp32 overflow",
    "rope element", "rope heads",
    "qk row decode", "qk row chunk", "qk head decode", "qk head chunk", "qk row 64 heads decode", "qk row 64 heads chunk",
    "qkv planes decode", "qkv planes chunk", "qkv fallback decode", "qkv fallback chunk", "qk decode_attention_fused",
    "swiglu vec", "swiglu scalar", "add vec", "add scalar", "quantized_embedding",
    "argmax vec parts 1", "argmax vec parts >1", "argmax vec parts 64", "argmax scalar parts 1", "argmax scalar parts >1",
    "argmax scalar parts 64", "argmax bf16", "argmax f16", "argmax f32",
    "append 16-byte bf16", "append 16-byte f32", "append 2-byte bf16", "append 4-byte f32",
}


def test_the_cases_reach_every_elementwise_cell(dev, capsys):
    """Each case asserts its route when it runs; this requires that together they reached every cell, and prints the
    error statistics they collected."""
    with capsys.disabled():
        print("\nelement-wise coverage:")
        for cell in sorted(REACHED):
            print(f"  {cell:32s} <- {REACHED[cell]}")
        print("element-wise errors (cell, dtype: max error/bound, max error in output ulps over outputs >= 1/8 of the largest):")
        for key in sorted(STATS):
            print(f"  {key[0]:28s} {key[1]:5s} {STATS[key][0]:7.4f} {STATS[key][1]:7.3f}")
        print(f"f32 unit-norm probes bit-exact (rsqrtf(1) == 1): {RSQRT_EXACT}")
    assert REQUIRED <= set(REACHED), sorted(REQUIRED - set(REACHED))
