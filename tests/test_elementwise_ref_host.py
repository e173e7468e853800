"""The float64 element-wise reference (tests/elementwise_ref.py), its error bounds and its probes, on the CPU.

fp32 emulations of rms_norm, rope and the two q/k norm + RoPE + K/V append kernels (row kernel: two pairs per lane and
two warp sums; per-head kernel: one pair per thread and a sum over the warp partials), in the kernels' order of
operations, must stay within the bounds on random and extreme inputs and be exact on the probes.  The same emulations
with one defect each (swapped pair layout, flipped sine, one norm weight for both halves, the angle taken from ctx - 1,
an fp32-formed frequency, eps outside the square root, K written to the neighbouring KV head or to slot tok - 1) must
fail the checks."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch


def _load(name, file):
    """A helper next to this file, by path: `tests` is no package of this project."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


er = _load("tiny_llm_b200_elementwise_ref", "elementwise_ref.py")
F64, F32, BF16, F16 = torch.float64, torch.float32, torch.bfloat16, torch.float16
f4 = np.float32


# ----------------------------------------------------------------- emulations --
def T(x, dtype):
    """fp32 numpy values stored as T, back as fp32 numpy."""
    return torch.from_numpy(np.asarray(x, dtype=f4)).to(dtype).float().numpy()


def warp_sum(v):
    """__shfl_xor butterfly over the last axis (32 lanes)."""
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = (v + v[..., lanes ^ o]).astype(f4)
    return v[..., 0]


def rsqrtf(m):
    with np.errstate(divide="ignore"):  # rsqrtf(0) = inf
        return (1.0 / np.sqrt(m.astype(np.float64))).astype(f4)


def inv_freq(half, base, fp32=False):
    e = -np.arange(half, dtype=np.float64) / half * np.log2(np.float64(er.f32(base)))
    return np.exp2(e.astype(f4)).astype(np.float64) if fp32 else np.exp2(e)


def sincos(pos, half, base, fp32_freq=False):
    angle = (np.asarray(pos, dtype=np.float64)[..., None] * inv_freq(half, base, fp32_freq)).astype(f4)
    a = angle.astype(np.float64)
    return np.sin(a).astype(f4), np.cos(a).astype(f4)


def emulate_rms_norm(x, w, eps, dtype, defect=None):
    """rms_norm_kernel<T, TPR, VEC>: per-thread sums over the thread's 16-byte chunks (or elements), a warp sum, for
    TPR 256 a second sum over the 8 warp partials; then x * inv * w."""
    x, w = x.float().numpy(), w.float().numpy()
    rows, dim = x.shape
    tpr, epv = (32 if dim <= 512 else 256), 16 // torch.tensor([], dtype=dtype).element_size()
    vec = dim % epv == 0
    idx = [[i + j for i in range(lane * epv, dim, tpr * epv) for j in range(epv)] if vec else list(range(lane, dim, tpr))
           for lane in range(tpr)]
    ss = np.zeros((rows, tpr), dtype=f4)
    for k in range(max(len(i) for i in idx)):
        col = np.array([i[k] if k < len(i) else -1 for i in idx])
        v = np.where(col >= 0, x[:, np.maximum(col, 0)], 0).astype(f4)
        ss = (ss + (v * v).astype(f4)).astype(f4)
    part = warp_sum(ss.reshape(rows, tpr // 32, 32))
    tot = warp_sum(np.pad(part, ((0, 0), (0, 32 - tpr // 32)))) if tpr > 32 else part[:, 0]
    m = (tot / f4(dim)).astype(f4)
    inv = (rsqrtf(m) + f4(er.f32(eps))).astype(f4) if defect == "eps-outside" else rsqrtf((m + f4(er.f32(eps))).astype(f4))
    return T((x * inv[:, None]).astype(f4) * w, dtype)


def emulate_rope(x, offsets, dims, base, traditional, dtype, defect=None):
    """rope_kernel: angle = fp32(pos * inv_freq) with inv_freq in double, fp32 products."""
    x = x.float().numpy().copy()
    B, L, H, D = x.shape
    half = dims // 2
    pos = offsets.numpy()[:, None] + np.arange(L)
    s, c = sincos(pos, half, base, defect == "f32-freq")
    s, c = s[:, :, None, :], c[:, :, None, :]
    if defect == "sin-sign":
        s = -s
    lay = (not traditional) if defect == "layout" else traditional
    i = np.arange(half)
    ri, ii = (2 * i, 2 * i + 1) if lay else (i, i + half)
    re, im = x[..., ri], x[..., ii]
    x[..., ri] = (re * c).astype(f4) - (im * s).astype(f4)
    x[..., ii] = (im * c).astype(f4) + (re * s).astype(f4)
    return T(x, dtype)


def emulate_qk(qkv, qw, kw, offsets, cl, bt, pages_k, pages_v, Hq, Hkv, base, eps, kernel, chunk=False, defect=None):
    """The fused q/k norm + RoPE + append.  kernel "row": lane l owns pairs (l, l + 64) and (l + 32, l + 96), the sum
    of squares is warp_sum(pairs 0..31) + warp_sum(pairs 32..63); "head": thread i owns pair i, the warp partials are
    summed by a second warp sum.  Writes into pages_k / pages_v (numpy, fp32 values of T) and returns q [R, Hq, D]."""
    dtype = qkv.dtype
    R = qkv.shape[0]
    H = Hq + 2 * Hkv
    D = qkv.shape[1] // H
    half = D // 2
    x = qkv.float().numpy().reshape(R, H, D)
    pos = (cl.numpy() - 1) if defect == "angle-ctx" else offsets.numpy()
    s, c = sincos(pos, half, base, defect == "f32-freq")
    s, c = s[:, None, :], c[:, None, :]
    if defect == "sin-sign":
        s = -s
    i = np.arange(half)
    ri, ii = (2 * i, 2 * i + 1) if defect == "layout" else (i, i + half)
    re, im = x[:, : Hq + Hkv][..., ri], x[:, : Hq + Hkv][..., ii]
    sq = ((re * re).astype(f4) + (im * im).astype(f4)).astype(f4)  # [R, Hq + Hkv, half]
    nw = -(-half // 32)
    part = warp_sum(np.pad(sq, ((0, 0), (0, 0), (0, 32 * nw - half))).reshape(R, Hq + Hkv, nw, 32))
    if kernel == "row":
        tot = (part[..., 0] + part[..., 1]).astype(f4)
    else:
        tot = warp_sum(np.pad(part, ((0, 0), (0, 0), (0, 32 - nw))))
    m = (tot / f4(D)).astype(f4)
    e = f4(er.f32(eps))
    inv = ((rsqrtf(m) + e) if defect == "eps-outside" else rsqrtf((m + e).astype(f4)))[..., None]
    w = np.stack([qw.float().numpy()] * Hq + [kw.float().numpy()] * Hkv)  # [Hq + Hkv, D]
    w_im = w[:, ri] if defect == "w-half" else w[:, ii]
    n_re = T((re * inv).astype(f4) * w[:, ri], dtype)
    n_im = T((im * inv).astype(f4) * w_im, dtype)
    y = x.copy()
    y[:, : Hq + Hkv, ri] = T((n_re * c).astype(f4) - (n_im * s).astype(f4), dtype)
    y[:, : Hq + Hkv, ii] = T((n_im * c).astype(f4) + (n_re * s).astype(f4), dtype)
    page = pages_k.shape[2]
    for b, pid, t in er.append_slots(cl, bt, page, pages_k.shape[0], chunk=chunk):
        kvh = np.arange(Hkv)
        if defect == "kv-head":
            kvh = (kvh + 1) % Hkv
        if defect == "slot":
            t = (t - 1) % page
        pages_k[pid, kvh, t] = y[b, Hq : Hq + Hkv]
        pages_v[pid, np.arange(Hkv), t] = y[b, Hq + Hkv :]
    return y[:, :Hq]


# ------------------------------------------------------------------ fixtures --
def rand_rows(shape, g, mode, dtype=BF16):
    x = torch.randn(*shape, generator=g, dtype=F64)
    if mode == "dynamic":  # entries from 2^-40 to 2^40 in one row (2^-12 to 2^12 in f16)
        e = 12 if dtype == F16 else 40
        x = x * torch.pow(2.0, torch.randint(-e, e + 1, shape, generator=g).to(F64))
    elif mode == "tiny":  # eps dominates the mean square
        x = x * 1e-4
    return x


def qk_setup(kernel, dtype, g, probe=None):
    """(qkv, qw, kw, offsets, cl, bt, Hq, Hkv, D, page): a decode batch whose offsets differ from ctx - 1, with an idle
    row, a row past the block table and page ids -1 and num_pages."""
    Hq, Hkv, D = (8, 2, 128) if kernel == "row" else (6, 2, 64)
    R, page, P, maxp = 8, 16, 12, 4
    H = Hq + 2 * Hkv
    if probe == "unit":
        x = er.unit_norm_rows(R, H, D, g)
    elif probe == "needle":
        x, _ = er.needle_rows(D, H, D)
        R = D
    else:
        x = rand_rows((R, H, D), g, probe or "gauss")
    qkv = x.reshape(R, H * D).to(dtype)
    qw, kw = (er.pow2_norm_weight(D, 0), er.pow2_norm_weight(D, 1)) if probe else (1 + 0.2 * torch.randn(D, generator=g), 1 + 0.2 * torch.randn(D, generator=g))
    cl = torch.randint(1, page * maxp, (R,), generator=g, dtype=torch.int32)
    cl[1], cl[2] = 0, page * maxp + 3  # idle, past the table
    offsets = torch.zeros(R, dtype=torch.int32) if probe == "unit" else (cl + 1000 + torch.arange(R, dtype=torch.int32))
    bt = torch.arange(R * maxp, dtype=torch.int32).view(R, maxp) % P
    bt[3, :], bt[4, :] = -1, P
    # distinct target slots per row: row b writes page b % P at slot b (pages are not shared between live rows)
    for b in range(R):
        if cl[b] > 0 and (cl[b] - 1) // page < maxp and b not in (3, 4):
            bt[b, (cl[b] - 1) // page] = b % P
            cl[b] = (cl[b] - 1) // page * page + (b // P) % page + 1
    return qkv.to(dtype), qw.to(dtype), kw.to(dtype), offsets, cl, bt, Hq, Hkv, D, page, P


def run_qk(kernel, dtype, probe, defect=None, seed=0, eps=1e-6):
    g = torch.Generator().manual_seed(seed)
    qkv, qw, kw, offsets, cl, bt, Hq, Hkv, D, page, P = qk_setup(kernel, dtype, g, probe)
    sentinel = torch.linspace(-3, 3, P * Hkv * page * D).view(P, Hkv, page, D).to(dtype)
    pk, pv = sentinel.float().numpy().copy(), sentinel.float().numpy().copy()
    q = emulate_qk(qkv, qw, kw, offsets, cl, bt, pk, pv, Hq, Hkv, 1e6, eps, kernel, defect=defect)
    ref = er.qk_norm_rope_ref(qkv, qw, kw, offsets, Hq, Hkv, 1e6, eps)
    slots = er.append_slots(cl, bt, page, P)
    return q, ref, sentinel, torch.from_numpy(pk).to(dtype), torch.from_numpy(pv).to(dtype), slots


def check_qk(q, ref, sentinel, pk, pv, slots, exact, what):
    if exact:
        er.assert_exact(torch.from_numpy(q), ref.q.out, f"{what} q")
        er.check_pages(sentinel, pk, slots, ref.k.out, f"{what} K")
    else:
        er.assert_within(torch.from_numpy(q), ref.q.pre, ref.q.tol, f"{what} q")
        er.check_pages(sentinel, pk, slots, None, f"{what} K", tol=ref.k.tol, pre=ref.k.pre)
        zero = ref.q.pre == 0
        er.assert_exact(torch.from_numpy(q)[zero], ref.q.pre[zero], f"{what} q zeros")
    er.check_pages(sentinel, pv, slots, ref.v, f"{what} V")


KERNELS = pytest.mark.parametrize("kernel", ["row", "head"])
QK_DTYPES = pytest.mark.parametrize("dtype", [BF16, F32], ids=["bf16", "f32"])


# ---------------------------------------------------------------------- bound --
@KERNELS
@QK_DTYPES
@pytest.mark.parametrize("mode", ["gauss", "dynamic", "tiny"])
def test_qk_emulations_stay_within_the_bound(kernel, dtype, mode):
    q, ref, sentinel, pk, pv, slots = run_qk(kernel, dtype, mode, seed=len(mode))
    assert len(slots) >= 4
    check_qk(q, ref, sentinel, pk, pv, slots, False, f"{kernel} {mode}")


@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("dim", [16, 129, 513, 2056, 4104])
@pytest.mark.parametrize("mode", ["gauss", "dynamic", "tiny"])
def test_rms_norm_emulation_stays_within_the_bound(dtype, dim, mode):
    g = torch.Generator().manual_seed(dim)
    x = rand_rows((4, dim), g, mode, dtype).to(dtype)
    w = (1 + 0.2 * torch.randn(dim, generator=g)).to(dtype)
    for eps in (1e-6, 1e-5):
        b = er.rms_norm_ref(x, w, eps, dtype)
        er.assert_within(torch.from_numpy(emulate_rms_norm(x, w, eps, dtype)), b.pre, b.tol, f"rms_norm {dim} {mode}")


@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
@pytest.mark.parametrize("traditional,dims", [(False, 64), (True, 64), (False, 32)])
def test_rope_emulation_stays_within_the_bound(dtype, traditional, dims):
    g = torch.Generator().manual_seed(dims + traditional)
    x = torch.randn(3, 2, 3, 64, generator=g).to(dtype)
    offsets = torch.tensor([0, 40959, 131071] if dtype != F32 else [4096, 40959, 1000000], dtype=torch.int32)
    b = er.rope_ref(x, offsets, dims, 1e4, traditional, dtype)
    er.assert_within(torch.from_numpy(emulate_rope(x, offsets, dims, 1e4, traditional, dtype)), b.pre, b.tol, "rope")


# --------------------------------------------------------------------- probes --
@KERNELS
@QK_DTYPES
def test_unit_norm_probes_are_exact_at_position_0(kernel, dtype):
    q, ref, sentinel, pk, pv, slots = run_qk(kernel, dtype, "unit", eps=0.0)
    check_qk(q, ref, sentinel, pk, pv, slots, True, f"{kernel} unit probe")


@KERNELS
@QK_DTYPES
def test_needle_probes_zero_everything_but_the_needle(kernel, dtype):
    q, ref, sentinel, pk, pv, slots = run_qk(kernel, dtype, "needle")
    assert int((ref.q.pre != 0).any(-1).sum()) > 0
    check_qk(q, ref, sentinel, pk, pv, slots, False, f"{kernel} needle probe")


def test_rms_norm_unit_rows_are_exact():
    g = torch.Generator().manual_seed(3)
    for dim in (128, 4096):
        x = er.unit_norm_rows(2, 1, dim, g).view(2, dim).to(BF16)
        w = er.pow2_norm_weight(dim, 0).to(BF16)
        er.assert_exact(torch.from_numpy(emulate_rms_norm(x, w, 0.0, BF16)), er.rms_norm_ref(x, w, 0.0, BF16).out, "rms_norm unit rows")


def test_round_to_handles_float32():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(10000, generator=g, dtype=F64) * 2.0 ** torch.randint(-140, 100, (10000,), generator=g)
    assert torch.equal(er.round_to(x, F32), x.float().double())


def test_argmax_reference_skips_nan():
    x = torch.tensor([[float("nan"), 1.0, 3.0, 3.0], [float("nan")] * 4, [float("-inf")] * 4, [float("nan"), float("-inf"), 0.0, 0.0]])
    x[3, 2:] = float("-inf")
    assert er.argmax_ref(x).tolist() == [2, 0, 0, 1]


# ------------------------------------------------------------------- defects --
QK_DEFECTS = ["layout", "sin-sign", "w-half", "angle-ctx", "eps-outside", "kv-head", "slot"]


@KERNELS
@pytest.mark.parametrize("defect", QK_DEFECTS)
def test_a_defective_fused_kernel_fails_the_checks(kernel, defect):
    """Each defect is caught by the exact probes or by the bound on needles, random or tiny rows (eps-outside)."""
    failed = []
    for probe, eps, exact in (("unit", 0.0, True), ("needle", 1e-6, False), ("gauss", 1e-6, False), ("tiny", 1e-5, False)):
        q, ref, sentinel, pk, pv, slots = run_qk(kernel, BF16, probe, defect=defect, eps=eps, seed=5)
        try:
            check_qk(q, ref, sentinel, pk, pv, slots, exact, f"{kernel} {defect} {probe}")
        except AssertionError:
            failed.append(probe)
    assert failed, f"{defect} passed every check"


@KERNELS
def test_an_fp32_formed_frequency_fails_in_f32(kernel):
    q, ref, sentinel, pk, pv, slots = run_qk(kernel, F32, "gauss", defect="f32-freq", seed=6)
    with pytest.raises(AssertionError, match="outside the error bound"):
        check_qk(q, ref, sentinel, pk, pv, slots, False, "f32 frequency")


@pytest.mark.parametrize("defect", ["layout", "sin-sign", "f32-freq"])
def test_a_defective_rope_fails_the_bound(defect):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 3, 2, 64, generator=g).to(F32)
    offsets = torch.tensor([4096, 40959], dtype=torch.int32)
    b = er.rope_ref(x, offsets, 64, 1e4, False, F32)
    with pytest.raises(AssertionError, match="outside the error bound"):
        er.assert_within(torch.from_numpy(emulate_rope(x, offsets, 64, 1e4, False, F32, defect)), b.pre, b.tol, defect)


def test_eps_outside_the_square_root_fails_the_rms_norm_bound():
    g = torch.Generator().manual_seed(4)
    for dtype in (BF16, F32):
        x = rand_rows((4, 128), g, "tiny").to(dtype)
        w = torch.ones(128).to(dtype)
        b = er.rms_norm_ref(x, w, 1e-5, dtype)
        with pytest.raises(AssertionError, match="outside the error bound"):
            er.assert_within(torch.from_numpy(emulate_rms_norm(x, w, 1e-5, dtype, "eps-outside")), b.pre, b.tol, "eps outside")
