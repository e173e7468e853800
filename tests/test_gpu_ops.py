"""Operator parity on an H100: every primitive of the extension, called through
the Python shim -> C ABI -> sm_90a kernels, against the CPU oracle on the same
seeded inputs.  Tolerances are written per test; integer / copy semantics are
bit-exact.  Full-size (BASELINE.json) cases use size-independent properties."""

import json
from math import prod
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import ops as oracle

pytestmark = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
ULP = {BF16: 2.0**-8, F16: 2.0**-11, F32: 2.0**-24}


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def gen(seed):
    return torch.Generator().manual_seed(seed)


def assert_close(got, want, rtol, atol, msg=""):
    torch.testing.assert_close(got.detach().cpu().to(F32), want.detach().cpu().to(F32), rtol=rtol, atol=atol, msg=lambda m: f"{msg}\n{m}")


def rand_packed(K, N, g, dtype=BF16, sigma=None):
    sigma = sigma if sigma is not None else 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
    scales = (torch.randn(K, N // 128, generator=g) * sigma).to(dtype)
    biases = (-7.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma).to(dtype)
    return words, scales, biases


# ----------------------------------------------------------------- W4A16 ----
QMM_SHAPES = [
    # (M, N, K)   test_week_2_day_3.py shapes first, then the Qwen3-4B / 0.6B projections
    (1, 128, 5), (3, 128, 5), (8, 128, 64), (1, 256, 96), (1, 2560, 1024), (8, 2560, 1024),
    (1, 2560, 4096), (1, 4096, 2560), (1, 2560, 9728), (1, 9728, 2560), (2, 1024, 3072), (5, 3072, 1024),
    (4, 2560, 1030), (7, 128, 17),
    # beyond the reference matvec limit: small decode batches and ragged tiles
    (9, 2560, 1024), (16, 2560, 1024), (17, 2560, 1032), (32, 2560, 1024), (10, 256, 96), (33, 256, 96),
    (64, 9728, 2560), (128, 256, 96), (40, 4096, 2560), (129, 2560, 1024), (300, 1024, 520), (512, 2560, 4096),
    # swap-AB split-reduction kernel: every token-column width (16/32/64/128), ragged feature tiles, split and unsplit reductions
    (12, 128, 40), (16, 4096, 2560), (24, 2560, 6144), (48, 2560, 19456), (64, 2560, 6144), (100, 9728, 2560), (128, 4096, 2560),
    (128, 2560, 1000), (77, 1024, 3072),
]


@pytest.mark.parametrize("shape", QMM_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
def test_quantized_matmul_matches_oracle(dev, shape, dtype):
    M, N, K = shape
    g = gen(M * 7919 + N + K)
    words, scales, biases = rand_packed(K, N, g, dtype)
    a = torch.randn(M, N, generator=g).to(dtype)
    want = oracle.quantized_matmul(scales, biases, 128, 4, a, words, True, use_simdgroup=False)  # fp32-exact weights
    # tensor-core GEMMs (M > 8: swap-AB split-reduction kernel up to 128 rows, 128 x 128 tiles above): weights
    # rounded to the activation dtype before the MMA, like the reference's tiled kernel (quantized_matmul.metal:183-194)
    w_rounded = oracle.dequantize_weights(words, scales, biases, 128, 4).float()
    want_tiled = (a.float() @ w_rounded.T).to(dtype)
    args = (scales.to(dev), biases.to(dev), 128, 4, a.to(dev), words.to(dev), True)
    scale_ref = float(want.float().abs().max()) + 1e-6
    # one output ulp of rounding disagreement + fp32 summation-order noise
    tol = dict(rtol=2 * ULP[dtype], atol=2e-3 * scale_ref)
    got = ext.quantized_matmul(*args)  # extension default: use_simdgroup=True
    assert got.dtype == dtype and tuple(got.shape) == (M, K)
    assert_close(got, want if M <= 8 else want_tiled, **tol, msg=f"stream/gemm {shape}")
    vanilla = ext.quantized_matmul(*args, use_simdgroup=False)
    assert_close(vanilla, want, **tol, msg=f"vanilla {shape}")
    split = ext.quantized_matmul(*args, use_simdgroup=True, use_split_k=True)
    # tiled/split variants may round weights / partials to the storage dtype (reference atol 1.0-1.5 at N=2560)
    assert_close(split, want, rtol=2e-2, atol=2e-2 * scale_ref, msg=f"split {shape}")


def test_identity_activations_return_dequantised_weights_bit_exact(dev):
    # test_week_2_day_3.py:74-118 identity case: eye(128) @ W^T
    g = gen(11)
    words, scales, biases = rand_packed(5, 128, g, sigma=0.1)
    want = oracle.dequantize_weights(words, scales, biases, 128, 4).T
    for kw in (dict(), dict(use_simdgroup=False), dict(use_simdgroup=True, use_split_k=True)):
        got = ext.quantized_matmul(scales.to(dev), biases.to(dev), 128, 4, torch.eye(128, dtype=BF16, device=dev), words.to(dev), True, **kw)
        assert torch.equal(got.cpu(), want), kw


def test_split_k_request_that_falls_back_is_bit_identical(dev):
    # test_week_2_day_7.py:80-109: a split request the policy declines must run the same kernel
    g = gen(12)
    words, scales, biases = rand_packed(2560, 256, g)
    a = torch.randn(128, 256, generator=g).to(BF16)
    args = (scales.to(dev), biases.to(dev), 128, 4, a.to(dev), words.to(dev), True)
    unsplit = ext.quantized_matmul(*args, use_simdgroup=True)
    requested = ext.quantized_matmul(*args, use_simdgroup=True, use_split_k=True)
    assert torch.equal(unsplit, requested)


def test_full_size_lm_head_one_hot_property(dev):
    """BASELINE size (tied head 2560 -> 151936): a one-hot activation must return
    column j of the dequantised table - exact arithmetic, so bit-exact up to rare
    fp32 ties; checked against torch ops on the GPU over all 151,936 rows."""
    g = gen(13)
    K, N = 151936, 2560
    words, scales, biases = rand_packed(K, N, g)
    wd, sd, bd = words.to(dev), scales.to(dev), biases.to(dev)
    for j in (0, 1, 129, 2047, 2559):
        a = torch.zeros(1, N, dtype=BF16, device=dev)
        a[0, j] = 1.0
        got = ext.quantized_matmul(sd, bd, 128, 4, a, wd, True)[0]
        code = ((wd[:, j // 8] >> (4 * (j % 8))) & 0xF).to(F32)
        want = (code * sd[:, j // 128].to(F32) + bd[:, j // 128].to(F32)).to(BF16)
        mismatch = (got != want).float().mean().item()
        assert mismatch < 1e-3, (j, mismatch)
        assert_close(got, want, rtol=ULP[BF16], atol=1e-6, msg=f"column {j}")
    # linearity in the activation at full size: f(2a) == 2 f(a) exactly (power-of-two scaling)
    a = torch.randn(3, N, generator=g).to(BF16).to(dev)
    y1 = ext.quantized_matmul(sd, bd, 128, 4, a, wd, True)
    y2 = ext.quantized_matmul(sd, bd, 128, 4, (a.float() * 2).to(BF16), wd, True)
    assert torch.equal((y1.float() * 2).to(BF16), y2)


def test_quantized_matmul_rejects_bad_arguments(dev):
    s = torch.zeros(4, 1, dtype=BF16, device=dev)
    a = torch.zeros(2, 128, dtype=BF16, device=dev)
    b = torch.zeros(4, 16, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError, match="b must be transposed"):
        ext.quantized_matmul(s, s, 128, 4, a, b, False)
    with pytest.raises(RuntimeError, match="must be contiguous"):
        ext.quantized_matmul(s, s, 128, 4, torch.zeros(128, 2, dtype=BF16, device=dev).T, b, True)
    with pytest.raises(RuntimeError, match="b must be uint32"):
        ext.quantized_matmul(s, s, 128, 4, a, b.to(torch.int64), True)
    out = ext.quantized_matmul(s, s, 128, 4, a[:0], b, True)
    assert tuple(out.shape) == (0, 4)


@pytest.mark.parametrize("index_dtype", [torch.int32, torch.uint32], ids=["i32", "u32"])
def test_quantized_embedding_is_bit_exact(dev, index_dtype):
    g = gen(21)
    words, scales, biases = rand_packed(517, 2560, g, sigma=0.05)
    idx = torch.randint(0, 517, (3, 9), generator=g).to(torch.int32)
    want = oracle.quantized_embedding(idx, scales, biases, words, 128, 4)
    idx_dev = idx.to(dev).view(index_dtype) if index_dtype == torch.uint32 else idx.to(dev)
    got = ext.quantized_embedding(idx_dev, scales.to(dev), biases.to(dev), words.to(dev).view(torch.uint32), 128, 4)
    assert tuple(got.shape) == (3, 9, 2560) and got.dtype == BF16
    assert torch.equal(got.cpu(), want)


# ------------------------------------------------------------ fused ops ------
@pytest.mark.parametrize("shape", [(1, 2560), (4, 1, 2560), (2, 3, 40, 128), (7, 16), (3, 1000), (2, 8192), (5, 129)], ids=str)
@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
def test_rms_norm_matches_oracle(dev, shape, dtype):
    g = gen(prod(shape))
    x = (torch.randn(*shape, generator=g) * 3).to(dtype)
    w = (1 + 0.1 * torch.randn(shape[-1], generator=g)).to(dtype)
    want = oracle.rms_norm(x, w, 1e-6)
    got = ext.rms_norm(x.to(dev), w.to(dev), 1e-6)
    assert got.dtype == dtype and got.shape == x.shape
    assert_close(got, want, rtol=2 * ULP[dtype] if dtype != F32 else 1e-5, atol=1e-6)


@pytest.mark.parametrize(
    "case",
    [
        dict(shape=(1, 1, 32, 128), dims=128, offsets=[0]),
        dict(shape=(2, 5, 8, 128), dims=128, offsets=[3, 4000]),
        dict(shape=(1, 7, 8, 128), dims=128, offsets=[32000]),
        dict(shape=(3, 4, 2, 16), dims=16, offsets=[3, 7, 0], traditional=True),
        dict(shape=(2, 9, 8, 4), dims=4, offsets=[1, 4]),
        dict(shape=(1, 3, 2, 16), dims=8, offsets=[5]),
        dict(shape=(1, 3, 2, 16), dims=8, offsets=[5], traditional=True),
        dict(shape=(1, 300, 32, 128), dims=128, offsets=[100]),                    # prefill-sized: per-(token, pair) kernel
        dict(shape=(2, 70, 8, 128), dims=128, offsets=[0, 5000]),
        dict(shape=(1, 80, 4, 16), dims=16, offsets=[9], traditional=True),
    ],
    ids=lambda c: f"{c['shape']}-d{c['dims']}{'-trad' if c.get('traditional') else ''}",
)
@pytest.mark.parametrize("dtype", [BF16, F32], ids=["bf16", "f32"])
def test_rope_matches_oracle(dev, case, dtype):
    g = gen(prod(case["shape"]))
    x = torch.randn(*case["shape"], generator=g).to(dtype)
    off = torch.tensor(case["offsets"], dtype=torch.int32)
    want = oracle.rope(x, off, case["dims"], 1000000.0, case.get("traditional", False))
    got = ext.rope(x.to(dev), off.to(dev), case["dims"], 1000000.0, case.get("traditional", False))
    # stated tolerance of the reference for this op: 2e-2 (test_week_2_day_4.py:51).  We hold 1 ulp plus
    # the fp32 angle noise of the reference arithmetic itself, position * 2^-23 rad (0.004 at 32K).
    far = max(case["offsets"]) + case["shape"][1]
    noise = 4.0 * far * 2.0**-23
    assert_close(got, want, rtol=2 * ULP[dtype] if dtype != F32 else 2e-4, atol=(4e-3 if dtype != F32 else 1e-5) + noise)


@pytest.mark.parametrize("n", [16, 9728, 3 * 9728, 1001])
@pytest.mark.parametrize("dtype", [BF16, F16, F32], ids=["bf16", "f16", "f32"])
def test_swiglu_and_add_match_oracle(dev, n, dtype):
    g = gen(n)
    a = (torch.randn(n, generator=g) * 4).to(dtype)
    b = torch.randn(n, generator=g).to(dtype)
    assert_close(ext.swiglu(a.to(dev), b.to(dev)), oracle.swiglu(a, b), rtol=2 * ULP[dtype] if dtype != F32 else 1e-5, atol=1e-6)
    assert torch.equal(ext.add(a.to(dev), b.to(dev)).cpu(), (a.float() + b.float()).to(dtype))


def test_dense_decode_attention_on_the_reference_fixture_sweep(dev):
    # test_week_2_day_5.py:119-163, tolerance 3e-2; plus the committed oracle checksums
    D, Hq = 128, 4
    ref = json.loads((Path(__file__).parent / "golden" / "decode_attention_fixture_checksums.json").read_text())

    def fixture(shape, phase):
        return torch.sin(torch.arange(prod(shape), dtype=F32) * 0.017 + phase).reshape(shape).to(BF16)

    shapes = [(1, s) for s in (1, 31, 32, 127, 128, 129, 255, 256)] + [(8, s) for s in (8, 31, 32, 127, 128, 129, 255, 256)]
    for L, S in shapes:
        for ratio in (1, 4):
            Hkv = Hq // ratio
            q, k, v = fixture((Hq, L, D), 0.1), fixture((Hkv, S, D), 0.7), fixture((Hkv, S, D), 1.3)
            explicit = torch.where(torch.arange(S) % 5 == 0, -2.0, 0.0).reshape(1, 1, S).expand(Hq, L, S).contiguous()
            for name, causal, mask in (("causal", True, torch.zeros(1)), ("mask", False, explicit)):
                want = oracle.decode_attention(q, k, v, mask, D**-0.5, causal, not causal, Hq, Hkv)
                got = ext.decode_attention(q.to(dev), k.to(dev), v.to(dev), mask.to(dev), D**-0.5, causal, not causal, Hq, Hkv)
                assert_close(got, want, rtol=2e-2, atol=1e-2, msg=f"L={L} S={S} gqa={ratio} {name}")
                key = f"L{L}_S{S}_g{ratio}_{name}"
                assert abs(float(got.float().sum()) - ref[key]) <= 3e-2 * max(1.0, abs(ref[key])), key


@pytest.mark.parametrize("dtype,D", [(F32, 4), (F32, 80), (F16, 64), (BF16, 256)], ids=["f32-4", "f32-80", "f16-64", "bf16-256"])
def test_dense_decode_attention_other_dtypes_and_dims(dev, dtype, D):
    g = gen(D)
    q = torch.randn(2 * 6, 2, D, generator=g).to(dtype)
    k = torch.randn(2 * 3, 37, D, generator=g).to(dtype)
    v = torch.randn(2 * 3, 37, D, generator=g).to(dtype)
    want = oracle.decode_attention(q, k, v, torch.zeros(1), D**-0.5, True, False, 6, 3)
    got = ext.decode_attention(q.to(dev), k.to(dev), v.to(dev), torch.zeros(1, device=dev), D**-0.5, True, False, 6, 3)
    assert_close(got, want, rtol=4 * ULP[dtype] if dtype != F32 else 1e-4, atol=2e-3 if dtype != F32 else 1e-5)


# ------------------------------------------------------------- paged KV ------
@pytest.mark.parametrize("dtype,D", [(F32, 4), (BF16, 128), (F32, 3), (BF16, 20)], ids=["f32-4", "bf16-128", "f32-3", "bf16-20"])
def test_paged_cache_update_is_an_exact_in_place_slice_write(dev, dtype, D):
    g = gen(D)
    pages = torch.randn(5, 2, 8, D, generator=g).to(dtype)
    vals = torch.randn(1, 2, 3, D, generator=g).to(dtype)
    want = oracle.paged_cache_update(pages.clone(), vals, 3, 4)
    pages_dev = pages.to(dev)
    out = ext.paged_cache_update(pages_dev, vals.to(dev), 3, 4)
    assert out is pages_dev, "the output aliases the input buffer (paged_attention.cpp:46-49)"
    assert torch.equal(pages_dev.cpu(), want)
    with pytest.raises(RuntimeError, match="outside page storage"):
        ext.paged_cache_update(pages_dev, vals.to(dev), 3, 6)


def test_paged_cache_append_decode_matches_per_row_updates(dev):
    g = gen(31)
    P, H, page, D, B = 9, 8, 16, 128, 5
    kp = torch.randn(P, H, page, D, generator=g).to(BF16)
    vp = torch.randn(P, H, page, D, generator=g).to(BF16)
    keys = torch.randn(B, H, 1, D, generator=g).to(BF16)
    values = torch.randn(B, H, 1, D, generator=g).to(BF16)
    ctx = torch.tensor([17, 0, 1, 32, 16], dtype=torch.int32)
    bt = torch.tensor([[4, 2, -1], [-1, -1, -1], [7, -1, -1], [0, 8, -1], [5, -1, -1]], dtype=torch.int32)
    want_k, want_v = kp.clone(), vp.clone()
    for b in range(B):
        if int(ctx[b]) > 0:
            tok = int(ctx[b]) - 1
            pid = int(bt[b, tok // page])
            oracle.paged_cache_update(want_k, keys[b : b + 1], pid, tok % page)
            oracle.paged_cache_update(want_v, values[b : b + 1], pid, tok % page)
    kd, vd = kp.to(dev), vp.to(dev)
    ext.paged_cache_append_decode(kd, vd, keys.to(dev), values.to(dev), bt.to(dev), ctx.to(dev))
    assert torch.equal(kd.cpu(), want_k) and torch.equal(vd.cpu(), want_v)


@pytest.mark.parametrize("dtype", [BF16, F32], ids=["bf16", "f32"])
@pytest.mark.parametrize("page,H,D,L,first", [(16, 2, 128, 70, 5), (128, 8, 128, 300, 0), (8, 3, 20, 33, 7)])
def test_paged_cache_append_chunk_equals_per_page_updates(dev, dtype, page, H, D, L, first):
    """One launch for a whole chunk (strided [1, H, L, D] view of a [1, L, H, D] projection output)
    against the reference's per-page paged_cache_update sequence."""
    g = gen(page + H + D + L)
    n_pages = (first + L + page - 1) // page + 3
    kp = torch.randn(n_pages, H, page, D, generator=g).to(dtype).to(dev)
    vp = torch.randn(n_pages, H, page, D, generator=g).to(dtype).to(dev)
    kp_ref, vp_ref = kp.clone(), vp.clone()
    keys = torch.randn(1, L, H, D, generator=g).to(dtype).to(dev).transpose(1, 2)    # [1, H, L, D], token stride H*D
    values = torch.randn(1, L, H, D, generator=g).to(dtype).to(dev).transpose(1, 2)
    order = torch.randperm(n_pages, generator=g).tolist()
    spans, done, slot = [], 0, first
    for pid in order:
        if done >= L:
            break
        take = min(page - slot, L - done)
        spans.append((pid, slot, take, done))
        ext.paged_cache_update(kp_ref, keys[:, :, done : done + take].contiguous(), pid, slot)
        ext.paged_cache_update(vp_ref, values[:, :, done : done + take].contiguous(), pid, slot)
        done += take
        slot = 0
    ext.paged_cache_append_chunk(kp, vp, keys, values, spans)
    assert torch.equal(kp, kp_ref) and torch.equal(vp, vp_ref)


def build_paged(g, lens, page, Hkv, D, dtype, scatter=True):
    """Random pages + block tables for requests of the given context lengths;
    page ids are shuffled so logical order != physical order."""
    need = [(n + page - 1) // page for n in lens]
    total = sum(need) + 2
    perm = torch.randperm(total, generator=g).tolist() if scatter else list(range(total))
    width = max(1, max(need))
    bt = torch.full((len(lens), width), -1, dtype=torch.int32)
    cursor = 0
    for b, n in enumerate(need):
        bt[b, :n] = torch.tensor(perm[cursor : cursor + n], dtype=torch.int32)
        cursor += n
    kp = torch.randn(total, Hkv, page, D, generator=g).to(dtype)
    vp = torch.randn(total, Hkv, page, D, generator=g).to(dtype)
    return kp, vp, bt, torch.tensor(lens, dtype=torch.int32)


PAGED_CASES = [
    # (dtype, D, page, Hq, Hkv, L, context lens)
    (F32, 4, 4, 4, 2, 1, [6]), (F32, 4, 4, 4, 2, 3, [6]), (F32, 4, 4, 4, 2, 1, [4, 0, 7]), (F32, 64, 16, 6, 3, 2, [33, 5]),
    (BF16, 128, 32, 8, 2, 1, [65]), (BF16, 128, 32, 4, 2, 9, [73]), (BF16, 128, 32, 4, 2, 65, [129]),
    (BF16, 128, 128, 32, 8, 1, [1]), (BF16, 128, 128, 32, 8, 1, [128]), (BF16, 128, 128, 32, 8, 1, [129]),
    (BF16, 128, 128, 32, 8, 1, [1000, 0, 17, 4097]), (BF16, 128, 128, 32, 8, 4, [900, 4]), (BF16, 128, 128, 32, 8, 8, [300]),
    (BF16, 128, 128, 16, 8, 1, [2500]), (BF16, 128, 16, 8, 8, 2, [77, 130]), (BF16, 128, 128, 32, 8, 128, [128]),
    (BF16, 128, 128, 32, 8, 40, [300]), (BF16, 128, 16, 8, 2, 70, [70, 200]), (BF16, 128, 128, 32, 8, 257, [600]),
    (BF16, 128, 64, 8, 8, 64, [64, 0, 500]), (BF16, 128, 32, 4, 1, 100, [40, 100]),
    # wgmma flash prefill (page % 64 == 0, Hq/Hkv divides 128): head ratios 1/2/4/8, chunk continuation (ctx > L),
    # L not a multiple of the 128/G-row query block, several requests, a 64-slot page
    (BF16, 128, 128, 16, 8, 200, [200]), (BF16, 128, 128, 16, 2, 130, [130, 400]), (BF16, 128, 64, 6, 6, 90, [90, 1000]),
    (BF16, 128, 128, 32, 8, 128, [4224]), (BF16, 128, 128, 32, 8, 33, [1025, 33]), (BF16, 128, 256, 8, 2, 300, [777]),
    (BF16, 128, 128, 32, 8, 1000, [1000]), (BF16, 64, 16, 4, 2, 1, [50]), (BF16, 64, 16, 4, 2, 5, [50]), (F32, 128, 8, 2, 1, 12, [40]),
]


@pytest.mark.parametrize("case", PAGED_CASES, ids=lambda c: f"{str(c[0])[6:]}-D{c[1]}-p{c[2]}-H{c[3]}/{c[4]}-L{c[5]}-ctx{'_'.join(map(str, c[6]))}")
@pytest.mark.parametrize("causal", [True, False], ids=["causal", "full"])
def test_paged_attention_matches_oracle(dev, case, causal):
    dtype, D, page, Hq, Hkv, L, lens = case
    if not causal and L > 8 and not (dtype == BF16 and D == 128 and page % 64 == 0):
        pytest.skip("non-causal prefill is never issued by the models (only the wgmma kernel takes it)")
    g = gen(D * 1000 + page + L + sum(lens))
    kp, vp, bt, cl = build_paged(g, lens, page, Hkv, D, dtype)
    B = len(lens)
    q = torch.randn(B * Hq, L, D, generator=g).to(dtype)
    scale = D**-0.5
    want = oracle.paged_attention(q, kp, vp, bt, cl, scale, causal, Hkv, Hq)
    got = ext.paged_attention(q.to(dev), kp.to(dev), vp.to(dev), bt.to(dev), cl.to(dev), scale, is_causal=causal, num_kv_heads=Hkv, num_heads=Hq)
    assert got.dtype == dtype and got.shape == q.shape
    tol = dict(rtol=1e-4, atol=1e-5) if dtype == F32 else dict(rtol=2e-2, atol=5e-3)  # reference: 2e-2 (test_week_3_day_5.py:61)
    assert_close(got, want, **tol)
    for b, n in enumerate(lens):
        if n == 0:
            assert torch.count_nonzero(got[b * Hq : (b + 1) * Hq]) == 0, "idle slot must be exact zeros"


def test_full_size_prefill_attention_properties(dev):
    """Config-3 size (Hq 32, Hkv 8, D 128, page 128, a 4096-token prompt in one chunk) through the
    tensor-core flash kernel: constant V rows come back unchanged (softmax weights sum to one), and
    identical K rows make every query the causal running mean of V."""
    g = gen(43)
    S, page, Hq, Hkv, D = 4096, 128, 32, 8, 128
    pages = S // page
    bt = torch.randperm(pages, generator=g).reshape(1, pages).to(torch.int32).to(dev)
    cl = torch.tensor([S], dtype=torch.int32, device=dev)
    q = torch.randn(Hq, S, D, generator=g).to(BF16).to(dev)
    kp = torch.randn(pages, Hkv, page, D, generator=g).to(BF16).to(dev)
    v_row = torch.randn(Hkv, 1, D, generator=g).to(BF16)
    vp = v_row[None].expand(pages, Hkv, page, D).contiguous().to(dev)
    out = ext.paged_attention(q, kp, vp, bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    want = v_row.repeat_interleave(Hq // Hkv, dim=0).expand(Hq, S, D)
    assert_close(out, want, rtol=4 * ULP[BF16], atol=1e-6, msg="constant V")
    vp2 = torch.randn(pages, Hkv, page, D, generator=g).to(BF16).to(dev)
    out2 = ext.paged_attention(q, torch.zeros_like(kp), vp2, bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    dense = vp2[bt[0].long()].permute(1, 0, 2, 3).reshape(Hkv, S, D).float()
    running = dense.cumsum(dim=1) / torch.arange(1, S + 1, device=dev, dtype=torch.float32)[None, :, None]
    assert_close(out2, running.repeat_interleave(Hq // Hkv, dim=0), rtol=2e-2, atol=4e-3, msg="causal running mean of V")


def test_full_size_prefill_attention_matches_oracle_on_sampled_rows(dev):
    """Config-3 size through the wgmma flash kernel, compared with the ORACLE: query row l of a causal
    chunk is exactly a decode query over the first ctx - L + l + 1 keys (bottom-right alignment,
    paged_attention.metal:158-160 / :411), so sampled rows are checked with the oracle's L == 1 path.
    Two shapes: the whole 4096-token prompt in one chunk, and a 512-token chunk that continues a
    3584-token context."""
    g = gen(47)
    page, Hq, Hkv, D = 128, 32, 8, 128
    for L, ctx in ((4096, 4096), (512, 4096)):
        pages = ctx // page
        bt = torch.randperm(pages, generator=g).reshape(1, pages).to(torch.int32)
        cl = torch.tensor([ctx], dtype=torch.int32)
        q = torch.randn(Hq, L, D, generator=g).to(BF16)
        kp = torch.randn(pages, Hkv, page, D, generator=g).to(BF16)
        vp = torch.randn(pages, Hkv, page, D, generator=g).to(BF16)
        out = ext.paged_attention(q.to(dev), kp.to(dev), vp.to(dev), bt.to(dev), cl.to(dev), D**-0.5, is_causal=True,
                                  num_kv_heads=Hkv, num_heads=Hq).cpu()
        for l in (0, 1, 31, 32, 63, 64, 127, 128, L // 2 - 1, L // 2, L - 65, L - 2, L - 1):
            seen = torch.tensor([ctx - L + l + 1], dtype=torch.int32)
            want = oracle.paged_attention(q[:, l : l + 1].contiguous(), kp, vp, bt, seen, D**-0.5, True, Hkv, Hq)
            assert_close(out[:, l : l + 1], want, rtol=2e-2, atol=5e-3, msg=f"L={L} ctx={ctx} row {l}")


def test_prefill_attention_ignores_pages_outside_the_block_table(dev):
    """Invalid page ids (-1 padding inside the visible range cannot occur after validation, attention.py:131-146,
    but the C ABI must not read through them): an id beyond the physical pages masks that page's keys."""
    g = gen(48)
    page, Hq, Hkv, D, L = 64, 8, 2, 128, 128
    kp = torch.randn(4, Hkv, page, D, generator=g).to(BF16)
    vp = torch.randn(4, Hkv, page, D, generator=g).to(BF16)
    q = torch.randn(Hq, L, D, generator=g).to(BF16)
    cl = torch.tensor([128], dtype=torch.int32)
    good = torch.tensor([[2, 1]], dtype=torch.int32)
    want = oracle.paged_attention(q, kp, vp, good, cl, D**-0.5, True, Hkv, Hq)
    got = ext.paged_attention(q.to(dev), kp.to(dev), vp.to(dev), good.to(dev), cl.to(dev), D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    assert_close(got, want, rtol=2e-2, atol=5e-3)
    # second page id out of range: queries 64.. see only their first 64 keys; launcher-level call (the Python layer rejects this table)
    bad = torch.tensor([[2, 99]], dtype=torch.int32)
    got_bad = ext.paged_attention(q.to(dev), kp.to(dev), vp.to(dev), bad.to(dev), cl.to(dev), D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq).cpu()
    first = oracle.paged_attention(q[:, :64].contiguous(), kp, vp, good[:, :1], torch.tensor([64], dtype=torch.int32), D**-0.5, True, Hkv, Hq)
    assert_close(got_bad[:, :64], first, rtol=2e-2, atol=5e-3)
    full_first_page = oracle.paged_attention(q[:, 64:].contiguous(), kp, vp, good[:, :1], torch.tensor([64], dtype=torch.int32), D**-0.5, False, Hkv, Hq)
    assert_close(got_bad[:, 64:], full_first_page, rtol=2e-2, atol=5e-3)


def test_full_size_decode_attention_properties(dev):
    """Config-2/5 size (Hq 32, Hkv 8, D 128, page 128, 8192-token context, split
    across CTAs): identical V rows must come back unchanged whatever the scores
    are (softmax weights sum to one), and identical K rows give the mean of V."""
    g = gen(41)
    S, page, Hq, Hkv, D, B = 8192, 128, 32, 8, 128, 2
    pages = S // page
    P = B * pages
    bt = torch.randperm(P, generator=g).reshape(B, pages).to(torch.int32)
    cl = torch.tensor([S, S - 77], dtype=torch.int32)
    q = torch.randn(B * Hq, 1, D, generator=g).to(BF16).to(dev)
    kp = torch.randn(P, Hkv, page, D, generator=g).to(BF16).to(dev)
    v_row = torch.randn(Hkv, 1, D, generator=g).to(BF16)
    vp = v_row[None].expand(P, Hkv, page, D).contiguous().to(dev)
    out = ext.paged_attention(q, kp, vp, bt.to(dev), cl.to(dev), D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    want = v_row[:, 0].repeat_interleave(Hq // Hkv, dim=0).repeat(B, 1)[:, None, :]
    assert_close(out, want, rtol=2 * ULP[BF16], atol=1e-6, msg="constant V")
    # uniform scores -> arithmetic mean of the visible V rows
    vp2 = torch.randn(P, Hkv, page, D, generator=g).to(BF16).to(dev)
    kp2 = torch.zeros_like(kp)
    out2 = ext.paged_attention(q, kp2, vp2, bt.to(dev), cl.to(dev), D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    for b in range(B):
        n = int(cl[b])
        dense = vp2[bt[b].long().to(dev)].permute(1, 0, 2, 3).reshape(Hkv, pages * page, D)[:, :n].float().mean(dim=1)
        assert_close(out2[b * Hq : (b + 1) * Hq, 0], dense.repeat_interleave(Hq // Hkv, dim=0), rtol=2e-2, atol=2e-3, msg=f"mean of V, row {b}")


def test_argmax_returns_the_first_maximum(dev):
    g = gen(51)
    logits = torch.randn(5, 151936, generator=g).to(BF16)
    logits[1, 77] = 50.0
    logits[1, 140000] = 50.0  # tie: first index wins, like mx.argmax / torch.argmax
    logits[3, 151935] = 60.0
    got = ext.argmax(logits.to(dev))
    assert got.dtype == torch.int32
    assert got.cpu().tolist() == torch.argmax(logits.float(), dim=-1).tolist()
    small = torch.randn(3, 128, generator=g)
    assert ext.argmax(small.to(dev)).cpu().tolist() == torch.argmax(small, dim=-1).tolist()


def test_launch_counter_counts_this_librarys_kernels(dev):
    before = ext.launch_count()
    ext.swiglu(torch.zeros(64, device=dev), torch.zeros(64, device=dev))
    torch.cuda.synchronize()
    assert ext.launch_count() == before + 1
    sms, major, minor = ext.device_info()
    assert (major, minor) == (9, 0) and sms >= 100
