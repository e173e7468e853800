"""Every 8-bit (W8A16) projection kernel and fused form against a float64 reference (tests/w8a16_ref.py).

Each case names the kernel it must reach (tl_quantized_matmul_route_bits).  Then:
  * exact probes: codes 0, 127, 128 and 255 in every needle column, needles at group and box boundaries, power-of-two
    scales: every path must be bit-exact (a dequantiser that is only right below 128 fails them);
  * random inputs, with a common activation mean and bias-dominated weights: within the derived error bound.
The embedding, residual_norm and qkv_project_rope_append are checked too."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


w8 = _load("tiny_llm_b200_w8a16_ref", "w8a16_ref.py")
wr = w8.wr

pytestmark = pytest.mark.gpu
BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
PATHS = {ext.W4_VANILLA: "vanilla", ext.W4_STREAM: "stream", ext.W4_SKINNY: "skinny", ext.W4_TILES: "tiles"}
NONE, RMS, SWI = wr.PRO_NONE, wr.PRO_RMSNORM, wr.PRO_SWIGLU
ENONE, ERES, EPAIRS = wr.EPI_NONE, wr.EPI_RESIDUAL, wr.EPI_SWIGLU_PAIRS


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def case(op, M, N, K, route, pro=NONE, epi=ENONE, simd=True):
    return dict(op=op, M=M, N=N, K=K, route=route, pro=pro, epi=epi, simd=simd)


CASES = [
    # streaming kernel: rows per pass 1, 2, 4, 8 (plain entry), 16 (a prologue keeps 9..128 rows on it) and 32 in five
    # passes (the fused entry keeps M > 128 on it)
    *[case("qmm", M, 512, 384, "stream") for M in (1, 2, 3, 4, 8)],
    case("fused", 16, 1024, 256, "stream", RMS),
    case("fused", 160, 512, 384, "stream"),
    # every prologue x epilogue of the streaming kernel, one pass and several
    *[case("fused", M, 512, 256, "stream", pro, epi) for M in (4, 136) for pro in (NONE, RMS, SWI) for epi in (ENONE, ERES, EPAIRS)],
    # the split-reduction wgmma kernel at each token tile, with splits, and its epilogues
    *[case("qmm", M, 4096, 1024, "skinny") for M in (9, 32, 64, 128)],
    *[case("fused", 24, 2560, 512, "skinny", NONE, epi) for epi in (ERES, EPAIRS)],
    case("resnorm", 24, 2560, 512, "skinny"),
    case("resnorm", 4, 512, 256, "stream"),
    # 128-token tiles, ragged M
    case("qmm", 200, 1024, 384, "tiles"),
    case("qmm", 128 + 64 + 3, 512, 256, "tiles"),
    # scalar control kernel
    case("qmm", 3, 512, 256, "vanilla", simd=False),
]
IDS = [f"{c['op']}-M{c['M']}-N{c['N']}-K{c['K']}-{c['route']}-p{c['pro']}e{c['epi']}" for c in CASES]


def route(c, words, scales, biases, p0, dtype):
    r = ext.quantized_matmul_route(c["M"], c["N"], c["K"], c["N"], c["pro"], c["op"] != "qmm", c["simd"], dtype, p0, words, scales, biases, bits=8)
    assert PATHS[r[0]] == c["route"], f"reached {PATHS[r[0]]} {r[1:]}"
    return r


def run(c, words, scales, biases, p0, p1=None, residual=None, eps=1e-6, norm_w=None):
    if c["op"] == "qmm":
        return ext.quantized_matmul(scales, biases, 128, 8, p0, words, True, use_simdgroup=c["simd"]), None
    if c["op"] == "resnorm":
        return ext.quantized_matmul_residual_norm(scales, biases, words, p0, residual, norm_w, eps)
    return ext.quantized_matmul_fused(scales, biases, words, p0, p1, residual, c["pro"], c["epi"], eps), None


def positions(N):
    """Needle columns: both ends of every group (128-byte box rows at 8 bits), the 16-byte chunk edges of the first
    group, and the last column."""
    pos = [p for g in range(N // 128) for p in (128 * g, 128 * g + 127)]
    return list(dict.fromkeys(pos + [16 * j + j % 16 for j in range(8)] + [N - 1]))


@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("c", [c for c in CASES if c["pro"] == NONE and c["epi"] in (ENONE, ERES)], ids=lambda c: f"{c['op']}-M{c['M']}-{c['route']}-e{c['epi']}")
def test_exact_probes(dev, c, dtype):
    g = torch.Generator().manual_seed(c["M"] * 7 + c["K"])
    res = c["epi"] == ERES or c["op"] == "resnorm"
    words, scales, biases, p0, residual, want = w8.exact_probes8(c["M"], c["N"], c["K"], dtype, g, positions(c["N"]), residual=res)
    words, scales, biases, p0 = words.to(dev), scales.to(dev), biases.to(dev), p0.to(dev)
    residual = None if residual is None else residual.to(dev)
    route(c, words, scales, biases, p0, dtype)
    norm_w = torch.ones(c["K"], dtype=dtype, device=dev) if c["op"] == "resnorm" else None
    out, _ = run(c, words, scales, biases, p0, residual=residual, norm_w=norm_w)
    wr.assert_exact(out.cpu(), want, f"{c['route']} exact probe")


def rand_inputs(c, dtype, g, dev):
    M, N, K = c["M"], c["N"], c["K"]
    codes = torch.randint(0, 256, (K, N), generator=g)
    # bias-dominated weights, small enough that a SwiGLU of two projections stays within fp16's range
    scales = (torch.rand(K, N // 128, generator=g) * 0.002 + 1e-4).to(dtype)
    biases = ((torch.rand(K, N // 128, generator=g) - 0.5) * 0.2).to(dtype)
    p0 = (torch.randn(M, N, generator=g) + 0.5).to(dtype)                   # a common activation mean
    p1 = None
    if c["pro"] == RMS:
        p1 = (1 + 0.1 * torch.randn(N, generator=g)).to(dtype)
    elif c["pro"] == SWI:
        p1 = torch.randn(M, N, generator=g).to(dtype)
    residual = torch.randn(M, K, generator=g).to(dtype) if c["epi"] == ERES or c["op"] == "resnorm" else None
    words = w8.pack_codes8(codes)
    return [None if t is None else t.to(dev) for t in (words, scales, biases, p0, p1, residual)]


@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_random_inputs_within_the_error_bound(dev, c, dtype):
    g = torch.Generator().manual_seed(c["M"] * 31 + c["K"] + c["pro"] * 3 + c["epi"])
    words, scales, biases, p0, p1, residual = rand_inputs(c, dtype, g, dev)
    r = route(c, words, scales, biases, p0, dtype)
    eps = 1e-6
    norm_w = (1 + 0.1 * torch.randn(c["K"], generator=g)).to(dtype).to(dev) if c["op"] == "resnorm" else None
    out, normed = run(c, words, scales, biases, p0, p1, residual, eps, norm_w)
    W = w8.weights8(words, scales, biases, rounded=c["route"] in ("skinny", "tiles"))
    ref = wr.reference(W, p0, p1=p1, prologue=c["pro"], epilogue=c["epi"], residual=residual, eps=eps, norm_weight=norm_w, norm_eps=1e-6)
    b = w8.error_bound(ref, W, c["route"], splits=r[1], gb_per_split=r[2])
    wr.assert_within(out, b.pre, b.tol, f"{c['route']} output")
    if normed is not None:
        wr.assert_within(normed, b.normed_pre, b.normed_tol, f"{c['route']} normed")


def test_the_cases_reach_every_8bit_route(dev):
    A = torch.empty(16, dtype=torch.uint8, device=dev)
    reached = set()
    for c in CASES:
        r = ext.quantized_matmul_route(c["M"], c["N"], c["K"], c["N"], c["pro"], c["op"] != "qmm", c["simd"], BF16, A, A, A, A, bits=8)
        assert PATHS[r[0]] == c["route"]
        reached.add(c["route"])
        if c["route"] == "skinny" and c["op"] == "qmm":
            assert r[1] > 1, "the skinny cases run split reductions"
        if c["route"] == "stream":
            assert r[4] == 1, "8-bit units hold one group"
    assert reached == {"vanilla", "stream", "skinny", "tiles"}
    rpp = {ext.quantized_matmul_route(M, 512, 384, 512, RMS, True, True, BF16, A, A, A, A, bits=8)[3] for M in (1, 2, 4, 8, 16, 40)}
    assert rpp == {1, 2, 4, 8, 16, 32}


@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
def test_embedding_rows_are_exact(dev, dtype):
    g = torch.Generator().manual_seed(3)
    vocab, dim = 300, 512
    codes = torch.randint(0, 256, (vocab, dim), generator=g)
    codes[:, ::37] = torch.tensor(w8.PROBE_CODES)[torch.arange(vocab) % 4][:, None]
    words = w8.pack_codes8(codes)
    scales = (torch.randn(vocab, dim // 128, generator=g) * 0.01).to(dtype)
    biases = torch.randn(vocab, dim // 128, generator=g).to(dtype)
    ids = torch.tensor([0, 299, 5, -1, 300, 127, 128, 255], dtype=torch.int32)
    got = ext.quantized_embedding(ids.to(dev), scales.to(dev), biases.to(dev), words.to(dev), 128, 8)
    assert torch.equal(got.cpu(), w8.embedding_ref(words, scales, biases, ids))


def test_qkv_project_rope_append_equals_the_two_calls(dev):
    """The composite at 8 bits (split planes at 9..128 rows, q|k|v scratch below) against quantized_matmul_fused then
    decode_qk_norm_rope_append, bit for bit."""
    g = torch.Generator().manual_seed(11)
    Hq, Hkv, D, N, page = 4, 2, 128, 512, 16
    K = (Hq + 2 * Hkv) * D
    words = w8.pack_codes8(torch.randint(0, 256, (K, N), generator=g)).to(dev)
    scales = (torch.rand(K, N // 128, generator=g) * 0.01).to(BF16).to(dev)
    biases = ((torch.rand(K, N // 128, generator=g) - 0.5) * 1.0).to(BF16).to(dev)
    qn = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16).to(dev)
    kn = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16).to(dev)
    for rows in (4, 24):
        p0 = torch.randn(rows, N, generator=g).to(BF16).to(dev)
        pages = rows * 2  # two pages of its own per row
        offsets = (torch.arange(rows, dtype=torch.int32, device=dev) * 3) % (2 * page)
        table = torch.arange(pages, dtype=torch.int32, device=dev).view(rows, 2)
        ctx = offsets + 1
        outs = []
        for fused in (True, False):
            kp = torch.zeros(pages, Hkv, page, D, dtype=BF16, device=dev)
            vp = torch.zeros_like(kp)
            if fused:
                q = ext.qkv_project_rope_append(scales, biases, words, p0, qn, kn, offsets, table, ctx, kp, vp, Hq, Hkv, 1e6, 1e-6)
            else:
                qkv = ext.quantized_matmul_fused(scales, biases, words, p0)
                q = ext.decode_qk_norm_rope_append(qkv, qn, kn, offsets, table, ctx, kp, vp, Hq, Hkv, 1e6, 1e-6)
            outs.append((q, kp, vp))
        for a, b in zip(*outs):
            assert torch.equal(a, b), f"rows {rows}"


def test_w8_and_w4_entries_refuse_widths_they_do_not_hold(dev):
    x = torch.randn(2, 256, dtype=BF16, device=dev)
    s = torch.ones(64, 2, dtype=BF16, device=dev)
    w6 = torch.zeros(64, 256 * 6 // 32, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError, match="4- or 8-bit"):
        ext.quantized_matmul_fused(s, s, w6, x)
    with pytest.raises(RuntimeError, match="bits must be 4 or 8"):
        ext.quantized_matmul(s, s, 128, 6, x, w6, True)
