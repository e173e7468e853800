"""Every 8-bit (W8A16) projection kernel and fused form against a float64 reference (tests/w8a16_ref.py).

Each case states the kernel it must reach and the launch facts it exists for (split count, length and cap, rows per
pass, one group per unit), checked through tl_quantized_matmul_route at bits = 8.  Then:
  * exact probes (w4a16_ref.exact_probes at bits = 8: codes 0, 127, 128 and 255 in every needle column, power-of-two
    scales, every prologue and epilogue, needles on every group offset and both sides of every split start): every path
    must be bit-exact (a dequantiser that is only right below 128 fails them);
  * random inputs, a large common activation mean and bias-dominated weights: within w8a16_ref.error_bound.
The largest error/bound ratio and the largest error in output ulps per path, dtype and inputs are printed by the
coverage test at the end.  Rows of the streaming kernel and of qkv_project_rope_append must not depend on how many rows
share the launch.  The embedding, the composite and the width refusals are checked too."""

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
NORM_EPS = 1e-6
MAX_ROUNDS = 24
LM = 151936
ADDR = 0x7F0000010000  # an aligned address for route queries
STATS = {}  # (path, dtype, inputs) -> [max error / bound, max output ulps, case with the largest ratio]


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def case(name, op, M, N, K, route, pro=NONE, epi=ENONE, pad=0, simd=True, facts=None, reaches=()):
    """op: "qmm" (quantized_matmul), "fused" (quantized_matmul_fused), "resnorm" (quantized_matmul_residual_norm).
    pad: row stride N + pad of the activations.  facts: a predicate on (splits, gb_per_split, rows_per_pass, units), the
    launch the case exists for."""
    return dict(name=name, op=op, M=M, N=N, K=K, route=route, pro=pro, epi=epi, pad=pad, simd=simd, facts=facts, reaches=reaches)


def table_case(op, M, N, K, route, pro=NONE, epi=ENONE, simd=True):
    """A case named by its shape (op-M-N-K-route-p<prologue>e<epilogue>); its exact-probe test keeps the shorter id
    op-M-route-e<epilogue> where that is unique (no prologue, a plain or residual epilogue)."""
    c = case(f"{op}-M{M}-N{N}-K{K}-{route}-p{pro}e{epi}", op, M, N, K, route, pro, epi, simd=simd)
    if pro == NONE and epi in (ENONE, ERES):
        c["probe_id"] = f"{op}-M{M}-{route}-e{epi}"
    return c


def route8(M, N, K, lda=None, pro=NONE, fused=False, simd=True, dtype=BF16):
    return ext.quantized_matmul_route(M, N, K, N if lda is None else lda, pro, fused, simd, dtype, ADDR, ADDR, ADDR, ADDR, bits=8)


def split_facts(N, many=None, ragged=None, cap=None):
    """many: more than one split; ragged: the last split is shorter (splits * gb_per_split > N / 128); cap: the split
    count is the policy's largest, min(16, groups / 2)."""
    G = N // 128

    def ok(s, gbps, rpp, u):
        return ((many is None or (s > 1) == many) and (ragged is None or (s > 1 and s * gbps > G) == ragged)
                and (cap is None or (s == min(16, G // 2)) == cap))
    return ok


def stream_facts(rpp):
    return lambda s, gbps, r, u: r == rpp and u == 1  # 8-bit units hold one group


def split_K(M, N, facts, candidates=(2560, 2048, 3072, 1536, 4096, 1024, 512, 256)):
    """A feature count whose split reduction over N has the launch facts ``facts`` on this device's SM count (2560 at
    N = 9728 on 132 SMs: 6 splits of 13 groups, the last of 11; 512: the cap of 16 splits of 5, the last of 1); the
    first candidate otherwise, which the case's facts then refuse."""
    for K in candidates:
        if facts(*route8(M, N, K)[1:]):
            return K
    return candidates[0]


CASES = [
    case("vanilla-ragged", "qmm", 3, 256, 40, "vanilla", simd=False, reaches=["vanilla ragged K"]),
    case("vanilla-2560", "qmm", 2, 2560, 130, "vanilla", simd=False),
    # streaming kernel: rows per pass 1, 2, 4, 8 (plain entry), 16 and 32 (fused entry), ragged K
    case("stream-m1", "qmm", 1, 2560, 1024, "stream", facts=stream_facts(1), reaches=["stream M=1"]),
    case("stream-m2", "qmm", 2, 1024, 256, "stream", facts=stream_facts(2), reaches=["stream M=2"]),
    case("stream-m3", "qmm", 3, 1024, 272, "stream", facts=stream_facts(4), reaches=["stream M=3"]),
    case("stream-m5-k40", "qmm", 5, 2560, 40, "stream", facts=stream_facts(8), reaches=["stream M=5", "stream K=40"]),
    case("stream-m8-k1030", "qmm", 8, 2560, 1030, "stream", facts=stream_facts(8), reaches=["stream M=8", "stream K=1030"]),
    case("stream-rpp16", "fused", 16, 1024, 256, "stream", pro=RMS, facts=stream_facts(16), reaches=["stream rpp 16 one pass"]),
    case("stream-rpp16-m17", "fused", 17, 4096, 200, "stream", pro=RMS, facts=stream_facts(16), reaches=["stream rpp 16 short last pass"]),
    case("stream-lda-m32", "fused", 32, 2560, 512, "stream", pad=8, facts=stream_facts(32), reaches=["stream rpp 32 one pass", "stream lda>N"]),
    case("stream-lda-m33", "fused", 33, 2560, 520, "stream", pad=64, facts=stream_facts(32), reaches=["stream rpp 32 short last pass"]),
    case("stream-m160", "fused", 160, 512, 384, "stream", facts=stream_facts(32), reaches=["stream rpp 32 five passes"]),
    # streaming fused forms: every prologue x epilogue pair, and prologues over several passes
    case("fused-none-none", "fused", 3, 2560, 1030, "stream", reaches=["stream none+none"]),
    case("fused-none-res", "fused", 3, 2560, 520, "stream", epi=ERES, reaches=["stream none+residual"]),
    case("fused-none-pairs", "fused", 2, 1024, 512, "stream", epi=EPAIRS, reaches=["stream none+pairs"]),
    case("fused-rms-none", "fused", 2, 2560, 1024, "stream", pro=RMS, reaches=["stream rmsnorm+none"]),
    case("fused-rms-res", "fused", 4, 2560, 264, "stream", pro=RMS, epi=ERES, reaches=["stream rmsnorm+residual"]),
    case("fused-rms-pairs", "fused", 8, 2560, 2 * 9728, "stream", pro=RMS, epi=EPAIRS, reaches=["stream rmsnorm+pairs 2560->2x9728"]),
    case("fused-swi-none", "fused", 2, 1024, 40, "stream", pro=SWI, reaches=["stream swiglu+none"]),
    case("fused-swi-res", "fused", 4, 9728, 2560, "stream", pro=SWI, epi=ERES, reaches=["stream swiglu+residual"]),
    case("fused-swi-pairs", "fused", 3, 1024, 512, "stream", pro=SWI, epi=EPAIRS, reaches=["stream swiglu+pairs"]),
    case("fused-swi-res-m40", "fused", 40, 1024, 264, "stream", pro=SWI, epi=ERES, facts=stream_facts(32), reaches=["stream prologue two passes"]),
    case("fused-rms-pairs-m136", "fused", 136, 512, 256, "stream", pro=RMS, epi=EPAIRS, facts=stream_facts(32), reaches=["stream pairs five passes"]),
    case("lmhead-stream-m1-1024", "fused", 1, 1024, LM, "stream", pro=RMS, reaches=["lm head rmsnorm M=1 N=1024"]),
    case("lmhead-stream-m8-1024", "fused", 8, 1024, LM, "stream", pro=RMS, reaches=["lm head rmsnorm M=8 N=1024"]),
    case("lmhead-stream-m1-2560", "fused", 1, 2560, LM, "stream", pro=RMS, reaches=["lm head rmsnorm M=1 N=2560"]),
    case("lmhead-stream-m8-2560", "fused", 8, 2560, LM, "stream", pro=RMS, reaches=["lm head rmsnorm M=8 N=2560"]),
    case("resnorm-stream", "resnorm", 4, 2560, 2560, "stream", reaches=["residual_norm stream"]),
    # swap-AB split-reduction kernel (one group per packed box at 8 bits): both sides of every token-column width, one
    # split, several, a ragged last split and the split cap, its epilogues
    case("skinny-m9", "qmm", 9, 2560, 1024, "skinny", facts=split_facts(2560, many=True), reaches=["skinny NT16 M=9", "skinny splits"]),
    case("skinny-m16-ragged", "qmm", 16, 9728, split_K(16, 9728, split_facts(9728, ragged=True, cap=False)), "skinny",
         facts=split_facts(9728, ragged=True, cap=False), reaches=["skinny NT16 M=16", "skinny ragged last split"]),
    case("skinny-m16-cap", "qmm", 16, 9728, split_K(16, 9728, split_facts(9728, cap=True), (512, 256, 1024, 128)), "skinny",
         facts=split_facts(9728, cap=True), reaches=["skinny split cap"]),
    case("skinny-m17", "qmm", 17, 2560, 9728, "skinny", facts=split_facts(2560, many=False), reaches=["skinny NT32 M=17", "skinny one split"]),
    case("skinny-m32", "qmm", 32, 1024, 3072, "skinny", reaches=["skinny NT32 M=32"]),
    case("skinny-m33", "qmm", 33, 2560, 1000, "skinny", facts=split_facts(2560, many=True), reaches=["skinny NT64 M=33", "skinny K=1000"]),
    case("skinny-m64", "qmm", 64, 4096, 2560, "skinny", reaches=["skinny NT64 M=64"]),
    case("skinny-m65", "qmm", 65, 2560, 1032, "skinny", reaches=["skinny NT128 M=65"]),
    case("skinny-m128", "qmm", 128, 2560, 1024, "skinny", reaches=["skinny NT128 M=128"]),
    case("skinny-res", "fused", 16, 2560, 1024, "skinny", epi=ERES, facts=split_facts(2560, many=True), reaches=["skinny residual splits"]),
    case("skinny-res-1split", "fused", 24, 2560, 9728, "skinny", epi=ERES, facts=split_facts(2560, many=False), reaches=["skinny residual one split"]),
    case("skinny-pairs", "fused", 64, 2560, 2 * 9728, "skinny", epi=EPAIRS, facts=split_facts(2560, many=False), reaches=["skinny pairs one split"]),
    case("skinny-pairs-splits", "fused", 16, 9728, 512, "skinny", epi=EPAIRS, facts=split_facts(9728, many=True), reaches=["skinny pairs splits"]),
    case("resnorm-reduce-norm", "resnorm", 16, 9728, 2560, "skinny", facts=split_facts(9728, many=True), reaches=["residual_norm reduce_norm"]),
    case("resnorm-fallback", "resnorm", 16, 2560, 6144, "skinny", facts=split_facts(2560, many=True), reaches=["residual_norm K=6144 fallback"]),
    case("lmhead-skinny-m16", "qmm", 16, 2560, LM, "skinny", reaches=["lm head skinny M=16"]),
    case("lmhead-skinny-m64", "qmm", 64, 2560, LM, "skinny", reaches=["lm head skinny M=64"]),
    # 128-token tiles, ragged M and K
    case("tiles-m129", "qmm", 129, 1024, 520, "tiles", reaches=["tiles M=129"]),
    case("tiles-m255", "qmm", 255, 2560, 200, "tiles", reaches=["tiles M=255"]),
    case("tiles-m256", "qmm", 256, 1024, 136, "tiles", reaches=["tiles M=256"]),
    case("tiles-m257", "qmm", 257, 1024, 300, "tiles", reaches=["tiles M=257"]),
    case("tiles-m1000", "qmm", 1000, 2560, 1030, "tiles", reaches=["tiles M=1000 ragged K"]),
    # the first 8-bit case table, kept under its ids: rows per pass 1..8 and 16, 32 in five passes, every prologue x
    # epilogue at 4 and 136 rows, the split-reduction kernel at each token tile, 128-token tiles and the scalar kernel
    *[table_case("qmm", M, 512, 384, "stream") for M in (1, 2, 3, 4, 8)],
    table_case("fused", 16, 1024, 256, "stream", RMS),
    table_case("fused", 160, 512, 384, "stream"),
    *[table_case("fused", M, 512, 256, "stream", pro, epi) for M in (4, 136) for pro in (NONE, RMS, SWI) for epi in (ENONE, ERES, EPAIRS)],
    *[table_case("qmm", M, 4096, 1024, "skinny") for M in (9, 32, 64, 128)],
    *[table_case("fused", 24, 2560, 512, "skinny", NONE, epi) for epi in (ERES, EPAIRS)],
    table_case("resnorm", 24, 2560, 512, "skinny"),
    table_case("resnorm", 4, 512, 256, "stream"),
    table_case("qmm", 200, 1024, 384, "tiles"),
    table_case("qmm", 128 + 64 + 3, 512, 256, "tiles"),
    table_case("qmm", 3, 512, 256, "vanilla", simd=False),
]
IDS = [c["name"] for c in CASES]
PROBE_IDS = [c.get("probe_id", c["name"]) for c in CASES]
DTYPES = pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])


def run(c, words, scales, biases, p0, p1, residual, eps, norm_w):
    """The case's entry point; asserts the route and its facts first.  Returns (out, normed or None, route facts)."""
    r = ext.quantized_matmul_route(c["M"], c["N"], c["K"], p0.stride(0), c["pro"], c["op"] != "qmm", c["simd"], p0.dtype, p0, words,
                                   scales, biases, bits=8)
    assert PATHS[r[0]] == c["route"], f"{c['name']}: reached {PATHS[r[0]]} {r[1:]}"
    if c["facts"] is not None:
        assert c["facts"](*r[1:]), f"{c['name']}: launch facts {r[1:]}"
    if c["op"] == "qmm":
        out, normed = ext.quantized_matmul(scales, biases, 128, 8, p0, words, True, use_simdgroup=c["simd"]), None
    elif c["op"] == "fused":
        out, normed = ext.quantized_matmul_fused(scales, biases, words, p0, p1, residual, c["pro"], c["epi"], eps), None
    else:
        out, normed = ext.quantized_matmul_residual_norm(scales, biases, words, p0, residual, norm_w, NORM_EPS)
    torch.cuda.synchronize()
    return out, normed, r


def epilogue(c):
    return ERES if c["op"] == "resnorm" else c["epi"]


def place_rows(x, lda, dev):
    """x [M, N] stored with row stride lda (a view into a wider buffer)."""
    M, N = x.shape
    buf = torch.full((M, lda), float("nan"), dtype=x.dtype, device=dev)
    buf[:, :N].copy_(x)
    return buf[:, :N]


def check_bound(c, dtype, W, ref, out, normed, r, label):
    """Asserts the bound and records (max error / bound, max error in output ulps of the plain projections over outputs
    not smaller than 1/8 of sum |a w|, where an output ulp measures the result and not a cancellation)."""
    b = w8.error_bound(ref, W, PATHS[r[0]], splits=r[1], gb_per_split=r[2])
    ratio = wr.assert_within(out, b.pre, b.tol, f"{c['name']} {label}")
    ul = 0.0
    if epilogue(c) == ENONE:
        big = b.pre.abs() >= ref.absacc / 8
        ul = float(torch.where(big, wr.ulps(out, b.pre, dtype), torch.zeros_like(b.pre)).max())
    if normed is not None:
        ratio = max(ratio, wr.assert_within(normed, b.normed_pre, b.normed_tol, f"{c['name']} {label} normed"))
    key = (PATHS[r[0]], str(dtype).split(".")[-1], label)
    old = STATS.get(key, [0.0, 0.0, ""])
    STATS[key] = [max(old[0], ratio), max(old[1], ul), c["name"] if ratio > old[0] else old[2]]


@DTYPES
@pytest.mark.parametrize("c", CASES, ids=PROBE_IDS)
def test_exact_probes(dev, c, dtype):
    M, N, K = c["M"], c["N"], c["K"]
    g = torch.Generator().manual_seed(len(c["name"]) * 131 + M + (dtype == F16))
    splits, gbps = 1, N // 128
    if c["route"] == "skinny":
        _, splits, gbps, _, _ = route8(M, N, K, fused=c["op"] != "qmm", dtype=dtype)
    bounds = [k * gbps * 128 for k in range(1, splits)]
    pairs = epilogue(c) == EPAIRS
    full = not pairs and c["pro"] == NONE and -(-len(wr.probe_positions(N, bounds)) // M) <= MAX_ROUNDS
    positions = wr.probe_positions(N, bounds, full=full)
    kw = dict(prologue=c["pro"], epilogue=epilogue(c), residual=epilogue(c) == ERES, lda=N + c["pad"], bits=8)
    weights, W = None, None
    norm_w = torch.ones(K, dtype=dtype, device=dev) if c["op"] == "resnorm" else None
    for rnd in range(min(MAX_ROUNDS, -(-len(positions) // M))):
        pos = positions[rnd * M :] + positions[: rnd * M]
        p = wr.exact_probes(M, N, K, dtype, g, pos, weights=weights, **kw)
        if weights is None:
            weights = (p.words.to(dev), p.scales.to(dev), p.biases.to(dev))
            W = w8.weights8(*weights, rounded=c["route"] in ("skinny", "tiles"))
        p0 = p.p0.to(dev) if c["pad"] == 0 else place_rows(p.p0, N + c["pad"], dev)
        p1 = None if p.p1 is None else (p.p1.to(dev) if p.p1.dim() == 1 or c["pad"] == 0 else place_rows(p.p1, N + c["pad"], dev))
        res = None if p.residual is None else p.residual.to(dev)
        out, normed, r = run(c, *weights, p0, p1, res, p.eps, norm_w)
        p.p0, p.p1, p.residual = p0, p1, res
        ref = wr.probe_reference(p, W, prologue=c["pro"], epilogue=epilogue(c), norm_weight=norm_w, norm_eps=NORM_EPS)
        wr.assert_exact(out, ref.out, f"{c['name']} {dtype} probe round {rnd} (rows' positions {p.positions[:4]}...)")
        if normed is not None:
            b = w8.error_bound(ref, W, PATHS[r[0]], splits=r[1], gb_per_split=r[2])
            wr.assert_within(normed, b.normed_pre, b.normed_tol, f"{c['name']} probe normed")


def rand_packed8(K, N, g, dtype, bias_scale=1.0):
    """Uniform 8-bit codes, scales and biases giving the weights of the 4-bit rand_packed (zero-centred codes)."""
    sigma = 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (K, N // 4), dtype=torch.int64, generator=g).to(torch.int32)
    scales = (torch.randn(K, N // 128, generator=g) * sigma / 17).to(dtype)
    biases = ((-127.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma) * bias_scale).to(dtype)
    return words, scales, biases


@DTYPES
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_random_inputs_within_the_error_bound(dev, c, dtype):
    M, N, K = c["M"], c["N"], c["K"]
    for mode in ("gauss", "mean", "bias"):
        g = torch.Generator().manual_seed(len(c["name"]) * 17 + len(mode) + (dtype == F16))
        words, scales, biases = (t.to(dev) for t in rand_packed8(K, N, g, dtype, bias_scale=16.0 if mode == "bias" else 1.0))
        x = torch.randn(M, N, generator=g) + (8.0 if mode == "mean" else 0.0)
        p1 = None
        if c["pro"] == RMS:
            p1 = (1.0 + 0.1 * torch.randn(N, generator=g)).to(dtype).to(dev)
        elif c["pro"] == SWI:
            p1 = place_rows(torch.randn(M, N, generator=g).to(dtype), N + c["pad"], dev)
        p0 = place_rows(x.to(dtype), N + c["pad"], dev)
        res = torch.randn(M, K, generator=g).to(dtype).to(dev) if epilogue(c) == ERES else None
        norm_w = (1.0 + 0.1 * torch.randn(K, generator=g)).to(dtype).to(dev) if c["op"] == "resnorm" else None
        eps = 1e-5
        out, normed, r = run(c, words, scales, biases, p0, p1, res, eps, norm_w)
        W = w8.weights8(words, scales, biases, rounded=c["route"] in ("skinny", "tiles"))
        ref = wr.reference(W, p0, p1=p1, prologue=c["pro"], epilogue=epilogue(c), residual=res, eps=eps, norm_weight=norm_w, norm_eps=NORM_EPS)
        check_bound(c, dtype, W, ref, out, normed, r, mode)
        del W, ref
        torch.cuda.empty_cache()


# ----------------------------------------------------------- row identity --
@DTYPES
@pytest.mark.parametrize("pro", [NONE, RMS], ids=["plain", "rmsnorm"])
def test_streaming_rows_equal_their_one_row_launch(dev, dtype, pro):
    """Every row of an M-row launch of the 8-bit streaming kernel (M = 2..8: 2, 4 and 8 rows per pass) equals the
    1-row launch of that row, bit for bit: the grid, the (chunk, unit) split over warps and the one-group units do not
    depend on M, and neither does any row's arithmetic."""
    g = torch.Generator().manual_seed(21 + pro)
    N, K = 2560, 1030
    words, scales, biases = (t.to(dev) for t in rand_packed8(K, N, g, dtype))
    x = (torch.randn(8, N, generator=g) + 0.5).to(dtype).to(dev)
    norm_w = (1.0 + 0.1 * torch.randn(N, generator=g)).to(dtype).to(dev) if pro == RMS else None

    def launch(a):
        r = route8(a.shape[0], N, K, pro=pro, fused=pro != NONE, dtype=dtype)
        assert PATHS[r[0]] == "stream" and r[4] == 1, r
        if pro == NONE:
            return ext.quantized_matmul(scales, biases, 128, 8, a, words, True)
        return ext.quantized_matmul_fused(scales, biases, words, a, norm_w, None, RMS, ENONE, 1e-6)

    single = [launch(x[i : i + 1]) for i in range(8)]
    for M in range(2, 9):
        out = launch(x[:M].contiguous())
        for i in range(M):
            assert torch.equal(out[i], single[i][0]), f"M={M}: row {i} differs from its 1-row launch"


@pytest.mark.parametrize("T", [2, 5, 8])
def test_qkv_project_rope_append_rows_equal_single_row_calls(dev, T):
    """A T-row qkv_project_rope_append at 8 bits (T positions of one sequence past 4K tokens, as a speculative verify
    pass writes them) against T calls of one row each: the same q rows and the same K and V pages, bit for bit."""
    g = torch.Generator().manual_seed(40 + T)
    Hq, Hkv, D, N, page = 16, 8, 128, 1024, 16
    K = (Hq + 2 * Hkv) * D
    words, scales, biases = (t.to(dev) for t in rand_packed8(K, N, g, BF16))
    qn = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16).to(dev)
    kn = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16).to(dev)
    ctx0 = 4093
    pages = (ctx0 + T) // page + 1
    p0 = torch.randn(T, N, generator=g).to(BF16).to(dev)
    offsets = torch.arange(ctx0, ctx0 + T, dtype=torch.int32, device=dev)
    table = torch.arange(pages, dtype=torch.int32, device=dev).repeat(T, 1)
    ctx = offsets + 1
    assert PATHS[route8(T, N, K, fused=True)[0]] == "stream"
    kp = torch.zeros(pages, Hkv, page, D, dtype=BF16, device=dev)
    vp = torch.zeros_like(kp)
    q = ext.qkv_project_rope_append(scales, biases, words, p0, qn, kn, offsets, table, ctx, kp, vp, Hq, Hkv, 1e6, 1e-6)
    kp1, vp1 = torch.zeros_like(kp), torch.zeros_like(vp)
    for i in range(T):
        q1 = ext.qkv_project_rope_append(scales, biases, words, p0[i : i + 1], qn, kn, offsets[i : i + 1], table[i : i + 1], ctx[i : i + 1],
                                         kp1, vp1, Hq, Hkv, 1e6, 1e-6)
        assert torch.equal(q[i], q1[0]), f"T={T}: q row {i}"
    assert torch.equal(kp, kp1), f"T={T}: K pages"
    assert torch.equal(vp, vp1), f"T={T}: V pages"


# ------------------------------------------------------------ other entries --
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


# ---------------------------------------------------------------- coverage --
REQUIRED = {
    "vanilla ragged K", "stream M=1", "stream M=2", "stream M=3", "stream M=5", "stream M=8", "stream K=40", "stream K=1030",
    "stream rpp 16 one pass", "stream rpp 16 short last pass", "stream rpp 32 one pass", "stream rpp 32 short last pass", "stream lda>N",
    "stream none+none", "stream none+residual", "stream none+pairs", "stream rmsnorm+none", "stream rmsnorm+residual",
    "stream rmsnorm+pairs 2560->2x9728", "stream swiglu+none", "stream swiglu+residual", "stream swiglu+pairs", "lm head rmsnorm M=1 N=1024",
    "lm head rmsnorm M=8 N=1024", "lm head rmsnorm M=1 N=2560", "lm head rmsnorm M=8 N=2560", "residual_norm stream", "skinny NT16 M=9",
    "skinny NT16 M=16", "skinny NT32 M=17", "skinny NT32 M=32", "skinny NT64 M=33", "skinny NT64 M=64", "skinny NT128 M=65",
    "skinny NT128 M=128", "skinny splits", "skinny one split", "skinny ragged last split", "skinny split cap", "skinny residual splits",
    "skinny residual one split", "skinny pairs one split", "skinny pairs splits", "residual_norm reduce_norm", "residual_norm K=6144 fallback",
    "lm head skinny M=16", "lm head skinny M=64", "tiles M=129", "tiles M=255", "tiles M=256", "tiles M=257", "tiles M=1000 ragged K",
}


def test_the_cases_reach_every_8bit_route(dev, capsys):
    """Each case asserts its route and launch facts when it runs; this checks the same on the current device for the
    case table as a whole, that together the cases reach every required cell, and prints the error statistics the
    other tests collected (max error / bound, max error in output ulps against the unrounded reference)."""
    reached = {}
    for c in CASES:
        r = route8(c["M"], c["N"], c["K"], lda=c["N"] + c["pad"], pro=c["pro"], fused=c["op"] != "qmm", simd=c["simd"])
        assert PATHS[r[0]] == c["route"], c["name"]
        assert c["facts"] is None or c["facts"](*r[1:]), (c["name"], r)
        if c["route"] == "stream":
            assert r[4] == 1, (c["name"], "8-bit units hold one group")
        # reduce_norm holds rows up to 4096 features; above, rms_norm follows the reduction
        if "residual_norm reduce_norm" in c["reaches"]:
            assert r[1] > 1 and c["K"] <= 4096, c["name"]
        if "residual_norm K=6144 fallback" in c["reaches"]:
            assert r[1] > 1 and c["K"] > 4096, c["name"]
        for label in c["reaches"]:
            reached.setdefault(label, c["name"])
    with capsys.disabled():
        print(f"\nW8A16 coverage ({torch.cuda.get_device_name()}):")
        for label in sorted(reached):
            print(f"  {label:36s} <- {reached[label]}")
        if STATS:
            print("W8A16 errors (path, dtype, inputs: max error/bound, max output ulps of plain projections, case with the "
                  "largest ratio):")
            for key in sorted(STATS):
                ratio, ul, who = STATS[key]
                print(f"  {key[0]:8s} {key[1]:9s} {key[2]:6s} {ratio:7.4f} {ul:7.3f}  {who}")
    assert REQUIRED <= set(reached), sorted(REQUIRED - set(reached))
