"""Every W4A16 projection kernel and fused form against a float64 reference (tests/w4a16_ref.py).

Each case states the kernel it must reach and the launch facts it exists for (split count and length, rows per pass,
columns per weight unit), checked through tl_quantized_matmul_route.  Then:
  * exact probes (power-of-two scales, integer biases, needle activations): every path must be bit-exact;
  * random inputs (Gaussian codes as in test_gpu_ops.rand_packed), a large common activation mean and bias-dominated
    weights: within error_bound, which has no absolute term.
The largest error/bound ratio and the largest error in output ulps per path and dtype are printed by the coverage test
at the end."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


def _load_w4a16_ref():
    """The helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    name = "tiny_llm_b200_w4a16_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("w4a16_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


wr = _load_w4a16_ref()

pytestmark = pytest.mark.gpu
BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
PATHS = {ext.W4_VANILLA: "vanilla", ext.W4_STREAM: "stream", ext.W4_SKINNY: "skinny", ext.W4_TILES: "tiles"}
NONE, RMS, SWI = wr.PRO_NONE, wr.PRO_RMSNORM, wr.PRO_SWIGLU
ENONE, ERES, EPAIRS = wr.EPI_NONE, wr.EPI_RESIDUAL, wr.EPI_SWIGLU_PAIRS
NORM_EPS = 1e-6
MAX_ROUNDS = 24
LM = 151936
STATS = {}  # (path, dtype, inputs) -> [max error / bound, max share of the accumulation bound, max output ulps, case]


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def case(name, op, M, N, K, route, pro=NONE, epi=ENONE, pad=0, simd=True, soff=0, facts=None, reaches=()):
    """op: "qmm" (quantized_matmul), "fused" (quantized_matmul_fused), "resnorm" (quantized_matmul_residual_norm).
    pad: row stride N + pad of the activations.  soff: the scales start 2 * soff bytes into their storage.  facts:
    a predicate on (splits, gb_per_split, rows_per_pass, units), the launch the case exists for."""
    return dict(name=name, op=op, M=M, N=N, K=K, route=route, pro=pro, epi=epi, pad=pad, simd=simd, soff=soff, facts=facts, reaches=reaches)


def split_facts(many=None, odd=None):
    def ok(s, gbps, rpp, u):
        return (many is None or (s > 1) == many) and (odd is None or (s > 1 and gbps % 2 == 1) == odd)
    return ok


def stream_facts(rpp, u=None):
    return lambda s, gbps, r, uu: r == rpp and (u is None or uu == u)


def odd_split_K(M, N, candidates=(2560, 2048, 3072, 1536, 4096, 1024)):
    """A feature count whose split reduction over N has an odd length (> 1 split), on this device's SM count: every
    second split then starts in the second half of a two-group TMA box.  2560 at N = 9728 on 132 SMs (6 splits of 13)."""
    A = 0x7F0000010000
    for K in candidates:
        _, s, gbps, _, _ = ext.quantized_matmul_route(M, N, K, N, NONE, False, True, BF16, A, A, A, A)
        if s > 1 and gbps % 2 == 1:
            return K
    return candidates[0]


CASES = [
    case("vanilla-ragged", "qmm", 3, 256, 40, "vanilla", simd=False, reaches=["vanilla ragged K"]),
    case("vanilla-2560", "qmm", 2, 2560, 130, "vanilla", simd=False),
    # streaming kernel
    case("stream-m1", "qmm", 1, 2560, 1024, "stream", facts=stream_facts(1, 2), reaches=["stream M=1", "stream U=2"]),
    case("stream-m2", "qmm", 2, 1024, 256, "stream", facts=stream_facts(2, 2), reaches=["stream M=2"]),
    case("stream-m3", "qmm", 3, 1024, 272, "stream", facts=stream_facts(4, 2), reaches=["stream M=3"]),
    case("stream-m5-k40", "qmm", 5, 2560, 40, "stream", facts=stream_facts(8, 2), reaches=["stream M=5", "stream K=40"]),
    case("stream-m8", "qmm", 8, 2560, 1030, "stream", facts=stream_facts(8, 2), reaches=["stream M=8"]),
    case("stream-n384", "qmm", 2, 384, 200, "stream", facts=stream_facts(2, 1), reaches=["stream U=1 N=384"]),
    case("stream-n1152", "qmm", 4, 1152, 100, "stream", facts=stream_facts(4, 1), reaches=["stream U=1 N=1152"]),
    case("stream-scales+2", "qmm", 2, 2560, 256, "stream", soff=1, facts=stream_facts(2, 1), reaches=["stream U=1 2-byte scales"]),
    case("stream-lda-m32", "fused", 32, 2560, 512, "stream", pad=8, facts=stream_facts(32, 1), reaches=["stream rpp 32 lda>N"]),
    case("stream-lda-m33", "fused", 33, 2560, 512, "stream", pad=64, facts=stream_facts(32, 1), reaches=["stream rpp 32 two passes"]),
    case("stream-9728-m16", "fused", 16, 9728, 320, "stream", pro=SWI, facts=stream_facts(8, 2), reaches=["stream rpp 8 two passes"]),
    case("stream-9728-m17", "fused", 17, 9728, 320, "stream", pro=SWI, facts=stream_facts(8, 1), reaches=["stream rpp 8 three passes"]),
    # streaming fused forms: every prologue x epilogue pair
    case("fused-none-res", "fused", 3, 2560, 512, "stream", epi=ERES, reaches=["stream none+residual"]),
    case("fused-none-pairs", "fused", 2, 1024, 512, "stream", epi=EPAIRS, reaches=["stream none+pairs"]),
    case("fused-rms-none", "fused", 2, 2560, 1024, "stream", pro=RMS, reaches=["stream rmsnorm+none"]),
    case("fused-rms-res", "fused", 4, 2560, 256, "stream", pro=RMS, epi=ERES, reaches=["stream rmsnorm+residual"]),
    case("fused-rms-pairs", "fused", 8, 2560, 2 * 9728, "stream", pro=RMS, epi=EPAIRS, reaches=["stream rmsnorm+pairs 2560->2x9728"]),
    case("fused-swi-none", "fused", 2, 1024, 256, "stream", pro=SWI, reaches=["stream swiglu+none"]),
    case("fused-swi-res", "fused", 4, 9728, 2560, "stream", pro=SWI, epi=ERES, reaches=["stream swiglu+residual"]),
    case("fused-swi-pairs", "fused", 3, 1024, 512, "stream", pro=SWI, epi=EPAIRS, reaches=["stream swiglu+pairs"]),
    case("fused-rms-m64", "fused", 64, 2560, 256, "stream", pro=RMS, pad=0, facts=stream_facts(32, 1), reaches=["stream prologue M>8"]),
    case("lmhead-stream-m1", "fused", 1, 2560, LM, "stream", pro=RMS, reaches=["lm head rmsnorm M=1"]),
    case("lmhead-stream-m8", "fused", 8, 2560, LM, "stream", pro=RMS, reaches=["lm head rmsnorm M=8"]),
    case("resnorm-stream", "resnorm", 4, 2560, 2560, "stream", reaches=["residual_norm stream"]),
    # swap-AB split-reduction kernel: every token-column width, one split and several
    case("skinny-m9", "qmm", 9, 2560, 1024, "skinny", facts=split_facts(many=True), reaches=["skinny NT16 M=9", "skinny splits"]),
    case("skinny-m16-odd", "qmm", 16, 9728, odd_split_K(16, 9728), "skinny", facts=split_facts(odd=True), reaches=["skinny NT16 M=16", "skinny odd split length"]),
    case("skinny-m17", "qmm", 17, 2560, 9728, "skinny", facts=split_facts(many=False), reaches=["skinny NT32 M=17", "skinny one split"]),
    case("skinny-m32", "qmm", 32, 1024, 3072, "skinny", reaches=["skinny NT32 M=32"]),
    case("skinny-m33", "qmm", 33, 2560, 1000, "skinny", facts=split_facts(many=True), reaches=["skinny NT64 M=33"]),
    case("skinny-m64", "qmm", 64, 4096, 2560, "skinny", reaches=["skinny NT64 M=64"]),
    case("skinny-m65", "qmm", 65, 2560, 1032, "skinny", reaches=["skinny NT128 M=65"]),
    case("skinny-m128", "qmm", 128, 2560, 1024, "skinny", reaches=["skinny NT128 M=128"]),
    case("skinny-res", "fused", 16, 2560, 1024, "skinny", epi=ERES, facts=split_facts(many=True), reaches=["skinny residual splits"]),
    case("skinny-res-1split", "fused", 24, 2560, 9728, "skinny", epi=ERES, facts=split_facts(many=False), reaches=["skinny residual one split"]),
    case("skinny-pairs", "fused", 64, 2560, 2 * 9728, "skinny", epi=EPAIRS, reaches=["skinny pairs"]),
    case("skinny-pairs-splits", "fused", 16, 9728, 512, "skinny", epi=EPAIRS, facts=split_facts(many=True), reaches=["skinny pairs splits"]),
    case("resnorm-reduce-norm", "resnorm", 16, 9728, 2560, "skinny", facts=split_facts(many=True), reaches=["residual_norm reduce_norm"]),
    case("resnorm-fallback", "resnorm", 16, 2560, 6144, "skinny", reaches=["residual_norm K=6144 fallback"]),
    case("lmhead-skinny-m16", "qmm", 16, 2560, LM, "skinny", reaches=["lm head skinny M=16"]),
    case("lmhead-skinny-m64", "qmm", 64, 2560, LM, "skinny", reaches=["lm head skinny M=64"]),
    # 128-token tiles
    case("tiles-m129", "qmm", 129, 1024, 520, "tiles", reaches=["tiles M=129"]),
    case("tiles-m255", "qmm", 255, 2560, 200, "tiles", reaches=["tiles M=255"]),
    case("tiles-m256", "qmm", 256, 1024, 136, "tiles", reaches=["tiles M=256"]),
    case("tiles-m257", "qmm", 257, 1024, 300, "tiles", reaches=["tiles M=257"]),
    case("tiles-m1000", "qmm", 1000, 2560, 1030, "tiles", reaches=["tiles M=1000 ragged K"]),
]
IDS = [c["name"] for c in CASES]
DTYPES = pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])


def place_scales(scales, soff):
    if not soff:
        return scales
    buf = torch.empty(scales.numel() + soff, dtype=scales.dtype, device=scales.device)
    buf[soff:].copy_(scales.reshape(-1))
    return buf[soff:].view(scales.shape)


def route_of(c, words, scales, biases, p0):
    return ext.quantized_matmul_route(c["M"], c["N"], c["K"], p0.stride(0), c["pro"], c["op"] != "qmm", c["simd"], p0.dtype, p0, words, scales,
                                      biases)


def run(c, words, scales, biases, p0, p1, residual, eps, norm_w):
    """The case's entry point; asserts the route and its facts first.  Returns (out, normed or None, route facts)."""
    r = route_of(c, words, scales, biases, p0)
    assert PATHS[r[0]] == c["route"], f"{c['name']}: reached {PATHS[r[0]]} {r[1:]}"
    if c["facts"] is not None:
        assert c["facts"](*r[1:]), f"{c['name']}: launch facts {r[1:]}"
    if c["op"] == "qmm":
        out, normed = ext.quantized_matmul(scales, biases, 128, 4, p0, words, True, use_simdgroup=c["simd"]), None
    elif c["op"] == "fused":
        out, normed = ext.quantized_matmul_fused(scales, biases, words, p0, p1, residual, c["pro"], c["epi"], eps), None
    else:
        out, normed = ext.quantized_matmul_residual_norm(scales, biases, words, p0, residual, norm_w, NORM_EPS)
    torch.cuda.synchronize()
    return out, normed, r


def epilogue(c):
    return ERES if c["op"] == "resnorm" else c["epi"]


def check_bound(c, dtype, W, ref, out, normed, r, label):
    """Asserts the bound and records (max error / bound; max share of the accumulation part of the bound used, i.e.
    (error - half an ulp) / (bound - half an ulp); max error in output ulps of the plain projections, over outputs not
    smaller than 1/8 of sum |a w|, where an output ulp measures the result and not a cancellation)."""
    b = wr.error_bound(ref, W, PATHS[r[0]], splits=r[1], gb_per_split=r[2])
    ratio = wr.assert_within(out, b.pre, b.tol, f"{c['name']} {label}")
    err = (out.to(F64) - b.pre).abs()
    hs = wr.spacing(b.pre, dtype) / 2
    share = float(torch.where(b.tol > hs, (err - hs).clamp(min=0) / (b.tol - hs), torch.zeros_like(err)).max())
    ul = 0.0
    if epilogue(c) == ENONE:
        big = b.pre.abs() >= ref.absacc / 8
        ul = float(torch.where(big, wr.ulps(out, b.pre, dtype), torch.zeros_like(err)).max())
    if normed is not None:
        ratio = max(ratio, wr.assert_within(normed, b.normed_pre, b.normed_tol, f"{c['name']} {label} normed"))
    key = (PATHS[r[0]], str(dtype).split(".")[-1], label)
    old = STATS.get(key, [0.0, 0.0, 0.0, ""])
    STATS[key] = [max(old[0], ratio), max(old[1], share), max(old[2], ul), c["name"] if share > old[1] else old[3]]


@pytest.mark.parametrize("c", CASES, ids=IDS)
@DTYPES
def test_exact_probes(dev, c, dtype):
    M, N, K = c["M"], c["N"], c["K"]
    g = torch.Generator().manual_seed(len(c["name"]) * 131 + M + (dtype == F16))
    path_route = c["route"]
    splits = 1
    if path_route == "skinny":
        A = 0x7F0000010000
        _, splits, gbps, _, _ = ext.quantized_matmul_route(M, N, K, N, NONE, c["op"] != "qmm", True, dtype, A, A, A, A)
    bounds = [k * gbps * 128 for k in range(1, splits)] if splits > 1 else []
    pairs = epilogue(c) == EPAIRS
    full = not pairs and c["pro"] == NONE and -(-len(wr.probe_positions(N, bounds)) // M) <= MAX_ROUNDS
    positions = wr.probe_positions(N, bounds, full=full)
    kw = dict(prologue=c["pro"], epilogue=epilogue(c), residual=epilogue(c) == ERES, lda=N + c["pad"])
    weights, W = None, None
    norm_w = torch.ones(K, dtype=dtype, device=dev) if c["op"] == "resnorm" else None
    for rnd in range(min(MAX_ROUNDS, -(-len(positions) // M))):
        pos = positions[rnd * M :] + positions[: rnd * M]
        p = wr.exact_probes(M, N, K, dtype, g, pos, weights=weights, **kw)
        if weights is None:
            weights = (p.words.to(dev), place_scales(p.scales.to(dev), c["soff"]), p.biases.to(dev))
            W = wr.Weights.build(*weights, rounded=path_route in ("skinny", "tiles"))
        p0 = p.p0.to(dev) if c["pad"] == 0 else place_rows(p.p0, N + c["pad"], dev)
        p1 = None if p.p1 is None else (p.p1.to(dev) if p.p1.dim() == 1 or c["pad"] == 0 else place_rows(p.p1, N + c["pad"], dev))
        res = None if p.residual is None else p.residual.to(dev)
        out, normed, r = run(c, *weights, p0, p1, res, p.eps, norm_w)
        p.p0, p.p1, p.residual = p0, p1, res
        ref = wr.probe_reference(p, W, prologue=c["pro"], epilogue=epilogue(c), norm_weight=norm_w, norm_eps=NORM_EPS)
        wr.assert_exact(out, ref.out, f"{c['name']} {dtype} probe round {rnd} (rows' positions {p.positions[:4]}...)")
        if normed is not None:
            b = wr.error_bound(ref, W, PATHS[r[0]], splits=r[1], gb_per_split=r[2])
            wr.assert_within(normed, b.normed_pre, b.normed_tol, f"{c['name']} probe normed")


def place_rows(x, lda, dev):
    """x [M, N] stored with row stride lda (a view into a wider buffer)."""
    M, N = x.shape
    buf = torch.full((M, lda), float("nan"), dtype=x.dtype, device=dev)
    buf[:, :N].copy_(x)
    return buf[:, :N]


def rand_packed(K, N, g, dtype, bias_scale=1.0):
    sigma = 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
    scales = (torch.randn(K, N // 128, generator=g) * sigma).to(dtype)
    biases = ((-7.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma) * bias_scale).to(dtype)
    return words, scales, biases


@pytest.mark.parametrize("c", CASES, ids=IDS)
@DTYPES
def test_random_and_adversarial_inputs(dev, c, dtype):
    M, N, K = c["M"], c["N"], c["K"]
    for mode in ("gauss", "mean", "bias"):
        g = torch.Generator().manual_seed(len(c["name"]) * 17 + len(mode) + (dtype == F16))
        words, scales, biases = rand_packed(K, N, g, dtype, bias_scale=16.0 if mode == "bias" else 1.0)
        words, scales, biases = words.to(dev), place_scales(scales.to(dev), c["soff"]), biases.to(dev)
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
        W = wr.Weights.build(words, scales, biases, rounded=c["route"] in ("skinny", "tiles"))
        ref = wr.reference(W, p0, p1=p1, prologue=c["pro"], epilogue=epilogue(c), residual=res, eps=eps, norm_weight=norm_w, norm_eps=NORM_EPS)
        check_bound(c, dtype, W, ref, out, normed, r, mode)
        del W, ref
        torch.cuda.empty_cache()


# ----------------------------------------------------------- shim validation --
def test_fused_forms_refuse_strided_weights(dev):
    """A strided view of b, scales or biases would be read as row-major: refused like quantized_matmul does."""
    g = torch.Generator().manual_seed(9)
    words, scales, biases = (t.to(dev) for t in rand_packed(64, 256, g, BF16))
    a = torch.randn(2, 256, generator=g).to(BF16).to(dev)
    res = torch.zeros(2, 64, dtype=BF16, device=dev)
    def strided(t):  # the same values with a column stride of 2
        v = torch.stack([t, t], dim=-1)[..., 0]
        assert not v.is_contiguous() and torch.equal(v, t)
        return v

    bad = dict(b=strided(words), scales=strided(scales), biases=strided(biases))
    for name, t in bad.items():
        args = dict(b=words, scales=scales, biases=biases)
        args[name] = t
        with pytest.raises(RuntimeError, match=f"{name} must be contiguous"):
            ext.quantized_matmul_fused(args["scales"], args["biases"], args["b"], a)
        with pytest.raises(RuntimeError, match=f"{name} must be contiguous"):
            ext.quantized_matmul_residual_norm(args["scales"], args["biases"], args["b"], a, res, torch.ones(64, dtype=BF16, device=dev), 1e-6)


# ---------------------------------------------------------------- coverage --
REQUIRED = {
    "vanilla ragged K", "stream M=1", "stream M=2", "stream M=3", "stream M=5", "stream M=8", "stream U=1 N=384", "stream U=1 N=1152",
    "stream U=1 2-byte scales", "stream U=2", "stream rpp 32 lda>N", "stream rpp 32 two passes", "stream rpp 8 two passes",
    "stream rpp 8 three passes", "stream K=40", "stream none+residual", "stream none+pairs", "stream rmsnorm+none", "stream rmsnorm+residual",
    "stream rmsnorm+pairs 2560->2x9728", "stream swiglu+none", "stream swiglu+residual", "stream swiglu+pairs", "lm head rmsnorm M=1",
    "lm head rmsnorm M=8", "skinny NT16 M=9", "skinny NT16 M=16", "skinny NT32 M=17", "skinny NT32 M=32", "skinny NT64 M=33",
    "skinny NT64 M=64", "skinny NT128 M=65", "skinny NT128 M=128", "skinny splits", "skinny one split", "skinny odd split length",
    "skinny residual splits", "skinny pairs", "residual_norm reduce_norm", "residual_norm K=6144 fallback", "lm head skinny M=16",
    "lm head skinny M=64", "tiles M=129", "tiles M=255", "tiles M=256", "tiles M=257", "tiles M=1000 ragged K",
}


def test_the_cases_reach_every_w4a16_path(dev, capsys):
    """Each case asserts its route and launch facts when it runs; this checks the same on the current device for the
    case table as a whole, that together the cases reach every required cell, and prints the error statistics the
    other tests collected (max error / bound, max error in output ulps against the unrounded reference)."""
    A = 0x7F0000010000
    reached = {}
    for c in CASES:
        r = ext.quantized_matmul_route(c["M"], c["N"], c["K"], c["N"] + c["pad"], c["pro"], c["op"] != "qmm", c["simd"], BF16, A, A,
                                       A + 2 * c["soff"], A)
        assert PATHS[r[0]] == c["route"], c["name"]
        assert c["facts"] is None or c["facts"](*r[1:]), (c["name"], r)
        if c["route"] == "skinny" and c["op"] == "resnorm" and "reduce_norm" in " ".join(c["reaches"]):
            assert r[1] > 1 and c["K"] <= 4096
        for label in c["reaches"]:
            reached.setdefault(label, c["name"])
    with capsys.disabled():
        print("\nW4A16 coverage:")
        for label in sorted(reached):
            print(f"  {label:36s} <- {reached[label]}")
        if STATS:
            print("W4A16 errors (path, dtype, inputs: max error/bound, max share of the accumulation bound, max output ulps of "
                  "plain projections, case with the largest share):")
            for key in sorted(STATS):
                ratio, share, ul, who = STATS[key]
                print(f"  {key[0]:8s} {key[1]:9s} {key[2]:6s} {ratio:7.4f} {share:7.4f} {ul:7.3f}  {who}")
    assert REQUIRED <= set(reached), sorted(REQUIRED - set(reached))
