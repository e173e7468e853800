"""The float64 W8A16 reference (tests/w8a16_ref.py), its error bound and the 8-bit exact probes, on the CPU.

An fp32 emulation of the 8-bit scalar kernel (sequential fma loop) and of the 8-bit streaming kernel (each code split
into nibbles, two shifted nibble sums per group combined as fma(16, d_h, d_l), summed in real fp32) must stay within
``w8a16_ref.error_bound`` on random and adversarial inputs, and be bit-exact on the probes of
``w4a16_ref.exact_probes(..., bits=8)``.  Kernels with a defect only 8-bit code has (codes >= 128 decoded as q - 128,
nibbles swapped, the high nibble weighted 8, the two 64-byte halves of a box row swapped) or any width has (a
neighbouring group's scale and bias, feature rows shifted at a tile edge, gate and up swapped) are simulated by the
reference on altered weights: the probe check must fail on each."""

import functools
import importlib.util
import sys
from dataclasses import replace
from pathlib import Path

import numpy as np
import pytest
import torch


def _load(name, file):
    """The helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


w8 = _load("tiny_llm_b200_w8a16_ref", "w8a16_ref.py")
wr = w8.wr
host4 = _load("tiny_llm_b200_w4a16_ref_host", "test_w4a16_ref_host.py")
BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
DTYPES = pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
activations = host4.activations


def rand_packed8(K, N, g, dtype, bias_scale=1.0):
    """Uniform 8-bit codes with scales and biases that give the weights of rand_packed (zero-centred codes); bias_scale
    > 1 makes the biases dominate the weights."""
    sigma = 1.0 / (4.717 * N**0.5)
    words = w8.pack_codes8(torch.randint(0, 256, (K, N), generator=g))
    scales = (torch.randn(K, N // 128, generator=g) * sigma / 17).to(dtype)
    biases = ((-127.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma) * bias_scale).to(dtype)
    return words, scales, biases


def fp32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32)


def emulate_vanilla8(words, scales, biases, a):
    """w4a16_vanilla_kernel<T, 8>: sum = fma(fma(code, s, b), a, sum) in fp32, codes in byte order (code * s is exact, so
    one rounding of the float64 value is the fma)."""
    q = w8.unpack_codes8(words).numpy().astype(np.float64)
    K, N = q.shape
    s = np.repeat(scales.double().numpy(), 128, axis=1)
    b = np.repeat(biases.double().numpy(), 128, axis=1)
    w = fp32(q * s + b).astype(np.float64)
    x = a.double().numpy()
    acc = np.zeros((x.shape[0], K), dtype=np.float32)
    for n in range(N):
        acc = fp32(acc.astype(np.float64) + w[None, :, n] * x[:, None, n])  # w a is exact in float64
    return torch.from_numpy(acc.astype(np.float64))


def group_sums(x):
    """sum(a) of every 128-column group as w4_stage forms it: per 8-element chunk ((e0 + e1) + (e2 + e3)) + ((e4 + e5) +
    (e6 + e7)), then a half-warp butterfly over the 16 chunks (xor 8, 4, 2, 1).  x [M, N] float32 -> [M, N/128]."""
    M, N = x.shape
    e = x.reshape(M, N // 128, 16, 8)
    c = ((e[..., 0] + e[..., 1]) + (e[..., 2] + e[..., 3])) + ((e[..., 4] + e[..., 5]) + (e[..., 6] + e[..., 7]))
    for sh in (8, 4, 2, 1):
        c = c + c[..., np.arange(16) ^ sh]
    return c[..., 0]


def emulate_stream8(words, scales, biases, a, dtype, dh_weight=16.0):
    """w8_consume with a sequential fp32 sum in place of the MMA: per group, for each nibble h and l
    d = -SHIFT * sum(a) + sum (SHIFT + nibble) a (the shift as the first accumulator input), then
    acc = fma(b, sum(a), fma(s, fma(16, d_h, d_l), acc))."""
    B = np.float32(wr.SHIFT[dtype])
    q = w8.unpack_codes8(words).numpy()
    K, N = q.shape
    nib = {"h": (q >> 4).astype(np.float32), "l": (q & 15).astype(np.float32)}
    s, b = scales.double().numpy(), biases.double().numpy()
    x = a.float().numpy()
    M = x.shape[0]
    asums = group_sums(x)
    acc = np.zeros((M, K), dtype=np.float32)
    for grp in range(N // 128):
        asum = asums[:, grp]
        d = {}
        for key, v in nib.items():
            dk = np.broadcast_to((-B * asum)[:, None], (M, K)).astype(np.float32)
            for n in range(128 * grp, 128 * grp + 128):
                dk = (dk + ((B + v[None, :, n]) * x[:, None, n]).astype(np.float32)).astype(np.float32)  # products exact
            d[key] = dk.astype(np.float64)
        t = fp32(dh_weight * d["h"] + d["l"]).astype(np.float64)
        acc = fp32(s[None, :, grp] * t + acc)
        acc = fp32(b[None, :, grp] * asum[:, None].astype(np.float64) + acc)
    return torch.from_numpy(acc.astype(np.float64))


def test_group_sums_follow_the_staging_order():
    g = torch.Generator().manual_seed(5)
    x = (torch.randn(2, 256, generator=g) * 2.0 ** torch.randint(-12, 12, (2, 256), generator=g)).numpy()
    got = group_sums(x.astype(np.float32))
    assert np.allclose(got, x.reshape(2, 2, 128).astype(np.float64).sum(-1), rtol=1e-5, atol=1e-3)


def test_unpack_matches_the_byte_layout_of_the_probe_words():
    g = torch.Generator().manual_seed(6)
    pos = wr.probe_positions(256)
    p = wr.exact_probes(4, 256, 32, BF16, g, pos, bits=8)
    codes = w8.unpack_codes8(p.words)
    assert torch.equal(codes, w8.unpack_codes8(w8.pack_codes8(codes)))
    assert int(codes.max()) <= 255 and p.words.shape == (32, 64)


# ------------------------------------------------------------------- bound --
def stream8_share(r, W, emu):
    """The smallest factor on the W4 scale coefficient that covers the emulation's accumulation error, over
    STREAM8_SCALE: (max over outputs of (error - bias part) / scale part at factor 1) / 18."""
    err = (emu - r.acc).abs()
    e_bias = wr.accumulation_error(r, replace(W, abs_s=torch.zeros_like(W.abs_s)), "stream")
    e_scale = wr.accumulation_error(r, replace(W, abs_b=torch.zeros_like(W.abs_b)), "stream")
    return float(((err - e_bias).clamp(min=0) / e_scale).max()) / w8.STREAM8_SCALE


@functools.lru_cache(maxsize=None)
def bound_case(dtype, mode):
    """(max error / bound of the scalar and the streaming emulation, share of STREAM8_SCALE the streaming one needs)."""
    g = torch.Generator().manual_seed(11 + len(mode))
    M, N, K = 3, 1024, 64
    words, scales, biases = rand_packed8(K, N, g, dtype, bias_scale=64.0 if mode == "bias" else 1.0)
    a = activations(mode, M, N, g, dtype)
    W = w8.weights8(words, scales, biases, rounded=False)
    r = wr.reference(W, a)
    stream = emulate_stream8(words, scales, biases, a, dtype)
    ratios = []
    for path, emu in (("vanilla", emulate_vanilla8(words, scales, biases, a)), ("stream", stream)):
        b = w8.error_bound(r, W, path)
        ratios.append(wr.assert_within(wr.round_to(emu, dtype), b.pre, b.tol, f"{path} {mode}"))
    return ratios, stream8_share(r, W, stream)


MODES = pytest.mark.parametrize("mode", ["gauss", "mean", "bias"])


@DTYPES
@MODES
def test_bound_holds_for_fp32_emulations(dtype, mode):
    ratios, share = bound_case(dtype, mode)
    assert max(ratios) <= 1.0 and share <= 1.0


def test_share_of_the_stream8_scale_the_emulation_uses(capsys):
    """Prints how much of STREAM8_SCALE = 18 the emulated streaming kernel needs on each kind of input."""
    rows = {(str(dt).split(".")[-1], mode): bound_case(dt, mode) for dt in (BF16, F16) for mode in ("gauss", "mean", "bias")}
    with capsys.disabled():
        print("\n8-bit emulations (dtype, inputs: max error / bound scalar, streaming; share of STREAM8_SCALE used):")
        for key, (ratios, share) in sorted(rows.items()):
            print(f"  {key[0]:9s} {key[1]:6s} {ratios[0]:7.4f} {ratios[1]:7.4f} {share:7.4f}")
    assert max(share for _, share in rows.values()) <= 1.0


def test_shift_term_is_what_the_streaming_emulation_needs_in_f16():
    """With a common activation mean the factorisation's cancellation error exceeds the plain accumulation bound."""
    g = torch.Generator().manual_seed(3)
    M, N, K = 2, 1024, 64
    words, scales, biases = rand_packed8(K, N, g, F16)
    a = activations("mean", M, N, g, F16)
    W = w8.weights8(words, scales, biases, rounded=False)
    r = wr.reference(W, a)
    err = (emulate_stream8(words, scales, biases, a, F16) - r.acc).abs()
    plain = (2 * (N // 128) + 20) * wr.U * r.absacc
    assert bool((err > plain).any())
    assert bool((err <= wr.accumulation_error(r, replace(W, abs_s=W.abs_s * w8.STREAM8_SCALE), "stream")).all())


# ------------------------------------------------------------------ probes --
N_P, K_P = 1024, 256
BOUNDS = (384, 640)


def probe_case(dtype, prologue=wr.PRO_NONE, epilogue=wr.EPI_NONE, residual=False, seed=0, **kw):
    g = torch.Generator().manual_seed(seed)
    pos = wr.probe_positions(N_P, boundaries=BOUNDS)
    return wr.exact_probes(len(pos), N_P, K_P, dtype, g, pos, prologue=prologue, epilogue=epilogue, residual=residual, bits=8, **kw), g, pos


@DTYPES
def test_probes_are_exact_for_the_emulated_kernels(dtype):
    p, _, _ = probe_case(dtype, seed=1)
    assert any(len(e) == 3 for e in p.positions), "multi-entry rows"
    W = w8.weights8(p.words, p.scales, p.biases, rounded=False)
    r = wr.probe_reference(p, W)
    wr.assert_exact(wr.round_to(emulate_vanilla8(p.words, p.scales, p.biases, p.p0), dtype), r.out, "vanilla")
    wr.assert_exact(wr.round_to(emulate_stream8(p.words, p.scales, p.biases, p.p0, dtype), dtype), r.out, "stream")
    Wt = w8.weights8(p.words, p.scales, p.biases, rounded=True)
    assert torch.equal(Wt.w, W.w), "the tensor-core rounding must leave probe weights unchanged"


@DTYPES
@pytest.mark.parametrize("prologue", [wr.PRO_NONE, wr.PRO_RMSNORM, wr.PRO_SWIGLU], ids=["none", "rmsnorm", "swiglu"])
@pytest.mark.parametrize("epilogue", [wr.EPI_NONE, wr.EPI_RESIDUAL, wr.EPI_SWIGLU_PAIRS], ids=["none", "residual", "pairs"])
def test_probes_hold_their_promise_for_every_form(dtype, prologue, epilogue):
    """probe_reference asserts that every accumulator, residual sum and gate * up product is a T number and that no
    prologue output is near a rounding midpoint; every needle column sees codes 0, 127, 128 and 255; the weights have at
    most 8 significant bits; a second round on the same weights (weights=, a row stride above N) keeps all of it."""
    res = epilogue == wr.EPI_RESIDUAL
    p, g, pos = probe_case(dtype, prologue, epilogue, residual=res, seed=2)
    W = w8.weights8(p.words, p.scales, p.biases, rounded=False)
    assert torch.equal(w8.weights8(p.words, p.scales, p.biases, rounded=True).w, W.w)
    codes = w8.unpack_codes8(p.words)
    for x in pos:
        assert set(codes[:, x].tolist()) == set(w8.PROBE_CODES), x
    r = wr.probe_reference(p, W, prologue=prologue, epilogue=epilogue)
    b = w8.error_bound(r, W, "stream")
    assert bool(((r.out - b.pre).abs() <= b.tol).all())
    if epilogue == wr.EPI_SWIGLU_PAIRS:
        assert bool((r.acc[:, wr.pairs_index(K_P // 2, r.acc.device)[0]] >= 32).any()), "some gates are open"
    M = 40
    again = wr.exact_probes(M, N_P, K_P, dtype, g, pos[M:] + pos[:M], prologue=prologue, epilogue=epilogue, residual=res,
                            lda=N_P + 64, weights=(p.words, p.scales, p.biases), bits=8)
    assert again.p0.stride(0) == N_P + 64
    wr.probe_reference(again, W, prologue=prologue, epilogue=epilogue)


@DTYPES
def test_probes_with_a_residual_use_large_residuals(dtype):
    """The residual of an 8-bit probe is chosen per output: it must not be all zeros or tiny."""
    p, _, _ = probe_case(dtype, epilogue=wr.EPI_RESIDUAL, residual=True, seed=3)
    W = w8.weights8(p.words, p.scales, p.biases, rounded=False)
    r = wr.probe_reference(p, W, epilogue=wr.EPI_RESIDUAL)
    ratio = r.residual.abs() / (r.acc.abs() + r.residual.abs()).clamp(min=1e-30)
    assert float((ratio > 0.5).double().mean()) > 0.25


# ------------------------------------------------------------- sensitivity --
def mutated_out(p, W, what, epilogue=wr.EPI_NONE):
    """The reference on the weights a defective kernel would use."""
    qi = w8.unpack_codes8(p.words)
    K, N = qi.shape
    G = N // 128
    q = qi.to(F64)
    s, b = p.scales.to(F64).clone(), p.biases.to(F64).clone()
    if what == "q-128":
        q = torch.where(qi >= 128, q - 128, q)
    elif what == "nibbles":
        q = ((qi & 15) * 16 + (qi >> 4)).to(F64)
    elif what == "dh-weight-8":
        q = ((qi >> 4) * 8 + (qi & 15)).to(F64)
    elif what == "neighbour-scale":
        s[:, 3], b[:, 3] = s[:, 4], b[:, 4]
    elif what == "box-halves":
        q = q.view(K, G, 2, 64).flip(2).reshape(K, N)
    w = (q.view(K, G, 128) * s[..., None] + b[..., None]).view(K, N)
    if what == "tile-edge":
        w[127] = W.w[128]
    elif what == "gate-up":
        w[0:8], w[8:16] = W.w[8:16].clone(), W.w[0:8].clone()
    Wm = wr.Weights(w, w.abs(), s.abs(), b.abs(), W.dtype, False)
    return wr.reference(Wm, p.p0, epilogue=epilogue, residual=p.residual).out


@DTYPES
@pytest.mark.parametrize("what", ["q-128", "nibbles", "dh-weight-8", "neighbour-scale", "box-halves", "tile-edge", "gate-up"])
def test_probe_check_catches_a_defective_kernel(dtype, what):
    epilogue = wr.EPI_SWIGLU_PAIRS if what == "gate-up" else wr.EPI_NONE
    p, _, _ = probe_case(dtype, epilogue=epilogue, seed=4)
    W = w8.weights8(p.words, p.scales, p.biases, rounded=False)
    want = wr.probe_reference(p, W, epilogue=epilogue).out
    wr.assert_exact(wr.reference(W, p.p0, epilogue=epilogue).out, want, "unchanged")
    with pytest.raises(AssertionError, match="differ from the exact probe result"):
        wr.assert_exact(mutated_out(p, W, what, epilogue), want, what)


@DTYPES
def test_the_streaming_emulation_with_the_high_nibble_weighted_8_fails_the_probes(dtype):
    """The same defect in the emulated arithmetic itself: fma(8, d_h, d_l)."""
    p, _, _ = probe_case(dtype, seed=5)
    W = w8.weights8(p.words, p.scales, p.biases, rounded=False)
    want = wr.probe_reference(p, W).out
    with pytest.raises(AssertionError, match="differ from the exact probe result"):
        wr.assert_exact(wr.round_to(emulate_stream8(p.words, p.scales, p.biases, p.p0, dtype, dh_weight=8.0), dtype), want, "dh 8")
