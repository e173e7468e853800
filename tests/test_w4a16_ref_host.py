"""The float64 W4A16 reference (tests/w4a16_ref.py), its error bound and its exact probes, on the CPU.

An fp32 emulation of the scalar kernel (sequential loop) and of the streaming kernel (the shifted-code factorisation,
summed in real fp32) must stay within the bound on random and adversarial inputs, and be bit-exact on the probes.
Kernels with a defect (swapped nibbles, a neighbouring group's scale, a group dropped or counted twice, feature rows
shifted at a tile edge, gate and up swapped) are simulated by the reference on altered weights: the probe check must
fail on each."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch


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
BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
DTYPES = pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])


def rand_packed(K, N, g, dtype, sigma=None, bias_scale=1.0):
    """Gaussian codes as in test_gpu_ops.rand_packed; bias_scale > 1 makes the biases dominate the weights."""
    sigma = sigma if sigma is not None else 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
    scales = (torch.randn(K, N // 128, generator=g) * sigma).to(dtype)
    biases = ((-7.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma) * bias_scale).to(dtype)
    return words, scales, biases


def emulate_vanilla(words, scales, biases, a):
    """w4a16_vanilla_kernel: sum += (code * s + b) * a in fp32, codes in order."""
    q = wr.unpack_codes(words).numpy().astype(np.float32)
    K, N = q.shape
    s = np.repeat(scales.float().numpy(), 128, axis=1)
    b = np.repeat(biases.float().numpy(), 128, axis=1)
    w = (q * s + b).astype(np.float32)
    x = a.float().numpy()
    acc = np.zeros((x.shape[0], K), dtype=np.float32)
    for n in range(N):
        acc = (acc + (w[None, :, n] * x[:, None, n]).astype(np.float32)).astype(np.float32)
    return torch.from_numpy(acc.astype(np.float64))


def emulate_stream(words, scales, biases, a, dtype):
    """The streaming kernel's arithmetic with a sequential fp32 sum in place of the MMA: per group
    d = -SHIFT * sum(a) + sum (SHIFT + q) a, then acc = fma(b, sum(a), fma(s, d, acc))."""
    B = np.float32(wr.SHIFT[dtype])
    q = wr.unpack_codes(words).numpy().astype(np.float32)
    K, N = q.shape
    s, b = scales.double().numpy(), biases.double().numpy()
    x = a.float().numpy()
    M = x.shape[0]
    acc = np.zeros((M, K), dtype=np.float32)
    for grp in range(N // 128):
        cols = slice(128 * grp, 128 * grp + 128)
        asum = np.zeros(M, dtype=np.float32)
        for n in range(128 * grp, 128 * grp + 128):
            asum = (asum + x[:, n]).astype(np.float32)
        d = np.broadcast_to((-B * asum)[:, None], (M, K)).astype(np.float32)
        for n in range(cols.start, cols.stop):
            d = (d + ((B + q[None, :, n]) * x[:, None, n]).astype(np.float32)).astype(np.float32)
        acc = (s[None, :, grp] * d.astype(np.float64) + acc).astype(np.float32)  # fma: s * d is exact in float64
        acc = (b[None, :, grp] * asum[:, None].astype(np.float64) + acc).astype(np.float32)
    return torch.from_numpy(acc.astype(np.float64))


def activations(mode, M, N, g, dtype):
    a = torch.randn(M, N, generator=g)
    if mode == "mean":
        a = a + 30.0  # a large common mean: the worst case of the shifted factorisation
    return a.to(dtype)


@DTYPES
@pytest.mark.parametrize("mode", ["gauss", "mean", "bias"])
def test_bound_holds_for_fp32_emulations(dtype, mode):
    g = torch.Generator().manual_seed(7 + len(mode))
    M, N, K = 3, 1024, 64
    words, scales, biases = rand_packed(K, N, g, dtype, bias_scale=64.0 if mode == "bias" else 1.0)
    a = activations(mode, M, N, g, dtype)
    W = wr.Weights.build(words, scales, biases, rounded=False)
    r = wr.reference(W, a)
    for path, emu in (("vanilla", emulate_vanilla(words, scales, biases, a)), ("stream", emulate_stream(words, scales, biases, a, dtype))):
        b = wr.error_bound(r, W, path)
        got = wr.round_to(emu, dtype)
        ratio = wr.assert_within(got, b.pre, b.tol, f"{path} {mode}")
        assert ratio <= 1.0


def test_shift_term_is_what_the_streaming_emulation_needs_in_f16():
    """With a common activation mean the factorisation's cancellation error exceeds the plain accumulation bound."""
    g = torch.Generator().manual_seed(3)
    M, N, K = 2, 1024, 64
    words, scales, biases = rand_packed(K, N, g, F16)
    a = activations("mean", M, N, g, F16)
    W = wr.Weights.build(words, scales, biases, rounded=False)
    r = wr.reference(W, a)
    err = (emulate_stream(words, scales, biases, a, F16) - r.acc).abs()
    plain = (2 * (N // 128) + 20) * wr.U * r.absacc
    assert bool((err > plain).any())
    assert bool((err <= wr.accumulation_error(r, W, "stream")).all())


def test_round_to_is_one_correct_rounding():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(10000, generator=g, dtype=F64) * 2.0 ** torch.randint(-30, 10, (10000,), generator=g)
    for dtype in (BF16, F16):
        x32 = x.float()  # float32 inputs: torch's conversion rounds once
        assert torch.equal(wr.round_to(x32.double(), dtype), x32.to(dtype).double())
    # a float64 value just above a bf16 midpoint that float32 rounds onto the midpoint
    mid = 1.0 + 2.0**-8
    assert float(wr.round_to(torch.tensor([mid + 2.0**-40], dtype=F64), BF16)) == 1.0 + 2.0**-7


# ------------------------------------------------------------------------ probes --
N_P, K_P = 1024, 256


def probe_case(dtype, prologue=wr.PRO_NONE, epilogue=wr.EPI_NONE, residual=False, seed=0):
    g = torch.Generator().manual_seed(seed)
    pos = wr.probe_positions(N_P, boundaries=(384, 640))
    p = wr.exact_probes(len(pos), N_P, K_P, dtype, g, pos, prologue=prologue, epilogue=epilogue, residual=residual)
    return p


@DTYPES
def test_probes_are_exact_for_the_emulated_kernels(dtype):
    p = probe_case(dtype, seed=1)
    W = wr.Weights.build(p.words, p.scales, p.biases, rounded=False)
    r = wr.probe_reference(p, W)
    wr.assert_exact(wr.round_to(emulate_vanilla(p.words, p.scales, p.biases, p.p0), dtype), r.out, "vanilla")
    wr.assert_exact(wr.round_to(emulate_stream(p.words, p.scales, p.biases, p.p0, dtype), dtype), r.out, "stream")
    Wt = wr.Weights.build(p.words, p.scales, p.biases, rounded=True)
    assert torch.equal(Wt.w, W.w), "the tensor-core rounding must leave probe weights unchanged"


@DTYPES
@pytest.mark.parametrize("prologue", [wr.PRO_NONE, wr.PRO_RMSNORM, wr.PRO_SWIGLU], ids=["none", "rmsnorm", "swiglu"])
@pytest.mark.parametrize("epilogue", [wr.EPI_NONE, wr.EPI_RESIDUAL, wr.EPI_SWIGLU_PAIRS], ids=["none", "residual", "pairs"])
def test_probes_hold_their_promise_for_every_form(dtype, prologue, epilogue):
    """probe_reference asserts that every accumulator, residual sum and gate * up product is a T number and that no
    prologue output is near a rounding midpoint."""
    p = probe_case(dtype, prologue, epilogue, residual=epilogue == wr.EPI_RESIDUAL, seed=2)
    W = wr.Weights.build(p.words, p.scales, p.biases, rounded=False)
    r = wr.probe_reference(p, W, prologue=prologue, epilogue=epilogue)
    b = wr.error_bound(r, W, "stream")
    assert bool(((r.out - b.pre).abs() <= b.tol).all())


def test_probes_cover_every_nibble_word_and_boundary():
    pos = wr.probe_positions(N_P, boundaries=(384,))
    offs = {x % 128 for x in pos}
    assert offs == set(range(128))
    assert {0, 127, N_P - 128, N_P - 1, 383, 384} <= set(pos)
    assert {x // 128 for x in pos} == set(range(N_P // 128))
    few = wr.probe_positions(N_P, full=False)
    assert {(x % 128) // 8 for x in few} == set(range(16)) and {x % 8 for x in few} == set(range(8))


# ------------------------------------------------------------------- sensitivity --
def swap_nibbles_1_2(words):
    w = words.to(torch.int64) & 0xFFFFFFFF
    n1, n2 = (w >> 4) & 0x000F000F, (w >> 8) & 0x000F000F  # nibbles 1, 5 and 2, 6
    w = (w & ~0x0FF00FF0) | (n1 << 8) | (n2 << 4)
    return torch.where(w >= 2**31, w - 2**32, w).to(torch.int32)


def mutated_out(p, W, dtype, what, epilogue=wr.EPI_NONE):
    words, scales, biases = p.words.clone(), p.scales.clone(), p.biases.clone()
    if what == "nibbles":
        words = swap_nibbles_1_2(words)
    elif what == "neighbour-scale":
        scales[:, 3], biases[:, 3] = scales[:, 4], biases[:, 4]
    Wm = wr.Weights.build(words, scales, biases, rounded=False)
    w = Wm.w
    if what == "drop-group":
        w[:, 2 * 128 : 3 * 128] = 0
    elif what == "group-twice":
        w[:, 5 * 128 : 6 * 128] *= 2
    elif what == "tile-edge":
        w[127] = W.w[128]
    elif what == "gate-up":
        w[0:8], w[8:16] = W.w[8:16].clone(), W.w[0:8].clone()
    return wr.reference(Wm, p.p0, epilogue=epilogue, residual=p.residual).out


@DTYPES
@pytest.mark.parametrize("what", ["nibbles", "neighbour-scale", "drop-group", "group-twice", "tile-edge", "gate-up"])
def test_probe_check_catches_a_defective_kernel(dtype, what):
    epilogue = wr.EPI_SWIGLU_PAIRS if what == "gate-up" else wr.EPI_NONE
    p = probe_case(dtype, epilogue=epilogue, seed=4)
    W = wr.Weights.build(p.words, p.scales, p.biases, rounded=False)
    want = wr.probe_reference(p, W, epilogue=epilogue).out
    wr.assert_exact(wr.reference(W, p.p0, epilogue=epilogue).out, want, "unchanged")
    with pytest.raises(AssertionError, match="differ from the exact probe result"):
        wr.assert_exact(mutated_out(p, W, dtype, what, epilogue), want, what)
