"""Float64 W4A16 reference, the error bound the projection kernels are held to, and exact probes.

``reference`` restates ``tl_quantized_matmul``, ``tl_quantized_matmul_fused`` (every prologue x epilogue) and
``tl_quantized_matmul_residual_norm`` (include/tiny_llm_b200.h) in float64 on the inputs' device, keeping the rounding
points the header states:

    weights      exact on the scalar and streaming kernels; T(code * scale + bias) on the tensor-core kernels (skinny
                 M = 9..128, tiles M > 128): one rounding of the exact value (``Weights(rounded=True)``)
    prologue     a = T(x * rsqrt(mean(x^2) + eps) * w)  or  a = T(silu(g) * u)
    epilogue     T(acc);  T(res + T(acc));  pairs T(silu(T(gate)) * T(up))
    normed       T(x * rsqrt(mean(x^2) + eps) * w) of the ROUNDED residual stream x

Intermediate values are float64 values of T numbers.  ``error_bound`` derives an elementwise tolerance from the kernel's
accumulation structure (its docstring has the derivation); it has no absolute term.  ``exact_probes`` builds inputs on
which every kernel's fp32 arithmetic is exact, so every path must match the reference bit for bit.

A single-rounding conversion ``round_to`` is written out here: ``Tensor.to(bfloat16)`` from float64 goes through
float32, which rounds twice.
"""

from __future__ import annotations

from dataclasses import dataclass

import torch

F64 = torch.float64
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
U = 2.0**-24  # fp32 unit roundoff
_P = {BF16: 8, F16: 11, F32: 24}  # significand bits
_EMIN = {BF16: -126, F16: -14, F32: -126}
# The streaming kernel feeds code q to the tensor cores as the exact number SHIFT + q and subtracts SHIFT * sum(a)
# through the accumulator input (w4a16_item.cuh).
SHIFT = {BF16: 128.0, F16: 1024.0}
PRO_NONE, PRO_RMSNORM, PRO_SWIGLU = 0, 1, 2
EPI_NONE, EPI_RESIDUAL, EPI_SWIGLU_PAIRS = 0, 1, 2
SILU_SLOPE = 1.1  # max |silu'(x)| = 1.0998 (at x ~ 2.4)
SWIGLU_REL = 8 * U  # fp32 g / (1 + expf(-g)) * u: expf (2 ulp = 4u), 1 + e (u), the division and the product (2u)


# ------------------------------------------------------------------ rounding --
def spacing(x, dtype):
    """Distance between neighbouring T numbers at |x| (float64 in, float64 out; subnormals included)."""
    _, e = torch.frexp(x.abs())
    e = torch.clamp(e.to(torch.int64) - 1, min=_EMIN[dtype])
    return torch.ldexp(torch.ones_like(x), e - (_P[dtype] - 1))


def round_to(x, dtype):
    """T(x): x float64 rounded once to the nearest T number (ties to even), returned as float64."""
    q = spacing(x, dtype)
    return torch.round(x / q) * q


def spread(x, err, dtype):
    """How far T(y) can be from T(x) for any |y - x| <= err: 0 unless x lies within err of a rounding midpoint."""
    r = round_to(x, dtype)
    return torch.maximum(round_to(x + err, dtype) - r, r - round_to(x - err, dtype))


def ulps(got, ref, dtype):
    """|got - ref| in units of T's spacing at ref."""
    return (got.to(F64) - ref).abs() / spacing(ref, dtype)


# ------------------------------------------------------------------- weights --
def unpack_codes(words):
    """[K, N/8] packed words -> [K, N] uint8 codes; code i of a word is (w >> 4i) & 15."""
    K, W = words.shape
    out = torch.empty(K, W * 8, dtype=torch.uint8, device=words.device)
    shifts = 4 * torch.arange(8, device=words.device, dtype=torch.int64)
    for k0 in range(0, K, 8192):
        w = words[k0 : k0 + 8192].to(torch.int64) & 0xFFFFFFFF
        out[k0 : k0 + 8192] = ((w[..., None] >> shifts) & 15).reshape(-1, W * 8).to(torch.uint8)
    return out


@dataclass
class Weights:
    """Dequantised weights in float64 on the words' device: w [K, N] (exact, or rounded once to T), |w|, |scale| and
    |bias| [K, N/128]."""

    w: torch.Tensor
    absw: torch.Tensor
    abs_s: torch.Tensor
    abs_b: torch.Tensor
    dtype: torch.dtype
    rounded: bool

    @classmethod
    def build(cls, words, scales, biases, rounded):
        K, G = scales.shape
        s, b = scales.to(F64), biases.to(F64)
        w = torch.empty(K, G * 128, dtype=F64, device=words.device)
        for k0 in range(0, K, 8192):
            q = unpack_codes(words[k0 : k0 + 8192]).to(F64).view(-1, G, 128)
            wk = q * s[k0 : k0 + 8192, :, None] + b[k0 : k0 + 8192, :, None]  # exact: |bias| and |code * scale| are within 2^24
            w[k0 : k0 + 8192] = (round_to(wk, scales.dtype) if rounded else wk).view(-1, G * 128)
        return cls(w, w.abs(), s.abs(), b.abs(), scales.dtype, rounded)


# ----------------------------------------------------------------- reference --
@dataclass
class Ref:
    """Float64 results with the rounding points of the header, and the magnitudes ``error_bound`` needs."""

    out: torch.Tensor          # T-rounded result (float64 values of T numbers): what out must equal on exact probes
    acc: torch.Tensor          # [M, K] exact projection of the (rounded) prologue output
    absacc: torch.Tensor       # [M, K] sum_n |a_n| |w_n|
    gsum: torch.Tensor         # [M, N/128] sum over each group of |a_n|
    amb: torch.Tensor          # [M, K] sum_n |w_n| spread(a_n): prologue outputs within the fp32 error of a midpoint
    epilogue: int
    residual: torch.Tensor | None = None
    normed: torch.Tensor | None = None
    norm_weight: torch.Tensor | None = None
    norm_eps: float = 0.0


def rms64(x, w, eps):
    """x * rsqrt(mean(x^2) + eps) * w in float64, and the inverse norm per row."""
    inv = 1.0 / torch.sqrt((x * x).mean(dim=-1, keepdim=True) + eps)
    return x * inv * w, inv


def ss_chain(n):
    """Longest chain of fp32 additions in a sum of squares of n values: the staging step of the streaming kernel (8
    per 16-byte chunk, 4 shuffles per group, one per group), the reduce_norm kernel (16 per thread, two 5-level warp
    sums) and rms_norm (n / 32 per thread, two warp sums) all stay below n / 32 + 26."""
    return n / 32 + 26


def prologue64(p0, p1, prologue, eps, dtype):
    """(a, spread) : the prologue output rounded to T, and how far the kernel's rounding of its fp32 value may be from
    it.  fp32 error of the prologue value p, relative to |p|:
      RMSNORM: the sum of squares (ss_chain(N) + 1 roundings), / N and + eps (2), rsqrtf (2 ulp = 4u) halve and add
               to a relative error of inv below ((ss_chain + 3) / 2 + 4) u; the two products add 2u;
      SWIGLU : expf (2 ulp = 4u), 1 + e (u), the division and the product (2u): 8u."""
    x = p0.to(F64)
    if prologue == PRO_NONE:
        return x, torch.zeros_like(x)
    if prologue == PRO_RMSNORM:
        p, _ = rms64(x, p1.to(F64), eps)
        rel = ((ss_chain(x.shape[-1]) + 3) / 2 + 6) * U
    else:
        up = p1.to(F64)
        p = x / (1.0 + torch.exp(-x)) * up
        rel = SWIGLU_REL
    return round_to(p, dtype), spread(p, rel * p.abs(), dtype)


def pairs_index(K2, device):
    """Rows of the gate and up halves of activation j in the interleaved gate|up weight (blocks of 8)."""
    j = torch.arange(K2, device=device)
    gate = (j // 8) * 16 + j % 8
    return gate, gate + 8


def silu64(x):
    return x / (1.0 + torch.exp(-x))


def reference(W, p0, *, p1=None, prologue=PRO_NONE, epilogue=EPI_NONE, residual=None, eps=0.0, norm_weight=None, norm_eps=0.0):
    """W: ``Weights``; p0 [M, N] (any row stride); p1 the prologue's second operand (norm weight [N] or up [M, N]);
    residual [M, K] for EPI_RESIDUAL; norm_weight [K] for the residual_norm form (implies EPI_RESIDUAL)."""
    dtype = W.dtype
    a, delta = prologue64(p0, p1, prologue, eps, dtype)
    acc = a @ W.w.T
    absacc = a.abs() @ W.absw.T
    amb = delta @ W.absw.T if bool(delta.any()) else torch.zeros_like(acc)
    gsum = a.abs().reshape(a.shape[0], -1, 128).sum(-1)
    r = Ref(out=None, acc=acc, absacc=absacc, gsum=gsum, amb=amb, epilogue=epilogue)
    if norm_weight is not None:
        epilogue = r.epilogue = EPI_RESIDUAL
    if epilogue == EPI_NONE:
        r.out = round_to(acc, dtype)
    elif epilogue == EPI_RESIDUAL:
        r.residual = residual.to(F64)
        r.out = round_to(r.residual + round_to(acc, dtype), dtype)
    else:
        gi, ui = pairs_index(acc.shape[1] // 2, acc.device)
        g, u = round_to(acc[:, gi], dtype), round_to(acc[:, ui], dtype)
        r.out = round_to(silu64(g) * u, dtype)
    if norm_weight is not None:
        r.norm_weight, r.norm_eps = norm_weight.to(F64), norm_eps
        r.normed = round_to(rms64(r.out, r.norm_weight, norm_eps)[0], dtype)
    return r


# --------------------------------------------------------------------- bound --
def accumulation_error(r, W, path, splits=1, gb_per_split=None):
    """Bound on |acc_kernel - acc| before any epilogue rounding (see error_bound)."""
    N = W.w.shape[1]
    G = N // 128
    if path == "vanilla":
        E = (N + 2) * U * r.absacc
    elif path == "stream":
        B = SHIFT[W.dtype]
        chain = 2 * G + 20
        coef_s = (chain * 15 + 32 * (2 * B + 15) + 8 * B) * U
        coef_b = (chain + 8) * U
        E = r.gsum @ (coef_s * W.abs_s + coef_b * W.abs_b).T
    elif path in ("skinny", "tiles"):
        gbps = G if path == "tiles" else gb_per_split
        E = (3 * 8 * gbps + splits + 2) * U * r.absacc
    else:
        raise ValueError(path)
    return E + r.amb


@dataclass
class Bound:
    """Elementwise tolerances: |out_kernel - pre| <= tol (pre: the reference value before the final rounding)."""

    pre: torch.Tensor
    tol: torch.Tensor
    normed_pre: torch.Tensor | None = None
    normed_tol: torch.Tensor | None = None


def error_bound(r, W, path, splits=1, gb_per_split=None, norm_chain=None):
    """Tolerance for a kernel on ``path`` ("vanilla" | "stream" | "skinny" | "tiles"; splits / gb_per_split from
    tl_quantized_matmul_route for "skinny").  u = 2^-24; every fp32 addition is off by at most u times its result,
    an MMA addition (which may truncate) by 2u; a chain of n additions of terms t_i is off by at most n u sum |t_i|.

    Accumulation (acc = sum_n a_n w_n, S = sum_n |a_n| |w_n|):
      vanilla: one thread, (code * s + b) * a added sequentially over N: (N + 2) u S.
      stream : per 128-group g, d_g = SHIFT * (-sum_g a) + sum_g (SHIFT + q) a (eight m16n8k16 MMAs with the shift in
               the accumulator input; products exact, each MMA <= 3u of the magnitudes it adds, which are below
               (2 SHIFT + 15) sum_g |a|; the fp32 tree sum of a adds 8u sum_g |a| per SHIFT), then
               acc += s_g d_g + b_g sum_g a (two fmas) in a per-warp chain over the groups and one over 16 warps:
               (2G + 20) u sum_g (15 |s_g| + |b_g|) sum_g |a|  +  sum_g |s_g| (32 (2 SHIFT + 15) + 8 SHIFT) u sum_g |a|
               + 8u |b_g| sum_g |a|.  The shift term is the cancellation of the factorisation: it grows with a common
               activation mean and is 8x larger in f16 (SHIFT 1024) than in bf16 (128).
      skinny / tiles: weights rounded to T (exact in the reference), 8 wgmma k16 steps per group over gb_per_split groups
               per split (G on tiles), then the partial planes in split order: (24 gb_per_split + splits + 2) u S.
    Prologue: the kernel's T(a_n) may differ from the reference's where a_n lies within its fp32 error of a rounding
      midpoint (``prologue64``): + sum_n |w_n| spread(a_n), over exactly those n.
    Epilogue: T(acc) may differ where acc lies within E of a midpoint: spread(acc, E).  residual: + u |res + T(acc)|
      for the fp32 add.  pairs: silu is 1.1-Lipschitz, so the gate spread costs 1.1 |up| dg, the up spread |silu(g)| du,
      and expf, 1 + e, the division and the product 8u |silu(g) up|; below gate = -87, where silu(gate) leaves fp32's
      normal range, |silu(g) up| itself.
    normed: x may differ by spread(pre_x, tol_x); then mean(x^2) moves by sum (2 |x| dx + dx^2) / K, which moves inv by
      half that relative to mean(x^2) + eps; the fp32 inv adds ((norm_chain + 3) / 2 + 4) u relative (norm_chain:
      ss_chain(K)), the two products 2u.
    Output: the final rounding, half the spacing of T at |pre| + E."""
    dtype = W.dtype
    E = accumulation_error(r, W, path, splits, gb_per_split)
    if r.epilogue == EPI_NONE:
        pre, Ep = r.acc, E
    elif r.epilogue == EPI_RESIDUAL:
        pre = r.residual + round_to(r.acc, dtype)
        Ep = spread(r.acc, E, dtype)
        Ep = Ep + U * (pre.abs() + Ep)
    else:
        gi, ui = pairs_index(r.acc.shape[1] // 2, r.acc.device)
        g, u = round_to(r.acc[:, gi], dtype), round_to(r.acc[:, ui], dtype)
        dg, du = spread(r.acc[:, gi], E[:, gi], dtype), spread(r.acc[:, ui], E[:, ui], dtype)
        pre = silu64(g) * u
        Ep = SILU_SLOPE * dg * (u.abs() + du) + silu64(g).abs() * du + SWIGLU_REL * pre.abs()
        # below gate = -87 silu(gate) = gate e^gate leaves fp32's normal range (expf(-gate) overflows near 88.7): the
        # kernel's quotient may be 0
        Ep = torch.where(g - dg < -87.0, Ep + pre.abs(), Ep)
    b = Bound(pre=pre, tol=Ep + spacing(pre.abs() + Ep, dtype) / 2)
    if r.normed is not None:
        K = r.out.shape[1]
        x, w = r.out, r.norm_weight
        dx = spread(pre, Ep, dtype)
        p, inv = rms64(x, w, r.norm_eps)
        ms = (x * x).mean(dim=-1, keepdim=True) + r.norm_eps
        dms = (2 * x.abs() * dx + dx * dx).mean(dim=-1, keepdim=True)
        chain = ss_chain(K) if norm_chain is None else norm_chain
        rel_inv = 1.01 * dms / (2 * ms) + ((chain + 3) / 2 + 4) * U
        En = w.abs() * inv * dx + (p.abs() + w.abs() * inv * dx) * (rel_inv + 2 * U)
        b.normed_pre, b.normed_tol = p, En + spacing(p.abs() + En, dtype) / 2
    return b


def assert_within(got, pre, tol, what):
    """Returns (max error in units of tol, max error in output ulps)."""
    err = (got.to(F64) - pre).abs()
    bad = err > tol
    if bool(bad.any()):
        worst = int((err - tol).flatten().argmax())
        where = [int(i) for i in torch.unravel_index(torch.tensor(worst), err.shape)]
        raise AssertionError(
            f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the error bound; worst at {where}: |got - ref| = "
            f"{float(err.flatten()[worst]):.4g} > bound {float(tol.flatten()[worst]):.4g} (ref {float(pre.flatten()[worst]):.5g})")
    return float((err / tol).max())


def assert_exact(got, want, what):
    got = got.to(F64)
    bad = got != want
    if bool(bad.any()):
        idx = bad.nonzero()[:8].tolist()
        first = tuple(idx[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ from the exact probe result; first at {idx}: "
                             f"got {float(got[first]):.6g}, want {float(want[first]):.6g}")


# -------------------------------------------------------------------- probes --
@dataclass
class Probe:
    """Inputs of one launch whose every result is exact in fp32 and representable in T."""

    words: torch.Tensor
    scales: torch.Tensor
    biases: torch.Tensor
    p0: torch.Tensor
    p1: torch.Tensor | None
    residual: torch.Tensor | None
    eps: float
    positions: list  # per row, the reduction positions of its needles


def probe_positions(N, boundaries=(), full=True):
    """Reduction positions worth a needle: every offset 0..127 of a group (every nibble of every word, and every column
    modulo 128), dealt over the groups (offset o in group 7 o mod G); or, with full=False, 16 offsets that still cover
    the 16 words and the 8 nibbles.  Then the first and last group's ends and both sides of each boundary (split starts)."""
    G = N // 128
    offsets = range(128) if full else [8 * w + (w % 8) for w in range(16)]
    pos = [128 * ((7 * o) % G) + o for o in offsets]
    pos += [0, 127, N - 128, N - 1]
    for x in boundaries:
        pos += [x - 1, x]
    return list(dict.fromkeys(p for p in pos if 0 <= p < N))


def _pow2(t):
    return torch.ldexp(torch.ones_like(t, dtype=torch.float32), t.to(torch.int64))


def exact_probes(M, N, K, dtype, g, positions, *, prologue=PRO_NONE, epilogue=EPI_NONE, residual=False, group_rows=True, lda=None,
                 weights=None):
    """Weights and needle activations on which every path is bit-exact.

    scales: powers of two 2^-(5 + (k + 2 grp) % 3), so neighbouring rows and neighbouring groups differ; biases -c s with
    an integer c in 0..15: every dequantised weight is (q - c) s, exact in bf16 and f16 and unchanged by the tensor-core
    rounding.  Row m of the activation takes the next position: one needle +-2^e (e in -2..3), or (every second row
    with group_rows and no prologue) three +-1 entries in that position's group.  Each output is then (q - c) s 2^e or s times an integer
    of at most 45: a few bits, exact in every fp32 sum the kernels form, and the shift of the streaming kernel
    ((SHIFT + q) 2^e, SHIFT sum(a)) stays exact too.
      RMSNORM prologue: x holds one +-1 per row; eps is the fp32 number that brings fl(1/N) + eps to 1/4, so inv = 2
        up to rsqrtf's error, and the norm weights are powers of two: a = +-2 w_n, a T number the fp32 value rounds to.
      SWIGLU prologue: gate 32 and up +-2^e / 32 at the needle (silu(32) = 32 in fp32 and within 2^-40 in float64),
        random gates with up = 0 elsewhere.
      SWIGLU_PAIRS epilogue: gate rows have q >= c and only q - c in {0, 8..15}, needles are +2^9 (after RMSNORM: x = 1 and
        w = 2^8): every gate output is 0 or >= 32, where silu(g) = g in fp32 and to 2^-45 in float64, and g * up has at
        most 8 significant bits (|g up| <= 240^2 < 65504).
      residual: s 2^e times an integer in -60..60, with the result still exact (at most 7 bits).
    positions: the reduction positions to cover (probe_positions); rows past them repeat from the start.
    weights: (words, scales, biases) of an earlier probe of the same form, to keep."""
    G = N // 128
    pairs = epilogue == EPI_SWIGLU_PAIRS
    kk = torch.arange(K)[:, None]
    gg = torch.arange(G)[None, :]
    s = _pow2(-(5 + (kk + 2 * gg) % 3)).expand(K, G).contiguous()
    if weights is not None:  # new activations for the same weights
        words, scales, biases = weights
    else:
        c = torch.randint(0, 16, (K, G), generator=g)
        if pairs:
            q = torch.randint(0, 16, (K, G, 128), generator=g)
            gate_rows = (torch.arange(K) % 16) < 8
            d = torch.randint(0, 9, (K, G, 128), generator=g)
            d = torch.where(d == 0, 0, d + 7)  # q - c in {0, 8..15}
            c_gate = torch.randint(0, 16, (K, G), generator=g)
            c = torch.where(gate_rows[:, None], torch.minimum(c_gate, 15 - d.amax(-1)), c)
            q = torch.where(gate_rows[:, None, None], c[..., None] + d, q)
            words = (q.reshape(K, N // 8, 8).to(torch.int64) << (4 * torch.arange(8))).sum(-1)
            words = torch.where(words >= 2**31, words - 2**32, words).to(torch.int32)
        else:  # uniform codes
            words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
        scales, biases = s.to(dtype), (-c * s).to(dtype)

    rows, mag = [], []
    pos = list(positions)
    i = 0
    multi = group_rows and prologue == PRO_NONE and not pairs
    for m in range(M):
        first = pos[i % len(pos)]
        i += 1
        ent = [first]
        if multi and m % 2 == 1:  # two more entries in the same group, at other offsets
            ent += [first - first % 128 + (first + d) % 128 for d in (37, 77)]
        rows.append(ent)
        if pairs:
            mag.append(2.0**9)
        elif len(ent) > 1 or prologue == PRO_RMSNORM:
            mag.append(1.0)
        else:
            mag.append(2.0 ** int(torch.randint(-2, 4, (1,), generator=g)))
    sign = lambda: 1.0 if pairs else (1.0 if bool(torch.randint(0, 2, (1,), generator=g)) else -1.0)  # noqa: E731

    lda = N if lda is None else lda
    p0 = torch.zeros(M, lda)
    p1 = None
    eps = 0.0
    if prologue == PRO_SWIGLU:
        p0 = torch.randn(M, lda, generator=g) * 4
        p1 = torch.zeros(M, lda)
    for m, ent in enumerate(rows):
        for n in ent:
            v = sign() * mag[m]
            if prologue == PRO_SWIGLU:
                p0[m, n], p1[m, n] = 32.0, v / 32.0
            elif prologue == PRO_RMSNORM:
                p0[m, n] = 1.0 if pairs else v
            else:
                p0[m, n] = v
    if prologue == PRO_RMSNORM:
        # norm weights: a = 2 w = 2^-1 .. 2^1 (2^9 everywhere for the pairs epilogue)
        p1 = (torch.full((N,), 2.0**8) if pairs else _pow2(torch.arange(N) % 3 - 2)).to(dtype)
        v = torch.tensor(1.0 / N, dtype=torch.float32)
        eps32 = (torch.tensor(0.25, dtype=F64) - v.to(F64)).to(torch.float32)
        assert float(eps32 + v) == 0.25
        eps = float(eps32)
    p0 = p0.to(dtype)
    p1 = None if p1 is None else p1.to(dtype)
    if lda != N:
        p0, p1 = p0[:, :N], (p1[:, :N] if p1 is not None and p1.dim() == 2 else p1)
    res = None
    if residual:
        grp = torch.tensor([ent[0] // 128 for ent in rows])
        unit = s[:, grp].T * torch.tensor(mag)[:, None]  # [M, K]
        res = (torch.randint(-60, 61, (M, K), generator=g) * unit).to(dtype)
    return Probe(words, scales, biases, p0, p1, res, eps, rows)


def probe_reference(probe, W, *, prologue=PRO_NONE, epilogue=EPI_NONE, norm_weight=None, norm_eps=0.0):
    """The reference on a probe, asserting that the probe is one: every accumulator and result is a T number."""
    dev = W.w.device
    r = reference(W, probe.p0.to(dev), p1=None if probe.p1 is None else probe.p1.to(dev), prologue=prologue, epilogue=epilogue,
                  residual=None if probe.residual is None else probe.residual.to(dev), eps=probe.eps, norm_weight=norm_weight,
                  norm_eps=norm_eps)
    assert bool((round_to(r.acc, W.dtype) == r.acc).all()), "probe accumulators are not T numbers"
    assert bool(r.amb.eq(0).all()), "probe prologue outputs are not clear of rounding midpoints"
    if epilogue == EPI_SWIGLU_PAIRS:
        gi, ui = pairs_index(r.acc.shape[1] // 2, dev)
        gate = r.acc[:, gi]
        assert bool(((gate == 0) | (gate >= 32)).all()), "probe gates must be 0 or >= 32"
        assert bool((round_to(gate * r.acc[:, ui], W.dtype) == gate * r.acc[:, ui]).all()), "probe gate * up is not a T number"
    elif epilogue == EPI_RESIDUAL or norm_weight is not None:
        total = r.residual + r.acc
        assert bool((round_to(total, W.dtype) == total).all()), "probe residual sums are not T numbers"
    return r
