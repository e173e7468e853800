"""Float64 reference for the element-wise kernels of elementwise.cu, the error bounds they are held to, and exact probes.

Each function restates one operator in float64 on the inputs' device and keeps the kernel's rounding points (T: the
activation dtype; fp32(.): one rounding to float32):

    rms_norm          T(x * rsqrt(mean(x^2) + eps) * w)
    rope              angle = fp32(pos * inv_freq), inv_freq = base^(-i / half) in double; T(re c - im s), T(im c + re s);
                      both pair layouts, and the tail [dims, D) copied
    q/k norm + RoPE   n = T(x * rsqrt(mean(x^2) + eps) * w), then y = T(rope(n)); V copied bit for bit (the decode, chunk
    + K/V append      and planes forms; the planes form first rounds q|k|v = T(sum of planes), which is what
                      quantized_matmul_fused returns for the same rows)
    swiglu            T(g / (1 + e^-g) * u)
    add               T(fp32(a + b))
    quantized_embed.  T(fp32(code * s + b)); ids < 0 or >= vocab give zero rows
    argmax            first index of the maximum; NaN is never picked, an all-NaN row gives 0
    paged append      row b writes token ctx - 1 to page block_table[b, (ctx - 1) // page]; ctx <= 0, a logical page
                      >= max_pages and a page id of -1 or >= num_pages write nothing

``add``, ``quantized_embedding`` and ``argmax`` have no rounding freedom: the kernels must equal the reference bit for
bit on any input.  The others come with an elementwise tolerance ``tol`` around the unrounded value ``pre`` (no
absolute term; the derivation is in ``norm64`` and ``rotate64``), and with exact probes: inputs on which every kernel's
fp32 arithmetic is exact (``unit_norm_rows``), or on which every output but one pair must be exactly zero
(``needle_rows``).

The rounding helpers (``spacing``, ``round_to``, ``spread``, ``rms64``, ``ss_chain``, the SwiGLU term) are the ones of
w4a16_ref.py next to this file.
"""

from __future__ import annotations

import importlib.util
import sys
from dataclasses import dataclass
from pathlib import Path

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
spacing, round_to, spread, rms64, ss_chain, silu64 = wr.spacing, wr.round_to, wr.spread, wr.rms64, wr.ss_chain, wr.silu64
assert_exact, ulps = wr.assert_exact, wr.ulps
F64, F32, BF16, F16 = torch.float64, torch.float32, torch.bfloat16, torch.float16
U = wr.U
RSQRT_REL = 4 * U     # rsqrtf, sincosf, expf: 2 ulp, and an fp32 ulp is at most 2u of the value
ANGLE_REL = 2.0**-46  # pos * inv_freq in double: device exp2(log2) and the host's pow differ in the last bits
SWIGLU_UNDERFLOW = -87.0


def f32(v: float) -> float:
    """The fp32 number a float argument of the C ABI becomes."""
    return float(torch.tensor(v, dtype=F32))


def to32(x):
    """fp32(x) of a float64 tensor, as float64 (one rounding)."""
    return x.to(F32).to(F64)


@dataclass
class Bound:
    """|kernel - pre| <= tol elementwise; ``out`` is the reference's own rounding of ``pre`` (what exact probes equal)."""

    out: torch.Tensor
    pre: torch.Tensor
    tol: torch.Tensor


def assert_within(got, pre, tol, what):
    """w4a16_ref.assert_within, and every value finite: a NaN compares false with any bound."""
    for name, t in (("kernel", got), ("reference", pre)):
        bad = ~torch.isfinite(t.to(F64))
        if bool(bad.any()):
            raise AssertionError(f"{what}: {int(bad.sum())} {name} values are not finite; first at {bad.nonzero()[:4].tolist()}")
    return wr.assert_within(got, pre, tol, what)


def finish(pre, E, dtype):
    """The final rounding: the kernel's fp32 value is within E of pre, so T of it is within E + half an ulp."""
    return Bound(round_to(pre, dtype), pre, E + spacing(pre.abs() + E, dtype) / 2)


# ------------------------------------------------------------------- RMSNorm --
def norm64(x, w, eps):
    """(pre, rel): x * rsqrt(mean(x^2) + eps) * w over the last axis in float64, eps as the fp32 the kernels get, and a
    bound on the relative error of the kernels' fp32 value of it.

    The sum of squares is a chain of fp32 additions of non-negative terms; its longest chain, plus the rounding of the
    square, is below ss_chain(n):
      rms_norm      : dim / TPR per thread (TPR 32 up to dim 512, else 256), a 5-level warp sum, and for TPR 256 a
                      second 5-level sum over the 8 warp partials;
      row kernel    : re^2 + im^2 of two pairs per lane, two 5-level warp sums added together (8 in all);
      per-head      : one pair per thread, a 5-level warp sum and a 5-level sum over up to 8 warp partials (12).
    So ss is within (ss_chain + 1) u ss, plus 2^-150 per square that underflows (n of them, divided by n in the mean).
    / n and + eps round once each: m = mean + eps is within ((chain + 2) u mean + 2^-150) / m + u relative.  rsqrt
    halves that and rsqrtf adds 2 ulp (4u); x * inv * w adds two roundings.  1.01 covers the higher-order terms."""
    x, w = x.to(F64), w.to(F64)
    n = x.shape[-1]
    e = f32(eps)
    ms = (x * x).mean(dim=-1, keepdim=True)
    m = ms + e
    pre = x / torch.sqrt(m) * w
    dm = ((ss_chain(n) + 2) * U * ms + 2.0**-150) / m + U
    return pre, 1.01 * (dm / 2 + RSQRT_REL + 2 * U)


def rms_norm_ref(x, w, eps, dtype):
    pre, rel = norm64(x, w, eps)
    return finish(pre, rel * pre.abs(), dtype)


# ---------------------------------------------------------------------- RoPE --
def inv_freq64(half, base, device=None):
    """base^(-i / half) in float64, base as the fp32 the kernels get (formed on the host, as rope_inv_freq_table does)."""
    b = torch.tensor(f32(base), dtype=F64)
    return torch.pow(b, -torch.arange(half, dtype=F64) / half).to(device)


def angles(pos, inv_freq):
    """pos [...] (int) -> (theta, dtheta) [..., half]: the fp32 angle fp32(pos * inv_freq) as float64, and how far the
    kernel's may be from it.  dtheta is 0 except where pos * inv_freq lies within its double-precision error of an fp32
    rounding midpoint: there the kernel may round to the neighbour."""
    p = pos.to(F64)[..., None] * inv_freq.to(pos.device)
    th = to32(p)
    err = p.abs() * ANGLE_REL
    return th, torch.maximum(to32(p + err) - th, th - to32(p - err))


def rotate64(re, im, dre, dim_, theta, dtheta):
    """(pre_re, pre_im, E_re, E_im) of the rotation T(re c - im s), T(im c + re s) with fp32 sincosf and fp32 products.
    re / im are the reference's inputs; the kernel's may differ by dre / dim_ (0 for stored inputs; the rounding
    ambiguity of n in the fused forms).  sincosf is within 2 ulp of sin / cos of the kernel's angle, which is within
    dtheta of theta (sin and cos are 1-Lipschitz).  The two products and the sum round at most three times, each within
    u of |re c| + |im s| (less with an fma)."""
    s, c = torch.sin(theta), torch.cos(theta)
    ds = 2 * spacing(s.abs(), F32) + dtheta
    dc = 2 * spacing(c.abs(), F32) + dtheta
    pre_re, pre_im = re * c - im * s, im * c + re * s
    are, aim = re.abs() + dre, im.abs() + dim_
    E_re = dre * c.abs() + dim_ * s.abs() + are * dc + aim * ds + 3 * U * (are * c.abs() + aim * s.abs())
    E_im = dim_ * c.abs() + dre * s.abs() + aim * dc + are * ds + 3 * U * (aim * c.abs() + are * s.abs())
    return pre_re, pre_im, E_re, E_im


def pair_index(D, dims, traditional, device=None):
    """Element indices (re, im) of the rotated pairs of a head."""
    i = torch.arange(dims // 2, device=device)
    return (2 * i, 2 * i + 1) if traditional else (i, i + dims // 2)


def rope_ref(x, offsets, dims, base, traditional, dtype):
    """x [B, L, H, D] (T), offsets [B]: position of x[b, l] is offsets[b] + l."""
    B, L, H, D = x.shape
    x64 = x.to(F64)
    pos = offsets.to(torch.int64)[:, None] + torch.arange(L, device=x.device)  # [B, L]
    th, dth = angles(pos, inv_freq64(dims // 2, base, x.device))
    th, dth = th[:, :, None, :], dth[:, :, None, :]  # one angle per (token, pair) for every head
    ri, ii = pair_index(D, dims, traditional, x.device)
    zero = torch.zeros((), dtype=F64, device=x.device)
    pre_re, pre_im, E_re, E_im = rotate64(x64[..., ri], x64[..., ii], zero, zero, th, dth)
    pre, E = x64.clone(), torch.zeros_like(x64)  # the tail [dims, D) is copied
    pre[..., ri], pre[..., ii], E[..., ri], E[..., ii] = pre_re, pre_im, E_re, E_im
    return finish(pre, E, dtype)


# --------------------------------------------------- q/k norm + RoPE + append --
@dataclass
class QkvRef:
    q: Bound   # [R, Hq, D]
    k: Bound   # [R, Hkv, D]
    v: torch.Tensor  # [R, Hkv, D]: the input's v heads, bit for bit


def qk_norm_rope_ref(qkv, q_norm_weight, k_norm_weight, offsets, Hq, Hkv, base, eps, inv_freq=None):
    """qkv [R, (Hq + 2 Hkv) * D] (T: its dtype); offsets [R] the RoPE position of each row (non-traditional RoPE over
    the whole head).  The normalised head n = T(x inv w) of the kernel may differ from round_to(pre_n) by
    spread(pre_n, rel |pre_n|): one T-ulp where pre_n lies within its fp32 error of a midpoint (a float32 n is not
    rounded again, and spread is then that error itself).  inv_freq: the frequency table of decode_attention_fused
    (default: the same float64 values the standalone kernels form)."""
    dtype = qkv.dtype
    R = qkv.shape[0]
    D = qkv.shape[1] // (Hq + 2 * Hkv)
    half = D // 2
    x = qkv.to(F64).view(R, Hq + 2 * Hkv, D)
    th, dth = angles(offsets.to(torch.int64), inv_freq64(half, base) if inv_freq is None else inv_freq.to(F64).cpu())
    th, dth = th[:, None, :], dth[:, None, :]
    out = []
    for heads, w in ((x[:, :Hq], q_norm_weight), (x[:, Hq : Hq + Hkv], k_norm_weight)):
        pre_n, rel = norm64(heads, w.to(qkv.device), eps)
        n, dn = round_to(pre_n, dtype), spread(pre_n, rel * pre_n.abs(), dtype)
        pr, pi, Er, Ei = rotate64(n[..., :half], n[..., half:], dn[..., :half], dn[..., half:], th, dth)
        out.append(finish(torch.cat([pr, pi], -1), torch.cat([Er, Ei], -1), dtype))
    return QkvRef(out[0], out[1], qkv.view(R, Hq + 2 * Hkv, D)[:, Hq + Hkv :])


# ------------------------------------------------------------ other operators --
def swiglu_ref(g, u, dtype):
    """SWIGLU_REL |pre| (w4a16_ref's prologue term); below g = -87, where silu(g) leaves fp32's normal range and
    expf(-g) overflows, the kernel's quotient may be 0: + |pre|."""
    g, u = g.to(F64), u.to(F64)
    pre = silu64(g) * u
    E = wr.SWIGLU_REL * pre.abs() + torch.where(g < SWIGLU_UNDERFLOW, pre.abs(), torch.zeros_like(pre))
    return finish(pre, E, dtype)


def add_ref(a, b, dtype):
    return round_to(to32(a.to(F64) + b.to(F64)), dtype)


def embedding_ref(indices, scales, biases, weight, dtype):
    """Rows of T(fp32(code * s + b)); an id < 0 or >= vocab gives a zero row."""
    vocab = weight.shape[0]
    ids = indices.to(torch.int64)
    ok = (ids >= 0) & (ids < vocab)
    rows = torch.where(ok, ids, torch.zeros_like(ids))
    codes = wr.unpack_codes(weight[rows]).to(F64)  # [T, dim]
    s = scales[rows].to(F64).repeat_interleave(128, dim=-1)
    b = biases[rows].to(F64).repeat_interleave(128, dim=-1)
    val = round_to(to32(codes * s + b), dtype)
    return torch.where(ok[:, None], val, torch.zeros_like(val))


def argmax_ref(logits):
    """First index of the row maximum over the non-NaN entries; 0 for an all-NaN row.  (The fp32 oracle follows
    torch.argmax, which picks a NaN: that behaviour is not pinned.)"""
    x = logits.to(F64)
    nan = torch.isnan(x)
    m = torch.where(nan, torch.full_like(x, float("-inf")), x).amax(dim=-1, keepdim=True)
    hit = (x == m) & ~nan
    first = torch.where(hit, torch.arange(x.shape[-1], device=x.device), x.shape[-1]).amin(dim=-1)
    return torch.where(first == x.shape[-1], torch.zeros_like(first), first)


def append_slots(context_lens, block_table, page_size, num_pages, chunk=False):
    """[(row, page id, slot)] the paged append writes: row b's token ctx - 1 (block_table: [rows, max_pages], or one
    [max_pages] row shared by every row of a chunk)."""
    cl = context_lens.tolist()
    bt = block_table.tolist()
    out = []
    for b, ctx in enumerate(cl):
        row = bt if chunk else bt[b]
        if ctx <= 0:
            continue
        tok = ctx - 1
        lp = tok // page_size
        if lp >= len(row):
            continue
        pid = row[lp]
        if 0 <= pid < num_pages:
            out.append((b, pid, tok - lp * page_size))
    return out


def check_pages(before, after, slots, rows, what, tol=None, pre=None):
    """Pages [P, H, page, D] after an append: every element outside the target slots keeps its bits; slot (b, pid, t)
    holds rows[b] [H, D] exactly, or, with tol / pre [rows, H, D], within the bound."""
    as_bits = (lambda t: t.view(torch.int16)) if before.element_size() == 2 else (lambda t: t.view(torch.int32))
    want = before.clone()
    for b, pid, t in slots:
        want[pid, :, t] = after[pid, :, t]
    bad = as_bits(want) != as_bits(after)
    if bool(bad.any()):
        raise AssertionError(f"{what}: {int(bad.sum())} page elements outside the target slots changed; first at "
                             f"{bad.nonzero()[:4].tolist()}")
    if slots:
        b_idx = [b for b, _, _ in slots]
        got = torch.stack([after[pid, :, t] for _, pid, t in slots])
        if tol is None:
            assert_exact(got, rows[b_idx].to(F64), f"{what}: appended rows")
            return 0.0
        return assert_within(got, pre[b_idx], tol[b_idx], f"{what}: appended rows")
    return 0.0


# -------------------------------------------------------------------- probes --
def unit_norm_rows(R, H, D, g):
    """[R, H, D] rows whose inverse norm is exactly 1 with eps = 0: entries +-1, +-2, +-8 and 0 with sum x^2 = D, in
    random places.  With power-of-two norm weights x * inv * w is then a T number the fp32 value equals, and at
    position 0 sincosf(0) = (0, 1) is exact: every form must match the reference bit for bit (given rsqrtf(1) = 1)."""
    x = torch.zeros(R * H, D)
    for r in range(R * H):
        k8 = int(torch.randint(0, 2, (1,), generator=g)) if D >= 64 else 0
        rest = D - 64 * k8
        k2 = int(torch.randint(0, rest // 8 + 1, (1,), generator=g))
        k1 = rest - 4 * k2
        vals = torch.tensor([8.0] * k8 + [2.0] * k2 + [1.0] * k1)
        sign = torch.where(torch.rand(len(vals), generator=g) < 0.5, -1.0, 1.0)
        where = torch.randperm(D, generator=g)[: len(vals)]
        x[r, where] = vals * sign
    assert bool(((x * x).sum(-1) == D).all())
    return x.view(R, H, D)


def pow2_norm_weight(D, which):
    """Power-of-two norm weights with w[i] != w[i + D/2]: 2^(i % 3 - 1) in the first half, 2^-(i % 3 + 2) (which=0) or
    2^-(i % 3 + 5) (which=1, the k weight) in the second (the longer first half of an odd D keeps the first rule)."""
    lo = torch.arange(D - D // 2)
    hi = torch.arange(D // 2)
    return torch.cat([torch.pow(2.0, (lo % 3 - 1).float()), torch.pow(2.0, -(hi % 3 + 2 + 3 * which).float())])


def needle_rows(R, H, D, value=1.0):
    """R rows of H heads holding one needle each: row r has +-value at element r % D of head r % H, and zeros elsewhere.
    R = D rows walk every element (the re and the im side of every pair, in either layout) and every head (H <= D).
    Returns (x, [(h, e)])."""
    x = torch.zeros(R, H, D)
    where = []
    for r in range(R):
        h, e = r % H, r % D
        x[r, h, e] = value if r % 2 == 0 else -value
        where.append((h, e))
    return x, where
