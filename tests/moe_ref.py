"""Float64 reference for the Qwen3-MoE kernels (moe.cu and the grouped form of w4a16_skinny.cu), the bounds they are
held to, and exact probes.

Each function restates one entry point of include/tiny_llm_b200.h in float64 on the inputs' device and keeps its
rounding points (T: the activation dtype; fp32(.): one rounding to float32):

    tl_moe_topk     probs = T(softmax_fp32(logits)): bounded (``softmax_ref``).  ids and scores are an exact function
                    of the probs the kernel returned (``select_ref``): the k largest, ties to the lower id, NaN below
                    every number; scores p_j, or with norm T(fp32(p_j / T(sum_fp32 p in slot order)))
    tl_moe_group    offsets, the stable argsort of the clamped ids and the tile table: exact (``group_ref``)
    tl_moe_gather   a copy: exact; with a norm weight rms_norm_ref of the gathered rows
    tl_moe_combine  T(fp32(res + T(sum_fp32 over slots in order of T(fp32(y_j s_j))))): exact on any finite input
                    (``combine_ref``; an explicit loop, since Tensor.sum does not fix its order)
    grouped W4A16   per expert w4a16_ref.reference: the wgmma route with weights rounded once to T and the "skinny"
                    bound of one split, the control route with exact weights and the "vanilla" bound; both epilogues

The rounding and bound helpers are those of w4a16_ref.py and elementwise_ref.py next to this file.
"""

from __future__ import annotations

import importlib.util
import math
import sys
from dataclasses import dataclass
from pathlib import Path

import torch


def _load(name, filename):
    """A helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(filename))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


wr = _load("tiny_llm_b200_w4a16_ref", "w4a16_ref.py")
er = _load("tiny_llm_b200_elementwise_ref", "elementwise_ref.py")
round_to, spread, spacing, to32 = wr.round_to, wr.spread, wr.spacing, er.to32
rms_norm_ref, swiglu_ref, assert_exact, assert_within = er.rms_norm_ref, er.swiglu_ref, wr.assert_exact, er.assert_within
F64, F32, F16, BF16 = torch.float64, torch.float32, torch.float16, torch.bfloat16
U = wr.U
EXPF_REL = 4 * U            # expf: 2 ulp, and an fp32 ulp is at most 2u of the value
EXPF_SUB = 2.0**-148        # 2 ulp of an fp32 subnormal
SUM_CHAIN = 13              # tl_moe_topk's sum of exponentials: 8 per lane, then 5 butterfly levels
EXP_FLOOR = -110.0          # below this exp(d) is far under fp32's smallest subnormal: the kernel's term is 0 or 2^-149
EPI_NONE, EPI_SWIGLU_PAIRS = wr.EPI_NONE, wr.EPI_SWIGLU_PAIRS


# ---------------------------------------------------------------------- top-k --
@dataclass
class Softmax:
    """probs the kernel may return: every T number in [lo, hi] (lo == hi == ``out`` unless ``pre`` lies within its
    error of a rounding midpoint); NaN where ``nan`` (the whole row)."""

    out: torch.Tensor
    pre: torch.Tensor
    tol: torch.Tensor
    lo: torch.Tensor
    hi: torch.Tensor
    nan: torch.Tensor  # [T] bool


def nan_rows(logits):
    """Rows whose fp32 softmax is NaN in tl_moe_topk: a NaN or +inf logit (x - m is NaN), or every logit -inf."""
    x = logits.to(F64)
    return torch.isnan(x).any(-1) | (x == math.inf).any(-1) | (x == -math.inf).all(-1)


def softmax_ref(logits, dtype=None, chain=SUM_CHAIN):
    """The float64 softmax of ``logits [T, E]`` and the bound of tl_moe_topk's probs.

    With d = x - m (m the row maximum) and e = exp(d), s = sum e, p = e / s:
      d    : the fp32 subtraction is within u |d| (exact for most 16-bit inputs; it matters for fp32 logits), which
             moves exp(d) by u |d| relative;
      e    : expf within 2 ulp: 4u relative, or 2^-148 for a subnormal result;
      s    : ``chain`` fp32 additions of positive terms: within chain u s, plus the terms' own errors;
      p    : (e + de) / (s + ds) is within (de + p ds) / (s - ds) of p; the fp32 division adds u |p| before the
             final rounding to a 16-bit T (for fp32 the division is that rounding).
    1.01 covers the higher-order terms.  Rows of ``nan_rows`` are NaN in the kernel and here."""
    dtype = logits.dtype if dtype is None else dtype
    x = logits.to(F64)
    nan = nan_rows(logits)
    x = torch.where(nan[:, None], torch.zeros_like(x), x)
    d = x - x.amax(-1, keepdim=True)
    live = d > EXP_FLOOR
    e = torch.where(live, torch.exp(d), torch.zeros_like(d))
    de = torch.where(live, e * 1.01 * (U * d.abs() + EXPF_REL), torch.zeros_like(d)) + EXPF_SUB
    s = e.sum(-1, keepdim=True)
    ds = de.sum(-1, keepdim=True) + 1.01 * chain * U * (s + de.sum(-1, keepdim=True))
    p = e / s
    E = 1.01 * (de + p * ds) / (s - ds)
    if dtype != F32:
        E = E + U * (p + E)
    lo, hi = round_to(p - E, dtype), round_to(p + E, dtype)
    out = round_to(p, dtype)
    nanv = torch.full_like(p, math.nan)
    pick = lambda t: torch.where(nan[:, None], nanv, t)  # noqa: E731
    tol = E + spacing(p + E, dtype) / 2
    return Softmax(pick(out), pick(p), pick(tol), pick(lo), pick(hi), nan)


def probs_within(got, sm: Softmax, what):
    """Asserts that the kernel's probs lie in [lo, hi] (NaN exactly on the NaN rows).  Returns the number of entries
    whose rounding the bound leaves open."""
    g = got.to(F64)
    gnan = torch.isnan(g)
    want_nan = sm.nan[:, None].expand_as(g)
    if not torch.equal(gnan, want_nan):
        bad = (gnan != want_nan).nonzero()[:4].tolist()
        raise AssertionError(f"{what}: NaN probabilities where the reference has none, or the reverse; first at {bad}")
    ok = gnan | ((g >= sm.lo) & (g <= sm.hi))
    if not bool(ok.all()):
        idx = (~ok).nonzero()[:4].tolist()
        r, c = idx[0]
        raise AssertionError(f"{what}: {int((~ok).sum())} probabilities outside the bound; first at {idx}: got {float(g[r, c]):.8g}, "
                             f"allowed [{float(sm.lo[r, c]):.8g}, {float(sm.hi[r, c]):.8g}] around {float(sm.pre[r, c]):.10g}")
    return int((sm.lo != sm.hi).sum())


def select_ref(probs, k, norm):
    """(ids int64 [T, k], scores float64 [T, k]) tl_moe_topk must return for the probs it returned: the k largest in
    descending order, ties to the lower id, a NaN below every number (so a NaN row gives 0..k-1); scores the picked
    probs, or with norm T(fp32(p_j / T(sum_fp32 p in slot order)))."""
    dtype = probs.dtype
    p = probs.to(F64).cpu()
    key = torch.where(torch.isnan(p), torch.full_like(p, -0.5), p)  # probabilities are >= 0
    ids = torch.sort(-key + 0.0, dim=-1, stable=True).indices[:, :k]  # + 0.0: one zero, not -0 and +0
    picked = torch.gather(p, -1, ids)
    if not norm:
        return ids, picked
    total = torch.zeros(p.shape[0], dtype=F64)
    for j in range(k):
        total = to32(total + picked[:, j])
    den = round_to(total, dtype)[:, None]
    return ids, round_to(to32(picked / den), dtype)


def same_or_both_nan(a, b):
    a, b = a.to(F64), b.to(F64)
    return (a == b) | (torch.isnan(a) & torch.isnan(b))


# ---------------------------------------------------------------------- group --
def group_ref(ids, E, nt):
    """(offsets [E + 1], perm [R], tiles or None) of tl_moe_group: ids clamped to [0, E) (the header's rule for ids
    outside it), perm the stable argsort, tiles {count, (expert, first sorted row) per nt-row piece}."""
    e = ids.to(torch.int64).clamp(0, E - 1)
    counts = torch.bincount(e, minlength=E)
    offsets = torch.cat([counts.new_zeros(1), torch.cumsum(counts, 0)])
    perm = torch.sort(e, stable=True).indices
    if nt <= 0:
        return offsets, perm, None
    per = (counts + nt - 1) // nt
    expert = torch.repeat_interleave(torch.arange(E, device=e.device), per)
    first = torch.repeat_interleave(offsets[:-1], per)
    piece = torch.arange(expert.numel(), device=e.device) - torch.repeat_interleave(torch.cumsum(per, 0) - per, per)
    body = torch.stack([expert, first + piece * nt], -1).reshape(-1)
    return offsets, perm, torch.cat([per.sum().reshape(1), body])


def tile_bound(R, E, nt):
    """The most tiles R rows can need over E experts: tl_moe_tile_table_size's (size - 1) / 2."""
    return (R + (nt - 1) * min(E, R)) // nt


# -------------------------------------------------------------------- combine --
def combine_ref(y, scores, residual=None):
    """tl_moe_combine's out, exactly: y [T k, H], scores [T, k], residual [T, H] (T numbers) -> float64 T numbers."""
    dtype = y.dtype
    T_, k = scores.shape
    yy = y.to(F64).view(T_, k, -1)
    s = scores.to(F64)
    acc = torch.zeros(T_, yy.shape[-1], dtype=F64, device=y.device)
    for j in range(k):  # slot order; each fp32 addition of two fp32 numbers, formed in float64, rounds once
        acc = to32(acc + round_to(to32(yy[:, j] * s[:, j, None]), dtype))
    r = round_to(acc, dtype)
    return r if residual is None else round_to(to32(residual.to(F64) + r), dtype)


def plant_cancellation(y, scores, rows):
    """Rows whose slot order shows in every dtype (k >= 3): slot products 2^-11, 2^15, -2^15 and 0 after them.  In
    slot order 2^-11 is absorbed by 2^15 (below half an fp32 ulp) and the row sums to 0; in any other order the big
    terms cancel first and it sums to 2^-11.  y [T k, H] and scores [T, k] are changed in place."""
    T_, k = scores.shape
    assert k >= 3
    yy = y.view(T_, k, -1)
    for t in rows:
        yy[t] = 0
        yy[t, 0], yy[t, 1], yy[t, 2] = 2.0**-11, 2.0**15, -(2.0**15)
        scores[t] = 1
    return y, scores


# --------------------------------------------------------------------- gather --
def gather_ref(x, perm, rows_per_source, norm_weight=None, eps=0.0):
    """The gathered rows (float64, exact) and, with a norm weight, rms_norm_ref of them (an elementwise_ref Bound)."""
    rows = x.to(F64)[perm.to(torch.int64) // rows_per_source]
    return rows, None if norm_weight is None else rms_norm_ref(rows, norm_weight, eps, x.dtype)


# ---------------------------------------------------------------- grouped GEMM --
@dataclass
class Grouped:
    """Sorted-row results of the grouped projection: ``out`` the reference's rounding (what probes must equal), and
    |kernel - pre| <= tol."""

    out: torch.Tensor
    pre: torch.Tensor
    tol: torch.Tensor


def grouped_reference(words, scales, biases, a, offsets, epilogue, wgmma, probe=False):
    """The grouped W4A16 projection of the expert-sorted rows ``a [R, N]`` by experts ``words [E, K, N/8]``,
    ``scales / biases [E, K, N/128]``; row j uses the expert whose segment of ``offsets`` holds it.  wgmma: weights
    T(code * s + b) (one __hfma2 rounding) and error_bound "skinny" with one split over all N / 128 group blocks; else
    the control kernel's exact weights and the "vanilla" bound.  probe: assert that every accumulator, gate and gate *
    up is a T number (w4a16_ref.probe_reference), so the kernel must equal ``out`` bit for bit."""
    E, K, _ = words.shape
    R, N = a.shape
    off = [int(v) for v in offsets.tolist()]
    width = K // 2 if epilogue == EPI_SWIGLU_PAIRS else K
    out, pre, tol = (torch.zeros(R, width, dtype=F64, device=a.device) for _ in range(3))
    for e in range(E):
        lo, hi = off[e], off[e + 1]
        if hi == lo:
            continue
        W = wr.Weights.build(words[e], scales[e], biases[e], rounded=wgmma)
        rows = a[lo:hi]
        if probe:
            r = wr.probe_reference(wr.Probe(None, None, None, rows, None, None, 0.0, []), W, epilogue=epilogue)
        else:
            r = wr.reference(W, rows, epilogue=epilogue)
        b = wr.error_bound(r, W, "skinny" if wgmma else "vanilla", splits=1, gb_per_split=N // 128)
        out[lo:hi], pre[lo:hi], tol[lo:hi] = r.out, b.pre, b.tol
        del W, r, b
    return Grouped(out, pre, tol)


def grouped_probes(T, N, E, K, dtype, g, positions, epilogue):
    """Exact probes for E experts: w4a16_ref.exact_probes over the E K stacked feature rows (K % 16 == 0 keeps the
    gate|up pattern of the pairs epilogue inside each expert), and T needle token rows.  Returns (words [E, K, N/8],
    scales, biases [E, K, N/128], a [T, N])."""
    p = wr.exact_probes(T, N, E * K, dtype, g, positions, epilogue=epilogue)
    return p.words.view(E, K, -1), p.scales.view(E, K, -1), p.biases.view(E, K, -1), p.p0
