"""Restatement of top-n-sigma, locally typical sampling and Mirostat 2.0 (DESIGN.md section 25), in numpy float64,
on top of ``penalties_ref`` (the penalised row and the top-k / top-p / min-p keep set) and ``dry_xtc_ref`` (XTC).

TEST INFRASTRUCTURE.  The kernel decides on 2^-40 fixed-point masses from fp32 ``expf``, on fixed-order double sums
and on distances rounded to fp32; this restatement decides on the exact float64 softmax.  The two agree except where
a decisive quantity lies within a small band of its boundary (the bands below, derived in DESIGN.md section 25), so
every function also reports whether the row came that near; such draws are counted, not compared.

Also here, for the host tests: ``hf_typical_keep`` (``transformers``' ``TypicalLogitsWarper`` step by step, in numpy)
and ``llama_mirostat_v2`` (llama.cpp's sorted-prefix loop for Mirostat 2.0, literally).
"""

from __future__ import annotations

import importlib.util
import math
import sys
from pathlib import Path

import numpy as np

from oracle import sampling as ref


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


penalties_ref = _load("tiny_llm_b200_penalties_ref", "penalties_ref.py")
dry_xtc_ref = _load("tiny_llm_b200_dry_xtc_ref", "dry_xtc_ref.py")

# |bound_kernel - bound| <= NSIGMA_BAND * max(1, |m|, |bound|): the kernel's double sums run in another order
NSIGMA_BAND = 2.0**-30
# typical: distances within TYPICAL_D_BAND of the boundary d*, or a boundary mass within TYPICAL_MASS_BAND of typical_p
TYPICAL_D_BAND = 2.0**-14
TYPICAL_MASS_BAND = 2.0**-18
# Mirostat: -log2 p_i within MIROSTAT_BAND of mu; mu' within MU_BAND_ETA * eta + 2 ulp (fp32) of the reference's
MIROSTAT_BAND = 2.0**-18
MU_BAND_ETA = 2.0**-16


def f32(v) -> float:
    return float(np.float32(v))


def ulp32(v) -> float:
    return float(np.spacing(np.float32(abs(v))))


def nsigma_bound(x3, n: float) -> float:
    """``m - n sigma`` over the finite entries of the row (population sigma), in float64."""
    x = np.asarray(x3, dtype=np.float64)
    F = x[np.isfinite(x)]
    mean = F.sum() / len(F)
    sigma = math.sqrt(((F - mean) ** 2).sum() / len(F))
    return float(F.max()) - float(n) * sigma


def nsigma_keep(x3, keep, n: float):
    """``(keep', near)``: the keep set with top-n-sigma's bound and whether a finite entry lies within the band of it."""
    if not n > 0:
        return keep, False
    x = np.asarray(x3, dtype=np.float64)
    b = nsigma_bound(x3, n)
    fin = np.isfinite(x)
    scale = max(1.0, abs(float(x[fin].max())), abs(b))
    near = bool(np.any(fin & (np.abs(x - b) <= NSIGMA_BAND * scale) & (x != x[fin].max())))
    with np.errstate(invalid="ignore"):
        return keep & (x >= b), near


def typical_distances(x3, keep):
    """``(p, d)`` over the keep set at T = 1: ``p_i`` the renormalised softmax, ``d_i = |-ln p_i - H|`` (inf outside)."""
    x = np.asarray(x3, dtype=np.float64)
    m = x[keep].max()
    z = np.where(keep, x - m, -np.inf)
    e = np.exp(z)
    p = e / e.sum()
    with np.errstate(divide="ignore", invalid="ignore"):
        logp = np.where(p > 0, np.log(np.where(p > 0, p, 1.0)), -np.inf)
        H = -np.sum(np.where(p > 0, p * logp, 0.0))
        d = np.where(keep, np.abs(-logp - H), np.inf)
    return p, d


def typical_keep(x3, keep, typical_p: float):
    """``(keep', near)``: keep i of the keep set while the mass of the entries with strictly smaller d is < typical_p."""
    if not 0 < typical_p < 1:
        return keep, False
    p, d = typical_distances(x3, keep)
    idx = np.flatnonzero(keep)
    order = idx[np.argsort(d[idx], kind="stable")]
    ds, ps = d[order], p[order]
    # mass(d < d_i) per entry, ties sharing the mass below their value
    below = np.zeros(len(order))
    acc, j = 0.0, 0
    while j < len(order):
        k = j
        while k < len(order) and ds[k] == ds[j]:
            k += 1
        below[j:k] = acc
        acc += ps[j:k].sum()
        j = k
    kept = below < typical_p
    out = np.zeros_like(keep)
    out[order[kept]] = True
    dstar = ds[kept].max()
    upto = ps[ds <= dstar].sum()
    under = ps[ds < dstar].sum()
    near = bool(np.any((ds != dstar) & (np.abs(ds - dstar) <= TYPICAL_D_BAND)))
    near |= abs(upto - typical_p) <= TYPICAL_MASS_BAND or abs(under - typical_p) <= TYPICAL_MASS_BAND
    return out, near


def mirostat_keep(x3, temperature: float, mu: float):
    """``(keep, p, near)``: the non-NaN entries with ``-log2 p_i <= mu`` at the temperature (the maximum always), the
    softmax p over the non-NaN entries, and whether some ``-log2 p_i`` lies within the band of mu."""
    x = np.asarray(x3, dtype=np.float64)
    ok = ~np.isnan(x)
    m = x[ok].max()
    with np.errstate(invalid="ignore", over="ignore"):
        z = np.where(ok, (x - m) / np.float64(temperature), -np.inf)
    e = np.exp(z)
    p = e / e.sum()
    with np.errstate(divide="ignore"):
        s = -np.log2(p)
    keep = ok & ((s <= mu) | (x == m))
    near = bool(np.any(ok & (x != m) & (np.abs(s - mu) <= MIROSTAT_BAND)))
    return keep, p, near


def mirostat_update(p, keep, token: int, mu: float, tau: float, eta: float) -> float:
    """``fl32(mu - eta (s - tau))``, s the surprise of ``token`` over the kept, renormalised mass."""
    s = math.log2(float(p[keep].sum())) - math.log2(float(p[token]))
    return f32(np.float64(np.float32(mu)) - np.float64(np.float32(eta)) * (s - np.float64(np.float32(tau))))


def sample_row(x, state, temperature, top_k, top_p, seed, pos, r=1.0, pres=0.0, freq=0.0, min_p=0.0, threshold=0.1, probability=0.0,
               typical_p=1.0, top_n_sigma=0.0, mirostat_tau=0.0, mirostat_eta=0.0, mu=0.0, allowed=None):
    """``(token, mu', near)`` of the penalised (with ``allowed``: constrained) draw with the truncation samplers on one
    fp32 row; ``mirostat_tau > 0`` runs Mirostat from ``mu`` (mu' is mu on the rows it leaves alone)."""
    x3 = penalties_ref.penalize(x, state, r, pres, freq)
    if allowed is not None:
        x3 = np.where(allowed, x3, np.float32(np.nan)).astype(np.float32)
    x64 = x3.astype(np.float64)
    ok = ~np.isnan(x64)
    if not temperature > 0 or not ok.any() or not np.isfinite(x64[ok].max()):
        return ref.greedy(x64), f32(mu), False
    if mirostat_tau > 0:
        keep, p, near = mirostat_keep(x3, temperature, mu)
        score = np.where(keep, ref.perturbed(x64, temperature, seed, pos), -np.inf)
        token = int(np.argmax(score))
        mu2 = mirostat_update(p, keep, token, mu, mirostat_tau, mirostat_eta) if pos > 0 else f32(mu)
        return token, mu2, near
    keep = penalties_ref.keep_set(x3, top_k, top_p, min_p, temperature)
    keep, near_n = nsigma_keep(x3, keep, top_n_sigma)
    keep, near_t = typical_keep(x3, keep, typical_p)
    keep, near_x = dry_xtc_ref.xtc_keep(x3, keep, temperature, threshold, probability, seed, pos)
    score = np.where(keep, ref.perturbed(x64, temperature, seed, pos), -np.inf)
    return int(np.argmax(score)), f32(mu), near_n or near_t or near_x


def mu_close(got: float, want: float, eta: float) -> bool:
    """Whether a kernel mu' lies within the documented band of the reference's."""
    return abs(got - want) <= MU_BAND_ETA * eta + 2 * ulp32(want)


# ----------------------------------------------------------------------------- outside restatements (host tests) --
def hf_typical_keep(scores, mass: float, min_tokens_to_keep: int = 1) -> np.ndarray:
    """``transformers``' ``TypicalLogitsWarper`` step by step, in numpy float64: the mask of the entries it leaves."""
    s = np.asarray(scores, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        normalized = s - np.logaddexp.reduce(s)
        p = np.exp(normalized)
        ent = -np.nansum(normalized * p)
        shifted = np.abs(-normalized - ent)
    order = np.argsort(shifted, kind="stable")
    sorted_scores = shifted[order]
    sorted_logits = s[order]
    sl = np.exp(sorted_logits - np.max(sorted_logits))
    cum = np.cumsum(sl / sl.sum())
    last_ind = min(int((cum < mass).sum()), len(s) - 1)
    remove_sorted = sorted_scores > sorted_scores[last_ind]
    remove_sorted[:min_tokens_to_keep] = False
    keep = np.ones(len(s), dtype=bool)
    keep[order[remove_sorted]] = False
    return keep


def llama_mirostat_v2(logits, temperature: float, mu: float, tau: float, eta: float, pick) -> tuple[int, float, np.ndarray]:
    """llama.cpp's ``llama_sampler_mirostat_v2_apply`` after its temperature sampler, literally: sort by logit
    descending, softmax, keep the prefix before the first ``-log2 p > mu`` (at least one), renormalise, draw with
    ``pick(indices, probs)``, then ``mu -= eta * (-log2 p_token - tau)``.  Returns ``(token, mu', kept ids)``."""
    x = np.asarray(logits, dtype=np.float64) / temperature
    order = np.argsort(-x, kind="stable")
    xs = x[order]
    p = np.exp(xs - xs[0])
    p /= p.sum()
    size = len(p)
    for i in range(len(p)):
        if -math.log2(p[i]) > mu:
            size = i
            break
    size = max(size, 1)
    q = p[:size] / p[:size].sum()
    idx = pick(order[:size], q)
    token = int(order[:size][idx])
    observed = -math.log2(q[idx])
    return token, mu - eta * (observed - tau), np.sort(order[:size])
