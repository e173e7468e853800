"""Planted-winner probes of top-n-sigma, locally typical sampling and Mirostat 2.0 (the ``TRUNC`` forms of
``sample_kernel``, DESIGN.md section 25).

TEST INFRASTRUCTURE.  ``truncation_ref`` compares random draws with a float64 restatement and skips every draw whose
decisive quantity lies inside a band around its boundary, so the kernel's exact decisions inside those bands are never
compared.  A probe here is a row built around one such boundary, with every other entry -inf (-inf entries do not enter
sigma, S or S_K, and cannot win the draw): a target entry on one side of it, and a (seed, position) searched so that the
target's float64 score ``x_t / T + g_t`` beats every other planted entry by ``keep_set_ref.MARGIN``.  The expected
token is then certain.

``trunc_rule`` restates the kernel's arithmetic rather than the float64 definition: 2^-40 fixed-point masses from fp32
``expf``, ``e_i z_i`` in 2^-4 fixed point, the typical distances rounded to fp32 and their four radix levels over the
distance keys, the n-sigma bound in double rounded up to fp32, and Mirostat's threshold ``min(S 2^-mu, 2^40)``.  ``expf``
is modelled as the correctly rounded value moved by ``shift`` ulps (-2, 0, +2; CUDA's ``expf`` is within 2 ulps), and
``expf(0)`` as exactly 1.  Every probe's token is the same under the three shifts, equals ``truncation_ref.sample_row``
and lies outside that module's bands (the host test checks all three).  ``variant`` names a defect of
``NSIGMA_VARIANTS``, ``TYPICAL_VARIANTS`` or ``MIROSTAT_VARIANTS`` restated as a change of the rule, so the host test
can show that every defect gets at least one probe wrong.

Mirostat's mu' is compared too: exactly on rows whose kept set is k ties of the maximum (``expf(0)`` is 1, so S_K is
k 2^40 and e_token 2^40), and elsewhere within the interval spanned by the ``expf`` shifts (S_K and e_token moved in
opposite directions) widened by one fp32 ulp for the double ``log2``.
"""

from __future__ import annotations

import importlib.util
import math
import sys
from dataclasses import dataclass
from fractions import Fraction
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


K = _load("tiny_llm_b200_keep_set_ref", "keep_set_ref.py")
RP = _load("tiny_llm_b200_rejection_probe_ref", "rejection_probe_ref.py")
TR = _load("tiny_llm_b200_truncation_ref", "truncation_ref.py")
X = RP.X
pref = K.pref

VOCABS = RP.XTC_VOCABS
DTYPES = K.DTYPES
MARGIN = K.MARGIN
SHIFTS = (-2, 0, 2)
SCALE = float(1 << 40)
MU_SENTINEL = -7.375  # mu of every non-Mirostat row: the kernel must leave it alone
ETA_JUNK = 0.75  # eta of every non-Mirostat row (tau 0 switches Mirostat off; eta must not be read as an update)

NSIGMA_VARIANTS = {
    "sample sigma": "sigma over |F| - 1 instead of |F|",
    "-inf counted": "-inf entries summed with the finite ones (the mean is -inf, the bound NaN)",
    "masked entries counted": "disallowed entries counted in the mean and sigma",
    "raw (unpenalised) row": "mean and sigma from the unpenalised row",
    "bound rounded to nearest": "the bound rounded to nearest fp32 instead of up",
    "> at the bound": "an entry exactly at the bound dropped",
    "bound replaces tau": "the n-sigma bound replacing the top-k / top-p / min-p threshold instead of joining it by max",
}
TYPICAL_VARIANTS = {
    "crossing entry dropped": "only entries with mass(d <= d_i) < typical_p kept (the smallest d still forced)",
    "ties split": "entries tied at d* kept in index order only until the mass reaches typical_p",
    "tempered masses": "d, S_K and z_bar from the masses at the row's temperature",
    "S_K and z_bar over the whole row": "S_K and z_bar summed over every non-NaN entry instead of the keep set",
    "radix prefix at the wrong shift": "each radix level's prefix compared at shift instead of shift + 8",
    "smallest d not forced": "the crossing entry dropped and an empty set drawn as the row maximum",
    "> at the crossing": "d* taken where the mass strictly exceeds typical_p S_K",
}
MIROSTAT_VARIANTS = {
    "> at the threshold": "e_i > S 2^-mu instead of >=",
    "no 2^40 cap": "the threshold not capped at the maximum's mass, so mu < 0 keeps nothing",
    "S over the top-k keep set": "S summed over the top-k / top-p / min-p keep set",
    "surprise over S": "mu' from log2 S instead of log2 S_K",
    "top-k, top-p and min-p applied": "the keep threshold applied on a Mirostat row",
    "typical and n-sigma applied": "typical and top-n-sigma applied on a Mirostat row",
    "XTC applied": "XTC applied on a Mirostat row",
    "penalties after Mirostat": "Mirostat on the unpenalised row",
    "S counts disallowed entries": "disallowed entries summed into S",
    "mu read from rank 0": "the drawn token's value read from rank 0's slice at token % slice",
    "mu read one entry on": "the drawn token's value read at token + 1",
    "mu written at position 0": "mu updated at position 0",
    "mu written on greedy rows": "mu updated on greedy rows and rows whose maximum is not finite",
    "mu written on non-Mirostat rows": "mu updated on rows with tau = 0",
}
VARIANTS = {**NSIGMA_VARIANTS, **TYPICAL_VARIANTS, **MIROSTAT_VARIANTS}


# ------------------------------------------------------------------------------------------------ the probe --
@dataclass(repr=False)
class TruncProbe(K.Probe):
    typical_p: float = 1.0
    n_sigma: float = 0.0
    tau: float = 0.0  # Mirostat's tau (> 0: the row runs Mirostat)
    eta: float = ETA_JUNK
    mu: float = MU_SENTINEL
    theta: float = 0.5
    q: float = 0.0
    mu_lo: float = math.nan  # mu' after the launch: [mu_lo, mu_hi], one value when exact
    mu_hi: float = math.nan

    @property
    def mirostat(self) -> bool:
        return self.tau > 0

    @property
    def mu_exact(self) -> bool:
        return self.mu_lo == self.mu_hi

    def __repr__(self) -> str:
        return (K.Probe.__repr__(self)[:-1] + f", typical_p={self.typical_p!r}, n={self.n_sigma!r}, tau={self.tau}, eta={self.eta}, "
                f"mu={self.mu!r}, mu'=[{self.mu_lo!r}, {self.mu_hi!r}])")


@dataclass
class Decision:
    token: int
    mu: float  # mu' (the row's mu when the kernel leaves it)
    keep: np.ndarray | None  # over the support (None: greedy)


def f32(v) -> np.float32:
    return np.float32(v)


def _nudge(v: np.float32, k: int) -> np.float32:
    for _ in range(abs(k)):
        v = np.nextafter(v, f32(np.inf) if k > 0 else f32(0))
    return v


def expf(z, shift: int = 0) -> np.ndarray:
    """fp32 ``expf`` of fp32 ``z``: the correctly rounded value moved ``shift`` ulps; exp(0) is exactly 1."""
    z = np.asarray(z, np.float32)
    e = np.exp(z.astype(np.float64)).astype(np.float32)
    if shift:
        e = np.array([f32(1) if zz == 0 else _nudge(f32(ee), shift) for zz, ee in zip(z, e)], np.float32)
    return e


def masses(z, shift: int = 0) -> list[int]:
    """``__float2ull_rn(expf(z) * 2^40)`` per entry, as Python ints."""
    e = expf(z, shift).astype(np.float64) * SCALE
    return [int(v) for v in np.rint(e)]


def fl_ru(b: float) -> np.float32:
    f = f32(b)
    if math.isfinite(b) and float(f) < b:
        f = np.nextafter(f, f32(np.inf))
    return f


def fl_rn(b: float) -> np.float32:
    return f32(b)


def dkey(d: np.ndarray) -> np.ndarray:
    return np.asarray(d, np.float32).view(np.uint32).astype(np.int64)


def split_byte(k1: int, k2: int) -> int:
    """The first byte (0 the top one) in which two 32-bit keys differ (4: equal)."""
    for level in range(4):
        s = 24 - 8 * level
        if (k1 >> s) & 0xFF != (k2 >> s) & 0xFF:
            return level
    return 4


# ------------------------------------------------------------------------------------------ the support --
class Support:
    """A probe's row reduced to the entries that are not background -inf: the staged values, the top-k / top-p /
    min-p keep set, and what a defect needs (raw values, the disallowed entries' values)."""

    def __init__(self, pr: TruncProbe):
        st = np.zeros(pr.V, np.int32) if pr.state is None else pr.state
        x3 = pref.penalize(pr.x, st, pr.r, pr.pres, pr.freq)
        pen = x3.copy()
        raw = np.asarray(pr.x, np.float32)
        if pr.allowed is not None:
            x3 = np.where(pr.allowed, x3, f32(np.nan)).astype(np.float32)
            raw = np.where(pr.allowed, raw, f32(np.nan)).astype(np.float32)
        self.J = np.flatnonzero(~(np.isneginf(pr.x) & (st == 0)))
        self.bg_inf = bool(np.any(np.isneginf(x3)))  # a non-NaN -inf entry (background or planted)
        self.x = x3[self.J]
        self.pen = pen[self.J]  # penalised, mask not applied
        self.raw = raw[self.J]
        self.full = x3
        ok = ~np.isnan(x3)
        self.point = not pr.T > 0 or not ok.any() or not np.isfinite(x3[ok].max())
        self.greedy = ref.greedy(x3.astype(np.float64))
        self.K0 = None if self.point else pref.keep_set(x3, pr.k, pr.p, pr.min_p, pr.T)[self.J]


def _support(pr: TruncProbe) -> Support:
    s = getattr(pr, "_support", None)
    if s is None:
        s = Support(pr)
        object.__setattr__(pr, "_support", s)
    return s


# ----------------------------------------------------------------------------------------------- n-sigma --
def nsigma_bound(x, m: float, n: float) -> float:
    """The kernel's bound in double: ``m - n sqrt(sum (x - mean)^2 / |F|)`` over the values ``x``."""
    v = np.asarray(x, np.float64)
    cnt = float(len(v))
    mean = float(v.sum()) / cnt
    sq = float(((v - mean) * (v - mean)).sum())
    return float(m) - float(f32(n)) * math.sqrt(sq / cnt)


def sums_exact(x) -> bool:
    """Whether the kernel's two double sums over the values ``x`` are exact in every order: every term and partial sum
    is a multiple of the smallest term's last bit and below 2^53 of them."""
    v = [float(t) for t in np.asarray(x, np.float64)]
    mean = sum(v) / len(v)
    for terms in (v, [(t - mean) * (t - mean) for t in v]):
        nz = [Fraction(t) for t in terms if t != 0]
        if not nz:
            continue
        unit = min(Fraction(1, q.denominator) if q.denominator > 1 else Fraction(2) ** (len(bin(q.numerator & -q.numerator)) - 3)
                   for q in nz)
        if sum(abs(q) for q in nz) >= unit * 2**53:
            return False
    return True


def _nsigma_keep(pr, s: Support, keep, m: float, variant):
    n = pr.n_sigma
    if not n > 0:
        return keep
    fin = np.isfinite(s.x)
    vals = s.x
    if variant == "-inf counted" and s.bg_inf:
        return np.zeros_like(keep)  # the bound is NaN: no key reaches it
    if variant == "masked entries counted":
        fin = np.isfinite(s.pen)
        vals = s.pen
    if variant == "raw (unpenalised) row":
        fin = np.isfinite(s.raw)
        vals = s.raw
    v = vals[fin].astype(np.float64)
    cnt = len(v)
    mean = float(v.sum()) / cnt
    sq = float(((v - mean) * (v - mean)).sum())
    if variant == "sample sigma":
        cnt -= 1
    sigma = math.sqrt(sq / cnt) if cnt > 0 else math.nan
    b = float(m) - float(f32(n)) * sigma
    if math.isnan(b):
        return np.zeros_like(keep)
    b32 = fl_rn(b) if variant == "bound rounded to nearest" else fl_ru(b)
    with np.errstate(invalid="ignore"):
        cut = s.x > b32 if variant == "> at the bound" else s.x >= b32
    if variant == "bound replaces tau":
        return ~np.isnan(s.x) & cut
    return keep & cut


# ----------------------------------------------------------------------------------------------- typical --
def radix_dstar(dk: np.ndarray, e: list[int], want: float, wrong_shift: bool = False, strict: bool = False) -> int:
    """The four ascending radix levels over the distance keys: the smallest key with (double) mass(key <= d*) >= want."""
    prefix, below = 0, 0
    for level in range(4):
        shift = 24 - 8 * level
        cs = shift if wrong_shift else shift + 8
        bins = [0] * 256
        for k_, e_ in zip(dk, e):
            if level == 0 or (int(k_) >> cs) == (prefix >> cs):
                bins[(int(k_) >> shift) & 0xFF] += e_
        acc = below
        for j in range(256):
            tot = float(acc + bins[j])
            if (tot > want) if strict else (tot >= want):
                prefix |= j << shift
                below = acc
                break
            acc += bins[j]
    return prefix


def typical_terms(x, keep, m, T: float, shift: int, tempered: bool = False):
    """``(z, e, se, zbar, d keys)`` over ``keep``: the kernel's fixed-point sums and fp32 distances."""
    z = (x - f32(m)).astype(np.float32)
    if tempered:
        z = (z / f32(T)).astype(np.float32)
    e = masses(np.where(keep, z, f32(0)), shift)
    se = sz = 0
    for i in np.flatnonzero(keep):
        se += e[i]
        if e[i]:
            sz += int(np.rint(float(e[i]) * float(z[i]) * 16.0))
    zbar = float(sz) * 0.0625 / float(se)
    with np.errstate(invalid="ignore"):
        d = np.abs(zbar - z.astype(np.float64)).astype(np.float32)
    return z, e, se, zbar, dkey(d)


def _typical_keep(pr, s: Support, keep, m, shift, variant):
    tp = pr.typical_p
    if not 0 < tp < 1:
        return keep
    ok = ~np.isnan(s.x)
    over = ok if variant == "S_K and z_bar over the whole row" else keep
    _, _, se, zbar, _ = typical_terms(s.x, over, m, pr.T, shift, variant == "tempered masses")
    z, e, _, _, _ = typical_terms(s.x, keep, m, pr.T, shift, variant == "tempered masses")
    with np.errstate(invalid="ignore"):
        d = np.abs(zbar - z.astype(np.float64)).astype(np.float32)
    dk = dkey(d)
    idx = np.flatnonzero(keep)
    want = float(f32(tp)) * float(se)
    dstar = radix_dstar(dk[idx], [e[i] for i in idx], want, variant == "radix prefix at the wrong shift",
                        variant == "> at the crossing")
    out = keep & (dk <= dstar)
    if variant in ("crossing entry dropped", "smallest d not forced"):
        out = keep & (dk < dstar)
        if variant == "crossing entry dropped":
            out |= keep & (dk == dk[idx].min())
    elif variant == "ties split":
        order = sorted(idx, key=lambda i: (dk[i], i))
        out = np.zeros_like(keep)
        acc = 0
        for i in order:
            out[i] = True
            acc += e[i]
            if float(acc) >= want:
                break
    return out


# ---------------------------------------------------------------------------------------------- Mirostat --
def _tempered(x, m, T):
    return ((x - f32(m)).astype(np.float32) / f32(T)).astype(np.float32)


def _mirostat_keep(pr, s: Support, m, shift, variant):
    x = s.raw if variant == "penalties after Mirostat" else s.x
    if variant == "penalties after Mirostat":
        m = np.nanmax(x)
    ok = ~np.isnan(x)
    e = masses(np.where(ok, _tempered(np.where(ok, x, m), m, pr.T), f32(0)), shift)
    over = ok
    if variant == "S over the top-k keep set":
        over = s.K0
    if variant == "S counts disallowed entries":
        over = ~np.isnan(s.pen)
        e_all = masses(_tempered(np.where(over, s.pen, m), m, pr.T), shift)
        S = sum(e_all[i] for i in np.flatnonzero(over))
    else:
        S = sum(e[i] for i in np.flatnonzero(over))
    thr = float(S) * 2.0 ** (-float(f32(pr.mu)))
    if variant != "no 2^40 cap":
        thr = min(thr, SCALE)
    ev = np.array([float(v) for v in e])
    keep = ok & ((ev > thr) if variant == "> at the threshold" else (ev >= thr))
    return keep, e, S


def mirostat_mu(pr, s: Support, token: int, S_K: int, e_tok: int) -> float:
    """``fl32(mu - eta (log2 S_K - log2 e_token - tau))`` in double."""
    lg = lambda v: math.log2(v) if v > 0 else -math.inf  # noqa: E731
    sur = lg(S_K) - lg(e_tok)
    if math.isnan(sur):
        return math.nan
    v = float(f32(pr.mu)) - float(f32(pr.eta)) * (sur - float(f32(pr.tau)))
    with np.errstate(over="ignore"):
        return float(f32(v))


# -------------------------------------------------------------------------------------------------- rule --
def trunc_rule(pr: TruncProbe, variant: str | None = None, shift: int = 0, pos: int | None = None, tok_shift: int | None = None) -> Decision:
    """The kernel's token and mu' for one probe (``tok_shift``: the token's own ``expf`` shift in the mu update)."""
    pos = pr.pos if pos is None else pos
    s = _support(pr)
    mu0 = float(f32(pr.mu))
    C, sl = K.plan(pr.V)
    if s.point:
        mu = mu0
        if pr.mirostat and variant == "mu written on greedy rows" and pr.pos > 0:
            mu = float(f32(mu0 - float(f32(pr.eta)) * (0.0 - float(f32(pr.tau)))))
        return Decision(s.greedy, mu, None)
    ok = ~np.isnan(s.x)
    m = float(np.max(s.x[ok]))
    first_max = int(s.J[np.flatnonzero(ok & (s.x == m))[0]])
    keep = s.K0.copy()
    S_K = 0
    if pr.mirostat:
        if variant == "typical and n-sigma applied":
            keep = _typical_keep(pr, s, _nsigma_keep(pr, s, ok.copy(), m, None), m, shift, None)
            mkeep, e, _ = _mirostat_keep(pr, s, m, shift, variant)
            keep = keep & mkeep
        else:
            keep, e, _ = _mirostat_keep(pr, s, m, shift, variant)
        if variant == "top-k, top-p and min-p applied":
            keep &= s.K0
        S_K = sum(e[i] for i in np.flatnonzero(keep))
        if variant == "XTC applied" and pr.q > 0:
            keep, _ = X.xtc_keep(s.x, keep, pr.T, pr.theta, pr.q, pr.seed, pos)
    else:
        keep = _nsigma_keep(pr, s, keep, m, variant)
        keep = _typical_keep(pr, s, keep, m, shift, variant)
    cand = np.flatnonzero(keep & np.isfinite(s.x))
    if len(cand) == 0:
        token = first_max
    else:
        sc = s.x[cand].astype(np.float64) / pr.T + K.gumbel_at(s.J[cand], pr.seed, pos)
        token = int(s.J[cand[int(np.argmax(sc))]])
    mu = mu0
    if pr.mirostat and (pos > 0 or variant == "mu written at position 0"):
        ts = shift if tok_shift is None else tok_shift
        read = token
        if variant == "mu read from rank 0":
            read = token % sl
        elif variant == "mu read one entry on":
            read = token + 1 if token + 1 < pr.V else token - 1
        xt = s.full[read]
        e_tok = 0 if np.isnan(xt) else masses(_tempered(np.array([xt], np.float32), m, pr.T), ts)[0]
        Sx = S_K
        if variant == "surprise over S":
            Sx = sum(masses(_tempered(np.where(ok, s.x, m), m, pr.T), shift)[i] for i in np.flatnonzero(ok))
        mu = mirostat_mu(pr, s, token, Sx, e_tok)
    elif not pr.mirostat and variant == "mu written on non-Mirostat rows" and pos > 0:
        z = _tempered(np.where(ok, s.x, m), m, pr.T)
        e = masses(z, shift)
        S_K = sum(e[i] for i in np.flatnonzero(keep))
        j = int(np.flatnonzero(s.J == token)[0])
        mu = float(f32(mu0 - float(f32(pr.eta)) * (math.log2(S_K) - math.log2(e[j]) if e[j] else math.inf)))
    return Decision(token, mu, keep)


def mu_interval(pr: TruncProbe) -> tuple[float, float]:
    """mu' over every pair of ``expf`` shifts (S_K's, the token's), widened by one fp32 ulp each way unless every pair
    gives the same double (then it is exact, provided the double is not within 2^-40 of an fp32 rounding point)."""
    vals = []
    for a in SHIFTS:
        for b in SHIFTS:
            vals.append(trunc_rule(pr, shift=a, tok_shift=b).mu)
    lo, hi = min(vals), max(vals)
    if lo == hi and _tie_row(pr):
        return lo, hi
    return float(np.nextafter(f32(lo), f32(-np.inf))), float(np.nextafter(f32(hi), f32(np.inf)))


def _tie_row(pr: TruncProbe) -> bool:
    """Every kept entry is a tie of the maximum, and mu' in double is far from an fp32 rounding point."""
    d = trunc_rule(pr)
    s = _support(pr)
    kept = s.x[d.keep]
    if not len(kept) or not np.all(kept == np.max(s.x[~np.isnan(s.x)])):
        return False
    k = len(kept)
    v = float(f32(pr.mu)) - float(f32(pr.eta)) * (math.log2(k) - float(f32(pr.tau)))
    f = f32(v)
    lo = float(np.nextafter(f, f32(-np.inf)))
    hi = float(np.nextafter(f, f32(np.inf)))
    mid_lo, mid_hi = (lo + float(f)) / 2, (float(f) + hi) / 2
    return min(abs(v - mid_lo), abs(v - mid_hi)) > 2.0**-40 * max(1.0, abs(v))


# -------------------------------------------------------------------------------------------------- settle --
def whole_row(pr: TruncProbe):
    """``truncation_ref.sample_row`` on the probe's whole row: ``(token, mu', near)``."""
    st = np.zeros(pr.V, np.int32) if pr.state is None else pr.state
    return TR.sample_row(pr.x, st, pr.T, pr.k, pr.p, pr.seed, pr.pos, pr.r, pr.pres, pr.freq, pr.min_p, pr.theta,
                         0.0 if pr.mirostat else pr.q, pr.typical_p, pr.n_sigma, pr.tau, pr.eta, pr.mu, pr.allowed)


def settle(pr: TruncProbe, seed: int, pos0: bool = False, tries: int = 1 << 17) -> TruncProbe:
    """Search positions at ``seed`` (or, ``pos0``, seeds at position 0) so that the target beats every other planted
    entry by MARGIN and the kept winner every other kept entry; fill ``want`` and mu'."""
    s = _support(pr)
    pr.seed = seed
    if s.point:
        pr.pos = 0 if pos0 else 1 + seed % 1000
    else:
        d = trunc_rule(pr, pos=1)
        live = np.flatnonzero(np.isfinite(s.x))
        tgt = int(np.flatnonzero(s.J[live] == pr.target)[0])
        kept = np.flatnonzero(d.keep[live])
        xs = s.x[live].astype(np.float64) / pr.T
        found = False
        if pos0:
            seeds = [seed + 7919 * j for j in range(4096)]
            for sd in seeds:
                g = K.gumbel_at(s.J[live], sd, 0)
                if _clear(xs + g, tgt, kept):
                    pr.seed, pr.pos, found = sd, 0, True
                    break
        else:
            start = 1 + (seed % 997) * 1000
            for b in range(0, tries, 4096):
                ps = np.arange(start + b, start + b + 4096)
                G = K.gumbel_at(s.J[live], seed, ps)
                for j in range(len(ps)):
                    if _clear(xs + G[j], tgt, kept):
                        pr.pos, found = int(ps[j]), True
                        break
                if found:
                    break
        assert found, f"no position settles {pr!r}"
    d = trunc_rule(pr)
    pr.want = d.token
    pr.inside = d.token == pr.target
    if pr.mirostat and not s.point and pr.pos > 0:
        pr.mu_lo, pr.mu_hi = mu_interval(pr)
    else:
        pr.mu_lo = pr.mu_hi = float(f32(pr.mu))
    return pr


def _clear(sc, tgt, kept) -> bool:
    o = np.argsort(-sc)
    if o[0] != tgt or (len(o) > 1 and sc[o[0]] - sc[o[1]] < MARGIN):
        return False
    if len(kept) > 1:
        k = np.sort(sc[kept])[::-1]
        if k[0] - k[1] < MARGIN:
            return False
    return True


# ------------------------------------------------------------------------------------------------ catalogue --
class Catalogue:
    """Every truncation probe of one (V, dtype); ``probes`` in a fixed order."""

    def __init__(self, V: int, dtype: str):
        self.V, self.dtype = V, dtype
        self.rows = K._Rows(V, dtype, seed=V * 17 + DTYPES.index(dtype) + 3)
        self.C, self.slice = K.plan(V)
        self.probes: list[TruncProbe] = []
        self.single()
        if V >= 8:
            self.nsigma()
            self.nsigma_against_other_bounds()
            self.nsigma_penalty_and_mask()
            self.typical_levels()
            self.typical_ties()
            self.typical_tiny()
            self.typical_separated()
            self.mirostat_sides()
            self.mirostat_ignores()
            self.mirostat_penalty_and_mask()
            self.sentinels()
        if V >= 4:
            self.mirostat_ties()

    # -- helpers
    def _g(self, v) -> float:
        return K.on_grid(v, self.dtype)

    def _row(self, vals, first=None):
        x = np.full(self.V, -np.inf, np.float32)
        idx = self.rows.spots(len(vals), first)
        x[idx] = [self._g(v) for v in vals]
        return x, idx

    def _spot(self, j: int) -> int:
        s = RP.slice_spots(self.V)
        return s[j % len(s)]

    def _add(self, pr: TruncProbe, pos0: bool = False) -> TruncProbe:
        pr = settle(pr, self.rows.seed64(), pos0)
        self.probes.append(pr)
        return pr

    def _probe(self, kind, x, target, idx, **kw) -> TruncProbe:
        return TruncProbe(kind, self.V, self.dtype, x.copy(), target, planted=list(idx), **kw)

    # -- every V
    def single(self) -> None:
        """One finite entry: sigma is 0 and the entry stays; typical keeps it; Mirostat's maximum always stays."""
        x, idx = self._row([1.5], first=self._spot(1))
        self._add(self._probe("nsigma one finite entry", x, idx[0], idx, n_sigma=1.0, T=0.8))
        self._add(self._probe("typical one finite entry", x, idx[0], idx, typical_p=0.3))

    # -- n-sigma
    def _nsigma_values(self, j: int):
        """Eight finite entries on the dtype grid whose double sums are exact in any order: the maximum, b_at and its
        dtype-grid neighbour below, and (fp32) an entry that cancels the neighbour's low bit in the sum; ``j`` moves
        one free entry, and with it sigma."""
        b_at = self._g(-1.25)
        b_below = K.next_below(b_at, self.dtype)
        low = b_at - b_below
        comp = float(f32(0.5 + low)) if self.dtype == "f32" else self._g(0.5)
        vals = [self._g(1.0), comp, self._g(0.25), self._g(j / 64), self._g(-0.375), self._g(-0.75), b_at, b_below]
        assert sums_exact(vals), vals
        return vals

    def _n_for(self, vals, lo: float, hi: float, n0: float) -> float | None:
        """An fp32 n whose bound m - n sigma (double) lies in (lo, hi], or None."""
        v = np.asarray(vals, np.float64)
        m = float(v.max())
        up = down = f32(n0)
        for _ in range(64):
            for cand in (up, down):
                b = nsigma_bound(v, m, float(cand))
                if lo < b <= hi:
                    return float(cand)
            up, down = np.nextafter(up, f32(np.inf)), np.nextafter(down, f32(0))
        return None

    def nsigma(self) -> None:
        def row_and_n(lo_u: float, hi_u: float):
            for j in range(40):
                vals = self._nsigma_values(j)
                b_at = vals[6]
                u = float(np.spacing(f32(abs(b_at))))
                n0 = (vals[0] - b_at) / (vals[0] - nsigma_bound(vals, vals[0], 1.0))
                n = self._n_for(vals, b_at + lo_u * u, b_at + hi_u * u, n0)
                if n is not None:
                    x, idx = self._row(vals, first=self._spot(j))
                    return x, idx, n
            raise AssertionError("no n-sigma row")

        T = (0.8, 1.0, 1.5)[DTYPES.index(self.dtype)]
        # the bound in (b_at - ulp, b_at]: rounded up it is b_at, which stays; its dtype-grid neighbour below goes
        x, idx, n_at = row_and_n(-1.0, 0.0)
        at, below = idx[6], idx[7]
        self._add(self._probe("nsigma at the bound", x, at, idx, n_sigma=n_at, T=T))
        self._add(self._probe("nsigma neighbour below", x, below, idx, n_sigma=n_at, T=T))
        # the bound in (b_at, b_at + ulp / 2): rounded up it drops b_at, rounded to nearest it would keep it
        x, idx, n_off = row_and_n(2.0**-30, 0.5 - 2.0**-30)
        self._add(self._probe("nsigma off the fp32 grid", x, idx[6], idx, n_sigma=n_off, T=T))
        # every finite entry equal: sigma 0, the bound is m and every tie stays
        ties = sorted(self.rows.spots(3, self._spot(-1)))
        x = np.full(self.V, -np.inf, np.float32)
        x[ties] = self._g(0.75)
        self._add(self._probe("nsigma all equal", x, ties[-1], ties, n_sigma=2.0))

    def _separating_n(self, pr: TruncProbe, variant: str, ns) -> TruncProbe | None:
        """The first n of ``ns`` at which the rule and ``variant`` disagree on keeping the target, the bound at least
        2^-10 from every finite entry."""
        s = _support(pr)
        for n in ns:
            pr.n_sigma = float(f32(n))
            ok = ~np.isnan(s.x)
            m = float(np.max(s.x[ok]))
            fin = np.isfinite(s.x)
            b = nsigma_bound(s.x[fin], m, pr.n_sigma)
            if np.min(np.abs(s.x[fin].astype(np.float64) - b)) < 2.0**-10:
                continue
            t = int(np.flatnonzero(s.J == pr.target)[0])
            good = _nsigma_keep(pr, s, s.K0.copy(), m, None)[t]
            bad = _nsigma_keep(pr, s, s.K0.copy(), m, variant)[t]
            if good != bad:
                return pr
        return None

    def nsigma_against_other_bounds(self) -> None:
        """The bound joins top-k / min-p by max: a target above the n-sigma bound but below min-p's (or top-k's) bound
        is dropped, one above min-p's but below n-sigma's too."""
        vals = [2.0, 1.5, 1.0, 0.5, 0.0, -0.5, -1.5, -3.0]
        x, idx = self._row(vals, first=self._spot(2))
        ns = [0.25 * j for j in range(1, 24)]
        pr = self._probe("nsigma below min-p's bound", x, idx[3], idx, min_p=K._min_p_for(self._g(2.0), 1.0, self._g(0.75)))
        assert self._separating_n(pr, "bound replaces tau", ns) is not None
        self._add(pr)
        pr = self._probe("nsigma below top-k's bound", x, idx[4], idx, k=4)
        assert self._separating_n(pr, "bound replaces tau", ns) is not None
        self._add(pr)
        pr = self._probe("nsigma above top-k's bound", x, idx[5], idx, k=7, n_sigma=1.0)
        s = _support(pr)
        assert s.K0[np.flatnonzero(s.J == idx[5])[0]] and not trunc_rule(pr, pos=1).keep[np.flatnonzero(s.J == idx[5])[0]]
        self._add(pr)

    def nsigma_penalty_and_mask(self) -> None:
        ns = [0.125 * j for j in range(1, 40)]
        # a prompt token at 3.0 becomes 1.0 under repetition 3: sigma and the maximum move
        vals = [3.0, 1.75, 1.25, 0.5, 0.0, -0.75, -1.5, -2.5]
        x, idx = self._row(vals, first=self._spot(3))
        st = np.zeros(self.V, np.int32)
        st[idx[0]] = pref.PROMPT
        for t in (idx[3], idx[4], idx[5]):
            pr = self._probe("nsigma penalty moves sigma", x, t, idx, r=3.0, state=st)
            if self._separating_n(pr, "raw (unpenalised) row", ns) is not None:
                self._add(pr)
                break
        else:
            raise AssertionError("no penalised n-sigma probe")
        # a disallowed entry at -6 would widen sigma
        vals = [1.5, 1.0, 0.5, 0.0, -0.5, -1.0, -6.0]
        x, idx = self._row(vals, first=self._spot(1))
        allowed = np.ones(self.V, bool)
        allowed[idx[6]] = False
        for t in (idx[3], idx[4], idx[5]):
            pr = self._probe("nsigma masked entry", x, t, idx[:6], allowed=allowed)
            if self._separating_n(pr, "masked entries counted", ns) is not None:
                self._add(pr)
                break
        else:
            raise AssertionError("no masked n-sigma probe")

    # -- typical
    def _typ_between(self, pr: TruncProbe, lo: float, hi: float) -> float:
        t = f32((lo + hi) / 2)
        assert lo + TR.TYPICAL_MASS_BAND * 2 < float(t) < hi - TR.TYPICAL_MASS_BAND * 2, (lo, hi)
        return float(t)

    def _masses_by_d(self, pr: TruncProbe):
        """Float64 ``(p, d)`` of truncation_ref over the support's keep set."""
        s = _support(pr)
        keep = TR.nsigma_keep(s.full, pref.keep_set(s.full, pr.k, pr.p, pr.min_p, pr.T), pr.n_sigma)[0]
        p, d = TR.typical_distances(s.full, keep)
        return p, d

    def typical_levels(self) -> None:
        """A boundary pair (a, b), d_a < d_b, whose distance keys first differ at byte L: typical_p between mass(d <
        d_a) and mass(d <= d_a) keeps a and drops b; between mass(d <= d_a) and mass(d <= d_b) it keeps b.  The pair
        sits near 0 with the maximum at 9, so z = x - 9 takes the fine grid of x near 0 in every dtype."""
        m = 9.0
        steps = {0: [0.25, 0.5], 1: [2.0**-4, 2.0**-3], 2: [2.0**-9, 2.0**-8], 3: [2.0**-13, 2.0**-12]}
        grid = np.unique(K.to_dtype(np.linspace(-2.5, 2.5, 4001), self.dtype))
        head = [self._g(v) for v in (m, m - 1, m - 2, m - 3)]
        for L in range(4):
            found = None
            for st_ in steps[L]:
                below = K.to_dtype(grid - st_, self.dtype)
                for xa, xb in zip(grid, below):
                    if not xb < xa:
                        continue
                    xc = np.array(head + [xa, xb], np.float32)
                    _, _, _, _, dk = typical_terms(xc, np.ones(6, bool), m, 1.0, 0)
                    if not dk[4] < dk[5] or split_byte(int(dk[4]), int(dk[5])) != L:
                        continue
                    p, d = TR.typical_distances(xc, np.ones(6, bool))
                    if not d[4] + TR.TYPICAL_D_BAND < d[5] or np.any((d[:4] > d[4] - TR.TYPICAL_D_BAND) & (d[:4] < d[5] + TR.TYPICAL_D_BAND)):
                        continue
                    if p[4] < 16 * TR.TYPICAL_MASS_BAND or p[5] < 16 * TR.TYPICAL_MASS_BAND:
                        continue
                    found = (float(xa), float(xb), p, d)
                    break
                if found:
                    break
            assert found, (L, self.V, self.dtype)
            xa, xb, p, d = found
            x, idx = self._row(head + [xa, xb], first=self._spot(L))
            a, b = idx[4], idx[5]
            below_a = float(p[d < d[4]].sum())
            t1 = self._typ_between(None, below_a, below_a + p[4])
            t2 = self._typ_between(None, below_a + p[4], below_a + p[4] + p[5])
            self._add(self._probe(f"typical level {L}", x, a, idx, T=3.0, typical_p=t1))
            self._add(self._probe(f"typical level {L}", x, b, idx, T=3.0, typical_p=t1))
            self._add(self._probe(f"typical level {L}", x, b, idx, T=3.0, typical_p=t2))

    def typical_ties(self) -> None:
        """Two entries with one logit (one d, bit for bit) on the first and the last rank, d* at them and typical_p
        below the mass of the first alone: both stay, and the later one is drawn."""
        ends = RP.slice_spots(self.V)
        t1, t2 = ends[0], ends[-1]
        others = [i for i in self.rows.spots(6) if i not in (t1, t2)][:3]
        x = np.full(self.V, -np.inf, np.float32)
        x[others] = [self._g(2.0), self._g(-0.5), self._g(-2.0)]
        x[[t1, t2]] = self._g(1.0)
        pr = self._probe("typical ties across ranks", x, t2, others + [t1, t2])
        p, d = self._masses_by_d(pr)
        below = p[d < d[t1]].sum()
        pr.typical_p = self._typ_between(pr, below, below + p[t1])
        self._add(pr)

    def typical_tiny(self) -> None:
        """typical_p below every mass: the entry nearest the entropy (not the maximum) is the only one left."""
        x, idx = self._row([1.0, 0.75, 0.5, 0.25, 0.0, -0.25], first=self._spot(1))
        pr = self._probe("typical tiny p", x, idx[0], idx, typical_p=0.01)
        p, d = self._masses_by_d(pr)
        j = int(np.argmin(np.where(np.isfinite(d), d, np.inf)))
        assert j != idx[0] and p[j] > 0.03
        pr.target = j
        self._add(pr)

    def _separating_typ(self, pr: TruncProbe, variant: str, targets) -> TruncProbe | None:
        """A typical_p at which the rule and ``variant`` disagree on keeping one of ``targets``: midpoints between the
        cumulative masses (in d order) of both rules, kept off the bands."""
        s = _support(pr)
        p, d = self._masses_by_d(pr)
        fin = np.flatnonzero(np.isfinite(d) & (p > 0))
        cums = sorted({float(p[d <= d[i]].sum()) for i in fin} | {0.0})
        cand = [(a + b) / 2 for a, b in zip(cums, cums[1:]) if b - a > 8 * TR.TYPICAL_MASS_BAND]
        cand += [c + sgn * 0.01 for c in cums for sgn in (-1, 1)]
        for t in targets:
            j = int(np.flatnonzero(s.J == t)[0])
            for c in sorted(set(cand)):
                if not 0.02 < c < 0.98:
                    continue
                pr.typical_p, pr.target = float(f32(c)), t
                if TR.typical_keep(s.full, TR.nsigma_keep(s.full, pref.keep_set(s.full, pr.k, pr.p, pr.min_p, pr.T), pr.n_sigma)[0],
                                   pr.typical_p)[1]:
                    continue
                good = trunc_rule(pr, pos=1).keep[j]
                bad = trunc_rule(pr, variant, pos=1).keep[j]
                if good != bad:
                    return pr
        return None

    def typical_separated(self) -> None:
        """Entries cut by top-k or n-sigma, counted in S_K and z_bar, would move d*; at T = 0.5 and 2 the tempered
        masses would keep another set."""
        vals = [1.0, 0.5, 0.25, -0.5, -0.5, -0.5, -0.5, -0.75]
        x, idx = self._row(vals, first=self._spot(2))
        for kind, kw in (("typical outside K: top-k", dict(k=3)), ("typical outside K: n-sigma", dict(n_sigma=0.5))):
            pr = self._probe(kind, x, idx[0], idx, **kw)
            assert self._separating_typ(pr, "S_K and z_bar over the whole row", idx[:3]) is not None, kind
            self._add(pr)
        vals = [1.0, 0.0, -0.5, -1.0, -2.0, -3.5]
        x, idx = self._row(vals, first=self._spot(3))
        for T in (0.5, 2.0):
            pr = self._probe(f"typical T = {T:g}", x, idx[0], idx, T=T)
            assert self._separating_typ(pr, "tempered masses", idx) is not None, T
            self._add(pr)

    # -- Mirostat
    def _surprise(self, pr: TruncProbe, j: int, over=None) -> float:
        s = _support(pr)
        x = s.full.astype(np.float64)
        ok = ~np.isnan(x)
        over = ok if over is None else over
        m = np.max(x[ok])
        e = np.where(ok, np.exp((np.where(ok, x, m) - m) / pr.T), 0.0)
        return float(-math.log2(e[j] / e[over].sum()))

    def mirostat_sides(self) -> None:
        vals = [1.0, 0.5, 0.0, -0.5, -1.5, -3.0]
        for j, T in enumerate((0.7, 1.0, 1.3)):
            x, idx = self._row(vals, first=self._spot(j))
            t = idx[3]
            base = self._probe("x", x, t, idx, T=T, tau=3.0, eta=0.1)
            sv = self._surprise(base, t)
            for name, mu in (("mirostat kept", sv + 0.05), ("mirostat dropped", sv - 0.05)):
                self._add(self._probe(name, x, t, idx, T=T, tau=float(f32(3.0 + j)), eta=float(f32(0.1 * (j + 1))), mu=float(f32(mu))))
        # S over the whole row: top-k 2 keeps {0, 1}; the target's surprise over them is below mu, over the row above
        x, idx = self._row(vals, first=self._spot(1))
        t = idx[2]
        base = self._probe("x", x, t, idx, k=2, tau=3.0, eta=0.2)
        s = _support(base)
        lo = self._surprise(base, t, pref.keep_set(s.full, 2, 0.0, 0.0, 1.0))
        hi = self._surprise(base, t)
        assert lo + 0.1 < hi
        self._add(self._probe("mirostat S over the row", x, t, idx, k=2, tau=3.0, eta=0.2, mu=float(f32((lo + hi) / 2))))

    def mirostat_ties(self) -> None:
        """k ties of the maximum, one on each rank (three at C = 1), and mu < 0: the cap keeps every tie, and mu' =
        fl32(mu - eta (log2 k - tau)) exactly, with the drawn tie on each rank.  The capped threshold is the ties' own
        mass 2^40, so ``>`` keeps nothing."""
        C, s = self.C, self.slice
        if C == 1:
            ties = sorted(self.rows.spots(3, self._spot(0)))
        else:
            ties = [int(self.rows.rng.integers(r * s, min(self.V, (r + 1) * s))) for r in range(C)]
        low = [i for i in self.rows.spots(len(ties) + 2) if i not in ties][:2] if self.V >= 8 else []
        x = np.full(self.V, -np.inf, np.float32)
        x[ties] = self._g(0.5)
        if low:
            x[low] = [self._g(0.25), self._g(-1.0)]
        for c, t in enumerate(ties):
            mu = -1.0 - 0.25 * c
            self._add(self._probe("mirostat ties mu < 0", x, t, ties + low, tau=float(f32(1.5 + 0.5 * c)), eta=0.125, mu=mu, T=1.0))

    def mirostat_ignores(self) -> None:
        """top-k 1, top-p, min-p, typical, n-sigma and XTC arrays on a Mirostat row are not read."""
        vals = [1.0, 0.75, 0.25, -0.25, -1.0]
        x, idx = self._row(vals, first=self._spot(2))
        kw = dict(k=1, p=0.2, min_p=0.9, typical_p=0.05, n_sigma=0.1, q=1.0, theta=0.05, tau=4.0, eta=0.3, mu=9.0)
        for t in (idx[0], idx[3]):
            self._add(self._probe("mirostat ignores the other samplers", x, t, idx, **kw))

    def mirostat_penalty_and_mask(self) -> None:
        vals = [2.0, 1.0, 0.5, 0.0, -1.0]
        x, idx = self._row(vals, first=self._spot(3))
        st = np.zeros(self.V, np.int32)
        st[idx[0]] = pref.PROMPT  # repetition 4: 2.0 -> 0.5
        pr = self._probe("x", x, idx[3], idx, r=4.0, state=st, tau=3.0, eta=0.1)
        sv = self._surprise(pr, idx[3])
        self._add(self._probe("mirostat after a penalty", x, idx[3], idx, r=4.0, state=st, tau=3.0, eta=0.1, mu=float(f32(sv + 0.05))))
        allowed = np.ones(self.V, bool)
        allowed[idx[0]] = False
        pr = self._probe("x", x, idx[3], idx[1:], allowed=allowed, tau=3.0, eta=0.1)
        sv = self._surprise(pr, idx[3])
        self._add(self._probe("mirostat after a mask", x, idx[3], idx[1:], allowed=allowed, tau=3.0, eta=0.1, mu=float(f32(sv + 0.05))))

    def sentinels(self) -> None:
        """mu stays at position 0, on greedy rows and on rows whose maximum is +inf."""
        vals = [1.0, 0.5, 0.0]
        x, idx = self._row(vals, first=self._spot(1))
        self._add(self._probe("mu at position 0", x, idx[1], idx, tau=3.0, eta=0.5, mu=2.5), pos0=True)
        self._add(self._probe("mu on a greedy row", x, idx[0], idx, T=0.0, tau=3.0, eta=0.5, mu=2.5))
        y = x.copy()
        y[idx[2]] = np.inf
        self._add(self._probe("mu with a non-finite maximum", y, idx[2], idx, tau=3.0, eta=0.5, mu=2.5))


FORMS = ("penalized off", "penalized on", "constrained + state")


def forms_of(pr: TruncProbe) -> tuple[str, ...]:
    if pr.allowed is not None:
        return ("constrained + state",)
    if pr.penalized or pr.state is not None:
        return ("penalized on", "constrained + state")
    return FORMS
