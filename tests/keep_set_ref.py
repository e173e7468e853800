"""Planted-winner probes of the sampling kernels' keep set (``tl_sample``, ``tl_sample_penalized``,
``tl_sample_constrained``; DESIGN.md sections 8, 8b and 8c).

TEST INFRASTRUCTURE.  A draw compared on random rows says little about the keep set ``{x >= tau}``: a threshold one
entry too loose or too tight changes the token only when that entry would have won the Gumbel argmax.  A probe is a
row built around one boundary (the k-th value, the top-p boundary v*, min-p's bound, a mask, a penalised value), a
target entry ``t`` on one side of it, and a (seed, position) searched so that ``t``'s float64 score ``x_t / T + g_t``
beats every other planted entry by at least ``MARGIN``:

* ``t`` in the reference keep set: the kernel must draw ``t``;
* ``t`` just outside it: the kernel must not draw ``t`` and must draw the reference's token, whose score beats every
  other kept planted entry by ``MARGIN`` as well.

Entries that are not planted (the background) are kept only when their best possible score, ``x / T + G_MAX``, is
below the winner's by ``MARGIN``.  ``MARGIN`` is far above the fp32 rounding of the kernel's scores, so each probe
asserts one token with ``==`` and a wrong threshold fails with certainty.  Top-k and min-p compare fp32 values exactly;
top-p probes keep every planted entry's mass above at least ``100 eps`` away from ``top_p`` (``eps`` as in the draw
tests' tolerance).

The reference is ``penalties_ref`` (the penalties and the min-p bound in fp32, keep set and draw in float64 through
``oracle.sampling``); a mask makes disallowed entries NaN, as the kernel does.
"""

from __future__ import annotations

import importlib.util
import math
import sys
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np

from oracle import sampling as ref

MARGIN = 0.25
G_MAX = -math.log(-math.log(1.0 - 2.0**-24))  # the largest Gumbel value the kernel's uniforms give
DTYPES = ("f32", "f16", "bf16")
FLT_MIN = float(np.finfo(np.float32).tiny)
MASK32 = 0xFFFFFFFF


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


pref = _load("tiny_llm_b200_penalties_ref", "penalties_ref.py")


# ------------------------------------------------------------------------------------------ values and keys --
def f32(v) -> np.float32:
    return np.float32(v)


def key(v) -> int:
    """The kernel's order-preserving 32-bit key of an fp32 value (+0 and -0 share one key)."""
    v = f32(v)
    b = int(np.array(0.0 if v == 0 else v, dtype=np.float32).view(np.uint32))
    return (~b) & MASK32 if b & 0x80000000 else b | 0x80000000


def from_key(k: int) -> float:
    b = k & 0x7FFFFFFF if k & 0x80000000 else (~k) & MASK32
    return float(np.array(b, dtype=np.uint32).view(np.float32))


def to_dtype(x, dtype: str) -> np.ndarray:
    """``x`` rounded to the dtype's grid, as fp32 values."""
    import torch

    x = np.asarray(x, dtype=np.float32)
    if dtype == "f32":
        return x.copy()
    t = torch.from_numpy(np.ascontiguousarray(x)).to(torch.float16 if dtype == "f16" else torch.bfloat16)
    return t.float().numpy()


def on_grid(v, dtype: str) -> float:
    return float(to_dtype([v], dtype)[0])


KEY_UNIT = {"f32": 1, "f16": 1 << 13, "bf16": 1 << 16}  # key step between neighbours of a normal value


def next_below(v, dtype: str) -> float:
    """The dtype's largest value below ``v`` (``v`` on the grid)."""
    if dtype == "f32":
        return float(np.nextafter(f32(v), f32(-np.inf)))
    if dtype == "f16":
        return float(np.nextafter(np.float16(v), np.float16(-np.inf)))
    b = int(np.array(f32(v)).view(np.uint32)) >> 16
    b = 0x8001 if v == 0 else (b - 1 if v > 0 else b + 1)
    return float(np.array(b << 16, dtype=np.uint32).view(np.float32))


def split_at_level(v0, level: int, dtype: str) -> tuple[float, float]:
    """``(a, b)``, neighbours on the dtype's grid near ``v0`` whose keys share the top ``level`` bytes and differ in
    byte ``level`` (byte 0 the top one): the radix select separates them at that level.  For fp16 and bf16, ``v0``
    must be positive (a negative value's key has its low bits set)."""
    k = key(on_grid(v0, dtype))
    shift = 8 * (3 - level)
    byte = (k >> shift) & 0xFF
    k = (k >> (shift + 8) << (shift + 8)) | ((byte or 0x80) << shift)  # the lower bytes zero: k - unit borrows in `level`
    a = from_key(k)
    b = from_key(k - KEY_UNIT[dtype])
    assert on_grid(a, dtype) == a and on_grid(b, dtype) == b and b < a
    assert key(a) >> (shift + 8) == key(b) >> (shift + 8) and (key(a) >> shift) & 0xFF != (key(b) >> shift) & 0xFF
    return a, b


# ------------------------------------------------------------------------------------------------- Philox --
def gumbel_at(indices, seed: int, pos) -> np.ndarray:
    """``g_i`` of ``oracle.sampling.gumbel`` at ``indices`` only: Philox4x32-10 at counters ``(i >> 2, pos, 0, 0)``.
    ``pos`` scalar -> ``[len(indices)]``; ``pos`` 1-D -> ``[len(pos), len(indices)]``."""
    idx = np.asarray(indices, dtype=np.int64).reshape(-1)
    ps = np.atleast_1d(np.asarray(pos, dtype=np.int64))
    ctr = np.zeros((len(ps), len(idx), 4), dtype=np.uint64)
    ctr[..., 0] = (idx >> 2)[None, :]
    ctr[..., 1] = (ps & MASK32)[:, None]
    words = ref.philox4x32_10(ctr, (seed & MASK32, (seed >> 32) & MASK32))
    w = np.take_along_axis(words, (idx & 3)[None, :, None], axis=2)[..., 0].astype(np.uint64)
    u = (2.0 * (w >> np.uint64(9)).astype(np.float64) + 1.0) * 2.0**-24
    g = -np.log(-np.log(u))
    return g if np.ndim(pos) else g[0]


# ------------------------------------------------------------------------------------------------- layout --
def plan(V: int) -> tuple[int, int]:
    """``sample_plan``: (cluster size C, slice length)."""
    c = min(-(-V // 4096), 8)
    return c, -(-(-(-V // c)) // 8) * 8


def boundary_spots(V: int) -> list[int]:
    """Entry 0, entry V - 1, the last entry of rank 0's slice and the first entry of rank C - 1."""
    C, s = plan(V)
    return sorted({0, V - 1, min(s - 1, V - 1), (C - 1) * s})


# ------------------------------------------------------------------------------------------------- probes --
@dataclass
class Probe:
    kind: str
    V: int
    dtype: str
    x: np.ndarray  # the raw row, fp32 values on the dtype's grid
    target: int
    T: float = 1.0  # fp32 values, as the kernel reads them
    k: int = 0
    p: float = 0.0
    min_p: float = 0.0
    r: float = 1.0
    pres: float = 0.0
    freq: float = 0.0
    state: np.ndarray | None = None  # int32 [V] token state (None: zeros)
    allowed: np.ndarray | None = None  # bool [V] (None: unconstrained)
    planted: list = field(default_factory=list)
    seed: int = 0
    pos: int = 0
    inside: bool = True
    want: int = -1
    keep: np.ndarray | None = None

    @property
    def penalized(self) -> bool:
        return self.r != 1.0 or self.pres != 0.0 or self.freq != 0.0 or self.min_p > 0.0

    def staged(self) -> np.ndarray:
        """The fp32 row every step of the kernel runs on: penalised, disallowed entries NaN."""
        st = np.zeros(self.V, np.int32) if self.state is None else self.state
        x3 = pref.penalize(self.x, st, self.r, self.pres, self.freq)
        if self.allowed is not None:
            x3 = np.where(self.allowed, x3, np.float32(np.nan)).astype(np.float32)
        return x3

    def __repr__(self) -> str:
        return (f"Probe({self.kind}, V={self.V}, {self.dtype}, t={self.target} {'in' if self.inside else 'out'}, "
                f"want={self.want}, T={self.T}, k={self.k}, p={self.p}, min_p={self.min_p}, r={self.r}, pres={self.pres}, "
                f"freq={self.freq}, seed={self.seed:#x}, pos={self.pos})")


def reference_keep(pr: Probe) -> tuple[np.ndarray | None, int | None]:
    """``(keep, greedy_token)``: the keep mask of a sampled row, or the token of a greedy / non-finite row."""
    x3 = pr.staged()
    x64 = x3.astype(np.float64)
    ok = ~np.isnan(x64)
    if not pr.T > 0 or not ok.any() or not np.isfinite(x64[ok].max()):
        return None, ref.greedy(x64)
    return pref.keep_set(x3, pr.k, pr.p, pr.min_p, pr.T), None


def _winner(scores: np.ndarray, cand: np.ndarray, rest: float) -> tuple[int, bool]:
    """Index into ``cand`` of the best score and whether it beats the others of ``cand`` and ``rest`` by MARGIN."""
    s = scores[cand]
    order = np.argsort(-s, kind="stable")
    best = s[order[0]]
    second = max(s[order[1]] if len(order) > 1 else -np.inf, rest)
    return int(cand[order[0]]), bool(best - second >= MARGIN)


def settle(pr: Probe, seeds=None, positions=None, tries: int = 1 << 16) -> Probe:
    """Fill ``pr.keep``, ``pr.inside`` and ``pr.want``, and search ``(seed, pos)`` so that the draw is certain.  With
    ``positions`` None the search runs over positions at ``seeds[0]``, otherwise over ``seeds`` at ``positions[0]``."""
    keep, greedy = reference_keep(pr)
    if keep is None:
        pr.keep, pr.inside, pr.want = None, greedy == pr.target, greedy
        pr.seed = seeds[0] if seeds else 0
        pr.pos = positions[0] if positions else 1
        return pr
    x64 = pr.staged().astype(np.float64)
    S = np.array(sorted(i for i in set(pr.planted) | {pr.target} if not np.isnan(x64[i])), dtype=np.int64)
    assert pr.target in S
    pr.keep, pr.inside = keep, bool(keep[pr.target])
    outside = keep.copy()
    outside[S] = False
    rest = float(x64[outside].max() / pr.T + G_MAX) if outside.any() else -np.inf
    kept = np.flatnonzero(keep[S])  # positions in S
    assert len(kept) > 0
    xs = x64[S] / pr.T
    every = np.arange(len(S))

    def ok(g) -> int | None:
        sc = xs + g
        w, clear = _winner(sc, every, -np.inf)
        if S[w] != pr.target or not clear:
            return None
        w, clear = _winner(sc, kept, rest)
        return int(S[w]) if clear else None

    if positions is None:
        seed = seeds[0]
        start = 1 + (seed % 997) * 1000
        for b in range(0, tries, 256):
            ps = np.arange(start + b, start + b + 256)
            G = gumbel_at(S, seed, ps)
            for j in range(len(ps)):
                w = ok(G[j])
                if w is not None:
                    pr.seed, pr.pos, pr.want = seed, int(ps[j]), w
                    return pr
    else:
        pos = positions[0]
        for seed in seeds:
            w = ok(gumbel_at(S, seed, pos))
            if w is not None:
                pr.seed, pr.pos, pr.want = seed, pos, w
                return pr
    raise AssertionError(f"no seed / position settles {pr!r}")


def draw(pr: Probe) -> int:
    """The reference token of a settled probe over the whole row (``penalties_ref.sample_row``)."""
    st = np.zeros(pr.V, np.int32) if pr.state is None else pr.state
    if pr.allowed is None:
        return pref.sample_row(pr.x, st, pr.T, pr.k, pr.p, pr.seed, pr.pos, pr.r, pr.pres, pr.freq, pr.min_p)
    x3 = pr.staged()
    x64 = x3.astype(np.float64)
    ok = ~np.isnan(x64)
    if not pr.T > 0 or not ok.any() or not np.isfinite(x64[ok].max()):
        return ref.greedy(x64)
    keep = pref.keep_set(x3, pr.k, pr.p, pr.min_p, pr.T)
    return int(np.argmax(np.where(keep, ref.perturbed(x64, pr.T, pr.seed, pr.pos), -np.inf)))


# ---------------------------------------------------------------------------------------------- catalogue --
class _Rows:
    """Rows of one (V, dtype): a low random background and planted entries at distinct indices spread over the
    slices."""

    def __init__(self, V: int, dtype: str, seed: int):
        self.V, self.dtype = V, dtype
        self.rng = np.random.default_rng(seed)
        self.C, self.slice = plan(V)

    def seed64(self) -> int:
        s = int(self.rng.integers(0, 1 << 63)) * 2 + int(self.rng.integers(0, 2))
        return s | (1 << 40)  # the key's high word set

    def background(self, lo=-60.0, hi=-45.0, fill=None) -> np.ndarray:
        if fill is not None:
            return np.full(self.V, fill, dtype=np.float32)
        return to_dtype(self.rng.uniform(lo, hi, self.V), self.dtype)

    def spots(self, n: int, first: int | None = None) -> list[int]:
        """``n`` distinct indices, ``first`` (when given) the first of them, the others on cycling ranks."""
        assert n <= self.V
        out = [] if first is None else [first]
        r = int(self.rng.integers(0, self.C))
        while len(out) < n:
            lo = r * self.slice
            hi = min(self.V, lo + self.slice)
            r = (r + 1) % self.C
            if lo >= hi:
                continue
            i = int(self.rng.integers(lo, hi))
            if i not in out:
                out.append(i)
        return out


def _eps(x3: np.ndarray) -> float:
    x = x3.astype(np.float64)
    ok = ~np.isnan(x)
    _, S = ref.mass_above(x)
    R = float(x[ok].max() - x[ok & np.isfinite(x)].min())
    return 2 * (2.0**-22 + R * 2.0**-24) + 2 * len(x) * 2.0**-40 / S


def _top_p_between(pr: Probe, lo_i: int, hi_i: int | None) -> float | None:
    """An fp32 ``top_p`` with the mass above entry ``lo_i`` below it and (``hi_i`` given) the mass above ``hi_i``
    above it, every planted entry's mass above at least 100 eps away from it; None when no such value exists."""
    x3 = pr.staged()
    M, _ = ref.mass_above(x3.astype(np.float64))
    lo = M[lo_i]
    hi = M[hi_i] if hi_i is not None else 1.0
    p = f32((lo + hi) / 2)
    e = 100 * _eps(x3)
    masses = [M[i] for i in set(pr.planted) | {pr.target} if np.isfinite(M[i])]
    if not 0 < p < 1 or any(abs(m - float(p)) < e for m in masses) or not lo < float(p) < hi:
        return None
    return float(p)


def _min_p_for(m: float, T: float, thr: float) -> float:
    """An fp32 min_p whose bound ``fl(m + fl(T log(min_p)))`` is exactly ``thr``."""
    base = f32(math.exp((thr - m) / T))
    bits = int(np.array(base).view(np.uint32))
    cand = (np.arange(-(1 << 14), 1 << 14, dtype=np.int64) + bits).astype(np.uint32).view(np.float32)
    cand = cand[(cand > 0) & (cand <= 1)]
    log_p = np.log(cand.astype(np.float64)).astype(np.float32)
    got = (f32(m) + (f32(T) * log_p).astype(np.float32)).astype(np.float32)
    hit = np.flatnonzero(got == f32(thr))
    assert len(hit), (m, T, thr)
    mp = float(cand[hit[len(hit) // 2]])
    assert pref.min_p_threshold(m, T, mp) == f32(thr)
    return mp


def _bucket_mate(P: float, make, dtype: str) -> tuple[float, int] | None:
    """A raw value on the grid of ``dtype`` and bf16 and a count whose penalised value shares P's 16-bit key bucket
    and lies below P (None when there is none)."""
    b = key(P) >> 16
    for c in (0, 1, 2, 3):
        ys = to_dtype(to_dtype(np.linspace(P - 0.75, P + 0.75, 4097), "bf16"), dtype)
        q = make(ys, c)
        qb = np.where(q == 0, np.float32(0), q).astype(np.float32).view(np.uint32).astype(np.int64)
        qk = np.where(qb & 0x80000000, ~qb & MASK32, qb | 0x80000000)  # key() of every entry
        hit = np.flatnonzero((q < P) & (qk >> 16 == b))
        if len(hit):
            return float(ys[hit[0]]), c
    return None


class Catalogue:
    """Every probe of one (V, dtype); ``probes`` in a fixed order."""

    def __init__(self, V: int, dtype: str):
        self.V, self.dtype = V, dtype
        self.rows = _Rows(V, dtype, seed=V * 7 + DTYPES.index(dtype))
        self.probes: list[Probe] = []
        if V == 1:
            for T in (0.0, 1.0):
                self._add(Probe("single", V, dtype, np.array([1.5], np.float32), 0, T=T, planted=[0]))
            return
        self.top_k_boundary()
        self.top_k_ties()
        self.top_k_counting()
        self.top_p_boundary()
        self.k_and_p_diverge()
        self.min_p()
        self.penalised()
        self.constrained()
        self.temperature()
        self.positions_and_seeds()

    # -- helpers
    def _add(self, pr: Probe, positions=None, seeds=None) -> None:
        if seeds is None:
            seeds = [self.rows.seed64()]
        self.probes.append(settle(pr, seeds=seeds, positions=positions))

    def _g(self, v) -> float:
        return on_grid(v, self.dtype)

    def _row(self, vals: list[float], first: int | None = None, **bg) -> tuple[np.ndarray, list[int]]:
        x = self.rows.background(**bg)
        idx = self.rows.spots(len(vals), first)
        x[idx] = vals
        return x, idx

    def _spot(self, j: int) -> int:
        s = boundary_spots(self.V)
        return s[j % len(s)]

    def _pair(self, kind, x, planted, inside_i, outside_i, **kw) -> None:
        for t in (inside_i, outside_i):
            self._add(Probe(kind, self.V, self.dtype, x.copy(), t, planted=planted, **kw))

    # -- the catalogue
    def top_k_boundary(self) -> None:
        bases = [1.53125, -0.71875, 2.875, -2.5625]
        levels = (0, 1, 2, 3) if self.dtype == "f32" else (None,)
        j = 0
        for a0 in bases:
            for level in levels:
                if level is None:
                    a = self._g(a0)
                    b = next_below(a, self.dtype)
                else:
                    a, b = split_at_level(a0, level, self.dtype)
                k = 1 + j % 4
                if k + 1 > self.V:
                    k = self.V - 1
                hs = [self._g(a + 0.25 * (i + 1)) for i in range(k - 1)]
                x, idx = self._row([a, b] + hs, first=self._spot(j))
                T = (0.7, 1.0, 1.3)[j % 3]
                self._pair("top-k boundary", x, idx, idx[0], idx[1], T=T, k=k)
                j += 1

    def top_k_ties(self) -> None:
        for j, a in enumerate((self._g(1.25), 0.0)):
            ties = boundary_spots(self.V)  # x_(k) tied on the slice edges of the first and last CTA
            others = [i for i in self.rows.spots(len(ties) + 2) if i not in ties][:2]
            order = [others[0]] + ties + [others[1]]
            x = self.rows.background()
            x[order] = [self._g(a + 0.5)] + [a] * len(ties) + [next_below(a, self.dtype)]
            k = 2
            if a == 0.0:
                x[ties[1::2]] = -0.0  # +0 and -0 are one value
            for t in ties + [order[-1]]:
                self._add(Probe("top-k ties", self.V, self.dtype, x.copy(), t, k=k, planted=order, T=1.0))

    def top_k_counting(self) -> None:
        V = self.V
        if V >= 8:
            # NaN entries at the boundary rank are not counted
            h1, h2, a = self._g(2.0), self._g(1.75), self._g(1.5)
            b = next_below(a, self.dtype)
            x, idx = self._row([h1, h2, np.nan, np.nan, a, b], first=self._spot(1))
            self._pair("top-k NaN", x, [idx[0], idx[1], idx[4], idx[5]], idx[4], idx[5], k=3)
            # -inf entries are counted: k beyond the finite entries keeps every finite one
            x, idx = self._row([self._g(1.0), self._g(0.75), self._g(0.5)], fill=-np.inf)
            self._add(Probe("top-k -inf", V, self.dtype, x, idx[2], k=5, planted=idx))
        # k at or above the non-NaN count keeps them all; one below drops the lowest
        n = min(3, V - 1)
        vals = [self._g(1.0 - 0.25 * i) for i in range(n)]
        x, idx = self._row(vals, first=self._spot(2), fill=np.nan)
        for k in (n, n + 1, max(1, n - 1)):
            if 0 < k < V:
                self._add(Probe("top-k count", V, self.dtype, x.copy(), idx[-1], k=k, planted=idx))
        if V <= 8:  # k = V - 1: the minimum alone is dropped; T = 1e30 leaves the draw to g over the whole row
            x = to_dtype(self.rows.rng.uniform(0.0, 0.5, V), self.dtype)
            lo = int(self.rows.rng.integers(0, V))
            x[lo] = self._g(-1.0)
            others = [i for i in range(V) if i != lo]
            pr = Probe("top-k V-1", V, self.dtype, x, lo, T=float(f32(1e30)), k=V - 1, planted=others)
            self._add(pr)

    def top_p_boundary(self) -> None:
        a = self._g(1.0)
        vals = [self._g(a - 0.5 * i) for i in range(5)]
        for j, t in enumerate((1, 2, 3)):
            x, idx = self._row(vals, first=self._spot(j))
            for inside in (True, False):
                pr = Probe("top-p boundary", self.V, self.dtype, x.copy(), idx[t], planted=idx, T=(0.8, 1.0, 1.2)[j])
                p = _top_p_between(pr, idx[t], idx[t + 1]) if inside else _top_p_between(pr, idx[t - 1], idx[t])
                assert p is not None
                pr.p = p
                self._add(pr)
        # the whole mass in one entry: only the maximum is kept, whatever g says
        x, idx = self._row([self._g(1.0), self._g(-199.0)], first=self._spot(3), fill=self._g(-200.0))
        self._add(Probe("top-p one entry", self.V, self.dtype, x, idx[1], p=0.5, T=float(f32(1e30)), planted=idx))

    def k_and_p_diverge(self) -> None:
        levels = {"f32": (1, 2, 3), "f16": (1, 2), "bf16": (1,)}[self.dtype]
        if self.V < 8:
            return
        for j, level in enumerate(levels):
            a, b = split_at_level(1.3 + 0.4 * j, level, self.dtype)
            hs = [self._g(a + 0.5), self._g(a + 1.0)]
            c = self._g(b - 1.0)
            x, idx = self._row(hs + [a, b, c], first=self._spot(j))
            ia, ib, ic = idx[2], idx[3], idx[4]
            for tighter in ("k", "p"):
                pr = Probe("k/p diverge", self.V, self.dtype, x.copy(), ia, planted=idx)
                if tighter == "k":  # top-k keeps H, H, A; top-p alone would keep B too
                    pr.k, pr.p = 3, _top_p_between(pr, ib, ic)
                else:  # top-p keeps H, H, A; top-k alone would keep B too
                    pr.k, pr.p = 4, _top_p_between(pr, ia, ib)
                assert pr.p is not None
                for t in (ia, ib):
                    q = Probe(pr.kind + f" {tighter} tighter L{level}", self.V, self.dtype, x.copy(), t, k=pr.k, p=pr.p, planted=idx)
                    self._add(q)

    def min_p(self) -> None:
        if self.V < 6:
            return
        for j, (T, k, p) in enumerate(((1.0, 0, 0.0), (0.7, 5, 0.0), (1.3, 0, 0.999), (1.0, 2, 0.0))):
            m, g_, e = self._g(2.0), self._g(1.75), self._g(1.5)
            f = next_below(e, self.dtype)
            x, idx = self._row([m, g_, e, f], first=self._spot(j))
            T = float(f32(T))
            for thr in (e, float(np.nextafter(f32(e), f32(np.inf)))):
                mp = _min_p_for(m, T, thr)
                self._pair("min-p", x, idx, idx[2], idx[3], T=T, k=k, p=p, min_p=mp)

    def penalised(self) -> None:
        """A penalised fp32 value P is x_(k) or v*; Q, raw or penalised, lies below it in its 16-bit key bucket."""
        if self.V < 8:
            return
        cases = [("repetition +", 2.0, dict(r=1.3)), ("repetition -", -1.1875, dict(r=1.3)), ("frequency +", 2.0, dict(freq=0.46)),
                 ("frequency -", -1.0, dict(freq=0.54)), ("presence +", 2.0, dict(pres=0.46)), ("presence -", -1.0, dict(pres=0.54))]
        for j, (name, raw, pen) in enumerate(cases):
            r, pres, freq = f32(pen.get("r", 1.0)), f32(pen.get("pres", 0.0)), f32(pen.get("freq", 0.0))
            c_p = 1

            rep = "r" in pen

            def state_of(c, rep=rep):  # c = 0: an unseen token; else a prompt token (repetition) or one drawn c times
                return 0 if c == 0 else (pref.PROMPT if rep else c)

            def make(y, c, r=r, pres=pres, freq=freq):
                y = np.atleast_1d(np.asarray(y, np.float32))
                q = pref.penalize(y, np.full(y.shape, state_of(c), np.int32), r, pres, freq)
                return q if len(q) > 1 else float(q[0])

            raw = self._g(raw)
            for _ in range(64):  # the first raw value from here down whose penalised value has a mate
                P = make(raw, c_p)
                mate = _bucket_mate(P, make, self.dtype)
                if mate is not None:
                    break
                raw = next_below(raw, "bf16")
            assert on_grid(P, "bf16") != P and mate is not None, name  # off the bf16 grid
            q_raw, q_c = mate
            H = self._g(P + 0.5)
            x, idx = self._row([raw, q_raw, H], first=self._spot(j))
            st = np.zeros(self.V, np.int32)
            st[idx[0]], st[idx[1]] = state_of(c_p), state_of(q_c)
            kw = dict(r=float(r), pres=float(pres), freq=float(freq), state=st)
            self._pair(f"penalised {name} top-k", x, idx, idx[0], idx[1], k=2, **kw)
            pr = Probe("x", self.V, self.dtype, x, idx[0], planted=idx, **kw)
            p = _top_p_between(pr, idx[0], idx[1])
            assert p is not None, name
            self._pair(f"penalised {name} top-p", x, idx, idx[0], idx[1], p=p, **kw)

    def constrained(self) -> None:
        if self.V < 12:
            return
        V = self.V
        # k counts allowed entries only; a disallowed entry sits at the boundary rank
        vals = [self._g(3.0), self._g(2.0), self._g(1.75), self._g(1.5), self._g(1.25), next_below(self._g(1.25), self.dtype)]
        x, idx = self._row(vals, first=self._spot(0))
        allowed = np.ones(V, bool)
        allowed[[idx[0], idx[3]]] = False  # 3.0 above everything, 1.5 at rank 4 of the raw row
        planted = [i for i in idx if allowed[i]]
        self._pair("mask k counts allowed", x, planted, idx[4], idx[5], k=3, allowed=allowed)
        # fewer allowed entries than k: every allowed entry is kept
        allowed = np.zeros(V, bool)
        allowed[idx[1:4]] = True
        self._add(Probe("mask fewer than k", V, self.dtype, x.copy(), idx[3], k=5, allowed=allowed, planted=idx[1:4]))
        # MASK with PEN: a penalised x_(k), a disallowed entry above it
        raw, r = self._g(2.0), f32(1.3)
        P = float(f32(raw) / r)
        x, idx = self._row([raw, self._g(1.53125), self._g(3.0), self._g(2.5)], first=self._spot(3))
        st = np.zeros(V, np.int32)
        st[idx[0]] = pref.PROMPT
        allowed = np.ones(V, bool)
        allowed[idx[2]] = False
        assert P > 1.53125
        self._pair("mask + penalised", x, [idx[0], idx[1], idx[3]], idx[0], idx[1], k=2, r=float(r), state=st, allowed=allowed)

    def temperature(self) -> None:
        temps = [1e-30, 1e-38, FLT_MIN, 1e-41, 1e-46]
        rowkinds = {"positive": (2.0, 30.0), "negative": (-30.0, -2.0), "mixed": (-15.0, 15.0)}
        for j, (name, (lo, hi)) in enumerate(rowkinds.items()):
            for i, T in enumerate(temps):
                M = self._g(hi + 1.0)
                x = self.rows.background(lo, hi)
                s = boundary_spots(self.V)  # not entry 0: the lowest index is what an all-inf score row returns
                idx = self.rows.spots(2, s[1 + (i + j) % (len(s) - 1)] if len(s) > 1 else None)
                x[idx] = [M, next_below(M, self.dtype)]
                self._add(Probe(f"temperature {T:g} {name}", self.V, self.dtype, x, idx[0], T=float(f32(T)), planted=idx))
            # T rounds to 0: greedy, the first of tied maxima
            x = self.rows.background(lo, hi)
            idx = sorted(self.rows.spots(2, self._spot(j)))
            x[idx] = self._g(hi + 1.0)
            self._add(Probe(f"temperature 1e-46 tie {name}", self.V, self.dtype, x, idx[0], T=float(f32(1e-46)), planted=idx))
            # T = 1e30: the argmax of g over the keep set
            if self.V >= 8:
                a = self._g((lo + hi) / 2)
                vals = [self._g(a + 0.5), self._g(a + 0.25), a, next_below(a, self.dtype)]
                x, idx = self._row(vals, first=self._spot(j + 1), lo=lo - 60, hi=lo - 45)
                self._pair(f"temperature 1e30 {name}", x, idx, idx[2], idx[3], T=float(f32(1e30)), k=3)

    def positions_and_seeds(self) -> None:
        if self.V < 4:
            return
        a = self._g(0.5)
        b = next_below(a, self.dtype)
        for j, pos in enumerate((0, 1, (1 << 31) - 1)):
            x, idx = self._row([a, b, self._g(0.75)], first=self._spot(j))
            seeds = [self.rows.seed64() | (0xFFFF << 48) for _ in range(4096)]
            for t in (idx[0], idx[1]):
                self._add(Probe(f"pos {pos}", self.V, self.dtype, x.copy(), t, k=2, planted=idx), positions=[pos], seeds=seeds)


# ---------------------------------------------------------------------------------------------- the forms --
FORMS = ("sample", "penalized off", "penalized on", "constrained", "constrained + state")


def forms_of(pr: Probe) -> tuple[str, ...]:
    """The kernel forms a probe runs in: a penalised probe needs the state, a masked one the constrained kernel."""
    if pr.allowed is not None:
        return ("constrained + state",) if pr.penalized or pr.state is not None else ("constrained", "constrained + state")
    if pr.penalized or pr.state is not None:
        return ("penalized on", "constrained + state")
    return FORMS
