"""Planted-winner probes of speculative sampling's accept / residual rule (``tl_speculative_sample``, DESIGN.md section
8d) and of XTC's exclusion (the XTC forms of ``sample_kernel``, section 24).

TEST INFRASTRUCTURE.  Both kernels decide on integers: 2^-40 fixed-point masses, 128-bit products and order keys.  A
probe is a row built so that the decision is certain, and a (seed, position) searched so that the token is too:

* Exact (plateau) rows.  Every kept entry is either at the row maximum m or at least max(30, 30 T) below it.  The
  kernel weighs a maximum exactly 2^40 (``expf(0)`` is 1) and the others exactly 0 (``expf(-30) 2^40`` is about 0.1),
  in the temperature masses and in section 8's temperature-free top-p masses alike.  So p_i and q_i are rationals,
  ``Fraction(M_i, n)`` with M the maxima of the keep set and n their count, and ``u q_d <= p_d`` is decided exactly
  (u, an odd multiple of 2^-24, never ties).  Point-mass rows are plateau rows with n = 1.
* Margin rows.  Any other row, where every decisive quantity (u q_d against p_d, each kept p_i against XTC's theta)
  stays at least ``REL`` = 2^-16 relative from its boundary, far above the 2^-20 bound of the kernels' masses, and
  every planted entry with p_i > q_i differs from q_i by more than that.

A residual or a Gumbel draw must beat every other candidate by ``keep_set_ref.MARGIN``, and the background (entries
not planted, 45-60 below the planted values) can never win.  The tokens are computed on the planted entries; the host
test checks every probe against the whole-row rules (``spec_sample_ref.rule_row``, ``dry_xtc_ref.xtc_sample_row``).

``spec_rule`` and ``xtc_rule`` take a ``variant``: a named defect (``SPEC_VARIANTS``, ``XTC_VARIANTS``) restated as a
change of the rule, so that the host test can show that every defect gets at least one probe wrong.
"""

from __future__ import annotations

import importlib.util
import math
import sys
from dataclasses import dataclass, field
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
R = _load("tiny_llm_b200_spec_sample_ref", "spec_sample_ref.py")
X = _load("tiny_llm_b200_dry_xtc_ref", "dry_xtc_ref.py")
pref = K.pref

SPEC_VOCABS = [1, 7, 4096, 4097, 8193, 12289, 16385, 20481, 24577, 28673, 151936, 204800]
XTC_VOCABS = SPEC_VOCABS + [409600]
DTYPES = K.DTYPES
MARGIN = K.MARGIN
REL = 2.0**-16
MASK32 = K.MASK32
U_ONE = 1 << 24  # u = u_odd / 2^24


# ------------------------------------------------------------------------------------------------- Philox --
def _key(seed: int) -> tuple[int, int]:
    return seed & MASK32, (seed >> 32) & MASK32


def u_odd_at(seed: int, positions, stream: int, word: int = 0) -> np.ndarray:
    """``2 (w >> 9) + 1`` of word ``word`` of Philox4x32-10 at counter ``(0, pos, stream, 0)``, for every position."""
    ps = np.atleast_1d(np.asarray(positions, dtype=np.int64))
    ctr = np.zeros((len(ps), 4), dtype=np.uint64)
    ctr[:, 1] = ps & MASK32
    ctr[:, 2] = stream
    w = ref.philox4x32_10(ctr, _key(seed))[:, word].astype(np.uint64)
    return (2 * (w >> np.uint64(9)) + 1).astype(np.int64)


def noise_at(indices, seed: int, pos: int, stream: int) -> np.ndarray:
    """Gumbel noise of word ``i % 4`` of Philox4x32-10 at counter ``(i >> 2, pos, stream, 0)`` at ``indices``."""
    idx = np.asarray(indices, dtype=np.int64).reshape(-1)
    ctr = np.zeros((len(idx), 4), dtype=np.uint64)
    ctr[:, 0] = idx >> 2
    ctr[:, 1] = pos & MASK32
    ctr[:, 2] = stream
    words = ref.philox4x32_10(ctr, _key(seed))
    w = words[np.arange(len(idx)), idx & 3]
    return -np.log(-np.log(R.to_uniform(w)))


def slice_spots(V: int) -> list[int]:
    """``boundary_spots`` and the first and last entry of every rank's slice."""
    C, s = K.plan(V)
    out = set(K.boundary_spots(V))
    for r in range(C):
        if r * s < V:
            out |= {r * s, min(V, (r + 1) * s) - 1}
    return sorted(out)


# ================================================================================ speculative sampling ==
SPEC_VARIANTS = {
    "acceptance uniform from stream 0": "the acceptance uniform drawn from the wrong stream",
    "acceptance uniform from word 1": "the acceptance uniform from the wrong Philox word",
    "acceptance uniform at position - 1": "the acceptance uniform at the wrong position",
    "p_d, q_d read from rank 0": "p_d / q_d read from the wrong CTA",
    "p_d, q_d read one entry on": "p_d / q_d read at the wrong offset",
    "no q_d > 0 guard": "a proposal outside the draft's keep set accepted",
    "p normalised over the whole row": "masses summed over the whole row instead of the keep set",
    "draft keeps by the target's tau": "the draft's keep set cut at the target's threshold",
    "top-p mass with temperature": "top-p computed on the tempered masses (section 8 keeps it temperature-free)",
    "masses without temperature": "p and q computed without the temperature",
    "residual set p_i >= q_i scored by log p_i": "a residual over p_i >= q_i with log p_i scores",
    "residual scored by log p_i": "residual scores log p_i in place of log(p_i - q_i)",
    "residual noise without the slice start": "residual noise counters from the slice-local index",
    "residual noise from stream 0": "residual noise from the draw's stream",
    "residual noise from stream 1": "residual noise from the acceptance stream",
    "last-maximum argmax": "the point mass at the last of tied maxima",
    "point mass weighs 2^-40": "a point-mass row mixed with a sampled one at the wrong scale",
    "(x - m) / T as x / T - m / T": "x / T overflowing for temperatures near the bottom of fp32",
    "64-bit products": "the acceptance products truncated to 64 bits",
}


@dataclass
class Dist:
    """One row's distribution: exact (``M`` the entries of mass 2^40, ``n`` their count) or float64 ``p``."""

    exact: bool
    p: np.ndarray
    keep: np.ndarray
    M: np.ndarray | None = None
    n: int = 1
    scale: int = 1  # the kernel's mass of one M entry, over 2^40 (a point mass weighs 1 against S = 1)

    def at(self, i: int):
        if not 0 <= i < len(self.p):
            return 0
        return Fraction(int(self.M[i]), self.n * self.scale) if self.exact else float(self.p[i])


def _last_greedy(x) -> int:
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    if not ok.any():
        return 0
    return int(np.flatnonzero(ok & (x == x[ok].max()))[-1])


def row_dist(x, T: float, k: int, p: float, exact: bool, variant: str | None = None, keep: np.ndarray | None = None) -> Dist:
    x = np.asarray(x, dtype=np.float64)
    V = len(x)
    ok = ~np.isnan(x)
    if R.is_point(x, T):
        a = _last_greedy(x) if variant == "last-maximum argmax" else ref.greedy(x)
        M = np.zeros(V, dtype=np.int64)
        M[a] = 1
        scale = 1 << 40 if variant == "point mass weighs 2^-40" else 1
        return Dist(True, M / scale, M.astype(bool), M, 1, scale)
    if keep is None:
        keep = ref.keep_set(x / T if variant == "top-p mass with temperature" and p else x, k, p)
    w = ok.copy() if variant == "p normalised over the whole row" else keep & ok
    m = x[ok].max()
    if exact:
        top = w & (x == m)
        below = w & ~top
        assert not below.any() or x[below].max() <= m - max(30.0, 30.0 * T), "not a plateau row"
        if variant == "(x - m) / T as x / T - m / T":
            with np.errstate(all="ignore"):
                z = np.float32(np.float32(m) / np.float32(T)) - (np.float32(x) / np.float32(T)).astype(np.float32)
            top &= z == 0  # inf - inf is NaN: the maxima lose their mass
        M = top.astype(np.int64)
        n = int(M.sum())
        if n == 0:
            return Dist(True, np.zeros(V), keep, M, 1)
        return Dist(True, M / n, keep, M, n)
    Tm = 1.0 if variant == "masses without temperature" else T
    e = np.where(w, np.exp((np.where(w, x, m) - m) / Tm), 0.0)
    return Dist(False, e / e.sum() if e.sum() > 0 else e, keep)


@dataclass
class SpecProbe:
    kind: str
    V: int
    dtype: str
    x: np.ndarray  # target row, fp32 values on the dtype's grid
    y: np.ndarray  # draft row
    d: int
    T: float = 1.0
    k: int = 0
    p: float = 0.0
    exact: bool = True
    planted: list = field(default_factory=list)
    seed: int = 0
    pos: int = 0
    want: int = -1
    accepted: bool = False

    def __repr__(self) -> str:
        return (f"SpecProbe({self.kind}, V={self.V}, {self.dtype}, d={self.d}, want={self.want} "
                f"{'accept' if self.accepted else 'reject'}, T={self.T}, k={self.k}, p={self.p}, seed={self.seed:#x}, pos={self.pos})")


@dataclass
class SpecDecision:
    token: int
    accepted: bool
    gap: float  # the residual's top-two gap (inf when accepted or a single candidate)
    rel: float  # |u q_d - p_d| / max(p_d, q_d) (inf on exact rows)


def spec_rule(pr: SpecProbe, variant: str | None = None, pos: int | None = None) -> SpecDecision:
    """The kernel's decision for one probe row, computed on the planted entries (and, for the residual of a margin row,
    every entry with p_i of at least 1e-12); ``variant`` restates one defect of ``SPEC_VARIANTS``."""
    pos = pr.pos if pos is None else pos
    V, seed, d = pr.V, pr.seed, pr.d
    P = row_dist(pr.x, pr.T, pr.k, pr.p, pr.exact, variant)
    keep_y = None
    if variant == "draft keeps by the target's tau" and not R.is_point(pr.x, pr.T) and not R.is_point(pr.y, pr.T):
        tau = np.asarray(pr.x, np.float64)[P.keep].min()
        keep_y = ~np.isnan(pr.y) & (np.asarray(pr.y, np.float64) >= tau)
    Q = row_dist(pr.y, pr.T, pr.k, pr.p, pr.exact, variant, keep=keep_y)
    rd = d
    if 0 <= d < V and variant == "p_d, q_d read from rank 0":
        rd = d % K.plan(V)[1]
    elif 0 <= d < V and variant == "p_d, q_d read one entry on":
        rd = d + 1 if d + 1 < V else d - 1
    pd, qd = P.at(rd), Q.at(rd)
    stream, word, upos = 1, 0, pos
    if variant == "acceptance uniform from stream 0":
        stream = 0
    elif variant == "acceptance uniform from word 1":
        word = 1
    elif variant == "acceptance uniform at position - 1":
        upos = pos - 1
    u_odd = int(u_odd_at(seed, [upos], stream, word)[0])
    rel = math.inf
    if variant == "64-bit products" and P.exact and Q.exact:
        one_p = 1 if R.is_point(pr.x, pr.T) else 1 << 40  # the kernel's mass of an M entry: a point mass weighs 1 of S = 1
        one_q = 1 if R.is_point(pr.y, pr.T) else 1 << 40
        e_p = int(P.M[rd]) * one_p if 0 <= rd < V else 0
        e_q = int(Q.M[rd]) * one_q if 0 <= rd < V else 0
        s_p, s_q = P.n * one_p, Q.n * one_q
        w64 = (1 << 64) - 1
        accept = e_q > 0 and (u_odd * e_q * s_p) & w64 <= ((e_p << 24) * s_q) & w64
    else:
        u = Fraction(u_odd, U_ONE) if P.exact else u_odd / U_ONE
        accept = (qd > 0 or variant == "no q_d > 0 guard") and u * qd <= pd
        if not P.exact and max(pd, qd) > 0:
            rel = abs(u * qd - pd) / max(pd, qd)
    if accept:
        return SpecDecision(d, True, math.inf, rel)
    # residual: argmax over {p_i > q_i} of log(p_i - q_i) + g_i
    if P.exact and Q.exact:
        a = P.M * (Q.n * Q.scale)
        b = Q.M * (P.n * P.scale)
        cand = (a >= b) & (P.M > 0) if variant == "residual set p_i >= q_i scored by log p_i" else a > b
        idx = np.flatnonzero(cand)
        den = P.n * P.scale * Q.n * Q.scale
        if variant in ("residual set p_i >= q_i scored by log p_i", "residual scored by log p_i"):
            base = np.array([math.log(int(P.M[i]) / (P.n * P.scale)) for i in idx])
        else:
            base = np.array([math.log(int(a[i] - b[i]) / den) for i in idx])
    else:
        cand = (P.p > Q.p) & (P.p >= 1e-12)
        if variant == "residual set p_i >= q_i scored by log p_i":
            cand = (P.p >= Q.p) & (P.p >= 1e-12)
        idx = np.flatnonzero(cand)
        if variant in ("residual set p_i >= q_i scored by log p_i", "residual scored by log p_i"):
            base = np.log(P.p[idx])
        else:
            base = np.log(P.p[idx] - Q.p[idx])
    if len(idx) == 0:
        return SpecDecision(_last_greedy(pr.x) if variant == "last-maximum argmax" else ref.greedy(pr.x), False, math.inf, rel)
    nstream = {"residual noise from stream 0": 0, "residual noise from stream 1": 1}.get(variant, 2)
    nidx = idx - (idx // K.plan(V)[1]) * K.plan(V)[1] if variant == "residual noise without the slice start" else idx
    g = noise_at(nidx, seed, pos, nstream)
    score = base + g
    order = np.argsort(-score, kind="stable")
    gap = float(score[order[0]] - score[order[1]]) if len(idx) > 1 else math.inf
    return SpecDecision(int(idx[order[0]]), False, gap, rel)


def _margin_row_ok(pr: SpecProbe) -> bool:
    """Every planted entry of a margin row has p_i and q_i equal or REL apart."""
    if pr.exact:
        return True
    P = row_dist(pr.x, pr.T, pr.k, pr.p, False)
    Q = row_dist(pr.y, pr.T, pr.k, pr.p, False)
    for i in pr.planted:
        a, b = P.p[i], Q.p[i]
        if max(a, b) > 1e-12 and 0 < abs(a - b) < REL * max(a, b):  # equal rows give equal masses in the kernel too
            return False
    return True


def settle_spec(pr: SpecProbe, seed: int, accept: bool | None, window=None, extra=None, tries: int = 1 << 21) -> SpecProbe:
    """Search positions at ``seed`` for a certain decision: accepted (or rejected) as asked, the acceptance uniform in
    ``window`` (a pair of bounds on u) when given, a residual winner ``MARGIN`` clear, margin rows ``REL`` clear, and
    ``extra(decision, position)`` true."""
    assert _margin_row_ok(pr), pr
    pr.seed = seed
    start = 1 + (seed % 991) * 4099
    for b in range(0, tries, 1 << 15):
        ps = np.arange(start + b, start + b + (1 << 15))
        u = u_odd_at(seed, ps, 1) / U_ONE
        if window is not None:
            ps = ps[(u > window[0]) & (u < window[1])]
        for p_ in ps[:256]:
            dec = spec_rule(pr, pos=int(p_))
            if accept is not None and dec.accepted != accept:
                continue
            if not dec.accepted and dec.gap < MARGIN:
                continue
            if dec.rel < REL or (extra is not None and not extra(dec, int(p_))):
                continue
            pr.pos, pr.want, pr.accepted = int(p_), dec.token, dec.accepted
            return pr
    raise AssertionError(f"no position settles {pr!r}")


class SpecCatalogue:
    """Every speculative-sampling probe of one (V, dtype); ``probes`` in a fixed order, then the bonus row."""

    def __init__(self, V: int, dtype: str):
        self.V, self.dtype = V, dtype
        self.rows = K._Rows(V, dtype, seed=V * 11 + DTYPES.index(dtype) + 1)
        self.C, self.slice = K.plan(V)
        self.probes: list[SpecProbe] = []
        self.outside()
        if V >= 7:
            self.accept_reject()
            self.margin()
            self.cuts()
            self.swapped_pair()
            self.residual_by_difference()
            self.point_mass()
            self.tiny_temperature()
        if V >= 2:
            self.flat()
        self.bonus = self._bonus()

    def _g(self, v) -> float:
        return K.on_grid(v, self.dtype)

    def _bg(self) -> np.ndarray:
        return self.rows.background(-60.0, -45.0)

    def _others(self, n: int, avoid) -> list[int]:
        out = []
        while len(out) < n:
            for i in self.rows.spots(n + len(avoid) + 1):
                if i not in avoid and i not in out and len(out) < n:
                    out.append(i)
        return out

    def _add(self, pr: SpecProbe, accept=None, window=None, extra=None) -> None:
        self.probes.append(settle_spec(pr, self.rows.seed64(), accept, window, extra))

    # -- exact rows
    def accept_reject(self) -> None:
        """d at every slice spot, p_d / q_d = n_y / n_x < 1; u just below it (accept) and just above it (reject), where
        the two residual candidates tie and the noise decides."""
        ratios = [(5, 2), (4, 3), (6, 5)]
        for j, d in enumerate(slice_spots(self.V)):
            nx, ny = ratios[j % 3]
            T = (0.7, 1.0, 1.3)[j % 3]
            hs = self._others(nx - 1 + ny - 1, [d])
            x, y = self._bg(), self._bg()
            x[[d] + hs[: nx - 1]] = 1.0
            y[[d] + hs[nx - 1:]] = 1.0
            r = ny / nx
            k = (0, nx + 1, 0)[j % 3]  # top-k and top-p that keep every maximum
            p = (0.0, 0.0, 0.9)[j % 3]
            for acc, win in ((True, (r - 0.125, r)), (False, (r, r + 0.125))):
                pr = SpecProbe("accept/reject", self.V, self.dtype, x.copy(), y.copy(), d, T=T, k=k, p=p, planted=[d] + hs)
                self._add(pr, acc, win)

    def outside(self) -> None:
        """d = -1 and d = V: rejected whatever u; the residual (or, where p == q, x's argmax) is the token."""
        V = self.V
        x = self._bg()
        y = x.copy()
        if V >= 3:
            a, b = self._others(2, [])
            x[a], y[b] = 1.0, 1.0
            x[b] = y[a] = self._g(x[a] - 50.0)
        else:
            a = 0
        for d in (-1, V):
            self._add(SpecProbe("d outside the row", V, self.dtype, x.copy(), y.copy(), d, planted=[a]), False, (0.0, 0.25))

    def swapped_pair(self) -> None:
        """y is x with a kept maximum a and a background entry z exchanged: S_p == S_q, the residual set is {a}, and the
        other maxima (p_i == q_i) are planted to win on noise alone."""
        for j in range(2):
            a = self.rows.spots(1, slice_spots(self.V)[-1 - j])[0] if self.C > 1 else self.rows.spots(1)[0]
            b, c, z = self._others(3, [a])
            x = self._bg()
            x[[a, b, c]] = 1.0
            y = x.copy()
            y[a], y[z] = x[z], x[a]
            pr = SpecProbe("swapped pair", self.V, self.dtype, x, y, z, T=(1.0, 0.7)[j], planted=[a, b, c, z])
            self._add(pr, False, None, lambda dec, pos, pr=pr, a=a, b=b, c=c: dec.token == a and  # the noise alone picks b or c
                      np.argmax(noise_at([a, b, c], pr.seed, pos, 2)) > 0)
            pr = SpecProbe("swapped pair", self.V, self.dtype, x.copy(), y.copy(), b, T=(1.0, 0.7)[j], planted=[a, b, c, z])
            self._add(pr, True)

    def residual_by_difference(self) -> None:
        """x's maxima {a, b} (p = 1/2), y's {a, c, e} (q_a = 1/3), d = c rejected: the residual weighs b (1/2) three times
        a (1/6), and the noise alone would pick a."""
        for j in range(2):
            a, b = self.rows.spots(2, slice_spots(self.V)[-1 - j])
            c, e = self._others(2, [a, b])
            x, y = self._bg(), self._bg()
            x[[a, b]] = 1.0
            y[[a, c, e]] = 1.0
            pr = SpecProbe("residual by the difference", self.V, self.dtype, x, y, c, T=(1.0, 1.3)[j], planted=[a, b, c, e])
            self._add(pr, False, None, lambda dec, pos, pr=pr, a=a, b=b: dec.token == b and noise_at([a, b], pr.seed, pos, 2)[0] >
                      noise_at([a, b], pr.seed, pos, 2)[1])

    def point_mass(self) -> None:
        V = self.V
        s = K.boundary_spots(V)
        lo, hi = s[0], s[-1]
        # T = 0: tied maxima on the first and the last rank; the first one is the point mass
        x = self._bg()
        x[[lo, hi]] = 1.0
        for d in (lo, hi):
            y = self._bg()
            y[d] = 1.0
            self._add(SpecProbe("point mass T=0 ties", V, self.dtype, x.copy(), y, d, T=0.0, planted=[lo, hi]), None)
        # +inf in y only: q is the point mass at e, p a plateau over {e, f}: accept iff u <= 1/2
        e, f = self._others(2, [])
        x = self._bg()
        x[[e, f]] = 1.0
        y = self._bg()
        y[e] = np.inf
        y[f] = 1.0
        for acc, win in ((True, (0.375, 0.5)), (False, (0.5, 0.625))):
            self._add(SpecProbe("point mass inf in y", V, self.dtype, x.copy(), y.copy(), e, planted=[e, f]), acc, win)
        # +inf in x only: p is the point mass at e; d = e is accepted, d = f rejected for e
        x = self._bg()
        x[e], x[f] = np.inf, 1.0
        y = self._bg()
        y[[e, f]] = 1.0
        for d in (e, f):
            self._add(SpecProbe("point mass inf in x", V, self.dtype, x.copy(), y.copy(), d, planted=[e, f]), d == e)
        # NaN at d in x only (p_d = 0, rejected), and in y only (q_d = 0, rejected even for a tiny u)
        g = self._others(1, [e, f])[0]
        x = self._bg()
        x[[e, f, g]] = 1.0
        x[e] = np.nan
        y = self._bg()
        y[[e, g]] = 1.0
        self._add(SpecProbe("NaN in x", V, self.dtype, x, y, e, planted=[e, f, g]), False)
        x = self._bg()
        x[[e, f]] = 1.0
        y = self._bg()
        y[f] = 1.0
        y[e] = np.nan
        self._add(SpecProbe("NaN in y", V, self.dtype, x, y, e, planted=[e, f]), False, (0.0, 0.25))

    def tiny_temperature(self) -> None:
        """Maxima at 30 with temperatures near the bottom of fp32: x / T overflows, (x - m) / T does not.  The proposal
        is the later maximum, accepted with p_d = q_d = 1/2."""
        for j, T in enumerate((1e-30, 1e-38, K.FLT_MIN, 1e-41, 1e-45)):
            h, d = sorted(self._others(2, []))
            x = self.rows.background(-30.0, -15.0)
            x[[h, d]] = 30.0
            y = self.rows.background(-30.0, -15.0)
            y[[h, d]] = 30.0
            self._add(SpecProbe(f"temperature {T:g}", self.V, self.dtype, x, y, d, T=float(np.float32(T)), planted=[h, d]), True)

    def flat(self) -> None:
        """Every entry at one value (S_p = V 2^40) against the same row with one entry z lowered (S_q = (V - 1) 2^40):
        accept iff u <= (V - 1) / V, the products near 2^122 at V = 204,800; a rejection's residual is z alone."""
        V = self.V
        x = np.full(V, self._g(0.5), dtype=np.float32)
        z, d = (self._others(2, []) if V > 2 else [0, 1])
        y = x.copy()
        y[z] = self._g(-60.0)
        r = (V - 1) / V
        for acc, win in ((True, (r - 0.125, r)), (False, (r, 1.0))):
            self._add(SpecProbe("flat", V, self.dtype, x.copy(), y.copy(), d, planted=[z, d]), acc, win)

    # -- margin rows
    def margin(self) -> None:
        """Four planted entries with different values in x and y, T = 0.7 and 1.3: u just inside and just outside
        p_d / q_d, so a mass computed without the temperature flips the decision."""
        for j, T in enumerate((0.7, 1.3)):
            idx = self.rows.spots(4, slice_spots(self.V)[j % len(slice_spots(self.V))])
            x, y = self._bg(), self._bg()
            x[idx] = [self._g(v) for v in (0.5, 1.0, 0.0, -0.5)]
            y[idx] = [self._g(v) for v in (1.0, 0.25, 0.5, -0.25)]
            d = idx[0]
            P, Q = row_dist(x, T, 0, 0.0, False), row_dist(y, T, 0, 0.0, False)
            r = P.p[d] / Q.p[d]
            for acc, win in ((True, (r * 0.94, r * (1 - 2 * REL))), (False, (r * (1 + 2 * REL), r * 1.06))):
                self._add(SpecProbe("margin accept/reject", self.V, self.dtype, x.copy(), y.copy(), d, T=T, exact=False, planted=idx), acc, win)

    def cuts(self) -> None:
        g = self._g
        # d cut from x by top-k (and by top-p): rejected even for a tiny u
        idx = self.rows.spots(4, slice_spots(self.V)[-1])
        a, b, d, e = idx
        x, y = self._bg(), self._bg()
        x[[a, b, d, e]] = [g(2.0), g(1.5), g(1.0), g(-1.0)]
        y[[a, b, d, e]] = [g(0.0), g(-0.5), g(1.0), g(0.5)]
        self._add(SpecProbe("d cut from x by top-k", self.V, self.dtype, x.copy(), y.copy(), d, k=2, exact=False, planted=idx), False, (0.0, 0.125))
        top_p = K._top_p_between(K.Probe("x", self.V, self.dtype, x.copy(), a, planted=[a, b, d, e]), b, d)
        if top_p is not None and ref.keep_set(y.astype(np.float64), 0, top_p)[d]:
            self._add(SpecProbe("d cut from x by top-p", self.V, self.dtype, x.copy(), y.copy(), d, p=top_p, exact=False, planted=idx), False,
                      (0.0, 0.125))
        # d cut from y by top-k, kept in x: q_d = 0
        x[[a, b, d, e]] = [g(1.0), g(-1.0), g(1.5), g(0.0)]
        y[[a, b, d, e]] = [g(2.0), g(1.5), g(1.0), g(-1.0)]
        self._add(SpecProbe("d cut from y by top-k", self.V, self.dtype, x.copy(), y.copy(), d, k=2, exact=False, planted=idx), False, (0.0, 1 / 16))
        # keep sets that differ: top-2 keeps {a, d} of x (threshold 0) and {d, b} of y; y cut at x's threshold would
        # keep e as well and lower q_d.  u lies between the two ratios p_d / q_d: rejected, where that cut accepts.
        x[[a, b, d, e]] = [g(1.0), g(-1.0), g(0.0), g(-1.0)]
        y[[a, b, d, e]] = [g(-2.0), g(0.875), g(1.0), g(0.5)]
        p_d = row_dist(x, 1.0, 2, 0.0, False).p[d]
        r = p_d / row_dist(y, 1.0, 2, 0.0, False).p[d]
        r_cut = p_d / row_dist(y, 1.0, 2, 0.0, False, keep=y >= x[d]).p[d]
        assert r * 1.2 < r_cut < 1
        self._add(SpecProbe("keep sets differ", self.V, self.dtype, x.copy(), y.copy(), d, k=2, exact=False, planted=idx), False,
                  (r * (1 + 4 * REL), r_cut * (1 - 4 * REL)))
        # top-p at T != 1: temperature-free top-p keeps d (T = 0.5) or cuts it (T = 2); y == x
        vals = [g(1.0), g(0.5), g(0.0), g(-0.5)]
        x[[a, b, d, e]] = vals
        Mf, _ = ref.mass_above(x.astype(np.float64))
        for T, keep_d in ((0.5, True), (2.0, False)):
            Mt, _ = ref.mass_above(x.astype(np.float64) / T)
            lo, hi = sorted((Mf[d], Mt[d]))
            top_p = float(np.float32((lo + hi) / 2))
            assert lo + 0.01 < top_p < hi - 0.01 and (Mf[d] < top_p) == keep_d
            self._add(SpecProbe("top-p at T != 1", self.V, self.dtype, x.copy(), x.copy(), d, T=T, p=top_p, exact=False, planted=idx), keep_d)

    def _bonus(self) -> SpecProbe:
        x = self._bg()
        idx = self.rows.spots(min(3, self.V))
        x[idx] = [self._g(1.0 - 0.25 * i) for i in range(len(idx))]
        seed = self.rows.seed64()
        pos = 1 + seed % 100_000
        want = ref.sample_row(x.astype(np.float64), 1.0, 0, 0.0, seed, pos)
        return SpecProbe("bonus", self.V, self.dtype, x, x, -1, planted=idx, seed=seed, pos=pos, want=want, accepted=True)


# ================================================================================================== XTC ==
XTC_VARIANTS = {
    "gate u <= q": "the gate fired at u == q (the rule is u < q)",
    "gate from stream 0": "the gate's uniform drawn from the wrong stream",
    "gate from word 1": "the gate's uniform from the wrong Philox word",
    "gate at position - 1": "the gate's uniform at the wrong position",
    "A removed whole": "every entry of A removed, the least likely too",
    "A needs three": "nothing removed when |A| = 2",
    "ties cut to one": "all but one of the ties at A's minimum removed",
    "A per CTA": "the count and the minimum taken from each CTA alone",
    "A's minimum from rank 0": "the minimum of A taken from rank 0's slice",
    "A over the whole row": "the shares normalised over the whole row instead of the keep set",
    "A without temperature": "the shares computed without the temperature",
    "A on unpenalised values": "the shares computed from the unpenalised row",
    "A counts disallowed entries": "disallowed entries counted in the shares and in A",
    "XTC at temperature 0": "XTC applied (at T = 1) before the greedy draw",
}


@dataclass(repr=False)
class XtcProbe(K.Probe):
    theta: float = 0.1
    q: float = 1.0
    pre: int = -1  # the token without XTC

    def __repr__(self) -> str:
        return K.Probe.__repr__(self)[:-1] + f", theta={self.theta}, q={self.q!r})"


def _xtc_u(seed: int, pos: int, stream: int = X.XTC_STREAM, word: int = 0) -> float:
    return int(u_odd_at(seed, [pos], stream, word)[0]) / U_ONE


def xtc_keep(pr: XtcProbe, variant: str | None = None, pos: int | None = None):
    """``(x3, keep, keep')``: the staged row, its keep set and the keep set after XTC."""
    pos = pr.pos if pos is None else pos
    V = pr.V
    st = np.zeros(V, np.int32) if pr.state is None else pr.state
    x3 = pr.staged()
    x64 = x3.astype(np.float64)
    ok = ~np.isnan(x64)
    if R.is_point(x64, pr.T):
        if variant == "XTC at temperature 0" and pr.T == 0 and ok.any() and np.isfinite(x64[ok].max()):
            T = 1.0
            keep = ok.copy()
        else:
            return x3, None, None
    else:
        T = pr.T
        keep = pref.keep_set(x3, pr.k, pr.p, pr.min_p, pr.T)
    stream, word, upos = X.XTC_STREAM, 0, pos
    if variant == "gate from stream 0":
        stream = 0
    elif variant == "gate from word 1":
        word = 1
    elif variant == "gate at position - 1":
        upos = pos - 1
    u = np.float32(_xtc_u(pr.seed, upos, stream, word))
    q = np.float32(pr.q)
    fire = u <= q if variant == "gate u <= q" else u < q
    if not fire:
        return x3, keep, keep
    xa, w = x64, keep.copy()
    if variant == "A on unpenalised values":
        xa = np.asarray(pr.x, np.float64)
        if pr.allowed is not None:
            xa = np.where(pr.allowed, xa, np.nan)
    if variant == "A counts disallowed entries" and pr.allowed is not None:
        xa = pref.penalize(pr.x, st, pr.r, pr.pres, pr.freq).astype(np.float64)
        w = keep | ~pr.allowed
    if variant == "A over the whole row":
        w = ~np.isnan(xa)
    Ta = 1.0 if variant == "A without temperature" else T
    m = xa[w].max()
    e = np.where(w, np.exp((np.where(w, xa, m) - m) / Ta), 0.0)
    share = e / e.sum()
    A = w & (share >= pr.theta)
    idx = np.flatnonzero(A)
    remove = np.zeros(V, bool)
    C, s = K.plan(V)
    groups = [idx[idx // s == r] for r in range(C)] if variant == "A per CTA" else [idx]
    for r, grp in enumerate(groups):
        mine = np.zeros(V, bool)
        if variant == "A per CTA":
            mine[r * s: (r + 1) * s] = True
        else:
            mine[:] = True
        if len(grp) >= (3 if variant == "A needs three" else 2):
            lowest = xa[grp].min()
            if variant == "A's minimum from rank 0":
                r0 = grp[grp < s]
                lowest = xa[r0].min() if len(r0) else np.inf
            if variant == "A removed whole":
                remove[grp] = True
            else:
                remove |= mine & keep & ~np.isnan(xa) & (xa > lowest)
                if variant == "ties cut to one":
                    ties = grp[xa[grp] == lowest]
                    remove[ties[1:]] = True
    return x3, keep, keep & ~remove


def xtc_rule(pr: XtcProbe, variant: str | None = None, pos: int | None = None) -> tuple[int, float, int, float]:
    """``(token, gap, pre, pre_gap)``: the draw after XTC over the planted entries and its top-two gap, and the same
    without XTC."""
    pos = pr.pos if pos is None else pos
    x3, keep, keep2 = xtc_keep(pr, variant, pos)
    x64 = x3.astype(np.float64)
    if keep is None:
        return ref.greedy(x64), math.inf, ref.greedy(x64), math.inf
    if pr.T == 0:  # the "XTC at temperature 0" variant: greedy over what it kept
        return int(np.argmax(np.where(keep2, x64, -np.inf))), math.inf, ref.greedy(x64), math.inf
    S = np.array(sorted(i for i in set(pr.planted) | {pr.target} if not np.isnan(x64[i])), dtype=np.int64)
    sc = x64[S] / pr.T + K.gumbel_at(S, pr.seed, pos)

    def best(kept):
        c = np.flatnonzero(kept[S])
        if len(c) == 0:
            return -1, -math.inf
        o = c[np.argsort(-sc[c], kind="stable")]
        return int(S[o[0]]), (sc[o[0]] - sc[o[1]] if len(o) > 1 else math.inf)

    t, gap = best(keep2)
    pre, pre_gap = best(keep)
    return t, gap, pre, pre_gap


def _xtc_margins_ok(pr: XtcProbe) -> bool:
    """Every kept share at least REL (relative) away from theta."""
    x3 = pr.staged()
    x64 = x3.astype(np.float64)
    if R.is_point(x64, pr.T):
        return True
    keep = pref.keep_set(x3, pr.k, pr.p, pr.min_p, pr.T)
    m = x64[keep].max()
    e = np.where(keep, np.exp((np.where(keep, x64, m) - m) / pr.T), 0.0)
    share = e / e.sum()
    return not np.any(keep & (np.abs(share - pr.theta) < REL * pr.theta))


def settle_xtc(pr: XtcProbe, seed: int, differ: bool | None = True, extra=None, tries: int = 1 << 16) -> XtcProbe:
    """Search positions at ``seed``: the draw after XTC ``MARGIN`` clear of every planted entry it keeps (and of the
    background's best score), and, with ``differ``, the draw without XTC another token, clear as well."""
    assert _xtc_margins_ok(pr), pr
    pr.seed = seed
    x64 = pr.staged().astype(np.float64)
    if R.is_point(x64, pr.T):
        pr.pos = 1 + seed % 1000
        pr.want = pr.pre = ref.greedy(x64)
        return pr
    _, keep, _ = xtc_keep(pr, None, 1)
    S = set(pr.planted) | {pr.target}
    bg = keep.copy()
    bg[list(S)] = False
    rest = float(x64[bg].max() / pr.T + K.G_MAX) if bg.any() else -math.inf
    start = 1 + (seed % 997) * 1000
    for p_ in range(start, start + tries):
        t, gap, pre, pre_gap = xtc_rule(pr, pos=p_)
        if t < 0 or gap < MARGIN or pre_gap < MARGIN:
            continue
        x_t = x64[t] / pr.T + K.gumbel_at([t], seed, p_)[0]
        if x_t - rest < MARGIN:
            continue
        if differ is not None and (pre != t) != differ:
            continue
        if extra is not None and not extra(t, pre):
            continue
        pr.pos, pr.want, pr.pre = p_, t, pre
        return pr
    raise AssertionError(f"no position settles {pr!r}")


class XtcCatalogue:
    """Every XTC probe of one (V, dtype)."""

    def __init__(self, V: int, dtype: str):
        self.V, self.dtype = V, dtype
        self.rows = K._Rows(V, dtype, seed=V * 13 + DTYPES.index(dtype) + 2)
        self.C, self.slice = K.plan(V)
        self.probes: list[XtcProbe] = []
        self.temperature_zero()
        if V >= 7:
            self.gate()
            self.sizes_of_a()
            self.ties()
            self.background_outside_k()
            self.penalty_and_mask()
        if self.C >= 2:
            self.one_per_rank()

    def _g(self, v) -> float:
        return K.on_grid(v, self.dtype)

    def _row(self, vals, first=None):
        x = self.rows.background(-60.0, -45.0)
        idx = self.rows.spots(len(vals), first)
        x[idx] = [self._g(v) for v in vals]
        return x, idx

    def _spot(self, j: int) -> int:
        s = slice_spots(self.V)
        return s[j % len(s)]

    def _add(self, pr: XtcProbe, differ=True, extra=None) -> XtcProbe:
        pr = settle_xtc(pr, self.rows.seed64(), differ, extra)
        self.probes.append(pr)
        return pr

    def gate(self) -> None:
        """A = {a, b} at theta 0.25; q = 1, q just above u, q == u (must not fire: the rule is u < q), q just below u."""
        for j in range(3):
            x, idx = self._row([1.0, 0.5, 0.0], first=self._spot(j))
            T = (1.0, 0.8, 1.2)[j]
            base = self._add(XtcProbe("gate q=1", self.V, self.dtype, x, idx[0], T=T, planted=idx, theta=0.25, q=1.0))
            u = np.float32(_xtc_u(base.seed, base.pos))
            for name, q, fires in (("gate q above u", np.nextafter(u, np.float32(2)), True), ("gate q == u", u, False),
                                   ("gate q below u", np.nextafter(u, np.float32(0)), False)):
                pr = XtcProbe(name, self.V, self.dtype, x.copy(), idx[0], T=T, planted=idx, theta=0.25, q=float(q), seed=base.seed,
                              pos=base.pos, pre=base.pre)
                pr.want = base.want if fires else base.pre
                self.probes.append(pr)

    def sizes_of_a(self) -> None:
        for j in range(2):
            # |A| = 1: the top entry stays and wins
            x, idx = self._row([1.0, 0.0, -0.5], first=self._spot(j + 1))
            self._add(XtcProbe("|A| = 1", self.V, self.dtype, x, idx[0], planted=idx, theta=0.3), None, lambda t, pre, a=idx[0]: t == a)
            # |A| = 2: the larger one, planted to win without XTC, is removed
            x, idx = self._row([1.0, 0.75], first=self._spot(j + 2))
            self._add(XtcProbe("|A| = 2", self.V, self.dtype, x, idx[0], planted=idx, theta=0.4))

    def ties(self) -> None:
        """A = {a, b1, b2}, b1 == b2 its minimum, b2 on a later rank: both ties stay, and b2 is the winner."""
        for j in range(2):
            x, idx = self._row([1.0, 0.5, 0.5], first=self._spot(j))
            a, b1, b2 = idx[0], *sorted(idx[1:])
            self._add(XtcProbe("ties at A's minimum", self.V, self.dtype, x, b2, planted=idx, theta=0.25), True,
                      lambda t, pre, b2=b2: t == b2)

    def one_per_rank(self) -> None:
        """One member of A per rank, the largest on rank 0 (which wins without XTC), the least likely on the last rank
        (the only one left)."""
        C, s = self.C, self.slice
        vals = [1.0 - 0.125 * r for r in range(C)]
        x = self.rows.background(-60.0, -45.0)
        idx = [int(self.rows.rng.integers(r * s, min(self.V, (r + 1) * s))) for r in range(C)]
        x[idx] = [self._g(v) for v in vals]
        e = np.exp(np.array(vals) - 1.0)
        theta = float(np.float32(0.9 * (e / e.sum()).min()))
        self._add(XtcProbe("one member of A per rank", self.V, self.dtype, x, idx[-1], planted=idx, theta=theta), True,
                  lambda t, pre, a=idx[0]: pre == a)

    def background_outside_k(self) -> None:
        """Entries cut by top-k, top-p or min-p would pull a below theta if the shares were taken over the whole row;
        theta between the T = 1 share and the T share."""
        vals = [1.0, 0.5, 0.25, 0.25, 0.25, 0.25]
        x, idx = self._row(vals, first=self._spot(0))
        a, b = idx[0], idx[1]
        self._add(XtcProbe("outside K: top-k", self.V, self.dtype, x.copy(), a, planted=idx, k=2, theta=0.3))
        top_p = K._top_p_between(K.Probe("x", self.V, self.dtype, x.copy(), a, planted=idx), b, idx[2])
        assert top_p is not None
        self._add(XtcProbe("outside K: top-p", self.V, self.dtype, x.copy(), a, planted=idx, p=top_p, theta=0.3))
        min_p = K._min_p_for(self._g(1.0), 1.0, self._g(0.5))  # the bound is b itself
        self._add(XtcProbe("outside K: min-p", self.V, self.dtype, x.copy(), a, planted=idx, min_p=min_p, theta=0.3))
        # temperature: p_b is 0.378 at T = 2 and 0.269 at T = 1 (theta 0.32: A = {a, b}); 0.119 at T = 0.5 (theta 0.2)
        x, idx = self._row([1.0, 0.0], first=self._spot(1))
        self._add(XtcProbe("theta between the T = 1 and T shares", self.V, self.dtype, x.copy(), idx[0], planted=idx, T=2.0, theta=0.32))
        self._add(XtcProbe("theta between the T = 1 and T shares", self.V, self.dtype, x.copy(), idx[0], planted=idx, T=0.5, theta=0.2),
                  None, lambda t, pre, a=idx[0]: t == a)
        self._add(XtcProbe("tiny T", self.V, self.dtype, x.copy(), idx[0], planted=idx, T=1e-30, theta=0.2), None,
                  lambda t, pre, a=idx[0]: t == a)

    def penalty_and_mask(self) -> None:
        # repetition 2 sends the prompt token a from 2.0 to 1.0: A = {b, c} on the penalised row, {a} on the raw one
        x, idx = self._row([2.0, 1.25, 1.125], first=self._spot(2))
        a, b, c = idx
        st = np.zeros(self.V, np.int32)
        st[a] = pref.PROMPT
        self._add(XtcProbe("penalty moves A", self.V, self.dtype, x, b, planted=idx, r=2.0, state=st, theta=0.31), True,
                  lambda t, pre, b=b: pre == b)
        # a disallowed h far above: XTC sees the allowed a and b only
        x, idx = self._row([3.0, 1.0, 0.75], first=self._spot(3))
        allowed = np.ones(self.V, bool)
        allowed[idx[0]] = False
        self._add(XtcProbe("mask hides an entry", self.V, self.dtype, x, idx[1], planted=idx[1:], allowed=allowed, theta=0.4), True,
                  lambda t, pre, a=idx[1]: pre == a)

    def temperature_zero(self) -> None:
        if self.V == 1:
            x = np.array([1.5], np.float32)
            self._add(XtcProbe("T = 0", 1, self.dtype, x, 0, T=0.0, planted=[0], theta=0.1), None)
            return
        x, idx = self._row([1.0, 0.75], first=self._spot(1))
        self._add(XtcProbe("T = 0", self.V, self.dtype, x, idx[0], T=0.0, planted=idx, theta=0.4), None)


XTC_FORMS = ("penalized off", "penalized on", "constrained + state")


def xtc_forms_of(pr: XtcProbe) -> tuple[str, ...]:
    if pr.allowed is not None:
        return ("constrained + state",)
    if pr.penalized or pr.state is not None:
        return ("penalized on", "constrained + state")
    return XTC_FORMS
