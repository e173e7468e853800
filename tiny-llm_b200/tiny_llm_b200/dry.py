"""DRY, "don't repeat yourself" (DESIGN.md section 24): ``SamplingParams.dry_multiplier``, ``dry_base``,
``dry_allowed_length``, ``dry_penalty_last_n`` and ``dry_sequence_breakers``, validated here and packed for
``tl_dry_penalty``.

A DRY row is one ``tl_dry_row``: int32 ``[ROW_WORDS]`` holding the flags, the allowed length, the window, the breaker
count, ``MAX_BREAKERS`` sorted breaker ids and ``MAX_MATCH`` fp32 penalties ``P[k] = fl32(m * b**k)`` (computed in
double, rounded once).  Beside it the request keeps its whole history on the device, ``capacity`` ids per row: the
prompt, then the generated ids, up to the step's input token, which each launch writes at index ``n - 1``."""

from __future__ import annotations

import math
import numbers

import numpy as np
import torch

MAX_MATCH = 64  # TL_DRY_MAX_MATCH
MAX_BREAKERS = 64  # TL_DRY_MAX_BREAKERS
ROW_WORDS = 4 + MAX_BREAKERS + MAX_MATCH  # int32 words of one tl_dry_row
FLAG_ON = 1


def _real(v) -> bool:
    return not isinstance(v, bool) and isinstance(v, numbers.Real) and math.isfinite(v)


def _int(v) -> bool:
    return not isinstance(v, bool) and isinstance(v, numbers.Integral)


def normalized_dry(p) -> dict:
    """The DRY fields of ``SamplingParams`` ``p`` validated and normalised (``ValueError`` naming the field)."""
    m = p.dry_multiplier
    if not _real(m) or m < 0:
        raise ValueError(f"dry_multiplier must be 0 (off) or a finite number > 0, got {m!r}")
    b = p.dry_base
    if not _real(b) or not b > 1:
        raise ValueError(f"dry_base must be a finite number > 1, got {b!r}")
    a = p.dry_allowed_length
    if not _int(a) or not 1 <= a < 1 << 31:
        raise ValueError(f"dry_allowed_length must be an int >= 1, got {a!r}")
    n = p.dry_penalty_last_n
    if not _int(n) or not 0 <= n < 1 << 31:
        raise ValueError(f"dry_penalty_last_n must be 0 (the whole history) or an int > 0, got {n!r}")
    brk = p.dry_sequence_breakers
    if isinstance(brk, (str, bytes)) or not hasattr(brk, "__iter__"):
        raise ValueError(f"dry_sequence_breakers must be a collection of token ids, got {type(brk).__name__}")
    ids = set()
    for t in brk:
        if not _int(t) or not 0 <= t < 1 << 31:
            raise ValueError(f"dry_sequence_breakers token ids must be ints in [0, 2**31), got {t!r}")
        ids.add(int(t))
    if len(ids) > MAX_BREAKERS:
        raise ValueError(f"dry_sequence_breakers holds at most {MAX_BREAKERS} ids, got {len(ids)}")
    return dict(dry_multiplier=float(m), dry_base=float(b), dry_allowed_length=int(a), dry_penalty_last_n=int(n),
                dry_sequence_breakers=tuple(sorted(ids)))


def penalty_table(multiplier: float, base: float, allowed_length: int) -> np.ndarray:
    """``P[k] = fl32(m * b**k)`` for ``k <= MAX_MATCH - a`` (+inf where it overflows fp32), 0 beyond: float32
    ``[MAX_MATCH]``."""
    out = np.zeros(MAX_MATCH, dtype=np.float32)
    for k in range(max(0, MAX_MATCH - allowed_length + 1)):
        try:
            v = multiplier * base**k
        except OverflowError:
            v = math.inf
        with np.errstate(over="ignore"):
            out[k] = np.float32(v)
    return out


def pack_row(p) -> np.ndarray:
    """The int32 ``[ROW_WORDS]`` ``tl_dry_row`` of ``SamplingParams`` ``p`` (zero when ``p`` is None or DRY is off)."""
    row = np.zeros(ROW_WORDS, dtype=np.int32)
    if p is None or not p.dry:
        return row
    brk = p.dry_sequence_breakers
    row[:4] = (FLAG_ON, p.dry_allowed_length, p.dry_penalty_last_n, len(brk))
    row[4 : 4 + len(brk)] = brk
    row[4 + MAX_BREAKERS :] = penalty_table(p.dry_multiplier, p.dry_base, p.dry_allowed_length).view(np.int32)
    return row


def unpack_row(row) -> dict:
    """The parameters a packed row carries (the inverse of ``pack_row``, for checks)."""
    row = np.asarray(row, dtype=np.int32)
    flags, a, n, nb = (int(v) for v in row[:4])
    return dict(flags=flags, dry_allowed_length=a, dry_penalty_last_n=n, dry_sequence_breakers=tuple(row[4 : 4 + nb].tolist()),
                penalty=row[4 + MAX_BREAKERS :].view(np.float32).copy())


class DryRows:
    """The ``tl_dry_penalty`` table of ``rows`` rows on ``device``: ``table`` (int32 ``[rows, ROW_WORDS]``, zero rows
    off), ``history`` (int32 ``[rows, capacity]``) and ``scratch`` (float32 ``[rows, capacity]``, the launch's
    per-end candidates)."""

    def __init__(self, rows: int, capacity: int, device):
        if capacity < 1:
            raise ValueError("a DRY history needs a capacity of at least one token")
        self.rows, self.capacity, self.device = rows, capacity, torch.device(device)
        self.table = torch.zeros((rows, ROW_WORDS), dtype=torch.int32, device=self.device)
        self.history = torch.zeros((rows, capacity), dtype=torch.int32, device=self.device)
        self.scratch = torch.zeros((rows, capacity), dtype=torch.float32, device=self.device)

    def set_row(self, r: int, p, history_ids) -> None:
        """Write request ``p``'s row ``r`` and its history (prompt then generated ids, the step's input token last: the
        launch writes that one again at index ``n - 1``).  A ``p`` without DRY clears the row."""
        if p is None or not p.dry:
            self.clear_row(r)
            return
        ids = [int(t) for t in history_ids]
        if len(ids) > self.capacity:
            raise ValueError(f"a DRY history of {len(ids)} tokens exceeds its capacity of {self.capacity}")
        self.table[r].copy_(torch.from_numpy(pack_row(p)))
        self.history[r].zero_()
        if ids:
            self.history[r, : len(ids)].copy_(torch.tensor(ids, dtype=torch.int32))

    def clear_row(self, r: int) -> None:
        self.table[r].zero_()
