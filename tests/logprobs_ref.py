"""Float64 restatement of ``tl_logprobs`` (DESIGN.md section 8a) and the error bound of its fp32 rounding points.

For one row ``x`` (the fp32 values the kernel reads):

* ``lse = m + log(sum_i exp(x_i - m))`` over the non-NaN entries, ``lp_i = x_i - lse``;
* ``rank(t) = 1 + #{i : x_i > x_t}`` (NaN entries never count); ``t = -1`` or a NaN ``x_t``: NaN and rank 0;
* top-N: the N largest non-NaN entries, descending, ties to the lower id; slots past them hold -1 and -inf;
* a row whose maximum is not finite (+inf, every non-NaN entry -inf, or every entry NaN): ``lse`` = that maximum (NaN
  when every entry is NaN) and NaN for every lp, ranks and ids as above.

``bound(x)`` is the largest difference the kernel's rounding points allow between its fp32 ``lp_i`` and ``lp_i`` here
(derivation in its docstring).  ``logprobs_like_ext`` has ``tiny_llm_ext_b200.logprobs``' surface on CPU tensors, for
host tests of the plumbing.
"""

from __future__ import annotations

import numpy as np

U = 2.0**-24  # unit roundoff of fp32
EXPF_ULP = 2  # CUDA expf: at most 2 ulp (CUDA C Programming Guide, mathematical functions, single precision)
LOGF_ULP = 1  # CUDA logf: at most 1 ulp


def row(x, target: int = -1, n: int = 0):
    """``(lse, lp, rank, ids [n], lps [n])`` of one row in float64."""
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    m = x[ok].max() if ok.any() else np.nan
    finite = bool(np.isfinite(m))
    if finite:
        lse = m + np.log(np.exp(x[ok] - m).sum())
    else:
        lse = m
    xt = x[target] if 0 <= target < len(x) else np.nan
    lp = xt - lse if finite and not np.isnan(xt) else np.nan
    rank = int((x[ok] > xt).sum()) + 1 if not np.isnan(xt) else 0
    order = np.lexsort((np.arange(len(x)), -np.where(ok, x, -np.inf)))  # value descending, id ascending
    order = order[ok[order]][:n]
    ids = np.full(n, -1, dtype=np.int64)
    lps = np.full(n, -np.inf)
    ids[: len(order)] = order
    lps[: len(order)] = (x[order] - lse) if finite else np.nan
    return float(lse), float(lp), rank, ids, lps


def logprobs(logits, targets=None, top_n=None, max_n: int = 0):
    """Row-wise ``row`` over ``logits [rows, V]`` -> numpy ``(lse, lp, rank, ids, lps)`` with the kernel's dtypes."""
    x = np.asarray(logits, dtype=np.float64)
    rows = x.shape[0]
    out = (np.empty(rows, np.float32), np.empty(rows, np.float32), np.empty(rows, np.int32), np.empty((rows, max_n), np.int32),
           np.empty((rows, max_n), np.float32))
    for r in range(rows):
        t = -1 if targets is None else int(targets[r])
        n = max_n if top_n is None else max(0, min(max_n, int(top_n[r])))
        lse, lp, rank, ids, lps = row(x[r], t, n)
        ids_full = np.full(max_n, -1, np.int64)
        lps_full = np.full(max_n, -np.inf)
        ids_full[:n], lps_full[:n] = ids, lps
        out[0][r], out[1][r], out[2][r], out[3][r], out[4][r] = lse, lp, rank, ids_full, lps_full
    return out


def bound(x):
    """Per-entry bound ``B_i`` on ``|lp_kernel(x_i) - lp_i|`` and the bound on ``|lse_kernel - lse|`` for a row with a
    finite maximum ``m``.  Rounding points of the kernel, with ``u = 2^-24``:

    1. ``d_i = fl(x_i - m)``: ``|d_i - (x_i - m)| <= u |x_i - m|``.
    2. ``e_i = expf(d_i)``: ``e_i = exp(d_i)(1 + a)``, ``|a| <= 2 ulp <= 2^-22``; with 1.,
       ``|e_i - exp(x_i - m)| <= exp(x_i - m) (exp(u |x_i - m|)(1 + 2^-22) - 1) =: E_i``.
    3. ``E_i = round(e_i 2^40)``: at most ``2^-41`` absolute per entry.
    4. ``S_fx`` exact; ``fl(S_fx) 2^-40 = S'(1 + b)``, ``|b| <= u``.
    So ``|S_k - S| <= dS := sum_i E_i + V 2^-41 + u (S + sum E_i + V 2^-41)`` and
    ``|log S_k - log S| <= -log(1 - dS / S) =: dL``.
    5. ``log_s = logf(S_k)``: ``+ 2^-23 |log S_k|`` (1 ulp).
    6. ``lp = fl(d_i - log_s)``: ``+ u |lp|`` (with 1. for ``d_i``); ``lse = fl(m + log_s)``: ``+ u |lse|``.
    Each bound is evaluated with a ``(1 + 2^-20)`` margin on ``|lp|``, ``|lse|`` and ``|log S|`` to cover the
    difference between the exact values and the float64 values the bound is computed from; there is no other term.
    """
    x = np.asarray(x, dtype=np.float64)
    ok = ~np.isnan(x)
    m = x[ok].max()
    d = np.abs(np.where(ok, x, m) - m)
    e = np.where(ok, np.exp(-d), 0.0)
    S = e.sum()
    V = int(ok.sum())
    live = ok & np.isfinite(d)  # -inf entries add exactly 0 (expf(-inf) = 0)
    E = np.where(live, e * np.expm1(U * np.where(live, d, 0.0) + np.log1p(2.0**-22)), 0.0)
    fix = V * 2.0**-41
    dS = E.sum() + fix + U * (S + E.sum() + fix)
    dL = -np.log1p(-dS / S)
    logS = np.log(S)
    grow = 1 + 2.0**-20
    log_s_err = dL + 2.0**-23 * (logS + dL) * grow
    lp = x - m - logS
    with np.errstate(invalid="ignore"):
        lp_bound = U * d + log_s_err + U * np.abs(lp) * grow + U * d * U  # the last term: 1.'s error inside 6.'s operand
    lse_bound = log_s_err + U * abs(m + logS) * grow
    return lp_bound, lse_bound


def logprobs_like_ext(logits, targets=None, top_n=None, max_n=0, out=None, out_index=None, stream=None):
    """``tiny_llm_ext_b200.logprobs``' surface on CPU tensors (test stand-in): the float64 values rounded to fp32."""
    import torch

    if out is not None:
        raise RuntimeError("logprobs stand-in: out / out_index are not supported")
    cols = logits.detach().float().cpu().numpy()
    t = None if targets is None else targets.detach().cpu().numpy()
    n = None if top_n is None else top_n.detach().cpu().numpy()
    return tuple(torch.from_numpy(a).to(logits.device) for a in logprobs(cols, t, n, max_n))
