"""Float64 attention reference and the error bound the attention kernels are held to.

``paged_reference`` restates ``tl_paged_attention`` (include/tiny_llm_b200.h): query row l of request b sees the keys
< min(clamp(ctx - L + l + 1, 0, ctx), max_pages * page_size) when causal, a key whose page id is < 0 or >= num_pages
is skipped, and a row that sees no key gives zeros.  ``dense_reference`` restates ``tl_decode_attention``.  Both work
in float64 from the exact inputs, on the inputs' device, and return besides the unrounded output

    A[r, d]   = sum_j p_j |v_jd|                                  the scale of any error in the probabilities
    smax[r]   = max over keys with p_j > 0 of |mask_j| + scale * sum_d |q_d k_jd|     bounds |s_j| and its fp32 error
    nvis[r]   = number of keys the row sees                        bounds the length of fp32 accumulation chains

``masked_reference`` takes an explicit key mask instead (``segment_visible`` builds the one of the segment-causal and
prefixed-segment entry points) and also returns V1, the sum of |v| over the visible keys.
``error_bound`` turns them into an elementwise tolerance (its docstring has the derivation).  ``check_needles``
compares a kernel with the reference on needle queries (``needle_queries``): a query that is a scaled copy of one key
puts almost all the probability on that key, so whether the kernel saw the key changes the output by O(1).
"""

from __future__ import annotations

import math

import torch

F64 = torch.float64
UNIT_ROUNDOFF = {torch.bfloat16: 2.0**-8, torch.float16: 2.0**-11, torch.float32: 2.0**-24}


def visible_keys(context_lens, L, causal, cap, ctx_delta=0, row_delta=0, clamp_first=False):
    """[B, L] number of keys row l of request b sees.  ``ctx_delta`` / ``row_delta`` move the context and the causal
    row, ``clamp_first`` clamps the context to the table before the causal shift: a correct check must fail against
    a reference changed by any of them (tests/test_attention_ref_host.py)."""
    ctx = context_lens.to(torch.int64).cpu()[:, None] + ctx_delta
    if clamp_first:
        ctx = ctx.clamp(max=cap)
    if causal:
        rows = torch.arange(L, dtype=torch.int64)[None, :] + row_delta
        vis = torch.minimum(torch.clamp(ctx - L + rows + 1, min=0), ctx.clamp(min=0))
    else:
        vis = ctx.clamp(min=0).expand(-1, L)
    return vis.clamp(max=cap)


def _softmax_stats(s, absum, V, out_rows, A_rows, smax_rows):
    """s, absum [..., S] (masked scores are -inf); V [S, D] broadcast over the leading dims."""
    m = s.amax(dim=-1, keepdim=True)
    m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    e = torch.exp(s - m)
    z = e.sum(dim=-1, keepdim=True)
    p = e / torch.where(z > 0, z, torch.ones_like(z))
    out_rows.copy_(p @ V)
    A_rows.copy_(p @ V.abs())
    smax_rows.copy_(torch.where(p > 0, absum, torch.zeros_like(absum)).amax(dim=-1))


def paged_reference(q, key_pages, value_pages, block_table, context_lens, scale, causal, num_kv_heads, num_heads, *, ctx_delta=0,
                    row_delta=0, clamp_first=False):
    """q [B*Hq, L, D]; pages [P, Hkv, page, D]; block_table int32 [B, max_pages]; context_lens int32 [B].
    Returns (out, A) float64 [B*Hq, L, D] and (smax float64, nvis int64) [B*Hq, L]."""
    rows, L, D = q.shape
    P, Hkv, page, _ = key_pages.shape
    B, max_pages = block_table.shape
    G = num_heads // num_kv_heads
    dev = q.device
    nvis = visible_keys(context_lens, L, causal, max_pages * page, ctx_delta, row_delta, clamp_first)
    out = torch.zeros(rows, L, D, dtype=F64, device=dev)
    A = torch.zeros_like(out)
    smax = torch.zeros(rows, L, dtype=F64, device=dev)
    ids = block_table.to(dev).to(torch.int64)
    live = (ids >= 0) & (ids < P)
    for b in range(B):
        S = int(nvis[b].max())
        if S == 0:
            continue
        npg = (S + page - 1) // page
        pid = ids[b, :npg].clamp(0, P - 1)
        K = key_pages[pid].to(F64).permute(1, 0, 2, 3).reshape(Hkv, npg * page, D)[:, :S]
        V = value_pages[pid].to(F64).permute(1, 0, 2, 3).reshape(Hkv, npg * page, D)[:, :S]
        key_ok = live[b, :npg].repeat_interleave(page)[:S]
        pos = torch.arange(S, device=dev)
        Qb = q[b * num_heads : (b + 1) * num_heads].to(F64).reshape(Hkv, G, L, D)
        nv = nvis[b].to(dev)
        chunk = max(1, (1 << 25) // (num_heads * S))
        for l0 in range(0, L, chunk):
            l1 = min(L, l0 + chunk)
            ok = key_ok[None, :] & (pos[None, :] < nv[l0:l1, None])  # [l, S]
            s = scale * (Qb[:, :, l0:l1] @ K.transpose(-1, -2)[:, None])  # [Hkv, G, l, S]
            s = s.masked_fill(~ok, float("-inf"))
            absum = abs(scale) * (Qb[:, :, l0:l1].abs() @ K.abs().transpose(-1, -2)[:, None])
            o = torch.empty(Hkv, G, l1 - l0, D, dtype=F64, device=dev)
            a = torch.empty_like(o)
            sm = torch.empty(Hkv, G, l1 - l0, dtype=F64, device=dev)
            _softmax_stats(s, absum, V[:, None], o, a, sm)
            out[b * num_heads : (b + 1) * num_heads, l0:l1] = o.reshape(num_heads, l1 - l0, D)
            A[b * num_heads : (b + 1) * num_heads, l0:l1] = a.reshape(num_heads, l1 - l0, D)
            smax[b * num_heads : (b + 1) * num_heads, l0:l1] = sm.reshape(num_heads, l1 - l0)
    nvis_rows = nvis.to(dev)[:, None, :].expand(B, num_heads, L).reshape(rows, L)
    return out, A, smax, nvis_rows


def dense_reference(q, k, v, mask, scale, causal, has_mask, num_heads, num_kv_heads):
    """tl_decode_attention: q [B*Hq, L, D], k/v [B*Hkv, S, D], mask fp32 [B*Hq, L, S]; key p is masked for row l
    when causal and p > S - L + l.  Same returns as paged_reference."""
    rows, L, D = q.shape
    S = k.shape[1]
    G = num_heads // num_kv_heads
    B = rows // num_heads
    Q = q.to(F64).reshape(B, num_kv_heads, G, L, D)
    K = k.to(F64).reshape(B, num_kv_heads, 1, S, D)
    V = v.to(F64).reshape(B, num_kv_heads, 1, S, D)
    s = scale * (Q @ K.transpose(-1, -2))
    absum = abs(scale) * (Q.abs() @ K.abs().transpose(-1, -2))
    if has_mask:
        mk = mask.to(F64).reshape(B, num_kv_heads, G, L, S)
        s = s + mk
        absum = absum + torch.where(torch.isfinite(mk), mk.abs(), torch.zeros_like(mk))
    pos = torch.arange(S, device=q.device)
    lim = S - L + torch.arange(L, device=q.device)
    if causal:
        s = s.masked_fill(pos[None, :] > lim[:, None], float("-inf"))
    out = torch.empty(B, num_kv_heads, G, L, D, dtype=F64, device=q.device)
    A = torch.empty_like(out)
    smax = torch.empty(B, num_kv_heads, G, L, dtype=F64, device=q.device)
    _softmax_stats(s, absum, V, out, A, smax)
    nvis = (torch.isfinite(s)).sum(dim=-1).reshape(rows, L)
    return out.reshape(rows, L, D), A.reshape(rows, L, D), smax.reshape(rows, L), nvis


def masked_reference(q, k, v, visible, scale, num_kv_heads):
    """Attention over an explicit key mask: q [Hq, L, D]; k / v [Hkv, S, D] in logical key order; visible bool
    [Hq or 1, L, S].  Returns (out, A, smax, nvis) as ``paged_reference`` does, plus V1 [Hq, L, D] = the sum of |v_jd|
    over the keys the row sees (the scale of P's absolute rounding floor, ``error_bound(p_dtype=float16)``).  Float64
    on q's device, chunked over rows so that L = S = 8192 fits."""
    Hq, L, D = q.shape
    S = k.shape[1]
    G = Hq // num_kv_heads
    dev = q.device
    Q = q.to(F64).reshape(num_kv_heads, G, L, D)
    K, V = k.to(dev).to(F64)[:, None], v.to(dev).to(F64)[:, None]  # [Hkv, 1, S, D]
    Kt, Ka, Va = K.transpose(-1, -2), K.abs().transpose(-1, -2), V.abs()
    vis = visible.to(dev)
    out = torch.zeros(Hq, L, D, dtype=F64, device=dev)
    A, V1 = torch.zeros_like(out), torch.zeros_like(out)
    smax = torch.zeros(Hq, L, dtype=F64, device=dev)
    nvis = torch.zeros(Hq, L, dtype=torch.int64, device=dev)
    chunk = max(1, (1 << 25) // (Hq * max(S, 1)))
    for l0 in range(0, L, chunk):
        l1 = min(L, l0 + chunk)
        ok = vis[:, l0:l1].expand(Hq, l1 - l0, S).reshape(num_kv_heads, G, l1 - l0, S)
        s = (scale * (Q[:, :, l0:l1] @ Kt)).masked_fill(~ok, float("-inf"))
        absum = abs(scale) * (Q[:, :, l0:l1].abs() @ Ka)
        o = torch.empty(num_kv_heads, G, l1 - l0, D, dtype=F64, device=dev)
        a = torch.empty_like(o)
        sm = torch.empty(num_kv_heads, G, l1 - l0, dtype=F64, device=dev)
        _softmax_stats(s, absum, V, o, a, sm)
        out[:, l0:l1] = o.reshape(Hq, l1 - l0, D)
        A[:, l0:l1] = a.reshape(Hq, l1 - l0, D)
        smax[:, l0:l1] = sm.reshape(Hq, l1 - l0)
        V1[:, l0:l1] = (ok.to(F64) @ Va).reshape(Hq, l1 - l0, D)
        nvis[:, l0:l1] = ok.sum(dim=-1).reshape(Hq, l1 - l0)
    return out, A, smax, nvis, V1


def live_keys(block_table, num_pages, page_size, S):
    """[S] bool: key j's page id block_table[j // page_size] is in [0, num_pages)."""
    ids = block_table.to(torch.int64).reshape(-1).cpu()[torch.arange(S) // page_size]
    return (ids >= 0) & (ids < num_pages)


def segment_visible(segment_start, key_live, prefix_start=None, prefix_end=None):
    """[1, L, L] bool: the keys row l of ``tl_paged_attention_segments`` (prefix_start None) or
    ``tl_paged_attention_prefixed_segments`` sees over one packed request whose keys are its L rows.  With
    lo = max(segment_start[l], 0): nothing when segment_start[l] > l; else [lo, l] and, prefixed, [max(prefix_start[l], 0),
    min(prefix_end[l], lo)); never a key whose page is not live (``live_keys``)."""
    seg = torch.as_tensor(segment_start, dtype=torch.int64).cpu()
    L = seg.shape[0]
    row = torch.arange(L)[:, None]
    key = torch.arange(L)[None, :]
    lo = seg.clamp(min=0)[:, None]
    own = seg[:, None] <= row
    vis = (key >= lo) & (key <= row)
    if prefix_start is not None:
        ps = torch.as_tensor(prefix_start, dtype=torch.int64).cpu().clamp(min=0)[:, None]
        pe = torch.minimum(torch.as_tensor(prefix_end, dtype=torch.int64).cpu()[:, None], lo)
        vis = vis | ((key >= ps) & (key < pe))
    return (vis & own & key_live[None, :])[None]


def error_bound(ref, A, smax, nvis, D, out_dtype, p_rounded, *, p_dtype=torch.bfloat16, V1=None):
    """Elementwise bound on |kernel - ref| for a kernel that computes scores and the softmax in fp32.

    Scores.  A score is a sum of D products; in fp32 (bf16 x bf16 products are exact, an MMA may truncate each
    addition) its error is at most (2D + 16) 2^-24 sum_d |q_d k_jd| scale, which also covers the scale multiply, the
    mask addition and subtracting the running maximum (each <= 2^-24 |s|).  ex2.approx / __expf add a relative
    error below 2^-21, i.e. an absolute error of 2^-21 in the exponent.  So every score the kernel exponentiates is
    off by at most delta = (2D + 16) 2^-24 smax + 2^-20.  Perturbing every score by at most delta changes each p_j
    by a factor in [e^-2delta, e^2delta], so the output moves by at most eps_s A with eps_s = e^(2 delta) - 1.

    P.  The tensor-core kernels (mma.sync flash, wgmma) round P to bf16 for P V while the row sum uses the unrounded
    P: at most 2^-8 A (bf16 unit roundoff, ``p_rounded``).  The fp16 form of the wgmma kernel (``p_dtype`` float16)
    rounds P to fp16, whose range ends where bf16's does not: in the units the row is finally normalised with, its
    largest p is >= 1 (the kept maximum lies at most 2^8 below the row's maximum and never above it; a rescale only
    scales earlier terms down), an fp16 p below 2^-14 is subnormal and one below 2^-25 rounds to 0.  So each p is off by
    at most 2^-11 p + 2^-25, and since sum p >= 1 the output by at most 2^-11 A + 2^-25 V1, V1 = sum over the visible
    keys of |v_jd| (``masked_reference``).  Example: a key at the row maximum with v_d = 0 and 4,000 keys 18 nats lower
    with v_d = 1 give ref_d = 6e-5 while every p of those keys (2^-26) rounds to 0.

    Accumulation.  O and the row sum are fp32 sums; no kernel adds more than nvis / 4 + 64 terms in one sequential
    chain (the row-wise and dense kernels' four warps are the narrowest split), each addition off by <= 2^-24
    relative, truncating MMA adds by 2^-23: (nvis / 4 + 64) 2^-23 A.

    Output.  Rounding to the output type: u |ref| (u = 2^-8 bf16, 2^-11 f16, 2^-24 f32); the division by the row
    sum adds 2^-23 |ref|.

    There is no absolute term: a row that sees nothing must be exactly zero."""
    delta = (2 * D + 16) * 2.0**-24 * smax + 2.0**-20
    eps_s = torch.expm1(2 * delta)
    n_acc = (nvis.to(F64) / 4 + 64) * 2.0**-23
    u_p = UNIT_ROUNDOFF[p_dtype] if p_rounded else 0.0
    u_out = UNIT_ROUNDOFF[out_dtype] + 2.0**-23
    tol = u_out * ref.abs() + (u_p + eps_s + n_acc)[..., None] * A
    if p_rounded and p_dtype == torch.float16:
        if V1 is None:
            raise ValueError("error_bound: fp16 P needs V1, the sum of |v| over the visible keys")
        tol = tol + 2.0**-25 * V1
    elif p_rounded and p_dtype != torch.bfloat16:
        raise ValueError(f"error_bound: no bound for P rounded to {p_dtype}")
    return tol


def assert_within(got, ref, tol, what):
    err = (got.to(F64) - ref).abs()
    bad = err > tol
    if bool(bad.any()):
        worst = int((err - tol).flatten().argmax())
        where = [int(i) for i in torch.unravel_index(torch.tensor(worst), err.shape)]
        raise AssertionError(
            f"{what}: {int(bad.sum())} of {bad.numel()} elements outside the error bound; worst at {where}: "
            f"|got - ref| = {float(err.flatten()[worst]):.3g} > bound {float(tol.flatten()[worst]):.3g} (ref {float(ref.flatten()[worst]):.4g})")


def paged_inputs(g, lens, page, Hkv, D, dtype, max_pages=None, holes=(), logical_keys=None, key_rms=1.0):
    """Random K/V pages for requests of the given context lengths -> (key_pages, value_pages, block_table,
    context_lens, storage), CPU tensors.  storage[b, lp] is the physical page of logical page lp of request b: every
    logical page up to the table's width has its own, shuffled.  The block table holds the pages with keys below
    min(ctx, capacity) and -1 after them.  ``holes``: (b, logical page, "neg" | "big") entries replaced by -1 / an id
    >= num_pages; their keys sit in physical page 0 / num_pages - 1, where a kernel that clamped the id would find
    them.  ``logical_keys`` [B, Hkv, max_pages * page, D] replaces the random keys."""
    B = len(lens)
    need = [(n + page - 1) // page for n in lens]
    width = max_pages if max_pages is not None else max(1, max(need))
    P = B * width + 2
    storage = torch.randperm(P, generator=g)[: B * width].reshape(B, width).to(torch.int32)
    for b, lp, kind in holes:
        phys = 0 if kind == "neg" else P - 1
        where = (storage == phys).nonzero()
        if len(where):
            storage[where[0, 0], where[0, 1]] = storage[b, lp]
        storage[b, lp] = phys
    bt = storage.clone()
    for b, n in enumerate(need):
        bt[b, min(n, width) :] = -1
    for b, lp, kind in holes:
        bt[b, lp] = -1 if kind == "neg" else P + 7
    kp = torch.randn(P, Hkv, page, D, generator=g) * key_rms
    vp = torch.randn(P, Hkv, page, D, generator=g)
    if logical_keys is not None:
        for b in range(B):
            kp[storage[b].long()] = logical_keys[b].reshape(Hkv, width, page, D).permute(1, 0, 2, 3).to(kp.dtype)
    return kp.to(dtype), vp.to(dtype), bt, torch.tensor(lens, dtype=torch.int32), storage


def needle_queries(key_pages, storage, targets, num_heads, num_kv_heads, scale, nats, dtype):
    """q [B*Hq, L, D] whose row (b, h, l) is the key at logical position targets[b, h, l] of request b (found through
    ``storage``, the physical page of every logical page, which may differ from the block table where the table masks
    a page), scaled so that its own score is ``nats`` and rounded to ``dtype``."""
    B, Hq, L = targets.shape
    P, Hkv, page, D = key_pages.shape
    G = num_heads // num_kv_heads
    t = targets.clamp(min=0).to(key_pages.device)
    st = storage.to(key_pages.device).to(torch.int64)
    pid = st.gather(1, (t // page).reshape(B, -1)).reshape(B, Hq, L)
    kvh = (torch.arange(Hq, device=t.device) // G)[None, :, None].expand(B, Hq, L)
    k = key_pages[pid, kvh, t % page].to(F64)  # [B, Hq, L, D]
    c = nats / (scale * (k * k).sum(dim=-1, keepdim=True))
    return (k * c).to(dtype).reshape(B * Hq, L, D)


def needle_values(value_pages, storage, targets, num_heads, num_kv_heads):
    """The value rows the needles point at, [B*Hq, L, D] float64."""
    B, Hq, L = targets.shape
    P, Hkv, page, D = value_pages.shape
    G = num_heads // num_kv_heads
    t = targets.clamp(min=0).to(value_pages.device)
    pid = storage.to(value_pages.device).to(torch.int64).gather(1, (t // page).reshape(B, -1)).reshape(B, Hq, L)
    kvh = (torch.arange(Hq, device=t.device) // G)[None, :, None].expand(B, Hq, L)
    return value_pages[pid, kvh, t % page].to(F64).reshape(B * Hq, L, D)


def needle_visible(block_table, num_pages, page_size, targets, nvis):
    """[B*Hq, L] bool: the needle's key is inside the row's visible range and its page id is live."""
    B, Hq, L = targets.shape
    t = targets.to(torch.int64).cpu()
    ids = block_table.to(torch.int64).cpu().gather(1, (t.clamp(min=0) // page_size).reshape(B, -1)).reshape(B, Hq, L)
    live = (ids >= 0) & (ids < num_pages)
    return ((t >= 0) & (t < nvis.cpu().reshape(B, Hq, L)) & live).reshape(B * Hq, L)


def check_needles(got, ref, A, tol, vneedle, visible, out_dtype, what):
    """A visible needle must come back as its value row within one ulp of the output type (the reference itself
    must equal it to 1e-9: otherwise the input is no needle).  An invisible one must match the reference over the
    other keys within ``tol``, and the value row must lie outside that bound on some element, so that a kernel that
    saw the needle would fail."""
    got = got.to(F64).reshape(ref.shape)
    vis = visible.to(ref.device)
    if bool(vis.any()):
        v, r, o = vneedle[vis], ref[vis], got[vis]
        assert float((r - v).abs().max()) <= 1e-9 * (1 + float(v.abs().max())), f"{what}: the inputs are not needles"
        ulp = 2 * UNIT_ROUNDOFF[out_dtype]
        err = (o - v).abs() - ulp * v.abs()
        if bool((err > 0).any()):
            rows = vis.nonzero()[(err > 0).any(dim=-1).nonzero()[:, 0]]
            raise AssertionError(f"{what}: {len(rows)} visible needles not returned (first query rows, positions {rows[:8].tolist()}); "
                                 f"worst |got - V| = {float((o - v).abs().max()):.3g}")
    hid = ~vis
    if bool(hid.any()):
        power = ((vneedle[hid] - ref[hid]).abs() - tol[hid]).amax(dim=-1)
        assert float(power.min()) > 0.05, f"{what}: an invisible needle's value row lies within the error bound (the check has no power)"
        err = (got[hid] - ref[hid]).abs() - tol[hid]
        if bool((err > 0).any()):
            rows = hid.nonzero()[(err > 0).any(dim=-1).nonzero()[:, 0]]
            raise AssertionError(f"{what}: {len(rows)} rows with an invisible needle outside the error bound (first query rows, positions "
                                 f"{rows[:8].tolist()}); worst excess {float(err.max()):.3g}")


def probe_positions(ctx, L, causal, page_size, cap, max_per_kind=256):
    """Key positions worth a needle for one request: (per-row list, shared list).  Per row l of a causal multi-row call:
    its last key and the first it must not see (ctx - L + l and ctx - L + l + 1 unless the block table clamps them).
    Shared: 0, the last visible key of the
    last row, ctx (the first invisible key) when it lies in a live page (ctx % page != 0), both sides of each page
    boundary and each 64-key tile boundary, and a sweep every 37 keys (crossing every split boundary whatever the split
    count).  Positions outside [0, cap) are dropped; a long list of boundaries is thinned evenly to max_per_kind."""

    def keep(ps):
        return [p for p in ps if 0 <= p < cap]

    def thin(ps):
        if len(ps) <= max_per_kind:
            return ps
        step = len(ps) / max_per_kind
        return [ps[int(i * step)] for i in range(max_per_kind)]

    vis = visible_keys(torch.tensor([ctx]), L, causal, cap)[0].tolist()
    per_row = [keep([vis[l] - 1, vis[l]]) if causal and L > 1 else [] for l in range(L)]
    end = min(ctx, cap)
    last = end - 1 if not causal else min(ctx - 1, cap - 1)
    shared = [0, last]
    if ctx % page_size != 0:
        shared.append(ctx)
    shared += thin([x + d for x in range(page_size, end + 1, page_size) for d in (-1, 0)])
    shared += thin([x + d for x in range(64, end + 1, 64) for d in (-1, 0)])
    shared += thin(list(range(0, end + 1, 37)))
    return per_row, list(dict.fromkeys(keep(shared)))


def assign_targets(per_row_lists, shared_lists, Hq, L, max_rounds, g):
    """Targets [rounds, B, Hq, L]: every row's own probes first, then the request's shared probes dealt over its rows
    and heads; empty slots get random positions among the request's first keys."""
    B = len(shared_lists)
    queues = [[list(per_row_lists[b][l]) for l in range(L)] for b in range(B)]
    for b in range(B):
        for i, p in enumerate(shared_lists[b]):
            queues[b][i % L].append(p)
    rounds = max(1, min(max_rounds, max(math.ceil(len(q) / Hq) for qs in queues for q in qs)))
    out = torch.empty(rounds, B, Hq, L, dtype=torch.int64)
    for b in range(B):
        hi = max([0] + shared_lists[b]) + 1
        fill = torch.randint(0, hi, (rounds, Hq, L), generator=g)
        for l in range(L):
            q = queues[b][l][: rounds * Hq]
            col = fill[:, :, l].reshape(-1).clone()
            col[: len(q)] = torch.tensor(q, dtype=torch.int64)
            out[:, b, :, l] = col.reshape(rounds, Hq)
    return out
