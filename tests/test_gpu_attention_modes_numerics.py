"""The masking modes of the wgmma flash kernel (attention_prefill_tc.cu) against the float64 bound of
tests/attention_ref.py: segment-causal attention (``tl_paged_attention_segments``, embeddings), prefixed-segment
attention (``tl_paged_attention_prefixed_segments``, reranking), both in bf16 and fp16, and shared-prefix decode
attention (``tl_shared_prefix_attention``, parallel sampling: prefix pass, suffix pass, merge).

Segment modes: the reference is ``masked_reference`` over the mask ``segment_visible`` states, at every head ratio
G = Hq / Hkv the ABI takes (1 to 128, so 128 down to 1 query positions per CTA), pages of 64, 128 and 256 slots,
L up to 8192, and block tables with -1 and out-of-range ids.  Needles (a query that is a 48-nat copy of one key) sit at
each row's segment start and the key before it (the previous segment's last), the row itself and the key after it,
the prefix bounds ps - 1, ps, pe - 1, pe, and the page and tile edges and a 37-key sweep inside each segment.  Score
cases run uniform to 200-nat scores and ramps that rescale every tile, in key order and, for prefixed rows, with the
prefix tiles (walked first) far below or far above the segment.  fp16 is held to the bound with P's absolute floor.

Shared prefix: the reference is ``paged_reference`` on each slot's whole table.  Needles at the last shared key, the
first private key, the shared run's tile edges and a 37-key sweep; a shared key targeted by every row of the launch must
reach exactly the rows of its group.  Each call asserts its launch count; the module ends with a coverage test."""

import importlib.util
import math
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


ar = _load("tiny_llm_b200_attention_ref", "attention_ref.py")

pytestmark = pytest.mark.gpu
BF16, F16 = torch.bfloat16, torch.float16
D, BN = 128, 64  # head dimension, keys per tile
MAX_ROUNDS = 12
SLOPE = 0.1  # nats per key: 6.4 per tile, above the kernel's 2^8 lazy-rescale threshold (5.5 nats)
NATS = 48.0
SCORE_MODES = ["uniform", "typical", "x8", "needle200", "ramp_up", "ramp_down"]


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


# ------------------------------------------------------------------ packed layouts --
def packed(lengths, L):
    """segment_start of consecutive segments from row 0; rows past them are padding (segment_start = L > row)."""
    seg, r = [], 0
    for n in lengths:
        seg += [r] * n
        r += n
    assert r <= L
    return seg + [L] * (L - r), [0] * L, [0] * L


def reranked(queries, L, pad_prefix=(0, 0)):
    """A reranking pass: per query (prefix rows, [document rows, ...]) its prefix is a segment of its own (no prefix
    range), each document a segment whose rows also see the query's prefix rows.  Padding rows get ``pad_prefix``."""
    seg, ps, pe, r = [], [], [], 0
    for plen, docs in queries:
        p0 = r
        seg += [p0] * plen
        ps += [0] * plen
        pe += [0] * plen
        r += plen
        for n in docs:
            seg += [r] * n
            ps += [p0] * n
            pe += [p0 + plen] * n
            r += n
    assert r <= L
    return seg + [L] * (L - r), ps + [pad_prefix[0]] * (L - r), pe + [pad_prefix[1]] * (L - r)


def _random_lengths(seed, total, lo, hi):
    g = torch.Generator().manual_seed(seed)
    out = []
    while sum(out) < total:
        out.append(int(torch.randint(lo, hi + 1, (1,), generator=g)))
    out[-1] -= sum(out) - total
    return [n for n in out if n > 0]


SEG_LAYOUTS = {
    # starts at 63, 64, 65, 127, 128, 129, 256 (page edges of 64 / 128 / 256), one-token segments, tail padding
    "edges": lambda L: packed([63, 1, 1, 62, 1, 1, 127, 2, 60, 5, 1, 190], L),
    # many segments inside single tiles
    "small": lambda L: packed([5, 7, 20, 10, 1, 1, 30, 3, 40, 17, 2, 9, 64, 11, 1, 33, 6], L),
    # segments of 1 to 300 rows crossing query blocks of every height
    "random": lambda L: packed(_random_lengths(L, L - 37, 1, 300), L),
}
PRE_LAYOUTS = {
    # prefix on tile edges [64, 128), an empty prefix, a query whose documents share CTAs with the previous query's
    "tiles": lambda L: reranked([(64, [30, 34]), (64, [50, 14, 64, 7]), (0, [20, 9]), (37, [3, 1, 90, 40])], L),
    # prefix hulls that straddle the first segment tile of a CTA, small documents of two queries in one CTA
    "straddle": lambda L: reranked([(100, [60, 1, 45]), (10, [5, 6]), (23, [7, 7, 7]), (150, [120, 33]), (5, [1, 1, 1])], L,
                                   pad_prefix=(0, 300)),
    "random": lambda L: reranked([(n, _random_lengths(n, 3 * n, 1, 90)) for n in _random_lengths(L, (L - 20) // 4, 5, 80)], L,
                                 pad_prefix=(10, 200)),
}


def _odd_rows(seg, ps, pe):
    """prefix_start < 0 on one document row, prefix_end past segment_start (clamped there) on another."""
    rows = [r for r in range(len(seg)) if ps[r] < pe[r] and seg[r] <= r]
    ps, pe = list(ps), list(pe)
    if rows:
        a, b = rows[len(rows) // 3], rows[2 * len(rows) // 3]
        ps[a] = -7
        pe[b] = seg[b] + 20
    return ps, pe


def case(name, mode, dtype, G, Hkv, page, L, layout, holes=(), reaches=()):
    return dict(name=name, mode=mode, dtype=dtype, G=G, Hkv=Hkv, Hq=G * Hkv, page=page, L=L, layout=layout, holes=holes, reaches=list(reaches))


HKV = {1: 4, 2: 4, 4: 2, 8: 2, 16: 1, 32: 1, 64: 1, 128: 1}
PAGES = [64, 128, 256]
CASES = []
for _dt, _dn in ((BF16, "bf16"), (F16, "f16")):
    for _i, _G in enumerate(HKV):
        _page = PAGES[(_i + (_dt == F16)) % 3]
        _sl = list(SEG_LAYOUTS)[_i % 3]
        CASES.append(case(f"seg-{_dn}-g{_G}-p{_page}-{_sl}", "segment", _dt, _G, HKV[_G], _page, 640, _sl))
        _pl = list(PRE_LAYOUTS)[(_i + 1) % 3]
        _page = PAGES[(_i + 2 * (_dt == F16)) % 3]
        CASES.append(case(f"pre-{_dn}-g{_G}-p{_page}-{_pl}", "prefixed", _dt, _G, HKV[_G], _page, 704, _pl))
CASES += [
    case("seg-bf16-holes", "segment", BF16, 4, 2, 64, 512, "random", holes=[(0, 2, "neg"), (0, 5, "big")], reaches=["table holes"]),
    case("pre-f16-holes", "prefixed", F16, 8, 2, 128, 640, "straddle", holes=[(0, 1, "big"), (0, 3, "neg")], reaches=["table holes"]),
    case("seg-bf16-8192-one", "segment", BF16, 8, 2, 256, 8192, "one", reaches=["L=8192 one segment"]),
    case("seg-f16-8192-many", "segment", F16, 16, 1, 128, 8192, "random", reaches=["L=8192 many segments"]),
    case("pre-bf16-8192-many", "prefixed", BF16, 4, 2, 64, 8192, "random", reaches=["L=8192 many segments"]),
]
BY_NAME = {c["name"]: c for c in CASES}


def layout(c):
    if c["layout"] == "one":
        return packed([c["L"]], c["L"])
    if c["mode"] == "segment":
        return SEG_LAYOUTS[c["layout"]](c["L"])
    seg, ps, pe = PRE_LAYOUTS[c["layout"]](c["L"])
    return (seg, *_odd_rows(seg, ps, pe))


def cta_facts(c, seg, ps, pe):
    """What the kernel's tile walk meets (restated from paged_prefill_tc_kernel, for the coverage labels only)."""
    L, RH = c["L"], BN * 2 // c["G"]
    facts = set()
    for q0 in range(0, L, RH):
        rows = range(q0, min(q0 + RH, L))
        key_end = rows[-1] + 1
        live = [r for r in rows if seg[r] <= r]
        if len({max(seg[r], 0) for r in live}) > 1:
            facts.add("rows of one CTA in different segments")
        if any(seg[r] > r for r in rows) and live:
            facts.add("padding rows beside live rows")
        if c["mode"] != "prefixed":
            continue
        tile_lo = min(min([max(seg[r], 0) for r in rows] + [key_end]) // BN, (key_end + BN - 1) // BN)
        hull = [(max(ps[r], 0), min(pe[r], key_end)) for r in live if max(ps[r], 0) < min(pe[r], key_end)]
        starts = {h[0] for h in hull}
        if len(starts) > 1:
            facts.add("two prefixes in one CTA")
        if hull and min(h[0] for h in hull) // BN < tile_lo < (max(h[1] for h in hull) + BN - 1) // BN:
            facts.add("prefix hull straddles tile_lo")
        if any(ps[r] < 0 for r in live):
            facts.add("prefix_start < 0")
        if any(pe[r] > max(seg[r], 0) and ps[r] < pe[r] for r in live):
            facts.add("prefix_end > segment_start")
        if any(ps[r] < pe[r] and seg[r] > r for r in rows):
            facts.add("padding rows with prefix ranges")
        if any(ps[r] == pe[r] and ps[r] > 0 for r in live):
            facts.add("empty prefix")
        if any(ps[r] < pe[r] and (ps[r] % BN == 0 or pe[r] % BN == 0) and ps[r] > 0 for r in live):
            facts.add("prefix on a tile edge")
    return facts


# ------------------------------------------------------------------ segment harness --
def seg_inputs(c, g, dev, logical_keys=None):
    L, page = c["L"], c["page"]
    max_pages = (L + page - 1) // page + 1  # one spare page: the table is wider than the pass
    kp, vp, bt, _, storage = ar.paged_inputs(g, [L], page, c["Hkv"], D, c["dtype"], max_pages=max_pages, holes=c["holes"],
                                             logical_keys=logical_keys)
    seg, ps, pe = (torch.tensor(x, dtype=torch.int32) for x in layout(c))
    live = ar.live_keys(bt[0], kp.shape[0], page, L)
    vis = ar.segment_visible(seg, live, *((ps, pe) if c["mode"] == "prefixed" else ()))
    idx = torch.arange(L)
    K = kp[storage[0, idx // page].long(), :, idx % page].permute(1, 0, 2).to(dev)  # logical order [Hkv, L, D]
    V = vp[storage[0, idx // page].long(), :, idx % page].permute(1, 0, 2).to(dev)
    return kp.to(dev), vp.to(dev), bt[0].contiguous().to(dev), storage, (seg, ps, pe), vis.to(dev), K, V


def call_segments(c, q, kp, vp, bt, lay, scale):
    seg, ps, pe = (x.to(q.device) for x in lay)
    torch.cuda.synchronize()
    before = ext.launch_count()
    if c["mode"] == "segment":
        out = ext.paged_attention_segments(q, kp, vp, bt, seg, scale, c["Hkv"], c["Hq"])
    else:
        out = ext.paged_attention_prefixed_segments(q, kp, vp, bt, seg, ps, pe, scale, c["Hkv"], c["Hq"])
    torch.cuda.synchronize()
    assert ext.launch_count() - before == 1, c["name"]
    return out.view(c["L"], c["Hq"], D).permute(1, 0, 2)  # [Hq, L, D]


def seg_bound(c, ref, A, smax, nvis, V1):
    return ar.error_bound(ref, A, smax, nvis, D, c["dtype"], True, p_dtype=c["dtype"], V1=V1)


def seg_probes(c, lay):
    """Per row: its own boundaries, then its segment's page / tile edges and sweep dealt over the segment's rows from
    the last one back (the rows that see most of it)."""
    seg, ps, pe = (x.tolist() for x in lay)
    L, page = c["L"], c["page"]
    own = []
    for l in range(L):
        p = [seg[l], seg[l] - 1, l, l + 1]
        if c["mode"] == "prefixed" and ps[l] < pe[l]:
            p += [ps[l], ps[l] - 1, pe[l] - 1, pe[l]]
        own.append([x for x in dict.fromkeys(p) if 0 <= x < L])
    segments = {}
    for l, s in enumerate(seg):
        if s <= l:
            segments.setdefault(s, []).append(l)
    for s0, rows in segments.items():
        s1 = rows[-1] + 1
        edges = [x + d for step in (page, BN) for x in range((s0 // step + 1) * step, s1, step) for d in (-1, 0)]
        edges += list(range(s0, s1, 37))
        for _, lp, _ in c["holes"]:
            edges += [x for x in (lp * page, lp * page + page // 2, lp * page + page - 1) if s0 <= x < s1]
        edges = [x for x in dict.fromkeys(edges) if max(s0, 0) <= x < s1]
        cap = max(48, len(rows))
        if len(edges) > cap:
            edges = [edges[int(j * len(edges) / cap)] for j in range(cap)]
        for j, x in enumerate(edges):
            own[rows[-1 - j % len(rows)]].append(x)
    return own


def seg_targets(c, own, g):
    """[rounds, Hq, L] needle positions; free slots get a random key of the row's segment."""
    Hq, L = c["Hq"], c["L"]
    rounds = max(1, min(MAX_ROUNDS, max(math.ceil(len(p) / Hq) for p in own)))
    out = (torch.rand(rounds, Hq, L, generator=g) * (torch.arange(L) + 1)).long()
    for l, p in enumerate(own):
        p = p[: rounds * Hq]
        col = out[:, :, l].reshape(-1).clone()
        col[: len(p)] = torch.tensor(p, dtype=torch.int64)
        out[:, :, l] = col.reshape(rounds, Hq)
    return out


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_segment_needles_see_exactly_the_visible_keys(dev, c):
    g = torch.Generator().manual_seed(len(c["name"]) * 1013 + c["L"] + c["G"])
    kp, vp, bt, storage, lay, vis, K, V = seg_inputs(c, g, dev)
    scale = D**-0.5
    for r, t in enumerate(seg_targets(c, seg_probes(c, lay), g)):
        q = ar.needle_queries(kp, storage, t[None], c["Hq"], c["Hkv"], scale, NATS, c["dtype"])
        got = call_segments(c, q, kp, vp, bt, lay, scale)
        ref, A, smax, nvis, V1 = ar.masked_reference(q, K, V, vis, scale, c["Hkv"])
        tol = seg_bound(c, ref, A, smax, nvis, V1)
        td = t.to(dev)
        needle_vis = vis[0][torch.arange(c["L"], device=dev)[None, :].expand_as(td), td]
        what = f"{c['name']} round {r}"
        ar.check_needles(got, ref, A, tol, ar.needle_values(vp, storage, t[None], c["Hq"], c["Hkv"]), needle_vis, c["dtype"], what)
        ar.assert_within(got, ref, tol, what)
        del ref, A, smax, nvis, V1, tol
    torch.cuda.empty_cache()


SEG_SCORE_CASES = ["seg-bf16-g1-p64-edges", "seg-f16-g8-p128-edges", "seg-bf16-g32-p256-random", "seg-f16-g128-p256-small",
                   "seg-bf16-holes", "pre-bf16-g1-p64-straddle", "pre-f16-g4-p128-tiles", "pre-bf16-g16-p128-random",
                   "pre-f16-g128-p64-random", "pre-f16-holes"]
PREFIX_MODES = ["prefix_low", "prefix_high"]


def _ramp_keys(c, g, a):
    """Keys whose scores against q = u (one unit direction per KV head) are a[j] + ~0.5 nat of noise."""
    Hkv, cap = c["Hkv"], ((c["L"] + c["page"] - 1) // c["page"] + 1) * c["page"]
    u = torch.randn(Hkv, D, generator=g).to(c["dtype"]).double()
    a = torch.cat([a, torch.zeros(cap - a.shape[0], dtype=torch.float64)])
    coef = a[None, :] / (D**-0.5 * (u * u).sum(-1, keepdim=True))
    keys = (u[:, None, :] * coef[..., None])[None] + 0.5 * torch.randn(1, Hkv, cap, D, generator=g, dtype=torch.float64)
    q = u.repeat_interleave(c["G"], dim=0)[:, None, :].expand(c["Hq"], c["L"], D)
    return keys, q


@pytest.mark.parametrize("mode", SCORE_MODES + PREFIX_MODES)
@pytest.mark.parametrize("name", SEG_SCORE_CASES)
def test_segment_score_magnitudes(dev, name, mode):
    c = BY_NAME[name]
    if mode in PREFIX_MODES and c["mode"] != "prefixed":
        pytest.skip("prefix-tile ramps need prefix ranges")
    g = torch.Generator().manual_seed(len(name) * 37 + len(mode))
    L, Hq, scale = c["L"], c["Hq"], D**-0.5
    q = torch.randn(Hq, L, D, generator=g)
    logical = None
    if mode == "uniform":
        logical = torch.zeros(1, c["Hkv"], ((L + c["page"] - 1) // c["page"] + 1) * c["page"], D)
    elif mode == "x8":
        q = q * 8
    elif mode.startswith("ramp"):
        logical, q = _ramp_keys(c, g, (SLOPE if mode == "ramp_up" else -SLOPE) * torch.arange(L, dtype=torch.float64))
    elif mode in PREFIX_MODES:
        # prefix keys (walked first) 30 nats below every segment key, the segments descending (a rescale on the first
        # segment tile, then none); or 24 nats above, the segments rising through them (rescales late in long passes)
        seg, ps, pe = layout(c)
        pre = torch.zeros(L, dtype=torch.bool)
        for r in range(L):
            if seg[r] <= r and ps[r] < pe[r]:
                pre[max(ps[r], 0) : min(pe[r], max(seg[r], 0))] = True
        j = torch.arange(L, dtype=torch.float64)
        if mode == "prefix_low":
            a = torch.where(pre, -SLOPE * L - 30.0, -SLOPE * j)
        else:
            a = torch.where(pre, torch.full_like(j, 24.0), SLOPE * (j - L / 2))
        logical, q = _ramp_keys(c, g, a)
    kp, vp, bt, storage, lay, vis, K, V = seg_inputs(c, g, dev, logical)
    if mode == "needle200":
        seg = lay[0].clamp(min=0).long()
        t = (seg + torch.rand(Hq, L, generator=g) * (torch.arange(L) - seg + 1).clamp(min=1)).long().clamp(max=L - 1)
        q = ar.needle_queries(kp, storage, t[None], Hq, c["Hkv"], scale, 200.0, c["dtype"])
    q = q.to(c["dtype"]).to(dev).contiguous()
    got = call_segments(c, q, kp, vp, bt, lay, scale)
    ref, A, smax, nvis, V1 = ar.masked_reference(q, K, V, vis, scale, c["Hkv"])
    ar.assert_within(got, ref, seg_bound(c, ref, A, smax, nvis, V1), f"{name} {mode}")


def test_fp16_probability_floor_on_the_gpu(dev):
    """The worked case of error_bound: every row's first key is its maximum with v_d = 0, the 4,000 keys after it lie
    18 nats lower with v_d = 1 and round to 0 as fp16 P.  Within the fp16 bound (2^-25 V1), which the bf16 form of the
    bound is not on the last rows."""
    L, Hkv, G, page = 4096, 1, 8, 128
    c = case("f16-floor", "segment", F16, G, Hkv, page, L, "one")
    g = torch.Generator().manual_seed(9)
    cap = ((L + page - 1) // page + 1) * page
    keys = torch.zeros(1, Hkv, cap, D)
    keys[0, :, 1:L, 0] = -18.0  # score q . k * scale = k_0 with q = 8 e_0 and scale 1/8
    kp, vp, bt, storage, lay, vis, K, V = seg_inputs(c, g, dev, keys)
    vd = 3
    for pid in range(kp.shape[0]):
        vp[pid, :, :, vd] = 1.0
    vp[int(storage[0, 0]), :, 0, vd] = 0.0
    V = vp[storage[0, torch.arange(L) // page].long(), :, torch.arange(L) % page].permute(1, 0, 2)
    q = torch.zeros(G * Hkv, L, D, dtype=F16, device=dev)
    q[..., 0] = 8.0
    got = call_segments(c, q, kp, vp, bt, lay, 0.125)
    ref, A, smax, nvis, V1 = ar.masked_reference(q, K, V, vis, 0.125, Hkv)
    ar.assert_within(got, ref, seg_bound(c, ref, A, smax, nvis, V1), "fp16 floor")
    old = ar.error_bound(ref, A, smax, nvis, D, F16, True)
    assert bool(((got.double() - ref).abs() > old).any()), "the fp16 P floor was not reached: the case has no power"


# ------------------------------------------------------------------ shared prefix --
def shared_layout(g, page, groups, lone, idle, sp, private, max_pages, short=(), holes=()):
    """Block tables and contexts: each group's slots share their first ``sp`` pages (``sp == max_pages``: all of their
    keys), then own up to ``private`` more keys.  ``short``: (group, slot) whose context ends inside the shared run;
    ``holes``: (slot, "neg" | "big"): the middle one of the slot's private pages gets the id -1 / one >= num_pages.  Returns tables, lens,
    descriptors, the number of physical pages and the logical page index of each physical page."""
    B = sum(groups) + lone + idle
    tables = torch.full((B, max_pages), -1, dtype=torch.int32)
    lens = torch.zeros(B, dtype=torch.int32)
    desc, logical, nxt, b = [], [], 0, 0

    def rnd(lo, hi):
        return int(torch.randint(lo, hi + 1, (1,), generator=g))

    for gi, count in enumerate(groups):
        shared = list(range(nxt, nxt + sp))
        logical += list(range(sp))
        nxt += sp
        for s in range(count):
            if (gi, s) in short:
                ctx = rnd(1, sp * page - 1)
            elif sp == max_pages:
                ctx = rnd((sp - 1) * page + 1, sp * page)
            else:
                ctx = sp * page + rnd(1, min(private, (max_pages - sp) * page))
            own = max(-(-ctx // page) - sp, 0)
            tables[b, :sp] = torch.tensor(shared, dtype=torch.int32)
            tables[b, sp : sp + own] = torch.arange(nxt, nxt + own, dtype=torch.int32)
            logical += list(range(sp, sp + own))
            nxt += own
            lens[b] = ctx
            b += 1
        desc.append((b - count, count, sp))
    for _ in range(lone):
        ctx = rnd(1, min(sp * page + private, max_pages * page))
        own = -(-ctx // page)
        tables[b, :own] = torch.arange(nxt, nxt + own, dtype=torch.int32)
        logical += list(range(own))
        nxt += own
        lens[b] = ctx
        b += 1
    P = nxt + 2  # physical pages 0 and P - 1 are where a clamped -1 / out-of-range id would land
    perm = torch.randperm(P - 2, generator=g).to(torch.int32) + 1
    tables = torch.where(tables >= 0, perm[tables.clamp(min=0).long()], tables)
    lp_of = torch.zeros(P, dtype=torch.int64)
    lp_of[perm.long()] = torch.tensor(logical, dtype=torch.int64)
    for slot, kind in holes:
        first = next((d[2] for d in desc if d[0] <= slot < d[0] + d[1]), 0)
        last = -(-int(lens[slot]) // page) - 1
        assert last >= first, "a hole needs a private page"
        tables[slot, (first + last) // 2] = -1 if kind == "neg" else P + 7
    return tables, lens, desc, P, lp_of


def scase(name, G, Hkv, page, groups, lone, idle, sp, private, max_pages, short=(), holes=(), reaches=()):
    return dict(name=name, G=G, Hkv=Hkv, Hq=G * Hkv, page=page, groups=groups, lone=lone, idle=idle, sp=sp, private=private,
                max_pages=max_pages, short=short, holes=holes, reaches=list(reaches))


SHARED_CASES = [
    scase("g1", 1, 8, 64, [8, 3], 1, 1, 3, 70, 5, short=[(1, 2)], holes=[(11, "neg")],
          reaches=["context ends in the shared run", "holes in private pages", "ungrouped and idle slots"]),
    scase("g2-cap", 2, 4, 128, [64], 1, 1, 2, 200, 4, reaches=["count*G = 128"]),
    scase("g4-cap", 4, 2, 64, [32], 2, 1, 4, 130, 8, short=[(0, 0), (0, 31)], holes=[(5, "big"), (33, "neg")],
          reaches=["count*G = 128", "context ends in the shared run", "holes in private pages"]),
    scase("g8-whole-table", 8, 2, 256, [16, 2], 1, 1, 3, 0, 3, short=[(1, 0)], reaches=["shared_pages == max_pages", "count*G = 128"]),
    scase("g16", 16, 1, 64, [8, 2], 1, 1, 2, 64, 5, holes=[(8, "big")], reaches=["count*G = 128"]),
    scase("g4-long", 4, 8, 64, [8], 1, 0, 64, 2000, 100, short=[(0, 3)], holes=[(2, "neg")], reaches=["both passes split"]),
]
SHARED_BY_NAME = {c["name"]: c for c in SHARED_CASES}


def wave_splits(base, max_tiles, max_splits, slots):
    """launch_shared_prefix_attention's split count (tc_wave_splits), restated."""
    best, best_cost = 1, None
    for sp in range(1, min(max_splits, max(max_tiles, 1)) + 1):
        tps = -(-max_tiles // sp)
        if -(-max_tiles // tps) != sp:
            continue
        cost = 4 * (-(-base * sp // slots)) * (tps + 3) + (8 + sp if sp > 1 else 0)
        if best_cost is None or cost < best_cost:
            best, best_cost = sp, cost
    return best


def shared_splits(c, B, dev):
    slots = torch.cuda.get_device_properties(dev).multi_processor_count
    max_tiles = c["max_pages"] * c["page"] // BN
    sp = wave_splits(c["Hkv"], max_tiles, 16, slots)
    return sp, wave_splits(B * c["Hkv"], max_tiles, 32 - sp, slots)


def shared_inputs(c, g, dev, key_fn=None):
    tables, lens, desc, P, lp_of = shared_layout(g, c["page"], c["groups"], c["lone"], c["idle"], c["sp"], c["private"], c["max_pages"],
                                                 c["short"], c["holes"])
    if key_fn is None:
        kp = torch.randn(P, c["Hkv"], c["page"], D, generator=g)
    else:
        kp = key_fn(lp_of)
    vp = torch.randn(P, c["Hkv"], c["page"], D, generator=g)
    return tables, lens, desc, P, lp_of, kp.to(BF16).to(dev), vp.to(BF16).to(dev)


def call_shared(c, q, kp, vp, tables, lens, desc, scale):
    dev = q.device
    B = tables.shape[0]
    groups = torch.tensor(desc or [(0, 0, 0)], dtype=torch.int32).view(-1, 3)
    need = ext.shared_prefix_attention_workspace(B, c["Hq"], c["Hkv"], c["page"], c["max_pages"])
    sp, ss = shared_splits(c, B, dev)
    assert need == B * c["Hq"] * (sp + ss) * (D + 2) * 4, (need, sp, ss)
    torch.cuda.synchronize()
    before = ext.launch_count()
    out = ext.shared_prefix_attention(q, kp, vp, tables.to(dev), lens.to(dev), groups.to(dev), groups.contiguous(), scale, c["Hkv"], c["Hq"])
    torch.cuda.synchronize()
    assert ext.launch_count() - before == 3, c["name"]  # prefix pass, suffix pass, merge
    return out


def shared_probe_rounds(c, tables, lens, desc, P, g):
    """[rounds, B, Hq, 2] physical (page, slot) targets.  Per slot, dealt over its heads: the last shared key, the first
    private key, the shared run's tile edges, its last key, the first key past it, a 37-key sweep and keys behind its
    holes' clamped ids.  Then the broadcast rounds, listed as (group, key position): every row of the launch targets
    one shared key of a group (its last, and for the first group also the first key of the second tile), which exactly
    the group's rows whose context passes it must see."""
    B, Hq, page = tables.shape[0], c["Hq"], c["page"]
    queues = []
    for b in range(B):
        n = int(lens[b])
        grp = next((d for d in desc if d[0] <= b < d[0] + d[1]), None)
        sk = grp[2] * page if grp else 0
        pos = [sk - 1, sk, n - 1, n] if grp else [n - 1, n, 0]
        pos += [x + d for x in range(BN, sk + 1, BN) for d in (-1, 0)][:40] + list(range(0, max(n, 1), 37))[:40]
        cells = []
        for p in dict.fromkeys(pos):
            if 0 <= p < c["max_pages"] * page and int(tables[b, p // page]) >= 0:
                cells.append((int(tables[b, p // page]) % P, p % page))
        if any(h[0] == b for h in c["holes"]):
            cells += [(0, 5), (P - 1, page - 1)]
        queues.append(cells)
    rounds = max(1, min(MAX_ROUNDS, max(math.ceil(len(q) / Hq) for q in queues)))
    out = torch.empty(rounds, B, Hq, 2, dtype=torch.int64)
    out[..., 0] = torch.randint(0, P, (rounds, B, Hq), generator=g)
    out[..., 1] = torch.randint(0, page, (rounds, B, Hq), generator=g)
    for b, cells in enumerate(queues):
        cells = cells[: rounds * Hq]
        flat = out[:, b].reshape(-1, 2).clone()
        if cells:
            flat[: len(cells)] = torch.tensor(cells, dtype=torch.int64)
        out[:, b] = flat.reshape(rounds, Hq, 2)
    broadcast = []
    for i, d in enumerate(x for x in desc if x[1] and x[2]):
        broadcast += [(d, d[2] * page - 1)] + ([(d, BN)] if i == 0 and BN < d[2] * page - 1 else [])
    for d, pos in broadcast:
        extra = torch.empty(1, B, Hq, 2, dtype=torch.int64)
        extra[..., 0], extra[..., 1] = int(tables[d[0], pos // page]), pos % page
        out = torch.cat([out, extra])
    return out, broadcast


def shared_needles(c, kp, vp, tables, lens, cells, scale):
    """q [B * Hq, 1, D] whose row is a 48-nat copy of the physical key cells[b, h]; its value rows; whether the row sees
    it (the key's page sits in the slot's table at a live id, before the slot's context)."""
    B, Hq, G, page = tables.shape[0], c["Hq"], c["G"], c["page"]
    kvh = (torch.arange(Hq) // G)[None, :].expand(B, Hq)
    pid, slot = cells[..., 0], cells[..., 1]
    k = kp[pid.to(kp.device), kvh.to(kp.device), slot.to(kp.device)].double()
    q = (k * (NATS / (scale * (k * k).sum(-1, keepdim=True)))).to(BF16).reshape(B * Hq, 1, D)
    v = vp[pid.to(kp.device), kvh.to(kp.device), slot.to(kp.device)].double().reshape(B * Hq, 1, D)
    vis = torch.zeros(B, Hq, dtype=torch.bool)
    for b in range(B):
        row = tables[b].long()
        for h in range(Hq):
            lp = (row == pid[b, h]).nonzero()
            vis[b, h] = bool(len(lp)) and int(lp[0, 0]) * page + int(slot[b, h]) < int(lens[b]) and 0 <= int(pid[b, h]) < kp.shape[0]
    return q, v, vis.reshape(B * Hq, 1)


@pytest.mark.parametrize("c", SHARED_CASES, ids=[c["name"] for c in SHARED_CASES])
def test_shared_prefix_needles(dev, c):
    g = torch.Generator().manual_seed(len(c["name"]) * 7919 + c["page"])
    tables, lens, desc, P, lp_of, kp, vp = shared_inputs(c, g, dev)
    scale = D**-0.5
    B = tables.shape[0]
    if "both passes split" in c["reaches"]:
        assert min(shared_splits(c, B, dev)) > 1
    cells, broadcast = shared_probe_rounds(c, tables, lens, desc, P, g)
    for r, cell in enumerate(cells):
        q, vneedle, vis = shared_needles(c, kp, vp, tables, lens, cell, scale)
        got = call_shared(c, q, kp, vp, tables, lens, desc, scale)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, tables.to(dev), lens.to(dev), scale, True, c["Hkv"], c["Hq"])
        tol = ar.error_bound(ref, A, smax, nvis, D, BF16, True)
        what = f"{c['name']} round {r}"
        if r >= len(cells) - len(broadcast):  # every row targets one shared key: exactly its group's rows see it
            (f, count, _), pos = broadcast[r - (len(cells) - len(broadcast))]
            want = torch.zeros(B, dtype=torch.bool)
            want[f : f + count] = lens[f : f + count] > pos
            assert torch.equal(vis.view(B, -1).all(dim=1), want) and torch.equal(vis.view(B, -1).any(dim=1), want), what
        ar.check_needles(got, ref, A, tol, vneedle.to(dev), vis.to(dev), BF16, what)
        ar.assert_within(got, ref, tol, what)
    idle = (lens == 0).repeat_interleave(c["Hq"])
    assert torch.equal(got[idle.to(dev)], torch.zeros_like(got[idle.to(dev)]))


SHARED_SCORE_CASES = ["g1", "g4-cap", "g8-whole-table", "g16", "g4-long"]


@pytest.mark.parametrize("mode", SCORE_MODES)
@pytest.mark.parametrize("name", SHARED_SCORE_CASES)
def test_shared_prefix_score_magnitudes(dev, name, mode):
    """ramp_down puts every row's maximum in the shared run (the suffix partials are far below it), ramp_up in the
    private run (the prefix partial is far below): the merge rescales one side by up to e^-200."""
    c = SHARED_BY_NAME[name]
    g = torch.Generator().manual_seed(len(name) * 41 + len(mode))
    Hkv, G, page, scale = c["Hkv"], c["G"], c["page"], D**-0.5
    u = torch.randn(Hkv, D, generator=g).to(BF16).double()

    def ramp(lp_of):
        pos = lp_of[:, None] * page + torch.arange(page)[None, :]  # [P, page] logical positions
        a = (SLOPE if mode == "ramp_up" else -SLOPE) * pos.double()
        coef = a[:, None, :] / (scale * (u * u).sum(-1))[None, :, None]  # [P, Hkv, page]
        return u[None, :, None, :] * coef[..., None] + 0.5 * torch.randn(*coef.shape, D, generator=g, dtype=torch.float64)

    key_fn = {"uniform": lambda lp: torch.zeros(lp.shape[0], Hkv, page, D), "ramp_up": ramp, "ramp_down": ramp}.get(mode)
    tables, lens, desc, P, lp_of, kp, vp = shared_inputs(c, g, dev, key_fn)
    B = tables.shape[0]
    q = torch.randn(B * c["Hq"], 1, D, generator=g)
    if mode == "x8":
        q = q * 8
    elif mode.startswith("ramp"):
        q = u.repeat_interleave(G, dim=0)[None].expand(B, c["Hq"], D).reshape(B * c["Hq"], 1, D)
    q = q.to(BF16).to(dev)
    if mode == "needle200":
        cells = torch.empty(B, c["Hq"], 2, dtype=torch.int64)
        for b in range(B):
            n = max(int(lens[b]), 1)
            p = (torch.rand(c["Hq"], generator=g) * n).long()
            ids = tables[b].long()[p // page]
            cells[b, :, 0] = torch.where((ids >= 0) & (ids < P), ids, torch.zeros_like(ids))  # a hole: some live page's key
            cells[b, :, 1] = p % page
        kq = kp[cells[..., 0].to(dev), (torch.arange(c["Hq"]) // G)[None].expand(B, -1).to(dev), cells[..., 1].to(dev)].double()
        q = (kq * (200.0 / (scale * (kq * kq).sum(-1, keepdim=True)))).to(BF16).reshape(B * c["Hq"], 1, D)
    got = call_shared(c, q, kp, vp, tables, lens, desc, scale)
    ref, A, smax, nvis = ar.paged_reference(q, kp, vp, tables.to(dev), lens.to(dev), scale, True, Hkv, c["Hq"])
    ar.assert_within(got, ref, ar.error_bound(ref, A, smax, nvis, D, BF16, True), f"{name} {mode}")


# ------------------------------------------------------------------ coverage --
REQUIRED = (
    {f"{m} {d} G={G}" for m in ("segment", "prefixed") for d in ("bf16", "f16") for G in HKV}
    | {f"{m} {d} page {p}" for m in ("segment", "prefixed") for d in ("bf16", "f16") for p in PAGES}
    | {f"shared bf16 G={G}" for G in (1, 2, 4, 8, 16)}
    | {"table holes", "L=8192 one segment", "L=8192 many segments", "rows of one CTA in different segments", "padding rows beside live rows",
       "two prefixes in one CTA", "prefix hull straddles tile_lo", "prefix_start < 0", "prefix_end > segment_start",
       "padding rows with prefix ranges", "empty prefix", "prefix on a tile edge", "count*G = 128", "context ends in the shared run",
       "shared_pages == max_pages", "holes in private pages", "ungrouped and idle slots", "both passes split"}
)


def test_the_cases_reach_every_mode_ratio_and_page_size(dev, capsys):
    """Each case above asserts its launch count; this checks that together they reach every mode x dtype x head ratio
    and page size, and the layouts each mode's tile walk and masks treat apart (restated from the kernel's tile walk)."""
    reached = {}
    for c in CASES:
        d = "bf16" if c["dtype"] == BF16 else "f16"
        labels = [f"{c['mode']} {d} G={c['G']}", f"{c['mode']} {d} page {c['page']}"] + c["reaches"]
        labels += sorted(cta_facts(c, *layout(c)))
        for label in labels:
            reached.setdefault(label, c["name"])
    for c in SHARED_CASES:
        assert c["G"] * max(c["groups"]) <= 128
        if c["G"] * max(c["groups"]) == 128:
            assert "count*G = 128" in c["reaches"], c["name"]
        for label in [f"shared bf16 G={c['G']}"] + c["reaches"]:
            reached.setdefault(label, c["name"])
    with capsys.disabled():
        print("\nattention mode coverage:")
        for label in sorted(reached):
            print(f"  {label:40s} <- {reached[label]}")
    assert REQUIRED <= set(reached), sorted(REQUIRED - set(reached))
