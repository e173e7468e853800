"""The float64 attention reference (tests/attention_ref.py) and its needle check, on the CPU.

A correct kernel is simulated by rounding the reference to bf16; a kernel with an off-by-one by a reference whose
context moved by one key or whose causal rows moved by one.  The check must pass the first and fail every other."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from oracle import ops as oracle


def _load_attention_ref():
    """The helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    name = "tiny_llm_b200_attention_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("attention_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


ar = _load_attention_ref()

BF16 = torch.bfloat16


def needle_case(lens, L, causal, page=16, max_pages=None, holes=(), seed=0, Hq=4, Hkv=2, D=128):
    g = torch.Generator().manual_seed(seed)
    kp, vp, bt, cl, storage = ar.paged_inputs(g, lens, page, Hkv, D, BF16, max_pages=max_pages, holes=holes)
    cap = bt.shape[1] * page
    per_row, shared = zip(*(ar.probe_positions(n, L, causal, page, cap) for n in lens))
    for b, lp, _ in holes:
        shared[b].append(lp * page + page // 2)
    targets = ar.assign_targets(per_row, shared, Hq, L, 64, g)
    return kp, vp, bt, cl, storage, targets


def run_check(kp, vp, bt, cl, storage, targets, L, causal, simulated, Hq=4, Hkv=2):
    scale = kp.shape[-1] ** -0.5
    for t in targets:
        q = ar.needle_queries(kp, storage, t, Hq, Hkv, scale, 48.0, BF16)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, scale, causal, Hkv, Hq)
        got = ar.paged_reference(q, kp, vp, bt, cl, scale, causal, Hkv, Hq, **simulated)[0].to(BF16)
        tol = ar.error_bound(ref, A, smax, nvis, kp.shape[-1], BF16, p_rounded=True)
        vis = ar.needle_visible(bt, kp.shape[0], kp.shape[2], t, nvis)
        ar.check_needles(got, ref, A, tol, ar.needle_values(vp, storage, t, Hq, Hkv), vis, BF16, "needles")


CASES = {
    "decode": dict(lens=[70, 45, 1], L=1, causal=True),
    "causal-4-rows": dict(lens=[70, 45], L=4, causal=True),
    "prefill": dict(lens=[40, 90], L=20, causal=True),
    "full": dict(lens=[70, 33], L=3, causal=False),
    "past-the-table": dict(lens=[86, 45], L=4, causal=True, max_pages=5),
    "holes": dict(lens=[70, 45], L=2, causal=True, holes=[(0, 1, "neg"), (1, 0, "big")]),
}


@pytest.mark.parametrize("name", list(CASES))
def test_needle_check_passes_a_correct_kernel(name):
    c = dict(CASES[name])
    L, causal = c.pop("L"), c.pop("causal")
    run_check(*needle_case(L=L, causal=causal, **c), L, causal, {})


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("shift", [dict(ctx_delta=1), dict(ctx_delta=-1), dict(row_delta=1), dict(row_delta=-1)], ids=["ctx+1", "ctx-1", "row+1", "row-1"])
def test_needle_check_catches_an_off_by_one(name, shift):
    c = dict(CASES[name])
    L, causal = c.pop("L"), c.pop("causal")
    if "row_delta" in shift and not (causal and L > 1):
        pytest.skip("a causal row shift needs a causal call with several rows")
    with pytest.raises(AssertionError, match="needle"):
        run_check(*needle_case(L=L, causal=causal, **c), L, causal, shift)


def test_needle_check_catches_clamping_the_context_before_the_causal_shift():
    """A context longer than the block table: rows of a multi-row causal call keep their alignment to the whole
    context.  Clamping the context to the table first moves every row's limit; the check must see it."""
    run_check(*needle_case(lens=[86, 45], L=4, causal=True, max_pages=5), 4, True, {})
    with pytest.raises(AssertionError, match="needle"):
        run_check(*needle_case(lens=[86, 45], L=4, causal=True, max_pages=5), 4, True, dict(clamp_first=True))


def test_needles_dominate_by_tens_of_nats():
    """At D = 128 and 8K random keys, a 48-nat needle returns its value row to 1e-12."""
    g = torch.Generator().manual_seed(3)
    kp, vp, bt, cl, storage = ar.paged_inputs(g, [8192], 128, 1, 128, BF16)
    t = torch.tensor([[[0, 4095, 8191, 77]]]).permute(0, 2, 1).reshape(1, 4, 1)
    q = ar.needle_queries(kp, storage, t, 4, 1, 128**-0.5, 48.0, BF16)
    ref = ar.paged_reference(q, kp, vp, bt, cl, 128**-0.5, True, 1, 4)[0]
    assert float((ref - ar.needle_values(vp, storage, t, 4, 1)).abs().max()) < 1e-9


def test_reference_agrees_with_the_oracle():
    """Same semantics as oracle.paged_attention wherever the oracle is defined (no id >= num_pages)."""
    g = torch.Generator().manual_seed(5)
    for dtype, L, causal, lens, mp in ((BF16, 1, True, [70, 0, 5], None), (torch.float32, 5, True, [40, 90], 4), (BF16, 12, False, [30, 2], None)):
        kp, vp, bt, cl, storage = ar.paged_inputs(g, lens, 16, 2, 128, dtype, max_pages=mp, holes=[(0, 1, "neg")])
        q = torch.randn(len(lens) * 4, L, 128, generator=g).to(dtype)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, 0.1, causal, 2, 4)
        want = oracle.paged_attention(q, kp, vp, bt, cl, 0.1, causal, 2, 4)
        torch.testing.assert_close(ref.to(dtype).float(), want.float(), rtol=2e-2, atol=1e-2)


def test_dense_reference_agrees_with_the_oracle():
    g = torch.Generator().manual_seed(6)
    q = torch.randn(8, 3, 64, generator=g)
    k = torch.randn(2, 50, 64, generator=g)
    v = torch.randn(2, 50, 64, generator=g)
    mask = torch.randn(8, 3, 50, generator=g)
    for causal, has_mask in ((True, False), (False, True), (True, True)):
        ref = ar.dense_reference(q, k, v, mask, 0.125, causal, has_mask, 4, 1)[0]
        want = oracle.decode_attention(q, k, v, mask, 0.125, causal, has_mask, 4, 1)
        torch.testing.assert_close(ref.float(), want, rtol=1e-5, atol=1e-6)


# ------------------------------------------------------- explicit masks, fp16 P --
def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


embed_ref = _load("tiny_llm_b200_embed_ref", "embed_ref.py")
rerank_ref = _load("tiny_llm_b200_rerank_ref", "rerank_ref.py")
F64 = torch.float64


def _logical(pages, storage, S):
    """[Hkv, S, D] keys (or values) of request 0 in logical order, through its physical pages."""
    page = pages.shape[2]
    return pages[storage[0, torch.arange(S) // page].long(), :, torch.arange(S) % page].permute(1, 0, 2)


def _close(got, want):
    torch.testing.assert_close(got, want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("L,ctx,max_pages,holes", [(1, 70, None, ()), (20, 90, None, [(0, 2, "neg")]), (5, 86, 5, [(0, 1, "big")])],
                         ids=["decode", "prefill-hole", "past-the-table"])
def test_masked_reference_equals_paged_reference_on_causal_layouts(L, ctx, max_pages, holes):
    g = torch.Generator().manual_seed(L + ctx)
    Hq, Hkv, D, page = 4, 2, 64, 16
    kp, vp, bt, cl, storage = ar.paged_inputs(g, [ctx], page, Hkv, D, BF16, max_pages=max_pages, holes=holes)
    S = bt.shape[1] * page
    q = torch.randn(Hq, L, D, generator=g).to(BF16)
    want = ar.paged_reference(q, kp, vp, bt, cl, 0.2, True, Hkv, Hq)
    n = ar.visible_keys(cl, L, True, S)[0]
    vis = (torch.arange(S)[None, :] < n[:, None]) & ar.live_keys(bt, kp.shape[0], page, S)[None, :]
    got = ar.masked_reference(q, _logical(kp, storage, S), _logical(vp, storage, S), vis[None], 0.2, Hkv)
    for a, b in zip(got[:3], want[:3]):
        _close(a, b)
    # nvis counts the keys seen: paged_reference's causal count less those behind dead pages
    assert torch.equal(got[3], vis.sum(dim=-1)[None].expand(Hq, L)) and bool((got[3] <= want[3]).all())
    assert torch.equal(got[4][:, :, 0] > 0, got[3] > 0)  # V1: a sum over the visible keys, nonzero where any is


def _packed(g, Hq, Hkv, L, D):
    return (torch.randn(Hq, L, D, generator=g, dtype=F64), torch.randn(Hkv, L, D, generator=g, dtype=F64),
            torch.randn(Hkv, L, D, generator=g, dtype=F64))


def test_masked_reference_equals_the_segment_reference():
    g = torch.Generator().manual_seed(11)
    L = 40
    seg = torch.tensor([0] * 7 + [7] * 13 + [20] + [21] * 15 + [L] * 4)  # segments of 7, 13, 1 and 15 rows, 4 padding rows
    seg[3] = -2  # a negative start reads as 0
    q, k, v = _packed(g, 6, 2, L, 16)
    vis = ar.segment_visible(seg, torch.ones(L, dtype=torch.bool))
    ref = ar.masked_reference(q, k, v, vis, 0.3, 2)[0]
    want = embed_ref.segment_attention_ref(q.numpy(), k.numpy(), v.numpy(), seg.clamp(min=0).numpy(), 0.3, 2)
    _close(ref.permute(1, 0, 2).reshape(L, -1), torch.from_numpy(want))
    assert torch.all(ref[:, L - 4 :] == 0)


def test_masked_reference_equals_the_prefixed_reference():
    g = torch.Generator().manual_seed(12)
    L = 48
    # a 10-row query prefix, its documents of 14 and 9 rows, a second 6-row prefix and its 5-row document, 4 padding rows
    seg = torch.tensor([0] * 10 + [10] * 14 + [24] * 9 + [33] * 6 + [39] * 5 + [L] * 4)
    ps = torch.tensor([0] * 10 + [0] * 14 + [0] * 9 + [33] * 6 + [33] * 5 + [0] * 4)
    pe = torch.tensor([0] * 10 + [10] * 14 + [10] * 9 + [33] * 6 + [39] * 5 + [10] * 4)
    ps[12], pe[12] = -3, 10  # prefix_start < 0 reads as 0
    pe[30] = 28  # prefix_end past segment_start (24) but not past the row: the clamp to segment_start applies
    q, k, v = _packed(g, 4, 4, L, 16)
    vis = ar.segment_visible(seg, torch.ones(L, dtype=torch.bool), ps, pe)
    ref = ar.masked_reference(q, k, v, vis, 0.25, 4)[0]
    want = rerank_ref.prefixed_attention_ref(q.numpy(), k.numpy(), v.numpy(), seg.numpy(), ps.numpy(), pe.numpy(), 0.25, 4)
    _close(ref.permute(1, 0, 2).reshape(L, -1), torch.from_numpy(want))
    # a prefix range that runs past the row itself stops at the segment start: no later key becomes visible
    pe[26] = 40
    row = ar.segment_visible(seg, torch.ones(L, dtype=torch.bool), ps, pe)[0, 26]
    assert row.nonzero()[:, 0].tolist() == list(range(0, 27))
    assert not bool(ar.segment_visible(seg, torch.ones(L, dtype=torch.bool), ps, pe)[0, L - 4 :].any())  # padding rows see nothing


def test_segment_visible_drops_keys_of_dead_pages():
    bt = torch.tensor([3, -1, 9, 2], dtype=torch.int32)
    live = ar.live_keys(bt, 9, 4, 16)
    assert live.tolist() == [True] * 4 + [False] * 8 + [True] * 4
    vis = ar.segment_visible(torch.zeros(16, dtype=torch.int64), live)[0]
    assert vis[15].nonzero()[:, 0].tolist() == [0, 1, 2, 3, 12, 13, 14, 15]


def _emulate_fp16_kernel(q, k, v, scale):
    """One row of the fp16 wgmma kernel: fp32 scores, 64-key tiles in key order, the kept maximum raised only past 2^8
    (log2 units), P = ex2(s - m) in fp32 rounded to fp16 for P V, fp32 row sum of the unrounded P, O / sum -> fp16."""
    s = (q.float() @ k.float().T) * (scale * 1.44269504089)
    o = torch.zeros(v.shape[1], dtype=torch.float32)
    m, l_sum = float("-inf"), torch.zeros((), dtype=torch.float32)
    for t0 in range(0, s.shape[0], 64):
        st = s[t0 : t0 + 64]
        tm = float(st.max())
        if tm > m + 8 or m == float("-inf"):
            if m != float("-inf"):
                alpha = torch.exp2(torch.tensor(m - tm, dtype=torch.float32))
                o, l_sum = o * alpha, l_sum * alpha
            m = tm
        p = torch.exp2(st - torch.tensor(m, dtype=torch.float32))
        l_sum = l_sum + p.sum()
        o = o + p.half().float() @ v[t0 : t0 + 64].float()
    return (o / l_sum).half()


def test_fp16_probability_floor_needs_the_absolute_term():
    """The worked case of error_bound: 4,000 keys 18 nats below the maximum flush to 0 in fp16 P.  The emulated kernel
    lies within the fp16 bound and outside the bf16-P form of it, by more than 100x."""
    n, D = 4000, 16
    k = torch.zeros(n + 1, D)
    k[1:, 0] = -18.0  # score = q . k with q = e_0 and scale 1
    v = torch.randn(n + 1, D, generator=torch.Generator().manual_seed(4)).half()
    v[0, 3], v[1:, 3] = 0.0, 1.0
    q = torch.zeros(1, D)
    q[0, 0] = 1.0
    ref, A, smax, nvis, V1 = ar.masked_reference(q[:, None].double(), k[None].double(), v[None].double(),
                                                 torch.ones(1, 1, n + 1, dtype=torch.bool), 1.0, 1)
    got = _emulate_fp16_kernel(q[0], k, v, 1.0).double()
    err = (got - ref[0, 0]).abs()
    assert got[3] == 0 and 5e-5 < float(ref[0, 0, 3]) < 7e-5
    new = ar.error_bound(ref, A, smax, nvis, D, torch.float16, True, p_dtype=torch.float16, V1=V1)[0, 0]
    old = ar.error_bound(ref, A, smax, nvis, D, torch.float16, True)[0, 0]
    assert bool((err <= new).all()), (err - new).max()
    assert float(err[3]) > 100 * float(old[3])


def test_error_bound_keeps_its_bf16_values():
    g = torch.Generator().manual_seed(8)
    ref, A = torch.randn(2, 3, 8, generator=g, dtype=F64), torch.rand(2, 3, 8, generator=g, dtype=F64)
    smax, nvis = torch.rand(2, 3, generator=g, dtype=F64) * 30, torch.randint(1, 5000, (2, 3), generator=g)
    for p_rounded, u_p in ((True, 2.0**-8), (False, 0.0)):
        delta = (2 * 128 + 16) * 2.0**-24 * smax + 2.0**-20
        want = (2.0**-8 + 2.0**-23) * ref.abs() + (u_p + torch.expm1(2 * delta) + (nvis / 4 + 64) * 2.0**-23)[..., None] * A
        assert torch.equal(ar.error_bound(ref, A, smax, nvis, 128, BF16, p_rounded), want)
    with pytest.raises(ValueError, match="V1"):
        ar.error_bound(ref, A, smax, nvis, 128, torch.float16, True, p_dtype=torch.float16)
