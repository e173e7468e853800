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
