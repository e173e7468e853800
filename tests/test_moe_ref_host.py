"""The float64 MoE reference (tests/moe_ref.py), its bounds and its exact probes, on the CPU.

An fp32 emulation of tl_moe_topk's softmax (per-lane sums and the butterfly) stays within the probs bound; the
selection rule agrees with oracle.moe.route_ref on planted ties and NaN rows; the combine restatement equals a plain
fp32 loop; the grouped probes are exact; and every bound rejects a planted one-ulp error away from a rounding midpoint."""

import importlib.util
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import moe as omoe


def _load_moe_ref():
    """The helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    name = "tiny_llm_b200_moe_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("moe_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


mr = _load_moe_ref()
wr = mr.wr
BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
ALL = pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])


def emulate_softmax(logits):
    """tl_moe_topk's fp32 arithmetic: lane l sums its entries l + 32 i in order, a 5-level xor butterfly adds the lanes,
    then one division per entry and the rounding to T."""
    x = logits.to(F32).numpy()
    T_, E = x.shape
    m = np.max(x, axis=1, keepdims=True)
    e = np.exp((x - m).astype(np.float32)).astype(np.float32)
    lanes = np.zeros((T_, 32), dtype=np.float32)
    for i in range(8):
        for lane in range(32):
            c = lane + 32 * i
            if c < E:
                lanes[:, lane] = (lanes[:, lane] + e[:, c]).astype(np.float32)
    for o in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ o]).astype(np.float32)
    p = (e / lanes[:, :1]).astype(np.float32)
    return torch.from_numpy(p).to(logits.dtype)


@ALL
@pytest.mark.parametrize("E", [3, 32, 129, 256])
def test_softmax_bound_holds_for_the_fp32_emulation(dtype, E):
    g = torch.Generator().manual_seed(E)
    logits = (torch.randn(64, E, generator=g) * torch.tensor([0.5, 4.0, 30.0, 100.0]).repeat(16)[:, None]).to(dtype)
    logits[0] = 0.25  # a uniform row
    logits[1, :] = -math.inf
    logits[1, E // 2] = 1.0  # one finite logit: p = 1 exactly, the rest 0
    got = emulate_softmax(logits)
    sm = mr.softmax_ref(logits)
    mr.probs_within(got, sm, f"emulated {dtype} E={E}")
    assert float(got[1, E // 2]) == 1.0


def test_softmax_marks_the_nan_rows():
    x = torch.zeros(4, 5)
    x[0, 2] = math.nan
    x[1, 3] = math.inf
    x[2] = -math.inf
    x[3, 1] = -math.inf  # an ordinary row: that entry's probability is 0
    sm = mr.softmax_ref(x)
    assert sm.nan.tolist() == [True, True, True, False]
    assert bool(torch.isnan(sm.lo[:3]).all()) and float(sm.out[3, 1]) == 0.0
    mr.probs_within(torch.softmax(x.double(), -1).float(), sm, "float64 softmax")


@pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])
def test_softmax_bound_rejects_one_ulp_away_from_a_midpoint(dtype):
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(32, 64, generator=g).to(dtype)
    sm = mr.softmax_ref(logits)
    got = sm.out.clone()
    mr.probs_within(got, sm, "reference")
    if dtype == F32:  # fp32 probs carry several ulps of the exp and sum chain: one ulp past the bound's edge
        r, c = 3, 7
        got[r, c] = sm.hi[r, c] + wr.spacing(sm.hi[r, c], dtype)
    else:
        clear = (sm.lo == sm.hi) & (sm.out > 0)
        assert int(clear.sum()) > 1000
        r, c = [int(v) for v in clear.nonzero()[7]]
        got[r, c] += wr.spacing(got[r, c], dtype)
    with pytest.raises(AssertionError, match="outside the bound"):
        mr.probs_within(got, sm, "one ulp up")


@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])
def test_selection_rule_matches_route_ref_on_ties_and_nan_rows(dtype, norm):
    E, k = 16, 4
    rows = [
        torch.full((E,), 0.5),                                    # all equal: ids 0..k-1
        torch.tensor([1.0, 3.0, 3.0, 0.0, 3.0] + [-2.0] * 11),    # ties at the top
        torch.tensor([4.0, 2.0, 2.0, 2.0, 2.0, 2.0] + [0.0] * 10),  # a tie straddling the k-th place
        torch.tensor([0.0] * 15 + [30.0]),                        # fp16 underflow: tied zeros after the first
        torch.full((E,), math.nan),                               # NaN rows
        torch.tensor([1.0, math.inf] + [0.0] * 14),
        torch.full((E,), -math.inf),
    ]
    logits = torch.stack(rows).to(dtype)
    probs, rids, rscores = omoe.route_ref(logits, k, norm)
    ids, scores = mr.select_ref(probs, k, norm)
    assert torch.equal(ids, rids)
    assert bool(mr.same_or_both_nan(scores, rscores).all())
    assert ids[0].tolist() == [0, 1, 2, 3] and ids[1].tolist()[:3] == [1, 2, 4] and ids[2].tolist() == [0, 1, 2, 3]
    assert ids[4].tolist() == [0, 1, 2, 3] and bool(torch.isnan(scores[4:]).all())


def test_selection_ranks_a_nan_below_every_number():
    p = torch.tensor([[math.nan, 0.0, 0.25, math.nan, 0.0]])
    ids, scores = mr.select_ref(p, 5, False)
    assert ids.tolist() == [[2, 1, 4, 0, 3]]


@ALL
@pytest.mark.parametrize("residual", [False, True])
def test_combine_restatement_equals_a_plain_fp32_loop(dtype, residual):
    g = torch.Generator().manual_seed(5)
    T_, k, H = 9, 8, 40
    y = (torch.randn(T_ * k, H, generator=g) * 3).to(dtype)
    s = torch.randn(T_, k, generator=g).to(dtype)
    s[0, 0], s[1, 1] = 0.0, -0.0
    s[2, 2] = torch.finfo(dtype).tiny / 4 if dtype != BF16 else 2.0**-130  # subnormal score
    res = torch.randn(T_, H, generator=g).to(dtype) if residual else None
    got = mr.combine_ref(y, s, res)
    want = np.zeros((T_, H), dtype=np.float32)
    yy = y.float().numpy().reshape(T_, k, H)
    ss = s.float().numpy()
    for t in range(T_):
        for i in range(H):
            acc = np.float32(0.0)
            for j in range(k):
                prod = np.float32(yy[t, j, i]) * np.float32(ss[t, j])  # numpy rounds the fp32 product once
                acc = np.float32(acc + np.float32(torch.tensor(float(prod), dtype=F32).to(dtype).float()))
            want[t, i] = acc
    r = torch.from_numpy(want).to(dtype)
    if residual:
        r = (res.float() + r.float()).to(dtype)
    mr.assert_exact(got, r.double(), "combine restatement")


def test_combine_restatement_catches_a_reversed_slot_sum():
    g = torch.Generator().manual_seed(6)
    T_, k, H = 16, 8, 256
    y = torch.randn(T_ * k, H, generator=g).to(BF16)
    s = torch.rand(T_, k, generator=g).to(BF16)
    mr.plant_cancellation(y, s, [3, 9])
    want = mr.combine_ref(y, s)
    assert float(want[3].abs().max()) == 0.0
    rev = mr.combine_ref(y.view(T_, k, H).flip(1).reshape(T_ * k, H), s.flip(1))
    with pytest.raises(AssertionError, match="differ"):
        mr.assert_exact(rev, want, "reversed")


def test_group_ref_clamps_and_tiles():
    ids = torch.tensor([3, -1, 3, 8, 2**31 - 1, 0, 3], dtype=torch.int32)
    offsets, perm, tiles = mr.group_ref(ids, 8, 2)
    assert offsets.tolist() == [0, 2, 2, 2, 5, 5, 5, 5, 7]
    assert perm.tolist() == [1, 5, 0, 2, 6, 3, 4]
    assert tiles.tolist() == [4, 0, 0, 3, 2, 3, 4, 7, 5]
    assert mr.tile_bound(7, 8, 2) >= 3


@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("epilogue", [mr.EPI_NONE, mr.EPI_SWIGLU_PAIRS], ids=["none", "pairs"])
def test_grouped_probes_are_exact(dtype, epilogue):
    g = torch.Generator().manual_seed(8)
    E, K, N, T_ = 4, 32, 384, 24
    words, scales, biases, a = mr.grouped_probes(T_, N, E, K, dtype, g, wr.probe_positions(N, full=False), epilogue)
    offsets = torch.tensor([0, 6, 6, 20, 24])
    for wgmma in (False, True):
        ref = mr.grouped_reference(words, scales, biases, a, offsets, epilogue, wgmma, probe=True)
        # any fp32 order of an exact sum: a plain per-expert float32 product, rounded once
        for e in range(E):
            lo, hi = int(offsets[e]), int(offsets[e + 1])
            W = wr.Weights.build(words[e], scales[e], biases[e], rounded=wgmma)
            acc = (a[lo:hi].float() @ W.w.float().T).double()
            if epilogue == mr.EPI_SWIGLU_PAIRS:
                gi, ui = wr.pairs_index(K // 2, acc.device)
                gate, up = wr.round_to(acc[:, gi], dtype), wr.round_to(acc[:, ui], dtype)
                acc = (gate.float() / (1 + torch.exp(-gate.float())) * up.float()).double()
            mr.assert_exact(wr.round_to(acc, dtype), ref.out[lo:hi], f"expert {e}")
        assert bool(((ref.out - ref.pre).abs() <= ref.tol).all())


@pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
def test_grouped_bound_rejects_one_ulp_and_a_swapped_gate_up(dtype):
    g = torch.Generator().manual_seed(9)
    E, K, N, T_ = 3, 32, 256, 12
    words = torch.randint(-(2**31), 2**31, (E, K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
    sigma = 1.0 / (4.717 * N**0.5)
    scales = (torch.randn(E, K, N // 128, generator=g) * sigma).to(dtype)
    biases = (-7.5 * scales.float() + torch.randn(E, K, N // 128, generator=g) * sigma).to(dtype)
    a = torch.randn(T_, N, generator=g).to(dtype)
    offsets = torch.tensor([0, 5, 5, 12])
    ref = mr.grouped_reference(words, scales, biases, a, offsets, mr.EPI_NONE, True)
    clear = wr.spread(ref.pre, ref.tol - wr.spacing(ref.pre.abs() + ref.tol, dtype) / 2, dtype) == 0
    r, c = [int(v) for v in clear.nonzero()[3]]
    got = ref.out.clone()
    wr.assert_within(got, ref.pre, ref.tol, "reference")
    got[r, c] += wr.spacing(got[r, c], dtype)
    with pytest.raises(AssertionError, match="outside the error bound"):
        wr.assert_within(got, ref.pre, ref.tol, "one ulp")
    # the pairs epilogue with gate and up read from each other's rows
    pairs = mr.grouped_reference(words, scales, biases, a, offsets, mr.EPI_SWIGLU_PAIRS, True)
    gi, ui = wr.pairs_index(K // 2, a.device)
    perm = torch.arange(K)
    perm[gi], perm[ui] = ui, gi
    swapped = mr.grouped_reference(words[:, perm], scales[:, perm], biases[:, perm], a, offsets, mr.EPI_SWIGLU_PAIRS, True)
    with pytest.raises(AssertionError, match="outside the error bound"):
        wr.assert_within(swapped.out, pairs.pre, pairs.tol, "gate/up swapped")


@pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])
def test_gather_norm_bound_rejects_one_ulp(dtype):
    g = torch.Generator().manual_seed(10)
    x = torch.randn(6, 513, generator=g).to(dtype)
    w = (1 + 0.1 * torch.randn(513, generator=g)).to(dtype)
    perm = torch.tensor([5, 0, 3, 3, 1, 2, 4, 0, 2, 1, 5, 4], dtype=torch.int32)
    rows, b = mr.gather_ref(x, perm, 2, w, 1e-6)
    assert torch.equal(rows, x.double()[perm.long() // 2])
    mr.assert_within(b.out, b.pre, b.tol, "reference")
    got = b.out.clone()
    if dtype == F32:  # fp32 outputs carry a few ulps of the sum-of-squares chain: one ulp past the bound's edge
        r, c = 4, 100
        edge = wr.round_to(b.pre[r, c] - b.tol[r, c], dtype)
        got[r, c] = edge - wr.spacing(edge, dtype)
    else:
        clear = (wr.spread(b.pre, b.tol - wr.spacing(b.pre.abs() + b.tol, dtype) / 2, dtype) == 0).nonzero()
        r, c = [int(v) for v in clear[11]]
        got[r, c] -= wr.spacing(got[r, c], dtype)
    with pytest.raises(AssertionError, match="outside the error bound"):
        mr.assert_within(got, b.pre, b.tol, "one ulp")
