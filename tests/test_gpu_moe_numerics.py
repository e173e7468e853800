"""Every Qwen3-MoE kernel against the float64 reference of tests/moe_ref.py.

  * tl_moe_topk: probs within the softmax bound (fp32, fp16, bf16; E from 1 to 256, off multiples of 32), ids and scores
    exact against the probs the kernel returned, and against oracle.moe.route_ref wherever the bound leaves no
    rounding open; planted ties, fp16 underflow, -inf logits and NaN rows;
  * tl_moe_group: offsets, perm and the tile table exact, the tile count within tl_moe_tile_table_size;
  * tl_moe_gather and tl_moe_combine: copies and slot sums bit for bit, their RMSNorm bit for bit tl_rms_norm's and
    within rms_norm_ref, on each (threads per row, vector or scalar) layout;
  * the grouped W4A16 GEMM: exact probes bit for bit and random inputs within error_bound on the wgmma route at every
    tile width and on the control route, both epilogues, rows scattered or sorted; a row's bits independent of the
    other rows;
  * route_topk, grouped_expert_linear and the Moe block, launch by launch.
Each case asserts the route or layout it exists for and records what it reached; the last test checks that together
they reached every entry of REQUIRED (run the module as a whole)."""

import importlib.util
import math
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import moe as omoe
from tiny_llm_b200 import Moe, QuantizedWeights, grouped_expert_linear, route_topk
from tiny_llm_b200.quantize import as_packed_i32, quantized_linear
from tiny_llm_b200.synthetic import quantize_w4


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
pytestmark = pytest.mark.gpu
BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
ALL = pytest.mark.parametrize("dtype", [F32, F16, BF16], ids=["f32", "f16", "bf16"])
HALF = pytest.mark.parametrize("dtype", [BF16, F16], ids=["bf16", "f16"])
EPS = 1e-6
REACHED = {}  # label -> first case that reached it


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def reach(label, who):
    REACHED.setdefault(label, who)


def name(dtype):
    return str(dtype).split(".")[-1]


def misplace(t, offset):
    """t's values in a buffer ``offset`` elements past a 16-byte boundary (a contiguous view)."""
    if offset == 0:
        return t.contiguous()
    buf = torch.empty(t.numel() + offset, dtype=t.dtype, device=t.device)
    buf[offset:].copy_(t.reshape(-1))
    return buf[offset:].view(t.shape)


def bits_equal(a, b):
    view = {2: torch.int16, 4: torch.int32}[a.element_size()]
    return torch.equal(a.contiguous().view(view), b.contiguous().view(view))


# ------------------------------------------------------------------------------------------------------ top-k --
def planted_rows(E, dtype, big):
    """Rows where selection goes wrong: all equal, ties across the k-th place, fp16 underflow (one 0 logit, the rest -30:
    in fp16 fewer than k probabilities are non-zero), -inf logits, and the NaN rows (a NaN logit, a +inf logit, every
    logit -inf); with ``big`` also ties at every slot (equal pairs)."""
    i = torch.arange(E, dtype=F32)
    rows = {"equal": torch.full((E,), 0.75)}
    straddle = torch.full((E,), -4.0)
    straddle[i.long() % 3 == 1] = 1.5
    straddle[E - 1] = 3.0
    rows["straddle"] = straddle
    under = torch.full((E,), -30.0)
    under[E // 2] = 0.0
    rows["underflow"] = under
    neg = torch.randn(E, generator=torch.Generator().manual_seed(E))
    neg[i.long() % 2 == 0] = -math.inf
    neg[E - 1] = 0.5
    rows["-inf"] = neg
    if big:
        rows["pairs"] = -(i // 2) * 0.25
    nan = torch.zeros(E)
    nan[E // 3] = math.nan
    rows["nan logit"] = nan
    pinf = torch.zeros(E)
    pinf[E - 1] = math.inf
    rows["+inf logit"] = pinf
    rows["all -inf"] = torch.full((E,), -math.inf)
    return list(rows), torch.stack(list(rows.values())).to(dtype)


def topk_logits(T_, E, dtype, g):
    """T rows: random logits at scales 0.5 to 30 (fp32 also 300), planted rows first (all of them at T = 4096, the
    seven but 'pairs' at T = 7)."""
    scale = torch.tensor([0.5, 2.0, 8.0, 30.0] + ([300.0] if dtype == F32 else []))
    x = torch.randn(T_, E, generator=g) * scale[torch.arange(T_) % len(scale)][:, None]
    x = x.to(dtype)
    labels = []
    if T_ >= 7:
        labels, rows = planted_rows(E, dtype, big=T_ > 7)
        x[: len(labels)] = rows
    return x, labels


def check_topk(dev, logits, labels, k, norm, sm, wide, what):
    probs, ids, scores = ext.moe_topk(logits, k, norm)
    open_ = mr.probs_within(probs.cpu(), sm, what)
    E = logits.shape[1]
    ids64 = ids.cpu().to(torch.int64)
    want_ids, want_scores = mr.select_ref(probs, k, norm)
    assert torch.equal(ids64, want_ids), f"{what}: ids are not the top-k of the returned probs"
    assert bool(mr.same_or_both_nan(scores.cpu(), want_scores).all()), f"{what}: scores"
    srt = ids64.sort(-1).values
    assert bool(((srt >= 0) & (srt < E)).all()) and bool((srt[:, 1:] != srt[:, :-1]).all()), f"{what}: k distinct experts"
    # the oracle's routing, wherever the bound (widened to a sequential sum over E) leaves no rounding open
    rp, rids, rs = omoe.route_ref(logits.cpu(), k, norm)
    clear = (wide.lo == wide.hi).all(-1) | wide.nan
    assert torch.equal(probs.cpu()[clear].to(F64).nan_to_num(7.0), rp[clear].to(F64).nan_to_num(7.0)), f"{what}: probs != route_ref"
    assert torch.equal(ids64[clear], rids[clear]), f"{what}: ids != route_ref"
    if not norm:
        assert bool(mr.same_or_both_nan(scores.cpu()[clear], rs[clear]).all()), f"{what}: scores != route_ref"
    for r, label in enumerate(labels):
        if label in ("equal", "nan logit", "+inf logit", "all -inf"):
            assert ids64[r].tolist() == list(range(k)), f"{what}: {label} row"
        if label in ("nan logit", "+inf logit", "all -inf"):
            assert bool(torch.isnan(scores[r].float()).all()), f"{what}: {label} row scores"
    if norm and k == 1:
        live = ~sm.nan
        assert bool((scores.cpu()[live].to(F64) == 1.0).all()), f"{what}: normalised k = 1 must score exactly 1"
        reach("topk normalised k=1", what)
    return probs, open_


TOPK_E = [1, 2, 3, 31, 32, 33, 60, 100, 128, 129, 255, 256]


def test_topk_nan_rows_name_k_distinct_experts(dev):
    """A row whose softmax is NaN gives ids 0..k-1 and NaN scores (route_ref's answer), not 0x7fffffff."""
    for dtype in (BF16, F16, F32):
        labels, rows = planted_rows(16, dtype, big=False)
        nan_rows = [i for i, lb in enumerate(labels) if lb in ("nan logit", "+inf logit", "all -inf")]
        x = rows[nan_rows].to(dev)
        for norm in (False, True):
            probs, ids, scores = ext.moe_topk(x, 4, norm)
            assert ids.cpu().tolist() == [[0, 1, 2, 3]] * len(nan_rows), f"{dtype} norm={norm}"
            assert bool(torch.isnan(scores.float()).all()) and bool(torch.isnan(probs.float()).all())
    reach("topk NaN rows", "nan rows")


@ALL
@pytest.mark.parametrize("E", TOPK_E)
def test_topk_against_the_float64_softmax(dev, dtype, E):
    g = torch.Generator().manual_seed(E * 7 + len(str(dtype)))
    ks = sorted({min(k, E) for k in (1, 2, 8)} | ({E} if E <= 8 else set()))
    for T_ in (1, 7, 4096):
        logits, labels = topk_logits(T_, E, dtype, g)
        ld = logits.to(dev)
        sm = mr.softmax_ref(ld)
        sm = mr.Softmax(*(t.cpu() for t in (sm.out, sm.pre, sm.tol, sm.lo, sm.hi, sm.nan)))
        wide = mr.softmax_ref(logits, chain=E + mr.SUM_CHAIN)
        first = None
        for k in ks:
            for norm in (False, True):
                what = f"topk {name(dtype)} E={E} T={T_} k={k} norm={norm}"
                probs, open_ = check_topk(dev, ld, labels, k, norm, sm, wide, what)
                if first is None:
                    first = probs
                assert bits_equal(probs, first), f"{what}: probs depend on k or norm"
        if T_ == 4096:
            reach(f"topk {name(dtype)}", f"E={E}")
            if labels and dtype == F16:
                r = labels.index("underflow")
                assert int((first[r] != 0).sum()) < min(8, E) or E < 8
                reach("topk fp16 underflow", f"E={E}")
    reach(f"topk E={E}", name(dtype))
    if E % 32:
        reach("topk E off a multiple of 32", f"E={E}")
    if E <= 8:
        reach("topk k=E", f"E={E}")


# ------------------------------------------------------------------------------------------------------ group --
def counts_to_ids(counts, g):
    ids = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    return ids[torch.randperm(ids.numel(), generator=g)].to(torch.int32)


def cycle_counts(R, E, pattern, first=0, last=None):
    """Counts following ``pattern`` over experts first..last, cut so that they sum to R (what is left goes to the
    first expert of the range)."""
    last = E - 1 if last is None else last
    counts, total, i = [0] * E, 0, 0
    span = list(range(first, last + 1))
    while total < R and span:
        e = span[i % len(span)]
        c = min(pattern[i % len(pattern)], R - total)
        counts[e] += c
        total += c
        i += 1
        if i > 100 * E and total < R:
            counts[span[0]] += R - total
            total = R
    return counts


def group_ids(dist, R, E, nt, g):
    n = max(nt, 16)
    if dist == "uniform":
        return torch.randint(0, E, (R,), generator=g, dtype=torch.int32)
    if dist == "single":
        return torch.full((R,), int(torch.randint(0, E, (1,), generator=g)), dtype=torch.int32)
    if dist == "tight":  # every expert 1 mod nt where R allows: the tile count at its bound
        if R <= E:
            return torch.randperm(E, generator=g)[:R].to(torch.int32)
        counts = [1] * E
        rest = R - E
        e = 0
        while rest >= n:
            counts[e % E] += n
            rest -= n
            e += 1
        counts[0] += rest
        return counts_to_ids(counts, g)
    if dist == "segments":
        return counts_to_ids(cycle_counts(R, E, [n - 1, n, n + 1]), g)
    if dist == "empty_ends":
        return torch.randint(1, E - 1, (R,), generator=g, dtype=torch.int32) if E >= 3 else torch.randint(0, E, (R,), generator=g, dtype=torch.int32)
    raise ValueError(dist)


def check_group(dev, ids, E, nt, what):
    offsets, perm, tiles = ext.moe_group(ids.to(dev), E, nt)
    wo, wp, wt = mr.group_ref(ids.to(dev), E, nt)
    assert torch.equal(offsets.to(torch.int64), wo), f"{what}: offsets"
    assert torch.equal(perm.to(torch.int64), wp), f"{what}: perm"
    if nt > 0:
        R = ids.numel()
        assert tiles.numel() == ext._lib.tl_moe_tile_table_size(R, E, nt)
        count = int(wt[0])
        assert count <= (tiles.numel() - 1) // 2 == mr.tile_bound(R, E, nt), f"{what}: {count} tiles"
        assert torch.equal(tiles[: wt.numel()].to(torch.int64), wt), f"{what}: tile table"
        return count
    assert tiles is None
    return None


@pytest.mark.parametrize("nt", [0, 16, 32, 64, 128])
@pytest.mark.parametrize("E", [1, 8, 128, 256])
def test_group_equals_a_stable_argsort(dev, nt, E):
    g = torch.Generator().manual_seed(nt * 1000 + E)
    for R in (0, 1, 31, 33, 1025, 2**20):
        for dist in ("uniform", "single", "tight", "segments", "empty_ends"):
            count = check_group(dev, group_ids(dist, R, E, nt, g), E, nt, f"group nt={nt} E={E} R={R} {dist}")
            if dist == "tight" and nt > 0 and (R <= E or (R - E) % nt == 0):
                assert count == mr.tile_bound(R, E, nt), f"nt={nt} E={E} R={R}: {count} tiles"
                reach("group tile count at its bound", f"nt={nt} E={E} R={R}")
    if nt > 0:  # R = E (nt + 1): every expert holds 1 mod nt rows
        R = E * (nt + 1)
        count = check_group(dev, counts_to_ids([nt + 1] * E, g), E, nt, f"group nt={nt} E={E} 1 mod nt")
        assert count == mr.tile_bound(R, E, nt) == 2 * E
    # ids outside [0, E) are clamped, as the header says: -1 to expert 0, E and 2^31 - 1 to expert E - 1
    ids = torch.randint(0, E, (1025,), generator=g, dtype=torch.int32)
    ids[::7], ids[3::11], ids[5::13] = -1, E, 2**31 - 1
    check_group(dev, ids, E, nt, f"group nt={nt} E={E} clamped ids")
    reach(f"group nt={nt}", f"E={E}")
    reach(f"group E={E}", f"nt={nt}")


# ----------------------------------------------------------------------------------------------------- gather --
@ALL
@pytest.mark.parametrize("H", [128, 256, 512, 513, 768, 2048, 4096, 6144])
def test_gather(dev, dtype, H):
    g = torch.Generator().manual_seed(H + len(str(dtype)))
    src = 37
    x0 = (torch.randn(src, H, generator=g) * 2).to(dtype).to(dev)
    w = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(dev)
    epv = 16 // x0.element_size()
    for rps in (1, 2, 8):
        R = src * rps
        perm = torch.randperm(R, generator=g).to(torch.int32).to(dev)
        for offset in (0, 1):
            x = misplace(x0, offset)
            what = f"gather {name(dtype)} H={H} rps={rps} offset={offset}"
            xs = ext.moe_gather(x, perm, rps)
            rows, _ = mr.gather_ref(x, perm, rps)
            assert bits_equal(xs, x[perm.long() // rps]) and torch.equal(xs.to(F64), rows), f"{what}: copy"
            xn = ext.moe_gather(x, perm, rps, w, EPS)
            tpr, vec = ext.rms_norm_route(H, dtype, x, w, xn)
            assert tpr == (32 if H <= 512 else 256) and vec == (offset == 0 and H % epv == 0), f"{what}: layout {tpr} {vec}"
            # tl_rms_norm on rows of the same alignment (a fresh aligned copy of a misaligned x would take the vector path)
            assert bits_equal(xn, ext.rms_norm(x, w, EPS)[perm.long() // rps]), f"{what}: normed != rms_norm"
            _, b = mr.gather_ref(x, perm, rps, w, EPS)
            mr.assert_within(xn, b.pre, b.tol, f"{what}: normed")
            reach(f"gather {name(dtype)} TPR{tpr} {'vec' if vec else 'scalar'}", what)


# ---------------------------------------------------------------------------------------------------- combine --
def subnormal(dtype):
    return {F32: 2.0**-140, F16: 2.0**-20, BF16: 2.0**-130}[dtype]


@ALL
@pytest.mark.parametrize("H", [64, 256, 512, 513, 2048, 4096])
def test_combine(dev, dtype, H):
    g = torch.Generator().manual_seed(H * 3 + len(str(dtype)))
    T_ = 19
    w0 = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(dev)
    epv = 16 // w0.element_size()
    for k in range(1, 9):
        y0 = (torch.randn(T_ * k, H, generator=g) * 2.0 ** torch.randint(-6, 6, (T_ * k, 1), generator=g)).to(dtype)
        s0 = torch.randn(T_, k, generator=g)
        s0[1], s0[2, 0], s0[3, -1] = -s0[1].abs(), 0.0, subnormal(dtype)  # negative, zero and subnormal scores
        s0 = s0.to(dtype)
        if k >= 3:  # rows whose slot order shows after the rounding to T
            mr.plant_cancellation(y0, s0, [0, 7])
        r0 = (torch.randn(T_, H, generator=g) * 4).to(dtype).to(dev)
        y0, s0 = y0.to(dev), s0.to(dev)
        for offset in (0, 1):
            y, s, r, w = (misplace(t, offset) for t in (y0, s0, r0, w0))
            for residual in (False, True):
                res = r if residual else None
                what = f"combine {name(dtype)} H={H} k={k} offset={offset} residual={residual}"
                out = ext.moe_combine(y, s, res)
                want = mr.combine_ref(y, s, res)
                mr.assert_exact(out, want, what)
                if k >= 3:
                    assert bool((out[0].to(F64) == (r[0].to(F64) if residual else 0.0)).all()), f"{what}: slot order"
                out2, normed = ext.moe_combine(y, s, res, w, EPS)
                assert bits_equal(out2, out), f"{what}: out with the norm"
                tpr, vec = ext.rms_norm_route(H, dtype, out2, w, normed)
                assert tpr == (32 if H <= 512 else 256) and vec == (offset == 0 and H % epv == 0), f"{what}: layout"
                assert bits_equal(normed, ext.rms_norm(out2, w, EPS)), f"{what}: normed != rms_norm"
                b = mr.rms_norm_ref(want, w, EPS, dtype)
                mr.assert_within(normed, b.pre, b.tol, f"{what}: normed")
                reach(f"combine {name(dtype)} TPR{tpr} {'vec' if vec else 'scalar'}", what)
    reach(f"combine {name(dtype)} k=1..8", f"H={H}")


def test_combine_refuses_a_norm_wider_than_4096(dev):
    y = torch.zeros(4, 4097, dtype=BF16, device=dev)
    s = torch.ones(2, 2, dtype=BF16, device=dev)
    with pytest.raises(RuntimeError, match="H <= 4096"):
        ext.moe_combine(y, s, None, torch.ones(4097, dtype=BF16, device=dev), EPS)
    assert ext._lib.tl_moe_combine(16, 16, None, 16, 0.0, 16, 16, 2, 2, 4097, 2, None) == -1  # refused before any access
    assert "4096" in ext._lib.tl_last_error().decode()
    ext.moe_combine(y, s)  # without the norm any width runs


# ----------------------------------------------------------------------------------------------- grouped GEMM --
def gcase(name_, T, k, E, N, K, dist, route="wgmma", nt=None, misalign=None, modes=("gauss", "mean", "bias"), pair_probes=True, reaches=()):
    """pair_probes=False: no exact probe with the pairs epilogue (its codes are drawn per weight on the host, seconds
    at 30B-A3B expert shapes; the other cases probe that epilogue at every tile width)."""
    return dict(name=name_, T=T, k=k, E=E, N=N, K=K, dist=dist, route=route, nt=nt, misalign=misalign, modes=modes, pair_probes=pair_probes,
                reaches=reaches)


SEG = lambda n: [0, n - 1, n, n + 1, n - 1, n, n + 1, 0]  # noqa: E731  segments of nt and nt +- 1, empty first and last experts
GCASES = [
    gcase("nt16-uniform", 40, 2, 16, 256, 256, "uniform", nt=16),
    gcase("nt16-one-expert", 200, 1, 64, 256, 128, "one", nt=16, reaches=["grouped many tiles of one expert"]),
    gcase("nt16-segments", 48, 2, 8, 256, 256, SEG(16), nt=16, reaches=["grouped segments nt+-1"]),
    gcase("nt32-uniform", 100, 8, 32, 512, 256, "uniform", nt=32),
    gcase("nt32-segments", 96, 2, 8, 384, 128, SEG(32), nt=32),
    gcase("nt64-segments", 96, 4, 8, 256, 256, SEG(64), nt=64),
    gcase("nt64-empty-ends", 200, 4, 16, 256, 128, "empty_ends", nt=64, reaches=["grouped empty first and last experts"]),
    gcase("nt128-segments", 96, 8, 8, 256, 128, SEG(128), nt=128),
    gcase("nt128-one-expert", 600, 1, 4, 256, 128, "one", nt=128),
    gcase("e256-k8", 64, 8, 256, 256, 256, "uniform", nt=16, reaches=["grouped E=256 k=8"]),
    gcase("30b-gate-up", 64, 8, 128, 2048, 1536, "uniform", nt=16, modes=("gauss", "mean"), pair_probes=False,
          reaches=["grouped 30B-A3B gate|up"]),
    gcase("30b-down", 64, 8, 128, 768, 2048, "uniform", nt=16, modes=("gauss", "bias"), pair_probes=False,
          reaches=["grouped 30B-A3B down"]),
    gcase("wide-4096", 300, 4, 16, 4096, 512, "uniform", nt=128, reaches=["grouped N=4096"]),
    gcase("control-k64", 6, 2, 3, 128, 64, "uniform", route="control", reaches=["grouped control K%128"]),
    gcase("control-k208", 20, 2, 5, 256, 208, "empty_ends", route="control"),
    gcase("control-misaligned-a", 30, 2, 8, 256, 128, "uniform", route="control", misalign="a", reaches=["grouped control misaligned a"]),
    gcase("control-misaligned-b", 30, 2, 8, 256, 128, "uniform", route="control", misalign="b", reaches=["grouped control misaligned b"]),
]
GIDS = [c["name"] for c in GCASES]


def case_ids(c, g):
    T, k, E = c["T"], c["k"], c["E"]
    if c["dist"] == "uniform":
        return torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)]).to(torch.int32)
    if c["dist"] == "one":
        return torch.full((T, k), int(torch.randint(0, E, (1,), generator=g)), dtype=torch.int32)
    if c["dist"] == "empty_ends":
        return torch.stack([1 + torch.randperm(E - 2, generator=g)[:k] for _ in range(T)]).to(torch.int32)
    ids = counts_to_ids(c["dist"], g)
    assert ids.numel() == T * k, c["name"]
    return ids.view(T, k)


def rand_experts(E, K, N, g, dtype, bias_scale=1.0):
    sigma = 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (E, K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
    scales = (torch.randn(E, K, N // 128, generator=g) * sigma).to(dtype)
    biases = ((-7.5 * scales.float() + torch.randn(E, K, N // 128, generator=g) * sigma) * bias_scale).to(dtype)
    return words, scales, biases


def run_grouped(c, words, scales, biases, a_tok, ids, epilogue, dev):
    """Group, gather and both grouped launches (scattered to t k + j and in sorted order) of one case; asserts the
    route.  Returns (scattered out, sorted out, sorted input rows, offsets, perm, tiles, nt)."""
    T, k, E, N, K = c["T"], c["k"], c["E"], c["N"], c["K"]
    b = misplace(words, 1) if c["misalign"] == "b" else words
    route, nt, max_tiles = ext.moe_grouped_matmul_route(T, k, E, N, K, epilogue, a_tok.dtype, a_tok, b)
    offsets, perm, tiles = ext.moe_group(ids.reshape(-1).to(dev), E, nt)
    xs = ext.moe_gather(a_tok, perm, k)
    if c["misalign"] == "a":
        xs = misplace(xs, 1)
    route, nt, max_tiles = ext.moe_grouped_matmul_route(T, k, E, N, K, epilogue, a_tok.dtype, xs, b)
    assert route == (ext.MOE_WGMMA if c["route"] == "wgmma" else ext.MOE_CONTROL), f"{c['name']}: route {route}"
    if c["route"] == "wgmma":
        assert nt == c["nt"] and max_tiles == mr.tile_bound(T * k, E, nt), f"{c['name']}: nt {nt}, max_tiles {max_tiles}"
    out = ext.moe_grouped_matmul(scales, biases, b, xs, offsets, tiles, k, out_index=perm, epilogue=epilogue)
    srt = ext.moe_grouped_matmul(scales, biases, b, xs, offsets, tiles, k, epilogue=epilogue)
    return out, srt, xs, offsets, perm, tiles, nt


def check_grouped(c, dtype, epilogue, out, srt, ref, perm, probe, what):
    scattered = torch.empty_like(ref.out)
    pre, tol = torch.empty_like(ref.pre), torch.empty_like(ref.tol)
    p = perm.long()
    scattered[p], pre[p], tol[p] = ref.out, ref.pre, ref.tol
    if probe:
        mr.assert_exact(srt, ref.out, f"{what} sorted")
        mr.assert_exact(out, scattered, f"{what} scattered")
    else:
        wr.assert_within(srt, ref.pre, ref.tol, f"{what} sorted")
        wr.assert_within(out, pre, tol, f"{what} scattered")


def case_facts(c, offsets, tiles, nt, what):
    R = c["T"] * c["k"]
    if nt > 0:
        count = int(tiles[0])
        last_start = int(tiles[2 * count])
        if last_start + nt > R:
            reach("grouped final tile past R", what)
        if c["dist"] == "one":
            assert count == -(-R // nt) > 1, f"{what}: {count} tiles of one expert"
        if isinstance(c["dist"], list):
            sizes = set((offsets[1:] - offsets[:-1]).tolist())
            assert {nt - 1, nt, nt + 1, 0} <= sizes, f"{what}: segments {sizes}"
    if c["dist"] in ("empty_ends",) or isinstance(c["dist"], list):
        counts = (offsets[1:] - offsets[:-1]).tolist()
        assert counts[0] == 0 and counts[-1] == 0, f"{what}: ends {counts[:2]} {counts[-2:]}"


@pytest.mark.parametrize("c", GCASES, ids=GIDS)
@HALF
@pytest.mark.parametrize("epilogue", [ext.EPI_NONE, ext.EPI_SWIGLU_PAIRS], ids=["none", "pairs"])
def test_grouped_matmul(dev, c, dtype, epilogue):
    T, k, E, N, K = c["T"], c["k"], c["E"], c["N"], c["K"]
    g = torch.Generator().manual_seed(len(c["name"]) * 101 + T + (dtype == F16) + 7 * epilogue)
    ids = case_ids(c, g)
    wgmma = c["route"] == "wgmma"
    label = f"{c['name']} {name(dtype)} {'pairs' if epilogue else 'none'}"
    # exact probes: bit for bit on every path
    if epilogue == ext.EPI_NONE or c["pair_probes"]:
        words, scales, biases, a = mr.grouped_probes(T, N, E, K, dtype, g, wr.probe_positions(N, full=False), epilogue)
        words, scales, biases, a = (t.to(dev) for t in (words, scales, biases, a))
        out, srt, xs, offsets, perm, tiles, nt = run_grouped(c, words, scales, biases, a, ids, epilogue, dev)
        ref = mr.grouped_reference(words, scales, biases, xs, offsets, epilogue, wgmma, probe=True)
        check_grouped(c, dtype, epilogue, out, srt, ref, perm, True, f"{label} probe")
    # random, large-mean and bias-dominated inputs: within error_bound
    for mode in c["modes"]:
        words, scales, biases = (t.to(dev) for t in rand_experts(E, K, N, g, dtype, bias_scale=16.0 if mode == "bias" else 1.0))
        a = (torch.randn(T, N, generator=g) + (8.0 if mode == "mean" else 0.0)).to(dtype).to(dev)
        out, srt, xs, offsets, perm, tiles, nt = run_grouped(c, words, scales, biases, a, ids, epilogue, dev)
        case_facts(c, offsets.cpu(), None if tiles is None else tiles.cpu(), nt, label)
        ref = mr.grouped_reference(words, scales, biases, xs, offsets, epilogue, wgmma)
        check_grouped(c, dtype, epilogue, out, srt, ref, perm, False, f"{label} {mode}")
        del ref
    # a row's bits depend on nothing but the row: the tokens in another order (other neighbours, other places in the
    # tiles), and the first token alone
    order = torch.randperm(T, generator=g)
    out2 = run_grouped(c, words, scales, biases, a[order.to(dev)], ids[order], epilogue, dev)[0]
    rows = (order[:, None] * k + torch.arange(k)).reshape(-1).to(dev)
    assert bits_equal(out2, out[rows]), f"{label}: rows moved with their neighbours"
    alone = dict(c, T=1)
    if wgmma:
        alone["nt"] = ext.moe_grouped_matmul_route(1, k, E, N, K, epilogue, dtype, a, words)[1]
    out1 = run_grouped(alone, words, scales, biases, a[:1], ids[:1], epilogue, dev)[0]
    assert bits_equal(out1, out[:k]), f"{label}: a row alone"
    reach(f"grouped {c['route']} {'NT' + str(nt) if wgmma else ''} {name(dtype)} {'pairs' if epilogue else 'none'}".replace("  ", " "), c["name"])
    for r in c["reaches"]:
        reach(r, label)
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------- entry points and block --
def quantized_experts(w):
    parts = [quantize_w4(w[e]) for e in range(w.shape[0])]
    return QuantizedWeights(scales=torch.stack([p[1] for p in parts]), biases=torch.stack([p[2] for p in parts]), group_size=128, bits=4,
                            weight=torch.stack([as_packed_i32(p[0]) for p in parts]))


def to_dev(q, dev):
    return QuantizedWeights(scales=q.scales.to(dev), biases=q.biases.to(dev), group_size=128, bits=4, weight=as_packed_i32(q.weight).to(dev))


@pytest.mark.parametrize("shape", ["task1", "wgmma"])
def test_grouped_expert_linear_on_the_device(dev, shape):
    """test_moe_host.py's task 1 inputs (64-wide experts: the control route) and a 256-wide form on the wgmma route."""
    g = torch.Generator().manual_seed(1)
    if shape == "task1":
        x = (torch.randn(2, 3, 128, generator=g) * 0.25).to(BF16)
        w = quantized_experts((torch.randn(3, 64, 128, generator=g) * 0.25).to(BF16))
        ids = torch.tensor([[2, 0, 1], [1, 2, 0]], dtype=torch.int32)
    else:
        x = (torch.randn(8, 16, 256, generator=g) * 0.25).to(BF16)
        w = quantized_experts((torch.randn(8, 256, 256, generator=g) * 0.25).to(BF16))
        ids = torch.randint(0, 8, (8, 16), generator=g, dtype=torch.int32)
    wd = to_dev(w, dev)
    out = grouped_expert_linear(x.to(dev), wd, ids.to(dev))
    E, K, N = wd.weight.shape[0], wd.weight.shape[1], wd.weight.shape[2] * 8
    flat = x.reshape(-1, N).to(dev)
    route = ext.moe_grouped_matmul_route(flat.shape[0], 1, E, N, K, ext.EPI_NONE, BF16, flat, wd.weight)[0]
    assert route == (ext.MOE_CONTROL if shape == "task1" else ext.MOE_WGMMA)
    offsets, perm, _ = mr.group_ref(ids.reshape(-1).to(dev), E, 0)
    ref = mr.grouped_reference(wd.weight, wd.scales, wd.biases, flat[perm], offsets, ext.EPI_NONE, route == ext.MOE_WGMMA)
    pre, tol = torch.empty_like(ref.pre), torch.empty_like(ref.tol)
    pre[perm], tol[perm] = ref.pre, ref.tol
    wr.assert_within(out.reshape(-1, K), pre, tol, f"grouped_expert_linear {shape}")
    reach(f"grouped_expert_linear {shape}", shape)


def test_route_topk_on_the_device(dev):
    """test_moe_host.py's task 2 inputs: the router projection, then tl_moe_topk held to the softmax bound and the
    selection rule on the logits that projection returned."""
    g = torch.Generator().manual_seed(2)
    x = (torch.randn(2, 2, 128, generator=g) * 0.25).to(BF16).to(dev)
    words, s, b = quantize_w4((torch.randn(4, 128, generator=g) * 0.25).to(BF16))
    router = QuantizedWeights(scales=s.to(dev), biases=b.to(dev), group_size=128, bits=4, weight=as_packed_i32(words).to(dev))
    logits = quantized_linear(x, router).reshape(-1, 4)
    for norm in (False, True):
        probs, ids, scores = route_topk(x, router, top_k=2, norm_topk_prob=norm)
        assert probs.shape == (2, 2, 4) and ids.shape == (2, 2, 2)
        sm = mr.softmax_ref(logits)
        mr.probs_within(probs.reshape(-1, 4), sm, "route_topk probs")
        want_ids, want_scores = mr.select_ref(probs.reshape(-1, 4), 2, norm)
        assert torch.equal(ids.reshape(-1, 2).cpu().long(), want_ids)
        mr.assert_exact(scores.reshape(-1, 2).cpu(), want_scores, "route_topk scores")
    reach("route_topk", "task 2")


def synthetic_experts(E, K, N, g):
    words, scales, biases = rand_experts(E, K, N, g, BF16)
    return QuantizedWeights(scales=scales, biases=biases, group_size=128, bits=4, weight=words)


@pytest.mark.parametrize("E, I, H, k, T", [(8, 128, 256, 2, 9), (128, 768, 2048, 8, 64)], ids=["tiny-moe-d128", "30b-a3b"])
def test_moe_block_launch_by_launch(dev, E, I, H, k, T):
    """Moe.__call__ equals its launches bit for bit, and each launch, fed the inputs it actually received, is held to
    its own bound: router logits -> top-k (softmax bound, exact selection) -> group (exact) -> gather (exact) ->
    gate|up with the pairs epilogue and down, scattered (error_bound of their route) -> combine (exact)."""
    g = torch.Generator().manual_seed(E + I)
    router = synthetic_experts(1, E, H, g)
    router = QuantizedWeights(scales=router.scales[0].to(dev), biases=router.biases[0].to(dev), group_size=128, bits=4,
                              weight=router.weight[0].to(dev))
    wg, wu, wd = (to_dev(synthetic_experts(E, o, i, g), dev) for o, i in ((I, H), (I, H), (H, I)))
    moe = Moe(router, wg, wu, wd, num_experts_per_tok=k, norm_topk_prob=True)
    h = torch.randn(T, H, generator=g).to(BF16).to(dev)
    out = moe(h)
    logits = quantized_linear(h, router)
    probs, ids, scores = ext.moe_topk(logits, k, True)
    mr.probs_within(probs, mr.softmax_ref(logits), "block top-k")
    want_ids, want_scores = mr.select_ref(probs, k, True)
    assert torch.equal(ids.cpu().long(), want_ids)
    mr.assert_exact(scores.cpu(), want_scores, "block scores")
    gu, dn = moe.w_gate_up, moe.w_down
    routes = [ext.moe_grouped_matmul_route(T, k, E, H, 2 * I, ext.EPI_SWIGLU_PAIRS, BF16, h, gu.weight),
              ext.moe_grouped_matmul_route(T, k, E, I, H, ext.EPI_NONE, BF16, h, dn.weight)]
    nt = max(r[1] for r in routes)
    offsets, perm, tiles = ext.moe_group(ids.reshape(-1).contiguous(), E, nt)
    wo, wp, wt = mr.group_ref(ids.reshape(-1), E, nt)
    assert torch.equal(offsets.long(), wo) and torch.equal(perm.long(), wp)
    xs = ext.moe_gather(h, perm, k)
    assert bits_equal(xs, h[perm.long() // k])
    act = ext.moe_grouped_matmul(gu.scales, gu.biases, gu.weight, xs, offsets, tiles if routes[0][0] == ext.MOE_WGMMA else None, k,
                                 epilogue=ext.EPI_SWIGLU_PAIRS)
    ref = mr.grouped_reference(gu.weight, gu.scales, gu.biases, xs, offsets, ext.EPI_SWIGLU_PAIRS, routes[0][0] == ext.MOE_WGMMA)
    wr.assert_within(act, ref.pre, ref.tol, "block gate|up")
    y = ext.moe_grouped_matmul(dn.scales, dn.biases, as_packed_i32(dn.weight), act, offsets, tiles if routes[1][0] == ext.MOE_WGMMA else None,
                               k, out_index=perm, epilogue=ext.EPI_NONE)
    ref = mr.grouped_reference(as_packed_i32(dn.weight), dn.scales, dn.biases, act, offsets, ext.EPI_NONE, routes[1][0] == ext.MOE_WGMMA)
    pre, tol = torch.empty_like(ref.pre), torch.empty_like(ref.tol)
    pre[perm.long()], tol[perm.long()] = ref.pre, ref.tol
    wr.assert_within(y, pre, tol, "block down")
    r = ext.moe_combine(y, scores)
    mr.assert_exact(r, mr.combine_ref(y, scores), "block combine")
    assert bits_equal(r, out), "Moe.__call__ is not its launches"
    reach(f"Moe block E={E}", f"routes {routes[0][0]} {routes[1][0]}")


# ---------------------------------------------------------------------------------------------------- coverage --
REQUIRED = {
    "topk NaN rows", "topk float32", "topk float16", "topk bfloat16", "topk fp16 underflow", "topk normalised k=1", "topk E off a multiple of 32",
    "topk k=E", *(f"topk E={e}" for e in TOPK_E),
    *(f"group nt={n}" for n in (0, 16, 32, 64, 128)), *(f"group E={e}" for e in (1, 8, 128, 256)), "group tile count at its bound",
    *(f"{op} {d} TPR{t} {v}" for op in ("gather", "combine") for d in ("float32", "float16", "bfloat16") for t in (32, 256)
      for v in ("vec", "scalar")),
    *(f"combine {d} k=1..8" for d in ("float32", "float16", "bfloat16")),
    *(f"grouped wgmma NT{n} {d} {e}" for n in (16, 32, 64, 128) for d in ("float16", "bfloat16") for e in ("none", "pairs")),
    *(f"grouped control {d} {e}" for d in ("float16", "bfloat16") for e in ("none", "pairs")),
    "grouped control K%128", "grouped control misaligned a", "grouped control misaligned b", "grouped many tiles of one expert",
    "grouped segments nt+-1", "grouped empty first and last experts", "grouped E=256 k=8", "grouped final tile past R",
    "grouped 30B-A3B gate|up", "grouped 30B-A3B down", "grouped N=4096",
    "grouped_expert_linear task1", "grouped_expert_linear wgmma", "route_topk", "Moe block E=8", "Moe block E=128",
}


def test_the_cases_reach_every_moe_branch(dev, capsys):
    """Each test above asserts the route or layout of every launch it makes and records the branches it reached; this
    lists them and checks that together they reach every entry of REQUIRED."""
    with capsys.disabled():
        print("\nMoE coverage:")
        for label in sorted(REACHED):
            print(f"  {label:44s} <- {REACHED[label]}")
    assert REQUIRED <= set(REACHED), sorted(REQUIRED - set(REACHED))
