"""Every attention kernel against a float64 reference with an error bound (tests/attention_ref.py).

Needle queries make every key matter at O(1): a visible needle must come back as its value row, an invisible one
must leave the output at the reference over the other keys.  Needles sit where kernels go wrong: the first and last
keys, the first invisible key, each causal row's boundary, both sides of page and 64-key tile boundaries, a sweep
every 37 keys (which crosses every split boundary), and keys behind block-table ids that are -1 or >= num_pages.
Score-magnitude cases (uniform, typical, x8, 200-nat needles, steep increasing and decreasing ramps) exercise the
running maximum, the lazy rescale of the wgmma kernel and the split merges.  Each case states the kernel it must
reach (checked through tl_paged_attention_route) and whether it splits (the merge is a second launch)."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


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

pytestmark = pytest.mark.gpu
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
ROUTES = {ext.PAGED_ROWWISE: "rowwise", ext.PAGED_GQA: "gqa", ext.PAGED_FLASH: "flash", ext.PAGED_WGMMA: "wgmma"}
OUT_ALIGNED = 256  # paged_attention allocates its output: always 16-byte aligned
MAX_ROUNDS = 32


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def case(name, dtype, D, page, Hq, Hkv, L, lens, route, launches, max_pages=None, causal=True, holes=(), q_offset=False, reaches=()):
    return dict(name=name, dtype=dtype, D=D, page=page, Hq=Hq, Hkv=Hkv, L=L, lens=lens, route=route, launches=launches,
                max_pages=max_pages, causal=causal, holes=holes, q_offset=q_offset, reaches=reaches)


# Split counts follow from the block table's width and the grid (launch_paged_gqa, launch_paged_prefill_tc); the
# cases that must split are far from the decision boundaries on a 114- or 132-SM H100.
CASES = [
    case("rowwise-f32", F32, 64, 16, 4, 2, 3, [70, 5], "rowwise", 1, holes=[(0, 1, "neg")], reaches=["rowwise f32"]),
    case("rowwise-f32-prefill", F32, 128, 8, 2, 1, 12, [40], "rowwise", 1),
    case("rowwise-f32-full", F32, 128, 8, 2, 1, 5, [40, 17], "rowwise", 1, causal=False),
    case("rowwise-bf16-d64", BF16, 64, 16, 8, 2, 2, [300, 1], "rowwise", 1, reaches=["rowwise bf16 D!=128"]),
    case("rowwise-bf16-unaligned-q", BF16, 128, 64, 8, 2, 2, [200, 64], "rowwise", 1, q_offset=True, reaches=["rowwise bf16 unaligned q"]),
    case("gqa-decode-causal4", BF16, 128, 16, 8, 2, 4, [100, 128], "gqa", 1, max_pages=8, reaches=["gqa"]),
    case("gqa-split", BF16, 128, 32, 32, 8, 1, [4097, 1000], "gqa", 2, holes=[(0, 3, "neg"), (1, 5, "big")], reaches=["gqa merge"]),
    case("gqa-split-full", BF16, 128, 32, 8, 2, 3, [1500, 1000], "gqa", 2, causal=False),
    case("gqa-split-cap", BF16, 128, 16, 32, 8, 1, [8000], "gqa", 2, max_pages=512, reaches=["gqa merge at PAGED_MAX_SPLITS"]),
    case("gqa-split-causal4", BF16, 128, 16, 8, 2, 4, [2000, 700], "gqa", 2),
    case("gqa-mixed", BF16, 128, 16, 8, 2, 1, [0, 1, 63, 64, 65, 2000], "gqa", 2),
    case("gqa-15-pages", BF16, 128, 64, 8, 2, 1, [900, 30], "gqa", 2, max_pages=15, reaches=["decode 15 pages of 64: gqa"]),
    case("gqa-gl256", BF16, 128, 64, 32, 1, 8, [1000], "gqa", 2, max_pages=16, reaches=["decode G*L=256: gqa"]),
    case("flash-p16", BF16, 128, 16, 8, 2, 70, [70, 200], "flash", 1, holes=[(1, 2, "neg")], reaches=["flash page 16"]),
    case("flash-p32", BF16, 128, 32, 4, 1, 100, [40, 100], "flash", 1, reaches=["flash page 32"]),
    case("flash-g3", BF16, 128, 64, 6, 2, 40, [300, 45], "flash", 1, holes=[(0, 1, "big")], reaches=["flash G=3"]),
    case("wgmma-prefill-g8", BF16, 128, 64, 16, 2, 130, [130, 400], "wgmma", 1, holes=[(1, 2, "big")], reaches=["wgmma prefill"]),
    case("wgmma-prefill-g4", BF16, 128, 128, 32, 8, 256, [1000], "wgmma", 1),
    case("wgmma-prefill-full", BF16, 128, 64, 8, 8, 70, [70, 300], "wgmma", 1, causal=False),
    case("wgmma-16-pages", BF16, 128, 64, 8, 2, 1, [900, 30], "wgmma", 2, max_pages=16, reaches=["decode 16 pages of 64: wgmma"]),
    case("wgmma-split", BF16, 128, 64, 32, 8, 1, [5000, 70], "wgmma", 2, holes=[(0, 10, "neg")], reaches=["wgmma merge"]),
    case("wgmma-gl128", BF16, 128, 64, 32, 2, 8, [1000], "wgmma", 2, max_pages=16, reaches=["decode G*L=128: wgmma"]),
    case("wgmma-decode-causal4", BF16, 128, 128, 16, 4, 4, [3000], "wgmma", 2),
    case("wgmma-mixed", BF16, 128, 64, 8, 2, 1, [0, 1, 63, 64, 65, 3000], "wgmma", 2),
    # contexts longer than the block table: the causal shift uses the whole context, the table clamps afterwards
    case("rowwise-past-table", F32, 64, 16, 4, 2, 4, [70, 20], "rowwise", 1, max_pages=4),
    case("gqa-past-table", BF16, 128, 16, 8, 2, 4, [131, 50], "gqa", 1, max_pages=8),
    case("gqa-split-past-table", BF16, 128, 16, 8, 2, 4, [1030, 300], "gqa", 2, max_pages=64),
    case("flash-past-table", BF16, 128, 32, 4, 1, 20, [70], "flash", 1, max_pages=2),
    case("wgmma-past-table", BF16, 128, 64, 8, 2, 20, [140], "wgmma", 1, max_pages=2),
    case("wgmma-split-past-table", BF16, 128, 64, 16, 4, 4, [1030, 500], "wgmma", 2, max_pages=16),
]
BY_NAME = {c["name"]: c for c in CASES}


def inputs(c, g, dev, logical_keys=None):
    kp, vp, bt, cl, storage = ar.paged_inputs(g, c["lens"], c["page"], c["Hkv"], c["D"], c["dtype"], max_pages=c["max_pages"], holes=c["holes"],
                                              logical_keys=logical_keys)
    return kp.to(dev), vp.to(dev), bt.to(dev), cl.to(dev), storage


def call_paged(c, q, kp, vp, bt, cl, scale):
    """paged_attention with the case's q placement; asserts the kernel it reached and its launch count."""
    if c["q_offset"]:  # 2 bytes past a 16-byte boundary, still contiguous
        buf = torch.empty(q.numel() + 1, dtype=q.dtype, device=q.device)
        buf[1:].copy_(q.reshape(-1))
        q = buf[1:].view(q.shape)
    rows, L, D = q.shape
    route = ext.paged_attention_route(q, kp, vp, OUT_ALIGNED, rows, L, D, kp.shape[0], kp.shape[2], bt.shape[1], c["Hkv"], c["Hq"], q.dtype)
    torch.cuda.synchronize()
    before = ext.launch_count()
    out = ext.paged_attention(q, kp, vp, bt, cl, scale, is_causal=c["causal"], num_kv_heads=c["Hkv"], num_heads=c["Hq"])
    torch.cuda.synchronize()
    launches = ext.launch_count() - before
    assert (ROUTES[route], launches) == (c["route"], c["launches"]), f"{c['name']}: reached {ROUTES[route]} with {launches} launches"
    return out


def bound(c, ref, A, smax, nvis):
    return ar.error_bound(ref, A, smax, nvis, c["D"], c["dtype"], p_rounded=c["route"] in ("flash", "wgmma"))


def probes(c):
    cap = (c["max_pages"] or max(1, max((n + c["page"] - 1) // c["page"] for n in c["lens"]))) * c["page"]
    per_row, shared = zip(*(ar.probe_positions(n, c["L"], c["causal"], c["page"], cap) for n in c["lens"]))
    shared = [list(s) for s in shared]
    for b, lp, _ in c["holes"]:
        shared[b] += [lp * c["page"], lp * c["page"] + c["page"] // 2, lp * c["page"] + c["page"] - 1]
    return per_row, shared


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_needles_see_exactly_the_visible_keys(dev, c):
    g = torch.Generator().manual_seed(len(c["name"]) * 1009 + sum(c["lens"]))
    kp, vp, bt, cl, storage = inputs(c, g, dev)
    scale = c["D"] ** -0.5
    per_row, shared = probes(c)
    targets = ar.assign_targets(per_row, shared, c["Hq"], c["L"], MAX_ROUNDS, g)
    for r, t in enumerate(targets):
        q = ar.needle_queries(kp, storage, t, c["Hq"], c["Hkv"], scale, 48.0, c["dtype"])
        got = call_paged(c, q, kp, vp, bt, cl, scale)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, scale, c["causal"], c["Hkv"], c["Hq"])
        tol = bound(c, ref, A, smax, nvis)
        vis = ar.needle_visible(bt, kp.shape[0], c["page"], t, nvis)
        what = f"{c['name']} round {r}"
        ar.check_needles(got, ref, A, tol, ar.needle_values(vp, storage, t, c["Hq"], c["Hkv"]), vis, c["dtype"], what)
        ar.assert_within(got, ref, tol, what)


SCORE_CASES = ["rowwise-f32", "rowwise-bf16-d64", "gqa-decode-causal4", "gqa-split", "gqa-mixed", "gqa-gl256", "flash-p16", "flash-g3",
               "wgmma-prefill-g8", "wgmma-split", "wgmma-mixed", "wgmma-decode-causal4", "gqa-split-past-table", "wgmma-past-table"]
SLOPE = 0.1  # nats per key: 6.4 per 64-key tile, above the wgmma kernel's 2^8 lazy-rescale threshold (5.5 nats)


@pytest.mark.parametrize("mode", ["uniform", "typical", "x8", "needle200", "ramp_up", "ramp_down"])
@pytest.mark.parametrize("name", SCORE_CASES)
def test_score_magnitudes(dev, name, mode):
    c = BY_NAME[name]
    g = torch.Generator().manual_seed(len(name) * 31 + len(mode))
    B, Hq, Hkv, L, D, page = len(c["lens"]), c["Hq"], c["Hkv"], c["L"], c["D"], c["page"]
    width = c["max_pages"] or max(1, max((n + page - 1) // page for n in c["lens"]))
    cap = width * page
    scale = D**-0.5
    logical = None
    q = torch.randn(B * Hq, L, D, generator=g)
    if mode == "uniform":
        logical = torch.zeros(B, Hkv, cap, D)
    elif mode == "x8":
        q = q * 8
    elif mode.startswith("ramp"):
        # scores scale * q . k_j = +-SLOPE * j (+ ~0.5 nat of noise): every tile and every split raises the running
        # maximum (ramp_up), or every split after the first lies far below the global maximum (ramp_down)
        u = torch.randn(Hkv, D, generator=g).to(c["dtype"]).double()
        a = (SLOPE if mode == "ramp_up" else -SLOPE) * torch.arange(cap, dtype=torch.float64)
        coef = a[None, :] / (scale * (u * u).sum(-1, keepdim=True))
        logical = (u[:, None, :] * coef[..., None])[None].expand(B, Hkv, cap, D) + 0.5 * torch.randn(B, Hkv, cap, D, generator=g, dtype=torch.float64)
        q = u.repeat_interleave(Hq // Hkv, dim=0)[None, :, None, :].expand(B, Hq, L, D).reshape(B * Hq, L, D)
    kp, vp, bt, cl, storage = inputs(c, g, dev, logical)
    if mode == "needle200":
        nv = ar.visible_keys(cl, L, c["causal"], cap)  # [B, L]
        t = (torch.rand(B, Hq, L, generator=g) * nv[:, None, :].clamp(min=1)).long()
        q = ar.needle_queries(kp, storage, t, Hq, Hkv, scale, 200.0, c["dtype"])
    q = q.to(c["dtype"]).to(dev)
    got = call_paged(c, q, kp, vp, bt, cl, scale)
    ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, scale, c["causal"], Hkv, Hq)
    ar.assert_within(got, ref, bound(c, ref, A, smax, nvis), f"{name} {mode}")


# ------------------------------------------------------------- token-major form --
def test_token_major_needles(dev):
    c = BY_NAME["wgmma-prefill-g8"]
    g = torch.Generator().manual_seed(77)
    kp, vp, bt, cl, storage = inputs(c, g, dev)
    B, Hq, Hkv, L, D = len(c["lens"]), c["Hq"], c["Hkv"], c["L"], c["D"]
    scale = D**-0.5
    per_row, shared = probes(c)
    for r, t in enumerate(ar.assign_targets(per_row, shared, Hq, L, MAX_ROUNDS, g)):
        q = ar.needle_queries(kp, storage, t, Hq, Hkv, scale, 48.0, BF16)
        # the token-major entry point takes only the wgmma kernel (otherwise the shim falls back to paged_attention)
        assert ext.paged_attention_route(q, kp, vp, OUT_ALIGNED, B * Hq, L, D, kp.shape[0], c["page"], bt.shape[1], Hkv, Hq, BF16) == ext.PAGED_WGMMA
        torch.cuda.synchronize()
        before = ext.launch_count()
        out = ext.paged_attention_token_major(q, kp, vp, bt, cl, scale, True, Hkv, Hq)
        torch.cuda.synchronize()
        assert ext.launch_count() - before == 1
        got = out.view(B, L, Hq, D).permute(0, 2, 1, 3).reshape(B * Hq, L, D)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, scale, True, Hkv, Hq)
        tol = ar.error_bound(ref, A, smax, nvis, D, BF16, p_rounded=True)
        vis = ar.needle_visible(bt, kp.shape[0], c["page"], t, nvis)
        ar.check_needles(got, ref, A, tol, ar.needle_values(vp, storage, t, Hq, Hkv), vis, BF16, f"token-major round {r}")


# -------------------------------------------------------------- fused decode kernel --
FUSED_CASES = [
    # (Hq, Hkv, page, contexts, max_context, launches): the split count follows from max_context and B * Hkv
    (8, 8, 64, [300, 129], 400, 1),
    (32, 8, 16, [3000, 70], 4096, 2),
    (8, 8, 128, [1500], 2048, 2),
]


@pytest.mark.parametrize("Hq,Hkv,page,contexts,max_context,launches", FUSED_CASES, ids=["one-split", "g4-splits", "splits"])
def test_fused_decode_needles(dev, Hq, Hkv, page, contexts, max_context, launches):
    """decode_attention_fused normalises and rotates q itself.  Its needles are built backwards: the target key is
    rotated back to the row's RoPE position in float64, and a constant q_norm weight scales the normalised row so the
    score is ~48 nats (the stored keys have rms 8, so q's score against itself - the appended key - stays ~3 nats).
    The k part of qkv repeats the q row and k_norm = q_norm: the kernel then appends, bit for bit, the q it used, and
    the reference reads it back from the cache."""
    g = torch.Generator().manual_seed(sum(contexts) + Hq)
    B, D, G, nats, eps, base = len(contexts), 128, Hq // Hkv, 48.0, 1e-6, 1e6
    max_pages = (max_context + page - 1) // page
    kp, vp, bt, cl, storage = ar.paged_inputs(g, contexts, page, Hkv, D, BF16, max_pages=max_pages, key_rms=8.0)
    kp, vp, bt, cl = kp.to(dev), vp.to(dev), bt.to(dev), cl.to(dev)
    scale = D**-0.5
    offsets = (cl - 1).to(torch.int32)
    freq = ext.rope_inv_freq_table(D, base, dev)
    w = torch.full((D,), nats / (scale * D * 8.0)).to(BF16).to(dev)
    cap = max_pages * page
    shared = [[p for p in ar.probe_positions(n, 1, True, page, cap)[1] if p != n - 1] for n in contexts]
    rounds = ar.assign_targets([[[]] for _ in contexts], shared, Hkv, 1, MAX_ROUNDS, g)  # [rounds, B, Hkv, 1]
    for r, tk in enumerate(rounds):
        tk = torch.where(tk == (cl.cpu() - 1)[:, None, None], torch.zeros_like(tk), tk)  # never the appended slot
        t = tk.repeat_interleave(G, dim=1)  # every query head of a KV group gets the group's needle
        k = ar.needle_values(kp, storage, tk, Hkv, Hkv)  # [B*Hkv, 1, D] target keys
        ang = offsets.double()[:, None, None] * freq[None, None, :]  # [B, 1, 64]
        cs, sn = torch.cos(ang), torch.sin(ang)
        kr = k.view(B, Hkv, D)
        re, im = kr[..., :64], kr[..., 64:]
        q_raw = torch.cat([re * cs + im * sn, im * cs - re * sn], dim=-1).to(BF16)  # RoPE^-1 at the row's position
        v_new = torch.randn(B, Hkv, D, generator=g).to(BF16).to(dev)
        qkv = torch.cat([q_raw.repeat_interleave(G, dim=1), q_raw, v_new], dim=1).reshape(B, (Hq + 2 * Hkv) * D).contiguous()
        torch.cuda.synchronize()
        before = ext.launch_count()
        got = ext.decode_attention_fused(qkv, w, w, offsets, bt, cl, freq, kp, vp, Hq, Hkv, eps, scale, max_context)
        torch.cuda.synchronize()
        assert ext.launch_count() - before == launches
        cur = (cl - 1).long()
        pid = bt.long().gather(1, (cur // page)[:, None])[:, 0]
        q_used = kp[pid, :, cur % page]  # [B, Hkv, D]: the appended key is the q the kernel used
        q = q_used.repeat_interleave(G, dim=1).reshape(B * Hq, 1, D)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, scale, True, Hkv, Hq)
        tol = ar.error_bound(ref, A, smax, nvis, D, BF16, p_rounded=False)
        vis = ar.needle_visible(bt, kp.shape[0], page, t, nvis)
        what = f"fused {Hq}/{Hkv} round {r}"
        ar.check_needles(got.view(B * Hq, 1, D), ref, A, tol, ar.needle_values(vp, storage, t, Hq, Hkv), vis, BF16, what)
        ar.assert_within(got.view(B * Hq, 1, D), ref, tol, what)


# ------------------------------------------------------------ dense decode_attention --
@pytest.mark.parametrize("dtype,D", [(F32, 80), (F16, 64), (BF16, 128), (BF16, 256)], ids=["f32-80", "f16-64", "bf16-128", "bf16-256"])
@pytest.mark.parametrize("mode", ["mask", "causal-mask", "x8-mask", "needles"])
def test_dense_decode_attention(dev, dtype, D, mode):
    """tl_decode_attention with masks holding -inf and large finite values (every row keeps a finite entry: an
    all-masked row divides 0 by 0), and causal needles at each row's last key and first hidden key."""
    g = torch.Generator().manual_seed(D + len(mode))
    B, Hq, Hkv, L, S = 2, 4, 2, 3, 300
    scale = D**-0.5
    k = torch.randn(B * Hkv, S, D, generator=g).to(dtype)
    v = torch.randn(B * Hkv, S, D, generator=g).to(dtype)
    q = torch.randn(B * Hq, L, D, generator=g) * (8 if mode.startswith("x8") else 1)
    causal, has_mask = mode != "mask", mode != "needles"
    mask = torch.zeros(B * Hq, L, S)
    if has_mask:
        r = torch.rand(B * Hq, L, S, generator=g)
        mask = torch.where(r < 0.3, float("-inf"), mask)
        mask = torch.where((r >= 0.3) & (r < 0.4), -1e4, mask)
        mask = torch.where((r >= 0.4) & (r < 0.45), 20.0, mask)
        mask = torch.where((r >= 0.45) & (r < 0.5), -60.0, mask)
        mask[..., 0] = 0.0
    vis = None
    if mode == "needles":
        lim = S - L + torch.arange(L)  # last key row l sees
        t = (lim[None, :] + (torch.arange(B * Hq) % 2)[:, None]).clamp(max=S - 1)  # odd rows: the first hidden key
        t[:, 0] = torch.where(torch.arange(B * Hq) % 4 == 3, 0, t[:, 0])
        kvrow = (torch.arange(B * Hq) // Hq) * Hkv + (torch.arange(B * Hq) % Hq) // (Hq // Hkv)
        kt = k.double()[kvrow[:, None], t]  # [B*Hq, L, D]
        q = kt * (48.0 / (scale * (kt * kt).sum(-1, keepdim=True)))
        vis = t <= lim[None, :]
        vneedle = v.double()[kvrow[:, None], t].to(dev)
    q = q.to(dtype)
    qd, kd, vd, md = q.to(dev), k.to(dev), v.to(dev), mask.to(dev)
    before = ext.launch_count()
    got = ext.decode_attention(qd, kd, vd, md if has_mask else torch.zeros(1, device=dev), scale, causal, has_mask, Hq, Hkv)
    torch.cuda.synchronize()
    assert ext.launch_count() - before == 1
    ref, A, smax, nvis = ar.dense_reference(qd, kd, vd, md, scale, causal, has_mask, Hq, Hkv)
    tol = ar.error_bound(ref, A, smax, nvis, D, dtype, p_rounded=False)
    if vis is not None:
        ar.check_needles(got, ref, A, tol, vneedle, vis.to(dev), dtype, f"dense {mode}")
    ar.assert_within(got, ref, tol, f"dense {dtype} D={D} {mode}")


# ---------------------------------------------------------------- kernel coverage --
REQUIRED = {
    "rowwise f32", "rowwise bf16 D!=128", "rowwise bf16 unaligned q", "gqa", "gqa merge", "gqa merge at PAGED_MAX_SPLITS",
    "flash page 16", "flash page 32", "flash G=3", "wgmma prefill", "wgmma merge", "decode 15 pages of 64: gqa",
    "decode 16 pages of 64: wgmma", "decode G*L=128: wgmma", "decode G*L=256: gqa",
}


def test_the_cases_reach_every_attention_kernel(dev, capsys):
    """Each case above asserts the kernel it reaches and whether it splits; this checks that together they reach every
    kernel of tl_paged_attention and every routing boundary, and that the routes the cases claim are the routes
    tl_paged_attention_route reports for their shapes.  The token-major form and the fused decode kernel (one split,
    several) have tests of their own above."""
    reached = {}
    for c in CASES:
        width = c["max_pages"] or max(1, max((n + c["page"] - 1) // c["page"] for n in c["lens"]))
        q = 0x10002 if c["q_offset"] else 0x10000
        r = ext.paged_attention_route(q, 0x20000, 0x30000, OUT_ALIGNED, len(c["lens"]) * c["Hq"], c["L"], c["D"], 1000, c["page"], width,
                                      c["Hkv"], c["Hq"], c["dtype"])
        assert ROUTES[r] == c["route"], c["name"]
        for label in c["reaches"]:
            reached.setdefault(label, c["name"])
    with capsys.disabled():
        print("\nattention kernel coverage:")
        for label in sorted(reached):
            print(f"  {label:34s} <- {reached[label]}")
    assert REQUIRED <= set(reached), sorted(REQUIRED - set(reached))
    assert [c[-1] for c in FUSED_CASES].count(1) >= 1 and [c[-1] for c in FUSED_CASES].count(2) >= 1
