"""Qwen3-MoE on the H100: every moe_* kernel against its exact restatement, the Moe block against the oracle, and the
MoE model on the operator path, the decode graph, the prefill graph and the batcher against the reference CPU path."""

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import moe as omoe
from oracle.model import greedy_decode
from tiny_llm_b200 import Moe, QuantizedWeights, Qwen3ModelWeek3
from tiny_llm_b200.synthetic import synthetic_qwen3, to_device

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


# ------------------------------------------------------------------------------------------------------ top-k --
def ambiguous_values(logits: torch.Tensor) -> torch.Tensor:
    """Probabilities the fp32 softmax may round either way: the float64 value lies within 2^-9 of a bf16 ulp (2^-16
    relative, well above the fp32 softmax's error) of a bf16 midpoint."""
    p64 = torch.softmax(logits.to(torch.float64), dim=-1)
    rounded = p64.to(BF).to(torch.float64)
    ulp = torch.ldexp(torch.ones_like(rounded), torch.frexp(rounded).exponent - 8)  # bf16 keeps 8 significant bits
    return (((p64 - rounded) / ulp).abs() - 0.5).abs() < 2.0**-9


@pytest.mark.parametrize("T", [1, 7, 64, 4096])
@pytest.mark.parametrize("E, k", [(8, 1), (8, 2), (64, 8), (128, 8), (256, 2), (256, 8)])
@pytest.mark.parametrize("norm", [False, True])
def test_topk_is_exact(dev, T, E, k, norm):
    g = torch.Generator().manual_seed(T * 1000 + E + k)
    logits = (torch.randn(T, E, generator=g) * 2).to(BF)
    if T >= 7:  # planted ties: equal logits give equal probs, the lower id must win
        logits[1, : E // 2] = logits[1, 0]
        logits[2, :] = 0.5
    probs, ids, scores = ext.moe_topk(logits.to(dev), k, norm)
    rp, rids, rs = omoe.route_ref(logits, k, norm)
    amb = ambiguous_values(logits)
    assert torch.equal(probs.cpu()[~amb], rp[~amb])
    # a row's selection can only move where one of its k + 1 largest probabilities may round either way
    order = torch.sort(-rp.to(torch.float64), dim=-1, stable=True).indices[:, : min(k + 1, E)]
    ok = ~torch.gather(amb, 1, order).any(dim=-1)
    assert torch.equal(ids.cpu().to(torch.int64)[ok], rids[ok])
    assert torch.equal(scores.cpu()[ok], rs[ok])
    if T >= 7:
        assert ids[2].tolist() == list(range(k))
    assert int((~ok).sum()) <= T // 10 + 1


# ------------------------------------------------------------------------------------------------------ group --
def tile_table(counts, nt):
    out, row = [], 0
    for e, c in enumerate(counts):
        for t in range((c + nt - 1) // nt):
            out += [e, row + t * nt]
        row += c
    return [len(out) // 2] + out


@pytest.mark.parametrize("case", ["segments", "one_expert", "random_big", "empty_experts"])
@pytest.mark.parametrize("nt", [16, 128])
def test_group_equals_a_stable_argsort(dev, case, nt):
    E = 16
    if case == "segments":
        sizes = [0, 1, nt - 1, nt, nt + 1, 3, 0, 2 * nt + 5] + [1] * 8
        ids = torch.cat([torch.full((s,), e, dtype=torch.int32) for e, s in enumerate(sizes)])
        ids = ids[torch.randperm(ids.numel(), generator=torch.Generator().manual_seed(0))]
    elif case == "one_expert":
        ids = torch.full((5000,), 7, dtype=torch.int32)
    elif case == "empty_experts":
        ids = torch.tensor([3, 3, 9], dtype=torch.int32)
    else:
        E = 128
        ids = torch.randint(0, E, (32768,), generator=torch.Generator().manual_seed(1), dtype=torch.int32)
    offsets, perm, tiles = ext.moe_group(ids.to(dev), E, nt)
    counts = torch.bincount(ids.to(torch.int64), minlength=E)
    assert offsets.cpu().tolist() == [0] + torch.cumsum(counts, 0).tolist()
    assert torch.equal(perm.cpu().to(torch.int64), torch.sort(ids.to(torch.int64), stable=True).indices)
    want = tile_table(counts.tolist(), nt)
    assert tiles.cpu().tolist()[: len(want)] == want


# --------------------------------------------------------------------------------------------- grouped matmul --
def probe_experts(E, K, N, gen):
    """Power-of-two scales and biases -c * s: every weight (code - c) * s is exact in bf16."""
    words = torch.randint(-(2**31), 2**31, (E, K, N // 8), generator=gen, dtype=torch.int64).to(torch.int32)
    s = 2.0 ** torch.randint(-6, -2, (E, K, N // 128), generator=gen).to(torch.float32)
    c = torch.randint(0, 16, (E, K, N // 128), generator=gen).to(torch.float32)
    return QuantizedWeights(scales=s.to(BF), biases=(-c * s).to(BF), group_size=128, bits=4, weight=words)


def dense_f32(w):
    return omoe.ops.dequantize_fp32(w.weight.reshape(-1, w.weight.shape[-1]), w.scales.reshape(-1, w.scales.shape[-1]),
                                    w.biases.reshape(-1, w.biases.shape[-1])).reshape(*w.weight.shape[:2], -1)


def run_grouped(w, a_tokens, ids, k, epilogue, scatter, dev):
    """a_tokens [T, N], ids [T, k] -> the grouped projection in original (t, j) row order (scatter) or sorted order."""
    E, K, words = w.weight.shape
    T = a_tokens.shape[0]
    route, nt, _ = ext.moe_grouped_matmul_route(T, k, E, words * 8, K, epilogue, BF, a_tokens, w.weight)
    offsets, perm, tiles = ext.moe_group(ids.reshape(-1).to(dev), E, nt)
    xs = ext.moe_gather(a_tokens.to(dev), perm, k)
    out = ext.moe_grouped_matmul(w.scales.to(dev), w.biases.to(dev), w.weight.to(dev), xs, offsets, tiles, k,
                                 out_index=perm if scatter else None, epilogue=epilogue)
    return route, nt, out, perm


def expected_rows(w, a_tokens, ids, k, epilogue):
    wd = dense_f32(w)
    rows = a_tokens.repeat_interleave(k, dim=0).to(torch.float32)
    e = ids.reshape(-1).to(torch.int64)
    acc = torch.einsum("rn,rkn->rk", rows.to(torch.float64), wd[e].to(torch.float64))
    if epilogue == ext.EPI_SWIGLU_PAIRS:
        R, K = acc.shape
        acc = acc.reshape(R, K // 16, 2, 8)
        return omoe.swiglu_once(acc[:, :, 0].to(BF), acc[:, :, 1].to(BF)).reshape(R, K // 2)
    return acc.to(BF)


@pytest.mark.parametrize("T, k, E, N, K, route", [
    (1, 8, 128, 2048, 256, ext.MOE_WGMMA),
    (64, 8, 128, 256, 256, ext.MOE_WGMMA),
    (512, 2, 8, 256, 128, ext.MOE_WGMMA),
    (512, 8, 64, 512, 128, ext.MOE_WGMMA),
    (6, 2, 3, 128, 64, ext.MOE_CONTROL),
])
@pytest.mark.parametrize("epilogue", [ext.EPI_NONE, ext.EPI_SWIGLU_PAIRS])
@pytest.mark.parametrize("scatter", [False, True])
def test_grouped_matmul_exact_probes(dev, T, k, E, N, K, route, epilogue, scatter):
    gen = torch.Generator().manual_seed(T + E + K)
    w = probe_experts(E, K, N, gen)
    # one power-of-two entry per row in each of up to 3 quantisation groups: every product is exact and so is their fp32
    # sum (multiples of 2^-9 below 2^5), which the wgmma kernel accumulates over several 128-wide group blocks
    a = torch.zeros(T, N)
    for grp in range(min(3, N // 128)):
        col = grp * (N // 128 // min(3, N // 128)) * 128 + torch.randint(0, 128, (T,), generator=gen)
        a[torch.arange(T), col] = 2.0 ** torch.randint(-3, 3, (T,), generator=gen).to(torch.float32)
    a = a.to(BF)
    ids = torch.stack([torch.randperm(E, generator=gen)[:k] for _ in range(T)]).to(torch.int32)
    got_route, nt, out, perm = run_grouped(w, a, ids, k, epilogue, scatter, dev)
    assert got_route == route and (nt > 0) == (route == ext.MOE_WGMMA)
    if route == ext.MOE_WGMMA:
        per = -(-T * k // E)
        assert nt == next(n for n in (16, 32, 64, 128) if n >= per or n == 128)
    want = expected_rows(w, a, ids, k, epilogue)
    if not scatter:
        want = want[perm.cpu().to(torch.int64)]
    assert torch.equal(out.cpu(), want)


@pytest.mark.parametrize("T, k, E, N, K", [(4, 8, 128, 2048, 1536), (300, 8, 128, 2048, 768), (33, 2, 8, 256, 256)])
def test_grouped_matmul_random_within_the_tiles_bound(dev, T, k, E, N, K):
    gen = torch.Generator().manual_seed(7)
    w = QuantizedWeights(**{key: v for key, v in vars(synthetic_experts(E, K, N, gen)).items()})
    a = torch.randn(T, N, generator=gen).to(BF)
    ids = torch.stack([torch.randperm(E, generator=gen)[:k] for _ in range(T)]).to(torch.int32)
    route, nt, out, _ = run_grouped(w, a, ids, k, ext.EPI_NONE, True, dev)
    assert route == ext.MOE_WGMMA
    wd = dense_f32(w).to(BF).to(torch.float64)  # the wgmma kernel rounds weights to bf16
    rows = a.repeat_interleave(k, dim=0).to(torch.float64)
    exact = torch.einsum("rn,rkn->rk", rows, wd[ids.reshape(-1).to(torch.int64)])
    mag = torch.einsum("rn,rkn->rk", rows.abs(), wd[ids.reshape(-1).to(torch.int64)].abs())
    err = (out.cpu().to(torch.float64) - exact).abs()
    assert bool((err <= exact.abs() * 2.0**-8 + mag * N * 2.0**-24 + 1e-30).all())


def synthetic_experts(E, K, N, gen):
    from types import SimpleNamespace

    sigma = 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (E, K, N // 8), dtype=torch.int64, generator=gen).to(torch.int32)
    scales = (torch.randn(E, K, N // 128, generator=gen) * sigma).to(BF)
    biases = (-7.5 * scales.to(torch.float32) + torch.randn(E, K, N // 128, generator=gen) * sigma).to(BF)
    return SimpleNamespace(weight=words, scales=scales, biases=biases, group_size=128, bits=4)


def test_grouped_matmul_row_is_independent_of_its_neighbours(dev):
    gen = torch.Generator().manual_seed(11)
    E, K, N, k = 16, 256, 512, 2
    w = QuantizedWeights(**vars(synthetic_experts(E, K, N, gen)))
    a = torch.randn(256, N, generator=gen).to(BF)
    ids = torch.stack([torch.randperm(E, generator=gen)[:k] for _ in range(256)]).to(torch.int32)
    _, _, alone, _ = run_grouped(w, a[:1], ids[:1], k, ext.EPI_SWIGLU_PAIRS, True, dev)
    for pos in (0, 100, 255):
        aa, ii = a.clone(), ids.clone()
        aa[[0, pos]], ii[[0, pos]] = aa[[pos, 0]], ii[[pos, 0]]
        _, _, full, _ = run_grouped(w, aa, ii, k, ext.EPI_SWIGLU_PAIRS, True, dev)
        assert torch.equal(full[pos * k:(pos + 1) * k].cpu(), alone.cpu())


# ----------------------------------------------------------------------------------------------------- combine --
@pytest.mark.parametrize("residual", [False, True])
def test_combine_is_exact(dev, residual):
    gen = torch.Generator().manual_seed(12)
    T, k, H = 37, 8, 2048
    y = torch.randn(T * k, H, generator=gen).to(BF)
    s = torch.rand(T, k, generator=gen).to(BF)
    x = torch.randn(T, H, generator=gen).to(BF)
    out = ext.moe_combine(y.to(dev), s.to(dev), x.to(dev) if residual else None)
    want = omoe.moe_combine(y, s, x if residual else None)
    assert torch.equal(out.cpu(), want)
    w = (1 + 0.1 * torch.randn(H, generator=gen)).to(BF)
    out2, normed = ext.moe_combine(y.to(dev), s.to(dev), x.to(dev), w.to(dev), 1e-6)
    ref_norm = ext.rms_norm(out2, w.to(dev), 1e-6)
    assert float((normed.float() - ref_norm.float()).abs().max()) <= float(ref_norm.float().abs().max()) * 2.0**-7


# -------------------------------------------------------------------------------------------------- Moe block --
@pytest.mark.parametrize("E, I, H, k, T", [(3, 128, 128, 2, 6), (128, 768, 2048, 8, 64), (8, 128, 256, 2, 5)])
def test_moe_block_against_the_oracle(dev, E, I, H, k, T):
    gen = torch.Generator().manual_seed(E + I)
    router = QuantizedWeights(**vars(synthetic_experts(1, E, H, gen)))
    router = QuantizedWeights(scales=router.scales[0], biases=router.biases[0], group_size=128, bits=4, weight=router.weight[0])
    wg, wu, wd = (QuantizedWeights(**vars(synthetic_experts(E, o, i, gen))) for o, i in ((I, H), (I, H), (H, I)))
    gpu = lambda q: QuantizedWeights(scales=q.scales.to(dev), biases=q.biases.to(dev), group_size=128, bits=4, weight=q.weight.to(dev))
    moe = Moe(gpu(router), gpu(wg), gpu(wu), gpu(wd), num_experts_per_tok=k, norm_topk_prob=True)
    h = torch.randn(T, H, generator=gen).to(BF)
    out = moe(h.to(dev)).cpu().to(torch.float64)
    dense = lambda q: dense_f32(q).to(BF)
    logits = (h.to(torch.float32) @ omoe.ops.dequantize_fp32(router.weight, router.scales, router.biases).T).to(BF)
    _, ids, scores = omoe.route_ref(logits, k, True)
    ref = omoe.experts_ref(h, ids, scores, dense(wg), dense(wu), dense(wd)).to(torch.float64)
    scale = float(ref.abs().max())
    assert float((out - ref).abs().max()) <= 0.05 * scale


# ------------------------------------------------------------------------------------------------------- model --
def teacher_forced_check(model, dev, prompt, ref_tokens, ref_lp, chunk=None, atol=0.25):
    """test_gpu_models.py's rule: the reference's top-4 log-probs within ``atol`` nat, the same argmax where its top-2
    margin exceeds 0.5 nat."""
    cache = model.create_kv_cache()
    try:
        offset = 0
        if chunk is not None:
            while len(prompt) - offset > chunk:
                model(torch.tensor([prompt[offset : offset + chunk]], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
                offset += chunk
        feed = prompt[offset:]
        for step, (tok, lp_ref) in enumerate(zip(ref_tokens, ref_lp)):
            out = model(torch.tensor([feed], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
            x = out[0, -1].to(torch.float32)
            lp = (x - torch.logsumexp(x, dim=-1)).cpu()
            top = torch.topk(lp_ref, 4)
            torch.testing.assert_close(lp[top.indices], top.values, rtol=0, atol=atol, msg=lambda m: f"step {step}: {m}")
            if float(top.values[0] - top.values[1]) > 0.5:
                assert int(torch.argmax(lp)) == tok, f"step {step}"
            offset += len(feed)
            feed = [tok]
    finally:
        for c in cache:
            c.release()


@pytest.fixture(scope="module")
def moe_pair(dev):
    kwargs = dict(seed=0, realistic=True, max_position_embeddings=512)
    cpu = synthetic_qwen3("tiny-moe-d128", **kwargs)
    gpu = to_device(synthetic_qwen3("tiny-moe-d128", **kwargs), dev)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11, 8, 1, 77, 402, 65, 9, 33, 210]
    tokens, lp = greedy_decode(omoe.ReferenceCpuMoeModel(cpu), prompt, 10, return_logprobs=True)
    return gpu, prompt, tokens, lp


@pytest.mark.parametrize("mode", ["operators", "decode_graph", "prefill_graph"])
def test_moe_model_tracks_the_reference_cpu_path(dev, moe_pair, mode):
    gpu, prompt, tokens, lp = moe_pair
    model = Qwen3ModelWeek3(gpu, page_size=128)
    if mode == "operators":
        model.use_decode_graph = False
        teacher_forced_check(model, dev, prompt, tokens, lp)
    elif mode == "decode_graph":
        teacher_forced_check(model, dev, prompt, tokens, lp)
        assert model._decode_engines, "the decode graph ran"
    else:
        model.prefill_graph_len = 8
        teacher_forced_check(model, dev, prompt, tokens, lp, chunk=8)
        assert model._prefill_engines, "the prefill graph ran"


def test_moe_batcher_matches_the_reference_greedy_tokens(dev, moe_pair):
    """Every generated token of every request (the first from prefill, the rest from the 16-slot decode graph) equals the
    reference's greedy token; a mismatch is excused only where the reference's top-2 margin is at most 0.5 nat, and the
    request's continuation is no longer comparable after it."""
    from tiny_llm_b200 import ContinuousBatcher

    gpu = moe_pair[0]
    model = Qwen3ModelWeek3(gpu, page_size=128)
    ref = omoe.ReferenceCpuMoeModel(synthetic_qwen3("tiny-moe-d128", seed=0, realistic=True, max_position_embeddings=512))
    g = torch.Generator().manual_seed(7)
    prompts = [torch.randint(1, 500, (n,), generator=g).tolist() for n in (5, 19, 3, 12, 8, 27)]
    budget = 8
    batcher = ContinuousBatcher(model, None, prompts, max_seq_len=128, batch_size=16, prefill_step=8, verbose=False, device=dev,
                                max_new_tokens=[budget] * len(prompts))
    results = dict(batcher.run())
    assert all(pool.used_page_ids == set() for pool in model.page_pools)
    assert model._decode_engines, "decode steps went through the graph"
    compared = 0
    for i, prompt in enumerate(prompts):
        got = [int(t) for t in results[i].split()]
        want, lps = greedy_decode(ref, prompt, budget, return_logprobs=True)
        assert len(got) == budget
        for step, (a, b, lp) in enumerate(zip(got, want, lps)):
            if a != b:
                top = torch.topk(lp, 2).values
                assert float(top[0] - top[1]) <= 0.5, f"request {i} token {step}: {a} != {b} at margin {float(top[0] - top[1]):.3f}"
                break
            compared += 1
    assert compared >= len(prompts) * budget // 2


def test_moe_model_is_not_a_verify_target_and_speculative_equals_greedy(dev, moe_pair):
    from tiny_llm_b200 import greedy_generate_ids, speculative_generate_ids

    gpu, prompt, _, _ = moe_pair
    target = Qwen3ModelWeek3(gpu, page_size=128)
    assert not target.verify_applies()
    draft = Qwen3ModelWeek3(to_device(synthetic_qwen3("tiny-d128", seed=1, max_position_embeddings=512), dev), page_size=128)
    greedy = greedy_generate_ids(target, prompt, 8, device=dev)
    spec, _ = speculative_generate_ids(draft, target, prompt, 8, 3, device=dev)
    assert spec == greedy


# ----------------------------------------------------------------------------------------------------- engines --
def wide_args():
    return dict(num_hidden_layers=2, vocab_size=4096, max_position_embeddings=4096)


@pytest.fixture(scope="module")
def wide_weights(dev):
    return synthetic_qwen3("qwen3-30b-a3b", seed=2, device=dev, **wide_args())


def wide_model(weights):
    return Qwen3ModelWeek3(weights, page_size=128)


@pytest.mark.parametrize("T", [1, 8, 16, 64, 256])
def test_every_engine_form_of_the_moe_layer_equals_the_operator_form(dev, wide_weights, T):
    """The three call forms of one sparse layer on the same rows, bit for bit: the operator path (rms_norm, Moe, add,
    next rms_norm), the matvec stack's (router with the RMSNorm prologue, norm fused into the gather) and the swap-AB
    stack's (combine returning the next norm)."""
    from tiny_llm_b200.engine import _moe_mlp

    model = wide_model(wide_weights)
    block, nxt = model.layers_inner[0], model.layers_inner[1].input_layernorm
    moe, ln2 = block.mlp, block.post_attention_layernorm
    x = (torch.randn(T, 2048, generator=torch.Generator().manual_seed(T)) * 3).to(BF).to(dev)
    w2, wn = ln2._weight_as(BF, dev), nxt._weight_as(BF, dev)
    h = ext.rms_norm(x, w2, ln2.eps)
    logits = ext.quantized_matmul(moe.w_router.scales, moe.w_router.biases, 128, 4, h, moe.w_router.weight, True)
    op = ext.add(x, moe(h))
    op_next = ext.rms_norm(op, wn, nxt.eps)
    if T <= 8:  # the matvec stack's rows: its router projection runs on the streaming kernel, as the operator path's does
        fused_logits = ext.quantized_matmul_fused(moe.w_router.scales, moe.w_router.biases, moe.w_router.weight, x, w2, prologue=ext.PRO_RMSNORM,
                                                  eps=ln2.eps)
        assert torch.equal(logits, fused_logits), "router: RMSNorm prologue != rms_norm then projection"
        assert torch.equal(_moe_mlp(moe, x, ln2=ln2), op), "matvec form"
    got, got_next = _moe_mlp(moe, x, h, nxt=nxt)
    assert torch.equal(got, op), "swap-AB form"
    assert torch.equal(got_next, op_next), "swap-AB form: next RMSNorm"
    assert torch.equal(_moe_mlp(moe, x, h), op), "operator-path form of the graph engines"


@pytest.mark.parametrize("B", [1, 8, 16, 64])
def test_decode_engine_matches_the_operator_path_at_30b_width(dev, wide_weights, B):
    from tiny_llm_b200 import BatchingKvCache

    g = torch.Generator().manual_seed(B)
    prompts = {slot: torch.randint(0, 4096, (5,), generator=g).tolist() for slot in range(0, B, max(1, B // 6))}
    outs = []
    for graph in (True, False):
        model = wide_model(wide_weights)
        model.use_decode_graph = graph
        tables = [BatchingKvCache(B, max_seq_len=256) for _ in range(model.num_hidden_layers)]
        for slot, ids in prompts.items():
            model.use_decode_graph = False
            cache = model.create_kv_cache()
            model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
            model.use_decode_graph = graph
            for layer_cache, table in zip(cache, tables):
                table.add_request(layer_cache, slot)
        tokens = torch.zeros((B, 1), dtype=torch.int32, device=dev)
        offsets = [5 if s in prompts else 0 for s in range(B)]
        seq = [model(tokens, [o + step * (o > 0) for o in offsets], tables, logits_to_keep=1).float().cpu() for step in range(3)]
        assert bool(model._decode_engines) == graph
        for table in tables:
            for slot in prompts:
                table.remove_request(slot)
        outs.append(seq)
    live = list(prompts)
    for a, b in zip(*outs):
        la, lb = (t[live, -1] - torch.logsumexp(t[live, -1], dim=-1, keepdim=True) for t in (a, b))
        assert float((la - lb).abs().max()) <= 0.25


def engine_run(weights, dev, B, slots, steps, grow_after=None):
    """``steps`` engine steps of a fresh model's B-slot decode engine with the requests ``slots`` (slot -> prompt),
    prefilled on the operator path; returns the logits of every step (and the engine)."""
    from tiny_llm_b200 import BatchingKvCache
    from tiny_llm_b200.engine import DecodeEngine

    model = wide_model(weights)
    engine = DecodeEngine(model, B, 256, dev)
    engine.reserve_pools()
    tables = [BatchingKvCache(B, max_seq_len=256) for _ in range(model.num_hidden_layers)]
    for slot, ids in slots.items():
        cache = model.create_kv_cache()
        model.use_decode_graph = False
        model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, slot)
    tokens = [7 * b + 1 if b in slots else 0 for b in range(B)]
    offsets = [len(slots[b]) if b in slots else 0 for b in range(B)]
    out = []
    for step in range(steps):
        if grow_after is not None and step == grow_after:
            engine.reserve_pools(2 * B * engine.max_pages + 7)  # new, larger slabs: the graphs must be re-captured
        logits, nxt = engine.step(tokens, offsets, tables)
        out.append(logits.clone())
        tokens = [int(t) if b in slots else 0 for b, t in enumerate(nxt.tolist())]
        offsets = [o + 1 if b in slots else 0 for b, o in enumerate(offsets)]
    return out, engine


def test_row_variant_gives_the_bits_of_the_full_step(dev, wide_weights):
    """B = 64 with 10 live slots replays the 16-row graph; adding slot 63 forces the full 64-row graph.  A row's result
    depends only on that row, so slots 0..9 get the same bits either way."""
    g = torch.Generator().manual_seed(64)
    slots = {b: torch.randint(0, 4096, (4 + b,), generator=g).tolist() for b in range(10)}
    small, e16 = engine_run(wide_weights, dev, 64, slots, 3)
    full, e64 = engine_run(wide_weights, dev, 64, {**slots, 63: [5, 6, 7]}, 3)
    assert e16.variant_replays[16] == 3 and e64.variant_replays[64] == 3
    for a, b in zip(small, full):
        assert torch.equal(a[:10], b[:10])


@pytest.mark.parametrize("B", [1, 16])
def test_decode_on_device_logs_the_tokens_of_step_calls(dev, wide_weights, B):
    from tiny_llm_b200 import BatchingKvCache

    steps = 24
    g = torch.Generator().manual_seed(24 + B)
    slots = {b: torch.randint(0, 4096, (6 + b,), generator=g).tolist() for b in range(0, B, 3)}

    def run(on_device):
        model = wide_model(wide_weights)
        engine = model.decode_engine(B, 256)
        tables = [BatchingKvCache(B, max_seq_len=256) for _ in range(model.num_hidden_layers)]
        for slot, ids in slots.items():
            cache = model.create_kv_cache()
            model.use_decode_graph = False
            model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
            for layer_cache, table in zip(cache, tables):
                table.add_request(layer_cache, slot)
        tokens = [3 * b + 2 if b in slots else 0 for b in range(B)]
        offsets = [len(slots[b]) if b in slots else 0 for b in range(B)]
        if on_device:
            return engine.decode_on_device(tokens, offsets, tables, steps).cpu().tolist()
        log = []
        for _ in range(steps):
            _, nxt = engine.step(tokens, offsets, tables)
            tokens = [int(t) if b in slots else 0 for b, t in enumerate(nxt.tolist())]
            offsets = [o + 1 if b in slots else 0 for b, o in enumerate(offsets)]
            log.append([t if b in slots else -1 for b, t in enumerate(tokens)])
        return log

    assert run(True) == run(False)


def test_recapture_after_slab_growth_gives_the_same_bits(dev, wide_weights):
    slots = {0: [11, 12, 13, 14], 3: [5, 9, 2]}
    base, e1 = engine_run(wide_weights, dev, 8, slots, 5)
    grown, e2 = engine_run(wide_weights, dev, 8, slots, 5, grow_after=2)
    assert e2.captures == e1.captures + 1
    for a, b in zip(base, grown):
        assert torch.equal(a, b)


@pytest.mark.parametrize("chunk, length", [(128, 128), (128, 2), (256, 256)])
def test_prefill_engine_matches_the_operator_path_at_30b_width(dev, wide_weights, chunk, length):
    """One prefill chunk through the graph (<= 128 rows: the swap-AB stack; 256: the > 128-row branch, a 2-token tail
    right-aligned in a 128-row chunk) against the operator path, logits within the model tolerance."""
    g = torch.Generator().manual_seed(chunk + length)
    ids = torch.randint(0, 4096, (length,), generator=g).tolist()
    out = []
    for graph in (True, False):
        model = wide_model(wide_weights)
        model.decode_engine(1, 4096)  # the page reservation the prefill graph needs
        model.prefill_graph_len = chunk if graph else 0
        cache = model.create_kv_cache()
        logits = model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)[0, -1].float().cpu()
        assert bool(model._prefill_engines) == graph
        for c in cache:
            c.release()
        out.append(logits - torch.logsumexp(logits, dim=-1))
    assert float((out[0] - out[1]).abs().max()) <= 0.25
