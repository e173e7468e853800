"""Round-2 parity additions (VERDICT r1, "close the parity gaps that are closable"): every test
compares the CUDA path with the CPU ORACLE (never GPU kernel against GPU kernel) at the sizes the
serving configurations run: long contexts with split/merge, 64-slot batches with idle slots, the
two-tile GEMM at the real down-projection shape, a full-depth Qwen3-4B step and the committed
config-1 trace (Qwen3-0.6B shape, 128 tokens)."""

import json
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import ops as oracle
from oracle.model import ReferenceCpuModel, greedy_decode
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.synthetic import synthetic_qwen3, to_device

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16
GOLDEN = Path(__file__).parent / "golden"


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def gen(seed):
    return torch.Generator().manual_seed(seed)


def logprobs(logits):
    x = logits.to(torch.float32)
    return x - torch.logsumexp(x, dim=-1, keepdim=True)


def rand_packed(K, N, g, sigma=None):
    sigma = sigma if sigma is not None else 1.0 / (4.717 * N**0.5)
    words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32)
    scales = (torch.randn(K, N // 128, generator=g) * sigma).to(BF16)
    biases = (-7.5 * scales.float() + torch.randn(K, N // 128, generator=g) * sigma).to(BF16)
    return words, scales, biases


# ------------------------------------------------------------------ attention at serving sizes --
@pytest.mark.parametrize("contexts", [[4100], [8192, 4097], [129, 0, 2500, 640]], ids=lambda c: "ctx" + "_".join(map(str, c)))
def test_fused_decode_attention_long_context_against_the_cpu_oracle(dev, contexts):
    """q/k rms_norm -> rope -> paged_cache_update -> paged_attention (qwen3_week3.py:62-105) in ONE launch,
    long enough that the KV range is split over CTAs and merged, against the oracle's operator sequence."""
    g = gen(sum(contexts))
    B, Hq, Hkv, D, page = len(contexts), 32, 8, 128, 128
    max_pages = (max(contexts) + page - 1) // page + 1
    P = B * max_pages
    qkv = torch.randn(B, (Hq + 2 * Hkv) * D, generator=g).to(BF16)
    qw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16)
    kw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16)
    ctx = torch.tensor(contexts, dtype=torch.int32)
    offsets = (ctx - 1).clamp_min(0)
    bt = torch.full((B, max_pages), -1, dtype=torch.int32)
    perm = torch.randperm(P, generator=g)
    for b, c in enumerate(contexts):
        n = (c + page - 1) // page
        bt[b, :n] = perm[b * max_pages : b * max_pages + n].to(torch.int32)
    kp = torch.randn(P, Hkv, page, D, generator=g).to(BF16)
    vp = torch.randn(P, Hkv, page, D, generator=g).to(BF16)
    scale = D**-0.5
    kp_ref, vp_ref = kp.clone(), vp.clone()
    q_in = qkv[:, : Hq * D].reshape(B, 1, Hq, D)
    k_in = qkv[:, Hq * D : (Hq + Hkv) * D].reshape(B, 1, Hkv, D)
    v_in = qkv[:, (Hq + Hkv) * D :].reshape(B, 1, Hkv, D)
    q_ref = oracle.rope(oracle.rms_norm(q_in, qw, 1e-6), offsets, D, 1e6)
    k_ref = oracle.rope(oracle.rms_norm(k_in, kw, 1e-6), offsets, D, 1e6)
    for b, c in enumerate(contexts):
        if c == 0:
            continue
        tok = c - 1
        pid = int(bt[b, tok // page])
        oracle.paged_cache_update(kp_ref, k_ref[b : b + 1].transpose(1, 2).contiguous(), pid, tok % page)
        oracle.paged_cache_update(vp_ref, v_in[b : b + 1].transpose(1, 2).contiguous(), pid, tok % page)
    want = oracle.paged_attention(q_ref.transpose(1, 2).reshape(B * Hq, 1, D).contiguous(), kp_ref, vp_ref, bt, ctx, scale, True, Hkv, Hq)
    kd, vd = kp.to(dev), vp.to(dev)
    got = ext.decode_attention_fused(qkv.to(dev), qw.to(dev), kw.to(dev), offsets.to(dev), bt.to(dev), ctx.to(dev),
                                     ext.rope_inv_freq_table(D, 1e6, dev), kd, vd, Hq, Hkv, 1e-6, scale, max(contexts))
    assert torch.equal(vd.cpu(), vp_ref)
    torch.testing.assert_close(kd.cpu().float(), kp_ref.float(), rtol=2**-7, atol=4e-3)
    torch.testing.assert_close(got.cpu().float().view(B * Hq, D), want.float().view(B * Hq, D), rtol=2e-2, atol=5e-3)  # test_week_3_day_5.py:61
    for b, c in enumerate(contexts):
        if c == 0:
            assert torch.count_nonzero(got[b]) == 0, "idle slot must be exact zeros"


@pytest.mark.parametrize("B,S", [(1, 4097), (1, 8192), (64, 4097)], ids=lambda v: str(v))
def test_paged_decode_attention_at_serving_sizes_matches_oracle(dev, B, S):
    """tl_paged_attention, L == 1, at the context lengths of configs 2/5 (one request checked in full for B = 64)."""
    g = gen(B * 10000 + S)
    Hq, Hkv, D, page = 32, 8, 128, 128
    pages = (S + page - 1) // page
    P = B * pages
    lens = [S - 13 * b if b % 5 else S for b in range(B)]
    bt = torch.randperm(P, generator=g).reshape(B, pages).to(torch.int32)
    cl = torch.tensor(lens, dtype=torch.int32)
    q = torch.randn(B * Hq, 1, D, generator=g).to(BF16)
    kp = torch.randn(P, Hkv, page, D, generator=g).to(BF16)
    vp = torch.randn(P, Hkv, page, D, generator=g).to(BF16)
    got = ext.paged_attention(q.to(dev), kp.to(dev), vp.to(dev), bt.to(dev), cl.to(dev), D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq).cpu()
    for b in sorted({0, B // 2, B - 1}):
        want = oracle.paged_attention(q[b * Hq : (b + 1) * Hq], kp, vp, bt[b : b + 1], cl[b : b + 1], D**-0.5, True, Hkv, Hq)
        torch.testing.assert_close(got[b * Hq : (b + 1) * Hq].float(), want.float(), rtol=2e-2, atol=5e-3, msg=lambda m: f"request {b}: {m}")


@pytest.mark.parametrize("B,L,ctx,Hq,Hkv,page", [(1, 128, 640, 32, 8, 128), (2, 100, 300, 16, 8, 64), (1, 40, 40, 8, 8, 128), (1, 4, 200, 32, 8, 128)])
def test_token_major_prefill_attention_is_the_transposed_head_major_result(dev, B, L, ctx, Hq, Hkv, page):
    """The chunked-prefill engine asks the wgmma kernel for [B * L, Hq * D] directly (the o-projection's layout):
    bit-identical to paged_attention + transpose; shapes the kernel does not take (here L = 4) fall back to exactly that."""
    g, D = gen(B * 1000 + L + ctx), 128
    pages = -(-ctx // page)
    kp = torch.randn(B * pages, Hkv, page, D, generator=g).to(BF16).to(dev)
    vp = torch.randn(B * pages, Hkv, page, D, generator=g).to(BF16).to(dev)
    q = torch.randn(B * Hq, L, D, generator=g).to(BF16).to(dev)
    bt = torch.randperm(B * pages, generator=g).reshape(B, pages).to(torch.int32).to(dev)
    cl = torch.tensor([ctx - 7 * b for b in range(B)], dtype=torch.int32).to(dev)
    want = ext.paged_attention(q, kp, vp, bt, cl, D**-0.5, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
    got = ext.paged_attention_token_major(q, kp, vp, bt, cl, D**-0.5, True, Hkv, Hq)
    assert got.shape == (B * L, Hq * D)
    assert torch.equal(got, want.view(B, Hq, L, D).transpose(1, 2).reshape(B * L, Hq * D))


@pytest.mark.parametrize("rows,chunk", [(64, False), (16, False), (128, True), (40, True), (4, False)])
def test_qkv_projection_feeding_rope_append_equals_the_two_calls(dev, rows, chunk):
    """q|k|v projection whose split-reduction planes go straight into q/k norm + RoPE + append (q|k|v never written):
    rotated queries and the appended K/V rows bit-identical to projection -> decode / chunk_qk_norm_rope_append
    (4 rows: the streaming projection, no planes - the call falls back to exactly those two launches)."""
    Hq, Hkv, D, N, page = 32, 8, 128, 2560, 128
    g = gen(rows * 3 + int(chunk))
    K = (Hq + 2 * Hkv) * D
    words, scales, biases = rand_packed(K, N, g)
    words, scales, biases = words.to(dev), scales.to(dev), biases.to(dev)
    h = torch.randn(rows, N, generator=g).to(BF16).to(dev)
    qw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16).to(dev)
    kw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF16).to(dev)
    if chunk:  # one request, `rows` consecutive tokens starting at position 200
        pages = 4
        bt = torch.tensor([3, 1, 0, 2], dtype=torch.int32, device=dev)
        offsets = torch.arange(200, 200 + rows, dtype=torch.int32, device=dev)
        ctx = offsets + 1
    else:  # one request per row, two idle rows
        pages = 2
        bt = torch.randperm(rows * pages, generator=g).reshape(rows, pages).to(torch.int32).to(dev)
        offsets = torch.tensor([(37 * r) % 250 for r in range(rows)], dtype=torch.int32, device=dev)
        ctx = offsets + 1
        ctx[1] = 0
        ctx[rows - 1] = 0
    P = (pages if chunk else rows * pages)
    outs = []
    for fused in (True, False):
        kp = torch.zeros(P, Hkv, page, D, dtype=BF16, device=dev)
        vp = torch.zeros_like(kp)
        if fused:
            q = ext.qkv_project_rope_append(scales, biases, words, h, qw, kw, offsets, bt, ctx, kp, vp, Hq, Hkv, 1e6, 1e-6, chunk=chunk)
        else:
            qkv = ext.quantized_matmul_fused(scales, biases, words, h)
            fn = ext.chunk_qk_norm_rope_append if chunk else ext.decode_qk_norm_rope_append
            q = fn(qkv, qw, kw, offsets, bt, ctx, kp, vp, Hq, Hkv, 1e6, 1e-6)
        outs.append((q, kp, vp))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ GEMM at the config-3 shapes --
# One CTA per output tile: the only form on Hopper (the CTA-pair form used Blackwell's cta_group::2).
@pytest.mark.parametrize("tiling", ["one-cta"])
@pytest.mark.parametrize("shape", [(4096, 9728, 2560), (4096, 2560, 19456 // 2), (4096, 4096, 2560), (1000, 256, 392)],
                         ids=lambda s: "x".join(map(str, s)))
def test_prefill_gemm_full_size_matches_oracle_on_sampled_rows(dev, shape, tiling):
    """M = 4096 at the Qwen3-4B down / gate / o shapes (and a ragged one: 1000 rows, 392 features) on the prefill
    kernel (128-token tiles, w4a16_skinny.cu): sampled token rows against the tiled kernel's arithmetic restated on the
    CPU (weights rounded to bf16 before the MMA, quantized_matmul.metal:183-194; fp32 accumulation), and two launches
    against each other bit for bit on the whole matrix (fixed accumulation order along the reduction)."""
    M, N, K = shape
    g = gen(M + N + K)
    words, scales, biases = rand_packed(K, N, g)
    a = torch.randn(M, N, generator=g).to(BF16)
    args = (scales.to(dev), biases.to(dev), 128, 4, a.to(dev), words.to(dev), True)
    got_dev = ext.quantized_matmul(*args)
    other = ext.quantized_matmul(*args)
    got = got_dev.cpu()
    rows = sorted({0, 1, 127, 128, 255, 256, M // 2 - 1, M // 2, M - 1})
    w = oracle.dequantize_weights(words, scales, biases, 128, 4).float()
    want = (a[rows].float() @ w.T).to(BF16)
    scale_ref = float(want.float().abs().max()) + 1e-6
    torch.testing.assert_close(got[rows].float(), want.float(), rtol=2 * 2.0**-8, atol=2e-3 * scale_ref)
    assert torch.equal(got_dev, other)


def test_reference_acceptance_shape_matvec_1x2560_to_1024(dev):
    """tests_refsol/test_week_2_day_3.py:179-196: the Qwen k_proj shape with Gaussian weights quantised to 4 bits,
    checked with the reference's own absolute tolerance (1.5) and with ours (2 output ulp) against the oracle."""
    from tiny_llm_b200.synthetic import quantize_w4

    g = gen(196)
    x = torch.randn(1, 2560, generator=g).to(BF16)
    weight = torch.randn(1024, 2560, generator=g).to(BF16)
    packed, scales, biases = quantize_w4(weight.float())
    words = packed.view(torch.int32) if packed.dtype == torch.uint32 else packed
    want = oracle.quantized_matmul(scales, biases, 128, 4, x, words, True, use_simdgroup=False)
    got = ext.quantized_matmul(scales.to(dev), biases.to(dev), 128, 4, x.to(dev), words.to(dev), True).cpu()
    torch.testing.assert_close(got.float(), want.float(), rtol=0, atol=1.5)  # the reference's bound
    torch.testing.assert_close(got.float(), want.float(), rtol=2 * 2.0**-8, atol=2e-3 * float(want.float().abs().max()))
    dense = (x.float() @ oracle.dequantize_weights(words, scales, biases, 128, 4).float().T)
    torch.testing.assert_close(got.float(), dense, rtol=2 * 2.0**-8, atol=2e-3 * float(dense.abs().max()))


# ------------------------------------------------------------------ engine at serving batch sizes --
@pytest.mark.parametrize("B", [8, 32, 64])
def test_engine_batch_with_idle_slots_matches_cpu_oracle(dev, B):
    """The CUDA-graph decode engine with B slots (every third one idle, different context lengths per slot),
    three steps, against the reference CPU path run request by request: teacher-forced log-probabilities of
    the oracle's top-4 candidates within 0.25 nat, block tables / page lens as the scheduler would see them."""
    kwargs = dict(seed=3, realistic=True, max_position_embeddings=512)
    cpu_ns = synthetic_qwen3("tiny-d128", **kwargs)
    gpu_ns = to_device(synthetic_qwen3("tiny-d128", **kwargs), dev)
    oracle_model = ReferenceCpuModel(cpu_ns)
    model = Qwen3ModelWeek3(gpu_ns, page_size=16)
    g = gen(B)
    steps = 3
    active = [b for b in range(B) if b % 3 != 1]
    prompts = {b: torch.randint(1, 500, (5 + (7 * b) % 40,), generator=g).tolist() for b in active}
    ref = {b: greedy_decode(oracle_model, prompts[b], steps + 1, return_logprobs=True) for b in active}
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=128) for _ in range(model.num_hidden_layers)]
    for b in active:
        cache = model.create_kv_cache()
        model(torch.tensor([prompts[b]], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, b)
    for step in range(steps):
        tokens = [ref[b][0][step] if b in prompts else 0 for b in range(B)]
        offsets = [len(prompts[b]) + step if b in prompts else 0 for b in range(B)]
        logits = model(torch.tensor(tokens, dtype=torch.int32, device=dev).reshape(B, 1), offsets, tables, logits_to_keep=1)
        lp = logprobs(logits[:, -1]).cpu()
        for b in active:
            top = torch.topk(ref[b][1][step + 1], 4)
            torch.testing.assert_close(lp[b][top.indices], top.values, rtol=0, atol=0.25, msg=lambda m: f"slot {b} step {step}: {m}")
    engine = model.decode_engine(B, 128)
    assert engine.graph_replays == steps, "the batched decode steps must have gone through the graph engine"
    for b in active:
        c0 = tables[0].kv_caches[b]
        n = len(prompts[b]) + steps
        assert c0.offset == n and sum(c0.page_lens) == n and len(c0.page_ids) == (n + 15) // 16
        assert all(t.kv_caches[b].page_ids == c0.page_ids and t.kv_caches[b].page_lens == c0.page_lens for t in tables)
    for table in tables:
        for b in active:
            table.remove_request(b)
    assert all(pool.used_page_ids == set() for pool in model.page_pools)


def test_serving_path_engine_matches_cpu_oracle(dev):
    """The step as the serving configurations run it - 32 slots behind 1024-token block tables (64-slot pages): more than
    16 K slot-tokens, so q|k|v projection + RoPE + append as one fused launch pair, attention on the wgmma streaming
    kernel with its split count from the table width, swap-AB projections with the RMSNorm folded into the reduction,
    and a 16-row step graph (occupied slots 0..12) - against the reference CPU path request by request: teacher-forced
    log-probabilities of the oracle's top-4 candidates within 0.25 nat over three steps."""
    kwargs = dict(seed=7, realistic=True, max_position_embeddings=2048)
    cpu_ns = synthetic_qwen3("tiny-d128", **kwargs)
    gpu_ns = to_device(synthetic_qwen3("tiny-d128", **kwargs), dev)
    oracle_model = ReferenceCpuModel(cpu_ns)
    model = Qwen3ModelWeek3(gpu_ns, page_size=64)
    B, steps, g = 32, 3, gen(321)
    active = [b for b in range(13) if b % 4 != 2]
    prompts = {b: torch.randint(1, 500, (9 + (13 * b) % 90,), generator=g).tolist() for b in active}
    ref = {b: greedy_decode(oracle_model, prompts[b], steps + 1, return_logprobs=True) for b in active}
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=1024) for _ in range(model.num_hidden_layers)]
    for b in active:
        cache = model.create_kv_cache()
        model(torch.tensor([prompts[b]], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, b)
    for step in range(steps):
        tokens = [ref[b][0][step] if b in prompts else 0 for b in range(B)]
        offsets = [len(prompts[b]) + step if b in prompts else 0 for b in range(B)]
        logits = model(torch.tensor(tokens, dtype=torch.int32, device=dev).reshape(B, 1), offsets, tables, logits_to_keep=1)
        lp = logprobs(logits[:, -1]).cpu()
        for b in active:
            top = torch.topk(ref[b][1][step + 1], 4)
            torch.testing.assert_close(lp[b][top.indices], top.values, rtol=0, atol=0.25, msg=lambda m: f"slot {b} step {step}: {m}")
    engine = model.decode_engine(B, 1024)
    assert engine.graph_replays == steps and not engine._attention_fused
    assert engine.variant_replays[16] == steps, "occupied slots 0..12: the 16-row graph must have been replayed"
    for table in tables:
        for b in active:
            table.remove_request(b)


def test_row_variant_graphs_give_the_bits_of_the_full_step(dev):
    """A 64-slot engine whose occupied slots are a short prefix replays the 16- or 32-row step graph: the logits of
    the occupied rows must be bit-identical to what the full 64-row graph produces (same kernels, same split counts),
    and a later step with a high slot occupied must pick the wide graph again."""
    ns = to_device(synthetic_qwen3("tiny-d128", seed=5, realistic=True, max_position_embeddings=512), dev)
    B, g = 64, gen(64)

    def run(variants: bool, slots):
        model = Qwen3ModelWeek3(ns, page_size=16)
        engine = DecodeEngine(model, B, 128, dev, _row_variants=variants)
        engine.reserve_pools()
        tables = [BatchingKvCache(max_active_requests=B, max_seq_len=128) for _ in range(model.num_hidden_layers)]
        prompts = {b: [3 + (11 * b + j) % 400 for j in range(4 + b % 7)] for b in slots}
        for b in slots:
            cache = model.create_kv_cache()
            model(torch.tensor([prompts[b]], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
            for layer_cache, table in zip(cache, tables):
                table.add_request(layer_cache, b)
        outs = []
        for step in range(2):
            tokens = [7 + b + step if b in prompts else 0 for b in range(B)]
            offsets = [len(prompts[b]) + step if b in prompts else 0 for b in range(B)]
            logits, _ = engine.step(tokens, offsets, tables)
            outs.append(logits.clone())
        for table in tables:
            for b in slots:
                table.remove_request(b)
        return outs, engine

    for slots, want_rows in (([0, 1, 2, 5, 9], 16), ([0, 3, 17, 30], 32), ([2, 40, 63], 64)):
        narrow, eng = run(True, slots)
        full, _ = run(False, slots)
        assert eng.variant_replays[want_rows] == 2 and sum(eng.variant_replays.values()) == 2
        for a, b in zip(narrow, full):
            assert torch.equal(a[slots], b[slots])


def test_engine_recapture_after_slab_growth_does_not_touch_released_pages(dev):
    """ADVICE r1: a second, larger engine moves the page slabs; the first engine then re-captures its graph.
    The warm-up passes of that capture must not append through stale metadata into pages that were released
    and handed to another request in the meantime."""
    ns = to_device(synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512), dev)
    model = Qwen3ModelWeek3(ns, page_size=8)
    ref = Qwen3ModelWeek3(ns, page_size=8)
    ref.use_decode_graph = False
    prompt_a, prompt_b = [5, 17, 3, 250, 99, 42, 7], [9, 2, 4, 6, 8, 10, 12, 14, 1]

    def prefill(m, prompt):
        cache = m.create_kv_cache()
        logits = m(torch.tensor([prompt], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
        return cache, int(torch.argmax(logits[0, -1].float()))

    small = DecodeEngine(model, 1, 64, dev)
    small.reserve_pools()
    cache_a, tok_a = prefill(model, prompt_a)
    small.step([tok_a], [len(prompt_a)], cache_a)  # captures; device metadata now describes request A
    for c in cache_a:
        c.release()  # A's pages go back to the free list (LIFO)
    cache_b, tok_b = prefill(model, prompt_b)  # ... and are handed to request B
    ref_cache_b, ref_tok_b = prefill(ref, prompt_b)
    assert tok_b == ref_tok_b
    big = DecodeEngine(model, 4, 256, dev)
    big.reserve_pools()  # slabs move: `small` must re-capture on its next step
    got, _ = small.step([tok_b], [len(prompt_b)], cache_b)
    want = ref(torch.tensor([[tok_b]], dtype=torch.int32, device=dev), len(prompt_b), ref_cache_b, logits_to_keep=1)
    torch.testing.assert_close(got.float().view(-1), want.float().view(-1), rtol=0, atol=0.06)
    for c in (*cache_b, *ref_cache_b):
        c.release()


# ------------------------------------------------------------------ whole models --
def test_qwen3_4b_full_depth_teacher_forced_against_cpu_oracle(dev):
    """All 36 layers at Qwen3-4B width (random W4 weights, seed 0): an 8-token prefill and two decode steps,
    log-probabilities of the reference CPU path's top-4 candidates within 0.25 nat.  ~1 minute of CPU time."""
    cpu_ns = synthetic_qwen3("qwen3-4b", seed=0)
    prompt = [1000, 20000, 300, 4567, 150000, 77, 88888, 2]
    tokens, lps = greedy_decode(ReferenceCpuModel(cpu_ns), prompt, 3, return_logprobs=True)
    model = Qwen3ModelWeek3(to_device(cpu_ns, dev), page_size=128)
    cache = model.create_kv_cache()
    feed, offset = prompt, 0
    for step, (tok, lp_ref) in enumerate(zip(tokens, lps)):
        out = model(torch.tensor([feed], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
        lp = logprobs(out[0, -1]).cpu()
        top = torch.topk(lp_ref, 4)
        torch.testing.assert_close(lp[top.indices], top.values, rtol=0, atol=0.25, msg=lambda m: f"step {step}: {m}")
        offset += len(feed)
        feed = [tok]
    for c in cache:
        c.release()


def test_config1_golden_trace_qwen3_0p6b_shape(dev):
    """BASELINE config 1: the committed 128-token greedy trace of the reference CPU path at Qwen3-0.6B shape
    (tests/golden/qwen3_0p6b_greedy_trace.json, written by make_golden.py --config1), replayed teacher-forced
    through the CUDA path: prefill of the 16-token prompt, then 127 steps through the decode engine."""
    golden = json.loads((GOLDEN / "qwen3_0p6b_greedy_trace.json").read_text())
    ns = synthetic_qwen3(golden["config"], seed=golden["seed"], device=dev)
    model = Qwen3ModelWeek3(ns, page_size=128)
    model.decode_graph_max_seq_len = 256
    cache = model.create_kv_cache()
    feed, offset = golden["prompt"], 0
    worst = 0.0
    for step, (ids, vals, ref_tok) in enumerate(zip(golden["top4_ids"], golden["top4_logprobs"], golden["tokens"])):
        out = model(torch.tensor([feed], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
        lp = logprobs(out[0, -1]).cpu()
        want = torch.tensor(vals)
        worst = max(worst, float((lp[ids] - want).abs().max()))
        torch.testing.assert_close(lp[ids], want, rtol=0, atol=0.25, msg=lambda m: f"step {step}: {m}")
        if vals[0] - vals[1] > 0.5:
            assert int(torch.argmax(lp)) == ref_tok, f"step {step}"
        offset += len(feed)
        feed = [ref_tok]
    assert model.decode_engine(1).graph_replays >= 127
    for c in cache:
        c.release()
    print(f"config-1 trace: worst top-4 log-prob deviation {worst:.4f} nat over {len(golden['tokens'])} steps")


# ------------------------------------------------------------------ chunked-prefill graph engine --
def test_prefill_chunk_graph_equals_the_operator_path(dev):
    """engine.PrefillEngine (one captured chunk, right-aligned tail chunks, device-driven K/V append) against the
    operator-by-operator path of the same model: logits of every chunk's last token, the pages written and the
    integer bookkeeping (page ids / page lens / offset, bit-exact), then a decode step on top of both caches."""
    ns = to_device(synthetic_qwen3("tiny-d128", seed=5, realistic=True, max_position_embeddings=512), dev)
    eager = Qwen3ModelWeek3(ns, page_size=64)
    eager.prefill_graph_len = 0
    graph = Qwen3ModelWeek3(ns, page_size=64)
    graph.prefill_graph_len = 32
    graph.decode_graph_max_seq_len = 256
    graph.prefill_engine(32).reserve_pools(16)
    for pool in eager.page_pools:
        pool.reserve(16, 2, 128, dtype=torch.bfloat16, device=dev)
    g = gen(77)
    prompt = torch.randint(1, 500, (77,), generator=g).tolist()  # chunks of 32, 32, 13 (the tail is right-aligned in 32 rows)
    ce, cg = eager.create_kv_cache(), graph.create_kv_cache()
    offset = 0
    while offset < len(prompt):
        ids = torch.tensor([prompt[offset : offset + 32]], dtype=torch.int32, device=dev)
        want = eager(ids, [offset], ce, logits_to_keep=1)
        got = graph(ids, [offset], cg, logits_to_keep=1)
        assert got.shape == want.shape
        torch.testing.assert_close(got.float(), want.float(), rtol=0, atol=0.08, msg=lambda m: f"chunk at {offset}: {m}")
        offset += ids.shape[1]
        for a, b in zip(ce, cg):
            assert a.page_ids == b.page_ids and a.page_lens == b.page_lens and a.offset == b.offset == offset
    assert graph.prefill_engine(32).replays == 3
    for layer, (pe, pg) in enumerate(zip(eager.page_pools, graph.page_pools)):
        for pid, fill in zip(ce[layer].page_ids, ce[layer].page_lens):
            torch.testing.assert_close(pg._key_pages[pid, :, :fill].float(), pe._key_pages[pid, :, :fill].float(), rtol=2**-6, atol=6e-2)
            torch.testing.assert_close(pg._value_pages[pid, :, :fill].float(), pe._value_pages[pid, :, :fill].float(), rtol=2**-6, atol=6e-2)
    tok = torch.tensor([[7]], dtype=torch.int32, device=dev)
    torch.testing.assert_close(graph(tok, len(prompt), cg, logits_to_keep=1).float(), eager(tok, len(prompt), ce, logits_to_keep=1).float(), rtol=0, atol=0.08)
    for c in (*ce, *cg):
        c.release()
