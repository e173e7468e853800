"""Model-level parity on an H100: the Week-2/Week-3 model code and the scheduler
running on the CUDA kernels, against the reference's CPU path (oracle.model) on
identical synthetic weights.  Stated tolerance: teacher-forced log-probabilities
of the reference's top-4 candidates within 0.25 nat (bf16 activations through
W4 weights; the reference itself accepts atol 2.0-2.5 against MLX,
tests_refsol/test_week_2_day_6.py:107-109), and the same argmax wherever the
reference's top-2 margin exceeds 0.5 nat."""

import pytest
import torch

from oracle.model import ReferenceCpuModel, greedy_decode
from tiny_llm_b200 import BatchingKvCache, ContinuousBatcher, Qwen3ModelWeek2, Qwen3ModelWeek3, greedy_generate_ids
from tiny_llm_b200.synthetic import synthetic_qwen3, to_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def logprobs(logits):
    x = logits.to(torch.float32)
    return x - torch.logsumexp(x, dim=-1, keepdim=True)


def teacher_forced_check(model, dev, prompt, ref_tokens, ref_lp, chunk=None, atol=0.25):
    cache = model.create_kv_cache()
    try:
        offset = 0
        if chunk is not None:  # chunked prefill of all but the last chunk, as the scheduler does
            while len(prompt) - offset > chunk:
                model(torch.tensor([prompt[offset : offset + chunk]], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
                offset += chunk
        feed = prompt[offset:]
        for step, (tok, lp_ref) in enumerate(zip(ref_tokens, ref_lp)):
            out = model(torch.tensor([feed], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
            lp = logprobs(out[0, -1]).cpu()
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
def tiny_pair(dev):
    kwargs = dict(seed=0, realistic=True, max_position_embeddings=512)
    cpu = synthetic_qwen3("tiny-d128", **kwargs)
    gpu = to_device(synthetic_qwen3("tiny-d128", **kwargs), dev)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11, 8, 1, 77, 402, 65, 9, 33, 210]
    tokens, lp = greedy_decode(ReferenceCpuModel(cpu), prompt, 10, return_logprobs=True)
    return gpu, prompt, tokens, lp


@pytest.mark.parametrize("page_size", [8, 128])
@pytest.mark.parametrize("chunk", [None, 4])
def test_week3_paged_model_tracks_the_reference_cpu_path(dev, tiny_pair, page_size, chunk):
    gpu, prompt, tokens, lp = tiny_pair
    teacher_forced_check(Qwen3ModelWeek3(gpu, page_size=page_size), dev, prompt, tokens, lp, chunk=chunk)


@pytest.mark.parametrize("checkpoint", ["kv-cache", "quantized-matvec", "swiglu", "decode-attention", "split-k"])
def test_week2_checkpoints_track_the_reference_cpu_path(dev, tiny_pair, checkpoint):
    gpu, prompt, tokens, lp = tiny_pair
    teacher_forced_check(Qwen3ModelWeek2(gpu, checkpoint=checkpoint), dev, prompt, tokens, lp)


def test_week3_dense_gather_fallback_tracks_the_reference(dev, tiny_pair):
    gpu, prompt, tokens, lp = tiny_pair
    teacher_forced_check(Qwen3ModelWeek3(gpu, page_size=8, enable_paged_attention=False), dev, prompt, tokens, lp)


def test_week3_incremental_decode_matches_week2_on_gpu(dev, tiny_pair):
    # test_week_3_day_4.py:325-345 (the reference holds 1e-3 on its own fp32-accumulating kernels;
    # here both sides round activations to bf16 in different kernels: 3e-2 on log-probs)
    gpu = tiny_pair[0]
    week2, week3 = Qwen3ModelWeek2(gpu), Qwen3ModelWeek3(gpu, page_size=4)
    inputs = torch.tensor([[1, 5, 7, 3, 9, 11]], dtype=torch.int32, device=dev)
    c2, c3 = week2.create_kv_cache(), week3.create_kv_cache()
    for offset in range(inputs.shape[1]):
        token = inputs[:, offset : offset + 1]
        torch.testing.assert_close(logprobs(week3(token, offset, c3)), logprobs(week2(token, offset, c2)), rtol=0, atol=3e-2)
    assert c3[0].page_ids == [0, 1] and c3[0].page_lens == [4, 2]


def test_qwen3_4b_width_two_layer_model_tracks_the_reference(dev):
    """BASELINE shapes (hidden 2560, 32/8 heads x 128, MLP 9728, vocab 151,936,
    tied head) with 2 layers so the CPU reference finishes in seconds."""
    kwargs = dict(seed=3, num_hidden_layers=2)
    cpu = synthetic_qwen3("qwen3-4b", **kwargs)
    prompt = [1000 + 37 * i for i in range(40)]
    tokens, lp = greedy_decode(ReferenceCpuModel(cpu), prompt, 4, return_logprobs=True)
    del cpu
    gpu = to_device(synthetic_qwen3("qwen3-4b", **kwargs), dev)
    teacher_forced_check(Qwen3ModelWeek3(gpu, page_size=128), dev, prompt, tokens, lp, chunk=16)


def test_batched_decode_rows_match_single_requests_and_idle_rows_are_ignored(dev, tiny_pair):
    gpu = tiny_pair[0]
    model = Qwen3ModelWeek3(gpu, page_size=8)
    prompts = {0: [1, 5, 7], 2: [9, 2, 4, 6, 8, 10, 12, 14, 16, 18, 20]}
    tables = [BatchingKvCache(3, max_seq_len=64) for _ in range(model.num_hidden_layers)]
    alone_logits = {}
    for slot, ids in prompts.items():
        cache = model.create_kv_cache()
        model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
        for layer_cache, table in zip(cache, tables):
            table.add_request(layer_cache, slot)
        alone = model.create_kv_cache()
        model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, alone, logits_to_keep=1)
        alone_logits[slot] = model(torch.tensor([[11]], dtype=torch.int32, device=dev), len(ids), alone, logits_to_keep=1)
        for c in alone:
            c.release()
    for step in range(3):  # a few steps so the batched append crosses a page boundary
        out = model(torch.tensor([[11], [0], [11]], dtype=torch.int32, device=dev), [3 + step, 0, 11 + step], tables, logits_to_keep=1)
        if step == 0:
            for slot in prompts:
                torch.testing.assert_close(logprobs(out[slot]), logprobs(alone_logits[slot][0]), rtol=0, atol=3e-2)
        assert torch.isfinite(out.float()).all()
    ctx = [tables[0].kv_caches[s].offset for s in (0, 2)]
    assert ctx == [6, 14]
    assert tables[0].kv_caches[2].page_ids == tables[1].kv_caches[2].page_ids


def test_continuous_batching_on_gpu_releases_everything_and_agrees_with_single_requests(dev, tiny_pair):
    gpu = tiny_pair[0]
    model = Qwen3ModelWeek3(gpu, page_size=8)
    g = torch.Generator().manual_seed(7)
    prompts = [torch.randint(1, 500, (n,), generator=g).tolist() for n in (5, 19, 3, 12, 8, 27)]
    budgets = [4, 3, 5, 2, 4, 3]
    batcher = ContinuousBatcher(model, None, prompts, max_seq_len=64, batch_size=3, prefill_step=8, verbose=False, device=dev, max_new_tokens=budgets)
    results = dict(batcher.run())
    assert sorted(results) == list(range(6))
    assert [len(results[i].split()) for i in range(6)] == budgets
    assert all(pool.used_page_ids == set() and pool.num_free_pages == pool.num_pages for pool in model.page_pools)
    assert batcher.prefill_tokens == sum(map(len, prompts))
    # First tokens come from (chunked) prefill of the same prompt; later ones may fork on near-ties.
    agree = 0
    for i, prompt in enumerate(prompts):
        solo = greedy_generate_ids(model, prompt, budgets[i], device=dev)
        agree += int(results[i].split()[0] == str(solo[0]))
    assert agree >= 5
