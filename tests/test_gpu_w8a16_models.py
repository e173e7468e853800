"""8-bit (W8A16) models on an H100: a tiny-d128 model with 8-bit weights against the CPU oracle (oracle.model, whose
dequantize_weights takes 8 bits) within the 4-bit parity tolerance, and the graph engines against the operator path
with the identities their 4-bit counterparts claim."""

import pytest
import torch

from oracle.model import ReferenceCpuModel, greedy_decode
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.synthetic import synthetic_qwen3, to_device

pytestmark = pytest.mark.gpu
PROMPT = [5, 17, 3, 250, 99, 42, 7, 300, 11, 8, 1, 77, 402, 65, 9, 33, 210]


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


@pytest.fixture(scope="module")
def tiny8(dev):
    kwargs = dict(seed=0, realistic=True, max_position_embeddings=512, bits=8)
    cpu = synthetic_qwen3("tiny-d128", **kwargs)
    return cpu, to_device(synthetic_qwen3("tiny-d128", **kwargs), dev)


def logprobs(logits):
    x = logits.to(torch.float32)
    return x - torch.logsumexp(x, dim=-1, keepdim=True)


@pytest.mark.parametrize("chunk", [None, 4])
def test_8bit_model_tracks_the_reference_cpu_path(dev, tiny8, chunk):
    cpu, gpu = tiny8
    assert gpu.model.layers[0].self_attn.q_proj.weight.shape[1] * 4 == 256
    tokens, ref_lp = greedy_decode(ReferenceCpuModel(cpu), PROMPT, 10, return_logprobs=True)
    model = Qwen3ModelWeek3(gpu, page_size=8)
    model.use_decode_graph = False
    cache = model.create_kv_cache()
    try:
        offset = 0
        if chunk is not None:
            while len(PROMPT) - offset > chunk:
                model(torch.tensor([PROMPT[offset : offset + chunk]], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)
                offset += chunk
        feed = PROMPT[offset:]
        for step, (tok, lp_ref) in enumerate(zip(tokens, ref_lp)):
            lp = logprobs(model(torch.tensor([feed], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)[0, -1]).cpu()
            top = torch.topk(lp_ref, 4)
            torch.testing.assert_close(lp[top.indices], top.values, rtol=0, atol=0.25, msg=lambda m: f"step {step}: {m}")
            if float(top.values[0] - top.values[1]) > 0.5:
                assert int(torch.argmax(lp)) == tok, f"step {step}"
            offset += len(feed)
            feed = [tok]
    finally:
        for c in cache:
            c.release()
    # greedy tokens through the public path (graph engines and chunked prefill) equal the oracle's up to the first step
    # whose top-2 margin is within the stated tolerance (0.5 nat): past a near-tie the continuations may legitimately part
    margins = [float(torch.topk(lp, 2).values[0] - torch.topk(lp, 2).values[1]) for lp in ref_lp]
    agree = next((i for i, m in enumerate(margins) if m <= 0.5), len(tokens))
    got = greedy_generate_ids(Qwen3ModelWeek3(gpu, page_size=8), PROMPT, 10, device=dev)
    assert got[:agree] == tokens[:agree]


def _prefill(model, dev, prompt):
    cache = model.create_kv_cache()
    was = model.use_decode_graph
    model.use_decode_graph = False
    logits = model(torch.tensor([prompt], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
    model.use_decode_graph = was
    return cache, int(torch.argmax(logits[0, -1].float()))


@pytest.mark.parametrize("mode", ["graph-unfused", "graph-fused"])
def test_8bit_decode_graph_matches_the_operator_path(dev, tiny8, mode):
    """The unfused step graph replays the operator path's launches: bit-identical, as at 4 bits.  The fused graph runs
    the 8-bit streaming and wgmma kernels with fused prologues and epilogues: within the 4-bit test's tolerance."""
    _, gpu = tiny8
    fused = mode != "graph-unfused"
    ref_model = Qwen3ModelWeek3(gpu, page_size=8)
    ref_model.use_decode_graph = False
    model = Qwen3ModelWeek3(gpu, page_size=8)
    engine = DecodeEngine(model, 1, 256, dev, fused=fused)
    engine.reserve_pools()
    ref_cache, tok = _prefill(ref_model, dev, PROMPT[:11])
    cache, tok2 = _prefill(model, dev, PROMPT[:11])
    assert tok == tok2
    offset = 11
    for step in range(12):
        want = ref_model(torch.tensor([[tok]], dtype=torch.int32, device=dev), offset, ref_cache, logits_to_keep=1)
        got, nxt = engine.step([tok], [offset], cache)
        if fused:
            torch.testing.assert_close(got.float().view_as(want), want.float(), rtol=0, atol=0.06)
        else:
            assert torch.equal(got.view_as(want), want), f"step {step}"
        assert int(nxt[0]) == int(torch.argmax(got.float().reshape(-1)))
        tok = int(torch.argmax(want[0, -1].float()))
        offset += 1
    for c in (*cache, *ref_cache):
        c.release()


def test_8bit_device_resident_loop_equals_host_loop(dev, tiny8):
    _, gpu = tiny8
    prompt, steps = [9, 2, 4, 6, 8, 10, 12], 16

    def run(on_device):
        model = Qwen3ModelWeek3(gpu, page_size=8)
        engine = DecodeEngine(model, 1, 256, dev)
        engine.reserve_pools()
        cache, tok = _prefill(model, dev, prompt)
        if on_device:
            out = engine.decode_on_device([tok], [len(prompt)], cache, steps).cpu().reshape(-1).tolist()
        else:
            out, offset = [], len(prompt)
            for _ in range(steps):
                _, nxt = engine.step([tok], [offset], cache)
                tok = int(nxt[0])
                out.append(tok)
                offset += 1
        for c in cache:
            c.release()
        return out

    assert run(True) == run(False)


def test_8bit_public_call_and_embeddings_run_on_the_8bit_kernels(dev, tiny8):
    """The public model call (decode graph on) gives the operator path's greedy tokens, and embed_ids pools the same
    hidden states wherever a prompt is placed."""
    from tiny_llm_b200.embed import embed_ids

    _, gpu = tiny8
    plain = Qwen3ModelWeek3(gpu, page_size=8)
    plain.use_decode_graph = False
    auto = Qwen3ModelWeek3(gpu, page_size=8)
    assert greedy_generate_ids(auto, PROMPT, 12, device=dev) == greedy_generate_ids(plain, PROMPT, 12, device=dev)
    model = Qwen3ModelWeek3(gpu, page_size=128)
    a = embed_ids(model, [PROMPT, [1, 2, 3]], max_tokens=256)
    b = embed_ids(model, [[7, 7], PROMPT], max_tokens=256)
    assert torch.equal(torch.as_tensor(a[0]), torch.as_tensor(b[1]))
