"""Qwen3-MoE checkpoints on the H100: the 8-bit group-64 router kernel (tl_moe_router) against float64 and by exact
probes, its RMSNorm prologue bit for bit against rms_norm, every engine form of a layer with such a router against
the operator form, and models saved and loaded from disk (both router layouts) against the in-memory model through
every serving path."""

import importlib.util
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import BatchingKvCache, ContinuousBatcher, Qwen3ModelWeek3, greedy_generate_ids
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.synthetic import pack_codes, synthetic_qwen3, to_device

pytestmark = pytest.mark.gpu
BF, F16 = torch.bfloat16, torch.float16
ROOT = Path(__file__).resolve().parent.parent
G64 = dict(router_bits=8, router_group_size=64)
LAYOUTS = {"g128": {}, "g64": G64}


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_moe_router_ref", "moe_router_ref.py")


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def random_router(E, H, dtype, g, dev):
    codes = torch.randint(0, 256, (E, H), generator=g)
    scales = (torch.randn(E, H // 64, generator=g) * 0.004).to(dtype)
    biases = (-127.5 * scales.float() + torch.randn(E, H // 64, generator=g) * 0.03).to(dtype)
    return pack_codes(codes, 8).view(torch.int32).to(dev), scales.to(dev), biases.to(dev)


# ------------------------------------------------------------------------------------------------- the kernel --
@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("E", [8, 128, 256])
@pytest.mark.parametrize("H", [256, 2048])
@pytest.mark.parametrize("T", [1, 2, 8, 9, 64, 128, 129, 4096])
def test_router_within_the_float64_bound(dev, dtype, E, H, T):
    g = torch.Generator().manual_seed(T * 7 + E + H)
    w, s, b = random_router(E, H, dtype, g, dev)
    x = (torch.randn(T, H, generator=g) * 2).to(dtype).to(dev)
    got = ext.moe_router(x, w, s, b)
    assert got.shape == (T, E) and got.dtype == dtype
    ref, bound = R.router_ref(x, w, s, b)
    err = (got.to(torch.float64) - ref).abs()
    assert bool((err <= bound).all()), f"max excess {float((err - bound).max())}"


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
def test_router_row_depends_only_on_that_row(dev, dtype):
    """The decode-sized (16 x 8) and prefill-sized (32 x 32) tiles give the same bits for the same row."""
    g = torch.Generator().manual_seed(5)
    w, s, b = random_router(128, 2048, dtype, g, dev)
    x = torch.randn(4096, 2048, generator=g).to(dtype).to(dev)
    full = ext.moe_router(x, w, s, b)
    for lo, hi in ((0, 1), (5, 13), (1000, 1129), (4000, 4096)):
        assert torch.equal(ext.moe_router(x[lo:hi].contiguous(), w, s, b), full[lo:hi]), (lo, hi)


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("T", [3, 2048])
def test_router_exact_probes(dev, dtype, T):
    """One non-zero input per row, at a group edge: the logit is exactly T(fp32(scale * code * a + bias * a)).  Codes
    0 / 128 / 255 at columns 63 / 64 / 127 / 128, plus bias-only (scale 0) and scale-only (bias 0) groups."""
    E, H = 8, 256
    probes = [(col, a) for col in (63, 64, 127, 128) for a in (1.0, -0.5, 3.0)]
    g = torch.Generator().manual_seed(1)
    codes = torch.randint(0, 256, (E, H), generator=g)
    codes[:, 63], codes[:, 64], codes[:, 127], codes[:, 128] = 0, 128, 255, 255
    codes[1:4, 64] = torch.tensor([0, 255, 7])
    scales = (torch.rand(E, H // 64, generator=g) * 0.25 + 0.01).to(dtype)
    biases = (torch.randn(E, H // 64, generator=g) * 2).to(dtype)
    scales[4, :] = 0  # bias-only expert
    biases[5, :] = 0  # scale-only expert
    x = torch.zeros(T, H, dtype=dtype)
    for t in range(T):
        col, a = probes[t % len(probes)]
        x[t, col] = a
    got = ext.moe_router(x.to(dev), pack_codes(codes, 8).view(torch.int32).to(dev), scales.to(dev), biases.to(dev)).cpu()
    for t in range(T):
        col, a = probes[t % len(probes)]
        grp = col // 64
        for e in range(E):
            want = R.probe_value(float(scales[e, grp]), int(codes[e, col]), float(biases[e, grp]), a, dtype)
            assert float(got[t, e]) == want, (t, e, col, a)


@pytest.mark.parametrize("dtype", [BF, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("H", [256, 2048])
@pytest.mark.parametrize("T", [1, 8, 64, 129, 4096])
def test_router_prologue_equals_rms_norm_then_router(dev, dtype, H, T):
    g = torch.Generator().manual_seed(T + H)
    w, s, b = random_router(128, H, dtype, g, dev)
    x = (torch.randn(T, H, generator=g) * 3).to(dtype).to(dev)
    nw = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).to(dev)
    want = ext.moe_router(ext.rms_norm(x, nw, 1e-6), w, s, b)
    assert torch.equal(ext.moe_router(x, w, s, b, nw, 1e-6), want)


# ------------------------------------------------------------------------------------------------- the layer --
def wide_args():
    return dict(num_hidden_layers=2, vocab_size=4096, max_position_embeddings=4096)


@pytest.fixture(scope="module")
def wide_g64(dev):
    return synthetic_qwen3("qwen3-30b-a3b", seed=2, device=dev, **G64, **wide_args())


@pytest.mark.parametrize("T", [1, 8, 16, 64, 256])
def test_every_engine_form_of_a_g64_router_layer_equals_the_operator_form(dev, wide_g64, T):
    from tiny_llm_b200.engine import _moe_mlp

    model = Qwen3ModelWeek3(wide_g64, page_size=128)
    block, nxt = model.layers_inner[0], model.layers_inner[1].input_layernorm
    moe, ln2 = block.mlp, block.post_attention_layernorm
    assert (moe.w_router.bits, moe.w_router.group_size) == (8, 64)
    x = (torch.randn(T, 2048, generator=torch.Generator().manual_seed(T)) * 3).to(BF).to(dev)
    w2, wn = ln2._weight_as(BF, dev), nxt._weight_as(BF, dev)
    h = ext.rms_norm(x, w2, ln2.eps)
    op = ext.add(x, moe(h))
    op_next = ext.rms_norm(op, wn, nxt.eps)
    if T <= 64:
        assert torch.equal(_moe_mlp(moe, x, ln2=ln2), op), "matvec form (router with the RMSNorm prologue)"
    got, got_next = _moe_mlp(moe, x, h, nxt=nxt)
    assert torch.equal(got, op), "swap-AB form"
    assert torch.equal(got_next, op_next), "swap-AB form: next RMSNorm"
    assert torch.equal(_moe_mlp(moe, x, h), op), "operator-path form of the graph engines"


# ------------------------------------------------------------------------------------------ loaded checkpoints --
PROMPT = [5, 17, 3, 250, 99, 42, 7, 300, 11, 8, 1, 77, 402, 65, 9, 33, 210]


@pytest.fixture(scope="module", params=sorted(LAYOUTS))
def pair(request, dev, tmp_path_factory):
    """(in-memory model namespace, the same saved and loaded, layout)."""
    ns = synthetic_qwen3("tiny-moe-d128", seed=0, realistic=True, max_position_embeddings=512, **LAYOUTS[request.param])
    path = tmp_path_factory.mktemp(f"tiny_moe_{request.param}")
    save_checkpoint(ns, path)
    return to_device(ns, dev), load_checkpoint(path, device=dev), request.param


def prefill_logits(model, dev, ids, graph_len=0):
    model.prefill_graph_len = graph_len
    cache = model.create_kv_cache()
    try:
        return model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1).float().cpu()
    finally:
        for c in cache:
            c.release()


def test_loaded_model_gives_the_operator_path_bits(dev, pair):
    mem, disk, layout = pair
    a, b = Qwen3ModelWeek3(mem, page_size=128), Qwen3ModelWeek3(disk, page_size=128)
    assert (b.layers_inner[1].mlp.w_router.group_size == 64) == (layout == "g64")
    assert torch.equal(prefill_logits(a, dev, PROMPT), prefill_logits(b, dev, PROMPT))


def test_loaded_model_gives_the_greedy_tokens_of_generate(dev, pair):
    mem, disk, _ = pair
    want = greedy_generate_ids(Qwen3ModelWeek3(mem, page_size=128), PROMPT, 12, device=dev)
    assert greedy_generate_ids(Qwen3ModelWeek3(disk, page_size=128), PROMPT, 12, device=dev) == want


def test_loaded_model_gives_the_prefill_graph_bits(dev, pair):
    mem, disk, _ = pair
    out = []
    for ns in (mem, disk):
        model = Qwen3ModelWeek3(ns, page_size=128)
        model.decode_engine(1, 512)  # the page reservation the prefill graph needs
        out.append(prefill_logits(model, dev, PROMPT, graph_len=32))  # the whole prompt is one chunk
        assert model._prefill_engines, "the prefill graph ran"
    assert torch.equal(out[0], out[1])


@pytest.mark.parametrize("B", [1, 4, 16])
def test_loaded_model_gives_the_decode_engine_bits(dev, pair, B):
    mem, disk, _ = pair
    slots = {b: [(7 * b + i) % 500 + 1 for i in range(3 + b)] for b in range(0, B, 3)}

    def run(ns):
        model = Qwen3ModelWeek3(ns, page_size=128)
        engine = model.decode_engine(B, 256)
        tables = [BatchingKvCache(B, max_seq_len=256) for _ in range(model.num_hidden_layers)]
        for slot, ids in slots.items():
            cache = model.create_kv_cache()
            model.use_decode_graph = False
            model(torch.tensor([ids], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
            for layer_cache, table in zip(cache, tables):
                table.add_request(layer_cache, slot)
        tokens = [5 * b + 1 if b in slots else 0 for b in range(B)]
        offsets = [len(slots[b]) if b in slots else 0 for b in range(B)]
        out = []
        for _ in range(4):
            logits, nxt = engine.step(tokens, offsets, tables)
            out.append(logits.float().cpu())
            tokens = [int(t) if b in slots else 0 for b, t in enumerate(nxt.tolist())]
            offsets = [o + 1 if b in slots else 0 for b, o in enumerate(offsets)]
        return out

    for a, b in zip(run(mem), run(disk)):
        assert torch.equal(a, b)


def test_loaded_model_gives_the_batcher_tokens(dev, pair):
    mem, disk, _ = pair
    g = torch.Generator().manual_seed(7)
    prompts = [torch.randint(1, 500, (n,), generator=g).tolist() for n in (5, 19, 3, 12)]

    def run(ns):
        model = Qwen3ModelWeek3(ns, page_size=128)
        batcher = ContinuousBatcher(model, None, prompts, max_seq_len=128, batch_size=16, prefill_step=8, verbose=False, device=dev,
                                    max_new_tokens=[8] * len(prompts))
        return dict(batcher.run())

    assert run(disk) == run(mem)


def test_saved_30b_a3b_shaped_model_tracks_the_operator_path(dev, tmp_path):
    """Two sparse layers of the Qwen3-30B-A3B shape with g64 routers, saved and loaded: the loaded model's operator path
    gives the in-memory model's bits, and its prefill graph tracks it within the model tolerance."""
    ns = synthetic_qwen3("qwen3-30b-a3b", seed=4, **G64, **wide_args())
    save_checkpoint(ns, tmp_path)
    mem, disk = to_device(ns, dev), load_checkpoint(tmp_path, device=dev)
    ids = torch.randint(0, 4096, (40,), generator=torch.Generator().manual_seed(4)).tolist()
    want = prefill_logits(Qwen3ModelWeek3(mem, page_size=128), dev, ids)
    assert torch.equal(prefill_logits(Qwen3ModelWeek3(disk, page_size=128), dev, ids), want)
    model = Qwen3ModelWeek3(disk, page_size=128)
    model.decode_engine(1, 4096)
    graph = prefill_logits(model, dev, ids, graph_len=128)
    assert model._prefill_engines
    norm = lambda t: t[0, -1] - torch.logsumexp(t[0, -1], dim=-1)
    assert float((norm(graph) - norm(want)).abs().max()) <= 0.25


def test_cli_generates_the_synthetic_tokens_from_a_saved_checkpoint(tmp_path):
    save_checkpoint(synthetic_qwen3("tiny-moe-d128", seed=0, realistic=True), tmp_path)

    def run(*source):
        cmd = [sys.executable, "-m", "tiny_llm_b200.cli", "generate", *source, "--prompt-ids", "5,17,3", "--max-new-tokens", "8"]
        env = {**os.environ, "PYTHONPATH": f"{ROOT}:{ROOT / 'tiny-llm_b200'}"}
        return subprocess.run(cmd, capture_output=True, text=True, check=True, cwd=ROOT, env=env).stdout

    assert run("--model", str(tmp_path)) == run("--synthetic", "tiny-moe-d128")
