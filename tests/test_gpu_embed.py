"""Text embeddings on the H100: the segment-causal attention kernel against a float64 reference with exact
key-visibility probes, ``tl_embed_pool`` against ``tl_rms_norm`` (bit for bit) and a float64 pooling reference, and
``embed_ids`` end to end against the operator path, bit-identical wherever a prompt lands, with every page returned."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import embed as embed_mod
from tiny_llm_b200 import embed_ids
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.qwen3_week3 import Qwen3ModelWeek3
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_embed_ref", "embed_ref.py")
DEV = "cuda:0"

# (lengths of the packed segments, rows): 1-token segments, segments crossing a 128-row query block and a page boundary
# at arbitrary starts, and tail padding rows.
LAYOUTS = {
    "mixed": ([1, 1, 70, 200, 3, 100, 1], 512),
    "aligned": ([64, 128, 1, 63, 191], 512),
    "one": ([300], 384),
}


def _segments(lengths, rows):
    seg = np.full(rows, rows, dtype=np.int32)
    r = 0
    for n in lengths:
        seg[r:r + n] = r
        r += n
    return seg, r


def _paged(k, v, page_size, gen):
    """Keys / values [Hkv, L, D] scattered over a permuted page table of a pool with spare pages."""
    Hkv, L, D = k.shape
    n = -(-L // page_size)
    P = n + 3
    table = torch.randperm(P, generator=gen)[:n].to(torch.int32)
    kp = torch.zeros((P, Hkv, page_size, D), dtype=k.dtype)
    vp = torch.full((P, Hkv, page_size, D), 0.0, dtype=v.dtype)
    for r in range(L):
        kp[table[r // page_size], :, r % page_size] = k[:, r]
        vp[table[r // page_size], :, r % page_size] = v[:, r]
    return kp.to(DEV), vp.to(DEV), table.to(DEV)


def _run_segments(q, k, v, seg, page_size, Hkv, gen, scale):
    kp, vp, table = _paged(k, v, page_size, gen)
    out = ext.paged_attention_segments(q.to(DEV), kp, vp, table, torch.from_numpy(seg).to(DEV), scale, Hkv, q.shape[0])
    torch.cuda.synchronize()
    return out.float().cpu()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("heads", [(16, 8), (32, 8)])
@pytest.mark.parametrize("page_size", [64, 128])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_segment_attention_matches_float64(dtype, heads, page_size, layout):
    Hq, Hkv = heads
    lengths, rows = LAYOUTS[layout]
    seg, used = _segments(lengths, rows)
    gen = torch.Generator().manual_seed(7)
    D = 128
    q = torch.randn((Hq, rows, D), generator=gen).to(dtype)
    k = torch.randn((Hkv, rows, D), generator=gen).to(dtype)
    v = torch.randn((Hkv, rows, D), generator=gen).to(dtype)
    scale = D ** -0.5
    got = _run_segments(q, k, v, seg, page_size, Hkv, gen, scale)
    want = R.segment_attention_ref(q.double().numpy(), k.double().numpy(), v.double().numpy(), seg, scale, Hkv)
    np.testing.assert_allclose(got.numpy(), want, rtol=2e-2, atol=2e-2)
    assert torch.all(got[used:] == 0), "padding rows see no key"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("page_size", [64, 128])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_segment_attention_exact_visibility(dtype, page_size, layout):
    """Exact probe: with all keys zero every visible key weighs exactly 1, so the output is the plain mean of the visible
    V rows.  V carries a sentinel of 1000 in dimension 1 on odd segments' keys and in dimension 2 on even ones': a row
    must read exactly 0 in its neighbours' dimension, and exactly the mean of its own visible keys everywhere."""
    Hq, Hkv, D = 16, 8, 128
    lengths, rows = LAYOUTS[layout]
    seg, used = _segments(lengths, rows)
    gen = torch.Generator().manual_seed(11)
    q = torch.randn((Hq, rows, D), generator=gen).to(dtype)
    k = torch.zeros((Hkv, rows, D), dtype=dtype)
    v = torch.randint(-4, 5, (Hkv, rows, D), generator=gen).to(dtype)
    seg_id = np.zeros(rows, dtype=np.int64)
    r = 0
    for j, n in enumerate(lengths):
        seg_id[r:r + n] = j
        r += n
    odd = torch.from_numpy(seg_id % 2 == 1)
    v[:, :, 0] = 1
    v[:, :, 1] = torch.where(odd, 1000.0, 0.0).to(dtype)
    v[:, :, 2] = torch.where(odd, 0.0, 1000.0).to(dtype)
    v[:, used:, :] = 30000.0 if dtype == torch.bfloat16 else 3000.0  # unwritten slots past the last segment
    got = _run_segments(q, k, v, seg, page_size, Hkv, gen, D ** -0.5).view(rows, Hq, D)
    want = torch.from_numpy(R.segment_attention_ref(q.double().numpy(), k.double().numpy(), v.double().numpy(), seg, D ** -0.5, Hkv))
    want = want.view(rows, Hq, D).to(dtype).float()
    live = torch.from_numpy(seg_id[:used])
    assert torch.all(got[:used, :, 0] == 1)
    assert torch.all(got[:used, :, 1][live % 2 == 0] == 0), "an even segment's row saw an odd segment's key"
    assert torch.all(got[:used, :, 2][live % 2 == 1] == 0), "an odd segment's row saw an even segment's key"
    ulp = 2.0 ** -7 if dtype == torch.bfloat16 else 2.0 ** -10
    torch.testing.assert_close(got[:used], want[:used], rtol=ulp, atol=1e-6)
    assert torch.all(got[used:] == 0)


def test_segment_attention_refuses_bad_shapes():
    q = torch.zeros((16, 128, 64), dtype=torch.bfloat16, device=DEV)
    kp = torch.zeros((4, 8, 64, 64), dtype=torch.bfloat16, device=DEV)
    seg = torch.zeros(128, dtype=torch.int32, device=DEV)
    table = torch.arange(2, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError, match="head dimension"):
        ext.paged_attention_segments(q, kp, kp, table, seg, 1.0, 8, 16)
    q = torch.zeros((16, 512, 128), dtype=torch.bfloat16, device=DEV)
    kp = torch.zeros((4, 8, 64, 128), dtype=torch.bfloat16, device=DEV)
    with pytest.raises(RuntimeError, match="do not fit"):
        ext.paged_attention_segments(q, kp, kp, table, torch.zeros(512, dtype=torch.int32, device=DEV), 1.0, 8, 16)


# ---------------------------------------------------------------- tl_embed_pool --
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("H", [256, 1024, 2560, 200])
def test_embed_pool_rows_are_rms_norm_bits(dtype, H):
    gen = torch.Generator().manual_seed(H)
    x = (torch.randn((37, H), generator=gen) * 3).to(dtype).to(DEV)
    w = (torch.rand(H, generator=gen) + 0.5).to(dtype).to(DEV)
    bounds = torch.arange(38, dtype=torch.int32, device=DEV)
    got = ext.embed_pool(x, w, 1e-6, bounds, "last", None, False)
    want = ext.rms_norm(x, w, 1e-6).float()
    assert torch.equal(got, want)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("H", [256, 1024, 2560])
@pytest.mark.parametrize("pooling", ["last", "mean"])
@pytest.mark.parametrize("dimensions", [None, 64, 100])
@pytest.mark.parametrize("normalize", [True, False])
def test_embed_pool_matches_float64(dtype, H, pooling, dimensions, normalize):
    gen = torch.Generator().manual_seed(3)
    rows = 300
    x = (torch.randn((rows, H), generator=gen) * 2).to(dtype).to(DEV)
    w = (torch.rand(H, generator=gen) + 0.5).to(dtype).to(DEV)
    bounds = np.array([0, 1, 2, 66, 67, 200, 200, 300], dtype=np.int32)  # one empty segment
    got = ext.embed_pool(x, w, 1e-6, torch.from_numpy(bounds).to(DEV), pooling, dimensions, normalize).double().cpu().numpy()
    normed = ext.rms_norm(x, w, 1e-6).double().cpu().numpy()
    want = R.pool_ref(normed, bounds, pooling, dimensions, normalize)
    scale = np.abs(want).max(axis=1, keepdims=True) + 1e-30
    assert np.all(np.abs(got - want) <= 1e-5 * scale), np.abs(got - want).max()
    assert np.all(got[5] == 0), "an empty segment pools to zeros"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("pooling", ["last", "mean"])
def test_embed_pool_zero_input_stays_zero(dtype, pooling):
    x = torch.zeros((10, 1024), dtype=dtype, device=DEV)
    w = torch.ones(1024, dtype=dtype, device=DEV)
    got = ext.embed_pool(x, w, 1e-6, torch.tensor([0, 4, 10], dtype=torch.int32, device=DEV), pooling, 512, True)
    assert torch.equal(got, torch.zeros_like(got))


# ---------------------------------------------------------------- embed_ids --
_MODELS = {}


def _model(name):
    if name not in _MODELS:
        ns = synthetic_qwen3(name, seed=0, device=DEV, realistic=name.startswith("tiny"))
        _MODELS[name] = (ns, Qwen3ModelWeek3(ns, page_size=128))
    return _MODELS[name][1]


def _operator_path(model, ids, pooling, dimensions):
    """The prompt alone through ``model.embedding`` and the ``layers_inner`` blocks as ``__call__`` runs them, then
    ``model.norm``, pooled in float64."""
    cache = model.create_kv_cache()
    try:
        h = model.embedding(torch.tensor([ids], dtype=torch.int32, device=DEV))
        for block, layer_cache in zip(model.layers_inner, cache):
            h = block(h, 0, layer_cache, mask="causal")
        normed = model.norm(h)[0].double().cpu().numpy()
    finally:
        for c in cache:
            c.release()
    return R.pool_ref(normed, [0, len(ids)], pooling, dimensions, True)[0]


def _prompts(vocab, lengths, seed):
    g = np.random.default_rng(seed)
    return [g.integers(0, vocab, size=n).tolist() for n in lengths]


@pytest.mark.parametrize("name", ["tiny-d128", "qwen3-0.6b"])
@pytest.mark.parametrize("pooling", ["last", "mean"])
def test_embed_ids_matches_operator_path(name, pooling):
    model = _model(name)
    prompts = _prompts(model.vocab_size, [1, 5, 64, 65, 130, 300], seed=1)
    got = embed_ids(model, prompts, pooling=pooling, dimensions=64 if pooling == "mean" else None, max_tokens=512).double().cpu().numpy()
    for i, p in enumerate(prompts):
        want = _operator_path(model, p, pooling, 64 if pooling == "mean" else None)
        cos = float(got[i] @ want / (np.linalg.norm(got[i]) * np.linalg.norm(want)))
        assert cos > 0.995, (i, len(p), cos)
        np.testing.assert_allclose(got[i], want, atol=2e-2, err_msg=f"prompt {i} ({len(p)} tokens)")
        assert abs(np.linalg.norm(got[i]) - 1.0) < 1e-5


@pytest.mark.parametrize("name", ["tiny-d128", "qwen3-0.6b"])
def test_embed_ids_bits_do_not_depend_on_placement(name):
    model = _model(name)
    a, b, c, p = _prompts(model.vocab_size, [37, 100, 3, 77], seed=2)
    alone = embed_ids(model, [p], max_tokens=512)
    among = embed_ids(model, [a, b, p, c], max_tokens=512)
    later = embed_ids(model, [b, c, a, b, p], max_tokens=256)  # p lands in the second pass, at another row
    assert torch.equal(alone[0], among[2])
    assert torch.equal(alone[0], embed_ids(model, [a, p], max_tokens=512)[1])
    assert torch.equal(embed_ids(model, [p], max_tokens=256)[0], later[4])
    for pooling in ("mean",):
        assert torch.equal(embed_ids(model, [p], pooling=pooling, max_tokens=512)[0],
                           embed_ids(model, [c, b, p], pooling=pooling, max_tokens=512)[2])


def test_embed_ids_input_order_and_many_passes():
    model = _model("tiny-d128")
    prompts = _prompts(model.vocab_size, [120, 5, 128, 60, 1, 128, 90, 33], seed=3)
    packed = embed_ids(model, prompts, max_tokens=256)
    for i, p in enumerate(prompts):
        assert torch.equal(packed[i], embed_ids(model, [p], max_tokens=256)[0])


def _available(model):
    return [p.pages_available() for p in model.page_pools]


def test_embed_ids_returns_every_page(monkeypatch):
    model = _model("tiny-d128")
    prompts = _prompts(model.vocab_size, [50, 200, 10, 130], seed=4)
    embed_ids(model, prompts, max_tokens=256)  # sizes the slabs
    before = _available(model)
    embed_ids(model, prompts, max_tokens=256)
    assert _available(model) == before
    with pytest.raises(ValueError, match="prompt 2 has 300 tokens"):
        embed_ids(model, prompts[:2] + [[1] * 300], max_tokens=256)
    with pytest.raises(ValueError, match="prompt 1"):
        embed_ids(model, [[1, 2], [model.vocab_size]], max_tokens=256)
    assert _available(model) == before
    calls = {"n": 0}
    real = ext.paged_attention_segments

    def failing(*a, **k):
        calls["n"] += 1
        if calls["n"] == 3:  # the second pass's first layer: the first pass returned its pages already
            raise RuntimeError("injected")
        return real(*a, **k)

    monkeypatch.setattr(embed_mod.ext, "paged_attention_segments", failing)
    with pytest.raises(RuntimeError, match="injected"):
        embed_ids(model, prompts, max_tokens=256)
    assert _available(model) == before


def test_embed_ids_refuses_adapters_and_bad_arguments():
    model = _model("tiny-d128")
    with pytest.raises(ValueError, match="multiple of 128"):
        embed_ids(model, [[1, 2]], max_tokens=200)
    with pytest.raises(ValueError, match="dimensions"):
        embed_ids(model, [[1, 2]], dimensions=model.hidden_size + 1)
    with pytest.raises(ValueError, match="pooling"):
        embed_ids(model, [[1, 2]], pooling="cls")


def test_qwen3model_checkpoint_embeds_the_same_bits(tmp_path):
    """``save_checkpoint`` of a synthetic model with its tensors renamed to the ``Qwen3Model`` layout (no ``model.``
    prefix, no ``lm_head``) loads and embeds to the same bits as the original."""
    from safetensors.torch import load_file, save_file

    ns = synthetic_qwen3("tiny-d128", seed=5, device="cpu", realistic=True)
    save_checkpoint(ns, tmp_path / "lm")
    save_checkpoint(ns, tmp_path / "embedding")
    tensors = load_file(str(tmp_path / "embedding" / "model.safetensors"))
    renamed = {k[len("model."):]: t for k, t in tensors.items() if k.startswith("model.")}
    save_file(renamed, str(tmp_path / "embedding" / "model.safetensors"))
    a = Qwen3ModelWeek3(load_checkpoint(tmp_path / "lm", device=DEV), page_size=128)
    b = Qwen3ModelWeek3(load_checkpoint(tmp_path / "embedding", device=DEV), page_size=128)
    prompts = _prompts(a.vocab_size, [9, 70], seed=6)
    assert torch.equal(embed_ids(a, prompts, max_tokens=256), embed_ids(b, prompts, max_tokens=256))


def test_cli_embed_prints_unit_vectors(capsys):
    from tiny_llm_b200 import cli

    assert cli.main(["embed", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3;9,2,4,8", "--dimensions", "64"]) == 0
    lines = [l for l in capsys.readouterr().out.splitlines() if l.startswith("[")]
    assert len(lines) == 2
    for line in lines:
        values = np.array([float(t) for t in line.split(": ", 1)[1].split()])
        assert values.shape == (64,) and abs(np.linalg.norm(values) - 1) < 1e-4
