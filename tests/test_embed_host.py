"""Text embeddings on the host: first-fit packing and the too-long-prompt error, the per-row positions, slots and
segment starts of a pass, the float64 pooling reference (last / mean, truncation, a zero vector), the CLI's
arguments, the model refusals, the C entries' argument errors and loading the ``Qwen3Model`` tensor naming."""

import argparse
import importlib.util
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import cli
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.embed import SEGMENT_ALIGN, _check_model, pack_prompts, pass_layout
from tiny_llm_b200.moe import Moe
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_embed_ref", "embed_ref.py")


def test_pack_first_fit_in_input_order():
    # aligned sizes 64, 256, 64, 192, 64, 128 in passes of 256
    assert pack_prompts([50, 200, 10, 130, 64, 100], 256) == [[0, 2, 4], [1], [3], [5]]
    assert pack_prompts([1] * 5, 256) == [[0, 1, 2, 3]] + [[4]]
    assert pack_prompts([256, 1, 255], 256) == [[0], [1], [2]]
    assert pack_prompts([], 128) == []


def test_pack_refuses_bad_prompts_and_sizes():
    with pytest.raises(ValueError, match=r"prompt 2 has 300 tokens, more than max_tokens=256"):
        pack_prompts([3, 4, 300, 5], 256)
    with pytest.raises(ValueError, match="prompt 1 is empty"):
        pack_prompts([3, 0], 256)
    for bad in (0, 100, 200, -128):
        with pytest.raises(ValueError, match="multiple of 128"):
            pack_prompts([3], bad)


def test_pass_layout_rows():
    offsets, ctxs, seg, bounds = pass_layout([3, 1, 70], 256)
    starts = [0, SEGMENT_ALIGN, 2 * SEGMENT_ALIGN]
    assert bounds.tolist() == [0, 3, 64, 65, 128, 198]
    for s, n in zip(starts, [3, 1, 70]):
        assert offsets[s:s + n].tolist() == list(range(n))  # RoPE positions within the prompt
        assert ctxs[s:s + n].tolist() == list(range(s + 1, s + n + 1))  # row r appends at slot r
        assert seg[s:s + n].tolist() == [s] * n
    pad = np.ones(256, dtype=bool)
    for s, n in zip(starts, [3, 1, 70]):
        pad[s:s + n] = False
    assert np.all(ctxs[pad] == 0) and np.all(offsets[pad] == 0) and np.all(seg[pad] == 256)
    assert np.all(seg[pad] > np.arange(256)[pad]), "padding rows see no key"
    with pytest.raises(ValueError):
        pass_layout([200, 100], 256)


def test_pool_reference():
    rows = np.array([[3.0, 4.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 0.0], [2.0, 2.0, 1.0]])
    np.testing.assert_allclose(R.pool_ref(rows, [0, 2, 4], "last", None, False), [[1, 0, 0], [2, 2, 1]])
    np.testing.assert_allclose(R.pool_ref(rows, [0, 2, 4], "mean", None, False), [[2, 2, 0], [1, 1, 0.5]])
    np.testing.assert_allclose(R.pool_ref(rows, [0, 1], "last", 2, True), [[0.6, 0.8]])
    np.testing.assert_allclose(R.pool_ref(rows, [2, 3], "last", None, True), [[0, 0, 0]])  # zero stays zero
    np.testing.assert_allclose(R.pool_ref(rows, [1, 1, 2], "mean", 2, True), [[0, 0], [1, 0]])  # empty segment: zeros


def test_segment_attention_reference_visibility():
    Hq, Hkv, L, D = 2, 1, 6, 4
    q = np.zeros((Hq, L, D))
    k = np.zeros((Hkv, L, D))
    v = np.arange(L, dtype=np.float64)[None, :, None].repeat(D, axis=2)
    seg = np.array([0, 0, 2, 2, 2, 6])
    out = R.segment_attention_ref(q, k, v, seg, 1.0, Hkv).reshape(L, Hq, D)[:, 0, 0]
    np.testing.assert_allclose(out, [0, 0.5, 2, 2.5, 3, 0])


def _args(argv):
    return argparse.Namespace(**{**dict(prompt_ids=None, prompt=None, prompts_file=None, append_eos=False), **argv})


def test_cli_embed_inputs(tmp_path):
    assert cli.embed_inputs(_args(dict(prompt_ids="5,17,3;9,2,4,8")), None) == [[5, 17, 3], [9, 2, 4, 8]]
    tok = SimpleNamespace(encode=lambda t, add_special_tokens=False: [len(w) for w in t.split()], eos_token_id=7)
    f = tmp_path / "p.txt"
    f.write_text("ab c\n\nxyz\n")
    assert cli.embed_inputs(_args(dict(prompt=["a bb"], prompts_file=str(f), append_eos=True)), tok) == [[1, 2, 7], [2, 1, 7], [3, 7]]
    with pytest.raises(SystemExit, match="tokenizer"):
        cli.embed_inputs(_args(dict(prompt=["hello"])), None)
    with pytest.raises(SystemExit, match="EOS"):
        cli.embed_inputs(_args(dict(prompt_ids="1,2", append_eos=True)), None)
    with pytest.raises(SystemExit, match="prompt 1 is empty"):
        cli.embed_inputs(_args(dict(prompt_ids="1,2;")), None)


def test_cli_embed_arguments(monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, "cmd_embed", lambda args: (seen.__setitem__("args", args), 0)[1])
    assert cli.main(["embed", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3;9,2,4,8", "--dimensions", "64", "--pooling", "mean",
                     "--no-normalize", "--max-tokens", "256", "--out", "e.npy"]) == 0
    a = seen["args"]
    assert (a.pooling, a.dimensions, a.no_normalize, a.max_tokens, a.out, a.prompt_ids) == ("mean", 64, True, 256, "e.npy", "5,17,3;9,2,4,8")
    with pytest.raises(SystemExit):
        cli.main(["embed", "--synthetic", "tiny-d128", "--pooling", "cls"])
    with pytest.raises(SystemExit):
        cli.main(["embed", "--synthetic", "tiny-d128", "--dimensions", "0"])


def test_refused_models():
    block = SimpleNamespace(mlp=Moe.__new__(Moe))
    with pytest.raises(ValueError, match="MoE"):
        _check_model(SimpleNamespace(layers_inner=[block], adapters=None), "cuda:0")
    block = SimpleNamespace(mlp=object())
    with pytest.raises(ValueError, match="adapters"):
        _check_model(SimpleNamespace(layers_inner=[block], adapters=object()), "cuda:0")


def test_c_entries_refuse_bad_arguments():
    lib = ext._lib
    null = None
    # tl_paged_attention_segments(q, K, V, table, seg, out, L, D, P, page_size, max_pages, scale, Hkv, Hq, dtype, stream)
    assert lib.tl_paged_attention_segments(null, null, null, null, null, null, 128, 128, 4, 64, 2, 1.0, 8, 16, 0, null) == -2
    assert lib.tl_paged_attention_segments(null, null, null, null, null, null, 128, 64, 4, 64, 2, 1.0, 8, 16, 2, null) == -1
    assert lib.tl_paged_attention_segments(null, null, null, null, null, null, 128, 128, 4, 96, 2, 1.0, 8, 16, 2, null) == -1
    assert lib.tl_paged_attention_segments(null, null, null, null, null, null, 128, 128, 4, 64, 2, 1.0, 8, 12, 2, null) == -1
    assert lib.tl_paged_attention_segments(null, null, null, null, null, null, 256, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1
    assert lib.tl_paged_attention_segments(null, null, null, null, null, null, 128, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # null
    assert lib.tl_paged_attention_segments(8, 16, 16, 16, 16, 16, 128, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # misaligned q
    # tl_embed_pool(x, w, eps, seg, n, rows, H, d, pooling, normalize, out, dtype, stream)
    assert lib.tl_embed_pool(null, null, 1e-6, null, 1, 4, 256, 64, 0, 1, null, 0, null) == -2
    assert lib.tl_embed_pool(null, null, 1e-6, null, 1, 4, 256, 0, 0, 1, null, 2, null) == -1
    assert lib.tl_embed_pool(null, null, 1e-6, null, 1, 4, 256, 257, 0, 1, null, 2, null) == -1
    assert lib.tl_embed_pool(null, null, 1e-6, null, 1, 4, 256, 64, 2, 1, null, 2, null) == -1
    assert lib.tl_embed_pool(null, null, 1e-6, null, 1, 4, 20000, 64, 0, 1, null, 2, null) == -1
    assert lib.tl_embed_pool(null, null, 1e-6, null, 1, 4, 256, 64, 0, 1, null, 2, null) == -1  # null
    assert lib.tl_embed_pool(null, null, 1e-6, null, 0, 4, 256, 64, 1, 1, null, 2, null) == 0  # nothing to pool


def test_load_qwen3model_naming(tmp_path):
    ns = synthetic_qwen3("tiny-d128", seed=1, realistic=True)
    save_checkpoint(ns, tmp_path / "lm")
    save_checkpoint(ns, tmp_path / "emb")
    from safetensors.torch import load_file, save_file

    tensors = load_file(str(tmp_path / "emb" / "model.safetensors"))
    assert "model.embed_tokens.weight" in tensors
    save_file({k[len("model."):]: t for k, t in tensors.items() if k.startswith("model.")}, str(tmp_path / "emb" / "model.safetensors"))
    a, b = load_checkpoint(tmp_path / "lm"), load_checkpoint(tmp_path / "emb")
    assert b.args.tie_word_embeddings and not hasattr(b, "lm_head")
    assert torch.equal(a.model.embed_tokens.weight, b.model.embed_tokens.weight)
    assert torch.equal(a.model.norm.weight, b.model.norm.weight)
    for la, lb in zip(a.model.layers, b.model.layers):
        for part in ("q_proj", "k_proj", "v_proj", "o_proj"):
            for f in ("weight", "scales", "biases"):
                assert torch.equal(getattr(getattr(la.self_attn, part), f), getattr(getattr(lb.self_attn, part), f))
        for part in ("gate_proj", "up_proj", "down_proj"):
            assert torch.equal(getattr(la.mlp, part).weight, getattr(lb.mlp, part).weight)
        assert torch.equal(la.input_layernorm.weight, lb.input_layernorm.weight)
        assert torch.equal(la.self_attn.k_norm.weight, lb.self_attn.k_norm.weight)
