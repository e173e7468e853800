"""Reranking on the host: group packing (input order, prefix repetition on overflow, 64-row alignment, refusals), the
per-row layout of a pass, ``split_shared_prefix``, the float64 references, the shim's argument checks, the C entries'
refusals and the CLI's arguments."""

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
from tiny_llm_b200.moe import Moe
from tiny_llm_b200.rerank import _check_model, group_layout, pack_groups, rerank_prompt, split_shared_prefix
from tiny_llm_b200.synthetic import pack_codes


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_rerank_ref", "rerank_ref.py")


# ---------------------------------------------------------------- packing --
def test_pack_groups_in_input_order():
    # query 0: prefix 70 (128 rows) + docs of 64, 192 and 64 rows; query 1: prefix 10 (64 rows) + one 64-row doc
    assert pack_groups([70, 10], [[5, 130, 64], [3]], 640) == [[(0, -1), (0, 0), (0, 1), (0, 2), (1, -1), (1, 0)]]
    assert pack_groups([70, 10], [[5, 130, 64], [3]], 512) == [[(0, -1), (0, 0), (0, 1), (0, 2)], [(1, -1), (1, 0)]]
    # no prefix: documents only
    assert pack_groups([0], [[5, 70]], 256) == [[(0, 0), (0, 1)]]
    assert pack_groups([], [], 128) == []
    assert pack_groups([5], [[]], 128) == []  # a query without documents lays out nothing


def test_pack_groups_repeat_the_prefix_on_overflow():
    # prefix 64 rows; docs 128, 64, 128 rows in passes of 256: [P d0 d1] then [P d2]
    assert pack_groups([64], [[100, 1, 128]], 256) == [[(0, -1), (0, 0), (0, 1)], [(0, -1), (0, 2)]]
    # one document per pass: the prefix in each
    assert pack_groups([64], [[150, 150, 150]], 256) == [[(0, -1), (0, 0)], [(0, -1), (0, 1)], [(0, -1), (0, 2)]]
    # a later small document goes back to the first pass holding its prefix that has room
    assert pack_groups([64], [[100, 128, 1]], 256) == [[(0, -1), (0, 0), (0, 2)], [(0, -1), (0, 1)]]
    # the next query fills the first pass with room for its prefix and document
    assert pack_groups([64, 1], [[64, 300], [1]], 384) == [[(0, -1), (0, 0), (1, -1), (1, 0)], [(0, -1), (0, 1)]]


def test_pack_groups_refusals():
    with pytest.raises(ValueError, match=r"query 1 document 2: a prefix of 100 tokens and a document of 150 tokens"):
        pack_groups([10, 100], [[1], [1, 2, 150]], 256)
    with pytest.raises(ValueError, match="query 0 document 1 is empty"):
        pack_groups([3], [[2, 0]], 256)
    for bad in (0, 100, -128):
        with pytest.raises(ValueError, match="multiple of 128"):
            pack_groups([1], [[1]], bad)


def test_group_layout_rows():
    P, docs = [70, 0], [[3, 64], [5]]
    entries = [(0, -1), (0, 0), (0, 1), (1, 0)]
    offsets, ctxs, seg, pst, pen, score, starts = group_layout(entries, P, docs, 512)
    assert starts == [0, 128, 192, 256]
    assert score.tolist() == [130, 255, 260]
    r = np.arange(512)
    live = np.zeros(512, dtype=bool)
    for s, n in zip(starts, [70, 3, 64, 5]):
        live[s:s + n] = True
        assert seg[s:s + n].tolist() == [s] * n
        assert ctxs[s:s + n].tolist() == list(range(s + 1, s + n + 1))
    assert offsets[0:70].tolist() == list(range(70)) and pst[0:70].tolist() == pen[0:70].tolist()  # prefix rows: no prefix
    assert offsets[128:131].tolist() == [70, 71, 72] and offsets[192:256].tolist() == list(range(70, 134))
    assert np.all(pst[128:131] == 0) and np.all(pen[128:131] == 70) and np.all(pen[192:256] == 70)
    assert offsets[256:261].tolist() == list(range(5)) and np.all(pst[256:261] == pen[256:261])  # no prefix
    assert np.all(ctxs[~live] == 0) and np.all(offsets[~live] == 0) and np.all(seg[~live] == 512)
    assert np.all(pst[~live] == pen[~live]) and np.all(seg[~live] > r[~live])
    assert np.all(pen <= seg)
    # a repeated prefix: the documents of the second pass point at the copy in that pass
    _, _, _, pst2, pen2, score2, starts2 = group_layout([(1, -1), (1, 0), (0, -1), (0, 0)], [64, 10], [[1], [2]], 256)
    assert starts2 == [0, 64, 128, 192] and score2.tolist() == [65, 192]
    assert pst2[64] == 0 and pen2[64] == 10 and pst2[192] == 128 and pen2[192] == 192


def test_split_shared_prefix():
    assert split_shared_prefix([[1, 2, 3, 4], [1, 2, 5], [1, 2, 3]]) == ([1, 2], [[3, 4], [5], [3]])
    assert split_shared_prefix([[7, 8, 9], [7, 8, 9]]) == ([7, 8], [[9], [9]])  # identical prompts keep one token each
    assert split_shared_prefix([[1, 2], [1]]) == ([], [[1, 2], [1]])  # a one-token prompt
    assert split_shared_prefix([[4, 5, 6]]) == ([4, 5], [[6]])
    assert split_shared_prefix([[1, 2], [3, 2]]) == ([], [[1, 2], [3, 2]])
    with pytest.raises(ValueError):
        split_shared_prefix([[1], []])
    with pytest.raises(ValueError):
        split_shared_prefix([])


def test_rerank_prompt_template():
    text = rerank_prompt("what is x", "x is y")
    assert text.startswith("<|im_start|>system\nJudge whether the Document meets the requirements")
    assert "<Instruct>: Given a web search query, retrieve relevant passages that answer the query\n<Query>: what is x\n<Document>: x is y" in text
    assert text.endswith("<|im_start|>assistant\n<think>\n\n</think>\n\n")
    assert "<Instruct>: mine\n" in rerank_prompt("q", "d", "mine")


# ---------------------------------------------------------------- references --
def test_prefixed_attention_reference_visibility():
    Hq, Hkv, L, D = 2, 1, 8, 4
    q = np.zeros((Hq, L, D))
    k = np.zeros((Hkv, L, D))
    v = np.arange(L, dtype=np.float64)[None, :, None].repeat(D, axis=2)
    seg = np.array([0, 0, 2, 2, 4, 4, 8, 8])
    ps = np.array([0, 0, 0, 0, 0, 0, 0, 0])
    pe = np.array([0, 0, 2, 2, 2, 2, 0, 0])
    out = R.prefixed_attention_ref(q, k, v, seg, ps, pe, 1.0, Hkv).reshape(L, Hq, D)[:, 0, 0]
    # row 3 sees 0, 1 (prefix) and 2, 3; row 5 sees 0, 1 and 4, 5; rows 6, 7 are padding
    np.testing.assert_allclose(out, [0, 0.5, 1, 1.5, 5 / 3, 2.5, 0, 0])


def test_head_weight_reference():
    codes = torch.tensor([[0, 15, 7, 1] * 32, [3] * 128])
    words = pack_codes(codes, 4)
    np.testing.assert_array_equal(R.unpack_codes(words, 4).numpy(), codes.numpy())
    scales = torch.tensor([[0.5], [2.0]], dtype=torch.bfloat16)
    biases = torch.tensor([[-1.0], [0.25]], dtype=torch.bfloat16)
    w = R.head_weights(words, scales, biases, 4)
    np.testing.assert_array_equal(w[0, :4], [-1.0, 6.5, 2.5, -0.5])
    assert np.all(w[1] == 6.25)
    logits, lp = R.select_logits_ref(np.ones((3, 128)), w, [2, 0], [1, 0])
    np.testing.assert_allclose(logits[0], [800.0, w[0].sum()])
    np.testing.assert_allclose(np.exp(lp).sum(axis=1), 1.0)


# ---------------------------------------------------------------- shim and C entries --
def test_shim_checks():
    x = torch.zeros((4, 256), dtype=torch.bfloat16)
    w = torch.zeros(256, dtype=torch.bfloat16)
    rows = torch.zeros(2, dtype=torch.int32)
    words = torch.zeros((10, 32), dtype=torch.int32)
    sc = torch.zeros((10, 2), dtype=torch.bfloat16)
    ids = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.select_logits(x, w, 1e-6, rows, words, sc, sc, ids)
    with pytest.raises(RuntimeError, match="1 to 32 token ids"):
        ext.select_logits(x, w, 1e-6, rows, words, sc, sc, torch.zeros(33, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="1 to 32 token ids"):
        ext.select_logits(x, w, 1e-6, rows, words, sc, sc, torch.zeros(0, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="4- or 8-bit"):
        ext.select_logits(x, w, 1e-6, rows, torch.zeros((10, 48), dtype=torch.int32), sc, sc, ids)  # 6 bits
    with pytest.raises(RuntimeError, match="scales and biases"):
        ext.select_logits(x, w, 1e-6, rows, words, sc.half(), sc.half(), ids)
    with pytest.raises(RuntimeError, match="int32"):
        ext.select_logits(x, w, 1e-6, rows.long(), words, sc, sc, ids)
    with pytest.raises(RuntimeError, match="float16 or bfloat16"):
        ext.select_logits(x.float(), w.float(), 1e-6, rows, words, sc, sc, ids)
    q = torch.zeros((16, 128, 128), dtype=torch.bfloat16)
    kp = torch.zeros((4, 8, 64, 128), dtype=torch.bfloat16)
    seg = torch.zeros(128, dtype=torch.int32)
    table = torch.arange(2, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="one entry per row"):
        ext.paged_attention_prefixed_segments(q, kp, kp, table, seg, seg, seg[:64], 1.0, 8, 16)
    with pytest.raises(RuntimeError, match="int32"):
        ext.paged_attention_prefixed_segments(q, kp, kp, table, seg, seg.long(), seg, 1.0, 8, 16)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.paged_attention_prefixed_segments(q, kp, kp, table, seg, seg, seg, 1.0, 8, 16)


def test_c_entries_refuse_bad_arguments():
    lib = ext._lib
    null = None
    # tl_paged_attention_prefixed_segments(q, K, V, table, seg, ps, pe, out, L, D, P, page_size, max_pages, scale, Hkv, Hq, dtype, stream)
    f = lib.tl_paged_attention_prefixed_segments
    assert f(null, null, null, null, null, null, null, null, 128, 128, 4, 64, 2, 1.0, 8, 16, 0, null) == -2  # fp32
    assert f(null, null, null, null, null, null, null, null, 128, 64, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # D
    assert f(null, null, null, null, null, null, null, null, 128, 128, 4, 96, 2, 1.0, 8, 16, 2, null) == -1  # page size
    assert f(null, null, null, null, null, null, null, null, 128, 128, 4, 64, 2, 1.0, 8, 12, 2, null) == -1  # head ratio
    assert f(null, null, null, null, null, null, null, null, 256, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # rows past the table
    assert f(16, 16, 16, 16, 16, null, 16, 16, 128, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # null prefix_start
    assert f(16, 16, 16, 16, 16, 16, null, 16, 128, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # null prefix_end
    assert f(8, 16, 16, 16, 16, 16, 16, 16, 128, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == -1  # misaligned q
    assert f(null, null, null, null, null, null, null, null, 0, 128, 4, 64, 2, 1.0, 8, 16, 2, null) == 0  # no rows
    # tl_select_logits(x, w, eps, rows, n, nrows, H, weight, scales, biases, V, bits, ids, m, logits, logprobs, dtype, stream)
    g = lib.tl_select_logits
    p = 16
    assert g(p, p, 1e-6, p, 2, 4, 256, p, p, p, 10, 4, p, 2, p, p, 0, null) == -2  # fp32
    assert g(p, p, 1e-6, p, 2, 4, 256, p, p, p, 10, 6, p, 2, p, p, 2, null) == -1  # bits
    assert g(p, p, 1e-6, p, 2, 4, 256, p, p, p, 10, 4, p, 0, p, p, 2, null) == -1  # m = 0
    assert g(p, p, 1e-6, p, 2, 4, 256, p, p, p, 10, 8, p, 33, p, p, 1, null) == -1  # m = 33
    assert g(p, p, 1e-6, p, 2, 4, 20480, p, p, p, 10, 4, p, 2, p, p, 2, null) == -1  # hidden size over the limit
    assert g(p, p, 1e-6, p, 2, 4, 200, p, p, p, 10, 4, p, 2, p, p, 2, null) == -1  # not a multiple of 128
    for i in (0, 1, 3, 7, 8, 9, 12, 14, 15):  # each pointer null in turn
        args = [p, p, 1e-6, p, 2, 4, 256, p, p, p, 10, 4, p, 2, p, p, 2, null]
        args[i] = null
        assert g(*args) == -1, i
    assert g(null, null, 1e-6, null, 0, 4, 256, null, null, null, 10, 4, null, 2, null, null, 2, null) == 0  # no rows


def test_refused_models():
    block = SimpleNamespace(mlp=Moe.__new__(Moe))
    with pytest.raises(ValueError, match="rerank: Qwen3-MoE"):
        _check_model(SimpleNamespace(layers_inner=[block], adapters=None), "cuda:0", "rerank")
    block = SimpleNamespace(mlp=object())
    with pytest.raises(ValueError, match="rerank: models with adapters"):
        _check_model(SimpleNamespace(layers_inner=[block], adapters=object()), "cuda:0", "rerank")


# ---------------------------------------------------------------- CLI --
def _args(argv):
    base = dict(prefix_ids=None, document_ids=None, query=None, document=None, documents_file=None, instruction=None, true_id=None,
                false_id=None)
    return argparse.Namespace(**{**base, **argv})


class _Tok:
    """Splits on spaces; a word's id is its length; "yes" and "no" are ids 100 and 101."""

    def encode(self, text, add_special_tokens=False):
        return [len(w) for w in text.split(" ")]

    def convert_tokens_to_ids(self, token):
        return {"yes": 100, "no": 101}[token]


def test_cli_rerank_inputs(tmp_path):
    got = cli.rerank_inputs(_args(dict(prefix_ids="5,17,3", document_ids="9,2;4,8,1", true_id=10, false_id=11)), None)
    assert got == ([5, 17, 3], [[9, 2], [4, 8, 1]], 10, 11)
    assert cli.rerank_inputs(_args(dict(document_ids="9;4", true_id=1, false_id=2)), None) == ([], [[9], [4]], 1, 2)
    f = tmp_path / "docs.txt"
    f.write_text("ab cd\n\nxyz\n")
    prefix, docs, t, n = cli.rerank_inputs(_args(dict(query="q", document=["a"], documents_file=str(f))), _Tok())
    whole = [_Tok().encode(rerank_prompt("q", d)) for d in ["a", "ab cd", "xyz"]]
    assert [prefix + d for d in docs] == whole and (t, n) == (100, 101)
    assert len(prefix) > 0
    with pytest.raises(SystemExit, match="tokenizer"):
        cli.rerank_inputs(_args(dict(query="q", document=["a"])), None)
    with pytest.raises(SystemExit, match="--true-id"):
        cli.rerank_inputs(_args(dict(document_ids="1,2")), None)
    with pytest.raises(SystemExit, match="document 1 is empty"):
        cli.rerank_inputs(_args(dict(document_ids="1,2;", true_id=1, false_id=2)), None)
    with pytest.raises(SystemExit, match="--query"):
        cli.rerank_inputs(_args(dict(document=["a"])), _Tok())


def test_cli_rerank_arguments(monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, "cmd_rerank", lambda args: (seen.__setitem__("args", args), 0)[1])
    assert cli.main(["rerank", "--synthetic", "tiny-d128", "--synthetic-bits", "8", "--prefix-ids", "5,17", "--document-ids", "9;4,8",
                     "--true-id", "10", "--false-id", "11", "--max-tokens", "256", "--device", "cuda:1"]) == 0
    a = seen["args"]
    assert (a.prefix_ids, a.document_ids, a.true_id, a.false_id, a.max_tokens, a.synthetic_bits, a.device) == \
        ("5,17", "9;4,8", 10, 11, 256, 8, "cuda:1")
    assert cli.main(["rerank", "--synthetic", "tiny-d128", "--query", "q", "--document", "a", "--document", "b", "--instruction", "i"]) == 0
    a = seen["args"]
    assert (a.query, a.document, a.instruction) == ("q", ["a", "b"], "i")
    with pytest.raises(SystemExit):
        cli.main(["rerank", "--synthetic", "tiny-d128", "--max-tokens", "0"])
    with pytest.raises(SystemExit):
        cli.main(["rerank", "--synthetic", "tiny-d128", "--true-id", "x"])
