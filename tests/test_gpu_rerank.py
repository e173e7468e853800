"""Reranking on the H100: prefixed-segment attention against a float64 reference with exact key-visibility probes and
bit for bit against segment attention when every prefix is empty, ``tl_select_logits`` against a float64 reference
built on ``tl_rms_norm``'s output, and ``rerank_ids`` end to end: bit-identical whether a prefix is shared and wherever
a document lands, against the model's own path, with every page returned."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import rerank as rerank_mod
from tiny_llm_b200 import rerank_ids
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.quantize import quantized_linear
from tiny_llm_b200.qwen3_week3 import Qwen3ModelWeek3
from tiny_llm_b200.rerank import group_layout
from tiny_llm_b200.synthetic import pack_codes, synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_rerank_ref", "rerank_ref.py")
DEV = "cuda:0"

# (prefix lengths, document lengths, entries in row order, rows): several documents per prefix, several prefixes per
# pass (one empty), lengths that are not multiples of 64, a prefix shorter than a tile, and tail padding.
LAYOUTS = {
    "multi": ([70, 0, 1], [[3, 64, 130], [5], [1, 200]],
              [(0, -1), (0, 0), (0, 1), (0, 2), (1, 0), (2, -1), (2, 0), (2, 1)], 1024),
    "one": ([130], [[64, 1, 100, 63]], [(0, -1), (0, 0), (0, 1), (0, 2), (0, 3)], 640),
}


def _layout(name):
    P, docs, entries, rows = LAYOUTS[name]
    offsets, ctxs, seg, pst, pen, score, starts = group_layout(entries, P, docs, rows)
    spans = [(s, s + (P[q] if d < 0 else docs[q][d]), q, d) for (q, d), s in zip(entries, starts)]
    return seg, pst, pen, spans, rows


def _paged(k, v, page_size, gen):
    """Keys / values [Hkv, L, D] scattered over a permuted page table of a pool with spare pages."""
    Hkv, L, D = k.shape
    n = -(-L // page_size)
    P = n + 3
    table = torch.randperm(P, generator=gen)[:n].to(torch.int32)
    kp = torch.zeros((P, Hkv, page_size, D), dtype=k.dtype)
    vp = torch.zeros((P, Hkv, page_size, D), dtype=v.dtype)
    for r in range(L):
        kp[table[r // page_size], :, r % page_size] = k[:, r]
        vp[table[r // page_size], :, r % page_size] = v[:, r]
    return kp.to(DEV), vp.to(DEV), table.to(DEV)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(DEV)


def _run(q, k, v, seg, pst, pen, page_size, Hkv, scale, seed=0):
    kp, vp, table = _paged(k, v, page_size, torch.Generator().manual_seed(seed))
    out = ext.paged_attention_prefixed_segments(q.to(DEV), kp, vp, table, _dev(seg), _dev(pst), _dev(pen), scale, Hkv, q.shape[0])
    torch.cuda.synchronize()
    return out.cpu()


def _qkv(Hq, Hkv, rows, dtype, seed):
    gen = torch.Generator().manual_seed(seed)
    D = 128
    return (torch.randn((Hq, rows, D), generator=gen).to(dtype), torch.randn((Hkv, rows, D), generator=gen).to(dtype),
            torch.randn((Hkv, rows, D), generator=gen).to(dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("heads", [(16, 8), (32, 8), (64, 8)])
@pytest.mark.parametrize("page_size", [64, 128])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_prefixed_attention_matches_float64(dtype, heads, page_size, layout):
    Hq, Hkv = heads
    seg, pst, pen, spans, rows = _layout(layout)
    q, k, v = _qkv(Hq, Hkv, rows, dtype, 7)
    scale = 128 ** -0.5
    got = _run(q, k, v, seg, pst, pen, page_size, Hkv, scale).float()
    want = R.prefixed_attention_ref(q.double().numpy(), k.double().numpy(), v.double().numpy(), seg, pst, pen, scale, Hkv)
    np.testing.assert_allclose(got.numpy(), want, rtol=2e-2, atol=2e-2)
    live = np.zeros(rows, dtype=bool)
    for a, b, _, _ in spans:
        live[a:b] = True
    assert torch.all(got[torch.from_numpy(~live)] == 0), "padding rows see no key"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("page_size", [64, 128])
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_prefixed_attention_exact_visibility(dtype, page_size, layout):
    """For every segment: a sentinel in K and V of every key its rows must not see (sibling documents, other queries'
    prefixes, alignment gaps, padding rows) leaves their output bit for bit unchanged; changing one key they must see
    (the first of their prefix, else their own first key) changes it."""
    Hq, Hkv = 32, 8
    seg, pst, pen, spans, rows = _layout(layout)
    q, k, v = _qkv(Hq, Hkv, rows, dtype, 11)
    big = 30000.0 if dtype == torch.bfloat16 else 3000.0
    scale = 128 ** -0.5
    base = _run(q, k, v, seg, pst, pen, page_size, Hkv, scale)
    for a, b, _, _ in spans:
        visible = np.zeros(rows, dtype=bool)
        visible[a:b] = True
        visible[pst[a]:pen[a]] = True
        hidden = torch.from_numpy(~visible)
        k2, v2 = k.clone(), v.clone()
        k2[:, hidden] = big
        v2[:, hidden] = -big
        probed = _run(q, k2, v2, seg, pst, pen, page_size, Hkv, scale)
        assert torch.equal(probed[a:b], base[a:b]), f"rows {a}..{b - 1} saw a key outside their prefix and segment"
        first = pst[a] if pen[a] > pst[a] else a
        v3 = v.clone()
        v3[:, first] = big
        changed = _run(q, k, v3, seg, pst, pen, page_size, Hkv, scale)
        assert not torch.equal(changed[b - 1], base[b - 1]), f"row {b - 1} did not see key {first}"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("heads", [(16, 8), (32, 8)])
def test_empty_prefixes_equal_segment_attention(dtype, heads):
    Hq, Hkv = heads
    seg, pst, pen, spans, rows = _layout("multi")
    q, k, v = _qkv(Hq, Hkv, rows, dtype, 5)
    zero = np.zeros(rows, dtype=np.int32)
    got = _run(q, k, v, seg, zero, zero, 128, Hkv, 0.088)
    kp, vp, table = _paged(k, v, 128, torch.Generator().manual_seed(0))
    want = ext.paged_attention_segments(q.to(DEV), kp, vp, table, _dev(seg), 0.088, Hkv, Hq).cpu()
    assert torch.equal(got, want)


def test_prefixed_attention_spans_two_prefixes_in_one_cta():
    """Head ratio 1: a CTA's 128 rows cover two 64-row blocks whose documents have different prefixes (the hull case)."""
    P, docs, entries, rows = [64, 64], [[64], [64]], [(0, -1), (1, -1), (0, 0), (1, 0)], 256
    offsets, ctxs, seg, pst, pen, score, starts = group_layout(entries, P, docs, rows)
    q, k, v = _qkv(8, 8, rows, torch.bfloat16, 3)
    got = _run(q, k, v, seg, pst, pen, 64, 8, 0.088).float()
    want = R.prefixed_attention_ref(q.double().numpy(), k.double().numpy(), v.double().numpy(), seg, pst, pen, 0.088, 8)
    np.testing.assert_allclose(got.numpy(), want, rtol=2e-2, atol=2e-2)


# ---------------------------------------------------------------- tl_select_logits --
def _head(V, H, bits, dtype, gen):
    codes = torch.randint(0, 1 << bits, (V, H), generator=gen)
    scales = (torch.rand((V, H // 128), generator=gen) * 0.02 + 0.001).to(dtype)
    biases = (-(1 << (bits - 1)) * scales.float() + torch.randn((V, H // 128), generator=gen) * 0.01).to(dtype)
    return pack_codes(codes, bits), scales, biases


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("m", [1, 2, 32])
@pytest.mark.parametrize("H", [256, 1024])
def test_select_logits_matches_float64(dtype, bits, m, H):
    gen = torch.Generator().manual_seed(bits * 100 + m + H)
    V, rows = 1000, 37
    words, scales, biases = _head(V, H, bits, dtype, gen)
    x = (torch.randn((rows, H), generator=gen) * 3).to(dtype)
    w = (torch.rand(H, generator=gen) + 0.5).to(dtype)
    ids = [0, V - 1] + torch.randint(0, V, (30,), generator=gen).tolist()
    ids = ids[:m] if m > 1 else [V - 1]
    row_index = [0, rows - 1, 5, 17, 5]
    logits, logprobs = ext.select_logits(x.to(DEV), w.to(DEV), 1e-6, _dev(row_index), words.to(DEV), scales.to(DEV), biases.to(DEV), _dev(ids))
    logits, logprobs = logits.double().cpu().numpy(), logprobs.double().cpu().numpy()
    normed = ext.rms_norm(x.to(DEV), w.to(DEV), 1e-6).double().cpu().numpy()
    W = R.head_weights(words, scales, biases, bits)
    want, _ = R.select_logits_ref(normed, W, row_index, ids)
    # one rounding to the dtype (half an ulp, at most 2^-9 / 2^-12 relative) after an fp32 sum whose error is bounded
    # by H * 2^-24 times the sum of the products' magnitudes
    mag = np.abs(normed[row_index]) @ np.abs(W[ids]).T
    rel = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11
    assert np.all(np.abs(logits - want) <= rel * np.abs(want) + H * 2.0 ** -24 * mag), np.abs(logits - want).max()
    assert np.all(logits == logits.astype(np.float32)), "logits are fp32"
    x_t = torch.from_numpy(logits).to(dtype).double().numpy()
    assert np.array_equal(x_t, logits), "logits hold dtype-rounded values"
    # the log-softmax of the kernel's own logits, to fp32 rounding
    np.testing.assert_allclose(logprobs, R.log_softmax(logits), rtol=0, atol=4e-7 * (1 + np.abs(logits).max()) * max(1, np.log2(m) + 1))
    assert np.array_equal(logits[2], logits[4]), "one row listed twice"


def test_select_logits_out_of_range_gives_nan():
    gen = torch.Generator().manual_seed(1)
    words, scales, biases = _head(50, 256, 4, torch.bfloat16, gen)
    x = torch.randn((4, 256), generator=gen).to(torch.bfloat16).to(DEV)
    w = torch.ones(256, dtype=torch.bfloat16, device=DEV)
    logits, logprobs = ext.select_logits(x, w, 1e-6, _dev([0, 4, -1]), words.to(DEV), scales.to(DEV), biases.to(DEV), _dev([3, 50]))
    logits, logprobs = logits.cpu(), logprobs.cpu()
    assert torch.isfinite(logits[0, 0]) and torch.isnan(logits[0, 1]) and torch.isnan(logprobs[0]).all()
    assert torch.isnan(logits[1:]).all() and torch.isnan(logprobs[1:]).all()


# ---------------------------------------------------------------- rerank_ids --
_MODELS = {}


def _model(name, bits=4, tied=True):
    key = (name, bits, tied)
    if key not in _MODELS:
        extra = {} if tied else {"tie_word_embeddings": False}
        ns = synthetic_qwen3(name, seed=0, device=DEV, realistic=name.startswith("tiny"), bits=bits, **extra)
        _MODELS[key] = Qwen3ModelWeek3(ns, page_size=128)
    return _MODELS[key]


def _ids(vocab, lengths, seed):
    g = np.random.default_rng(seed)
    return [g.integers(0, vocab, size=n).tolist() for n in lengths]


def _model_path_logits(model, ids, true_id, false_id):
    """The whole prompt alone through ``model.embedding``, the blocks as ``__call__`` runs them, ``model.norm`` and the
    full LM head: float64 (logit(false_id), logit(true_id)) of the last row."""
    cache = model.create_kv_cache()
    try:
        h = model.embedding(torch.tensor([ids], dtype=torch.int32, device=DEV))
        for block, layer_cache in zip(model.layers_inner, cache):
            h = block(h, 0, layer_cache, mask="causal")
        h = model.norm(h[:, -1:])
        logits = quantized_linear(h, model.w_lm_head) if model.w_lm_head is not None else model.embedding.as_linear(h)
        row = logits.reshape(-1).double().cpu()
    finally:
        for c in cache:
            c.release()
    return float(row[false_id]), float(row[true_id])


@pytest.mark.parametrize("name,bits,tied", [("tiny-d128", 4, True), ("tiny-d128", 4, False), ("tiny-d128", 8, True), ("qwen3-0.6b", 4, True)])
def test_rerank_ids_matches_model_path(name, bits, tied):
    """Scores against the model's own path.  The comparison is on the logit difference d = logit(true) - logit(false),
    recovered from the score as log(p / (1 - p)).  Both paths round each logit to bf16 (half an ulp, 2^-9 relative), so
    rounding alone moves d by up to 2^-8 (|l_true| + |l_false|); the bf16 hidden states of the two kernel paths
    (packed wgmma prefill and attention against the operator path) differ by a few bf16 ulps per layer, which a
    further 2% of (1 + |l_true| + |l_false|) covers."""
    model = _model(name, bits, tied)
    V = model.vocab_size
    prefix, *docs = _ids(V, [70, 1, 5, 64, 65, 130], seed=1)
    true_id, false_id = 7, V - 2
    got = rerank_ids(model, [(prefix, docs), ([], docs[:2])], true_id, false_id, max_tokens=512)
    assert [g.shape[0] for g in got] == [5, 2]
    for qi, (pre, ds) in enumerate([(prefix, docs), ([], docs[:2])]):
        p = got[qi].double().cpu().numpy()
        assert np.all((p > 0) & (p < 1))
        for di, d in enumerate(ds):
            lf, lt = _model_path_logits(model, pre + d, true_id, false_id)
            want = lt - lf
            have = np.log(p[di] / (1 - p[di]))
            assert abs(have - want) <= 2.0 ** -8 * (abs(lt) + abs(lf)) + 0.02 * (1 + abs(lt) + abs(lf)), (qi, di, have, want, lt, lf)


@pytest.mark.parametrize("name", ["tiny-d128", "qwen3-0.6b"])
def test_rerank_ids_bits_do_not_depend_on_sharing_or_placement(name):
    model = _model(name)
    V = model.vocab_size
    prefix, a, b, c, d, other = _ids(V, [100, 37, 100, 3, 150, 20], seed=2)
    t, f = 11, 12
    shared = rerank_ids(model, [(prefix, [a, b, c, d])], t, f, max_tokens=512)[0]
    alone = rerank_ids(model, [(prefix, [x]) for x in (a, b, c, d)], t, f, max_tokens=512)
    assert torch.equal(shared, torch.cat(alone)), "sharing the prefix changed a score"
    # other siblings, another order, another query in the pass first
    moved = rerank_ids(model, [(other, [c, a]), (prefix, [d, c, b, a])], t, f, max_tokens=512)[1]
    assert torch.equal(moved, shared.flip(0))
    # an overflowing group: [P a b] [P c d] ... d lands in a later pass with its prefix repeated
    over = rerank_ids(model, [(prefix, [b, a, b, d, c])], t, f, max_tokens=512)[0]
    assert torch.equal(over[3], shared[3]) and torch.equal(over[4], shared[2]) and torch.equal(over[0], over[2])


def _available(model):
    return [p.pages_available() for p in model.page_pools]


def test_rerank_ids_returns_every_page(monkeypatch):
    model = _model("tiny-d128")
    V = model.vocab_size
    prefix, *docs = _ids(V, [64, 100, 10, 130, 50], seed=4)  # three passes of 256 rows
    rerank_ids(model, [(prefix, docs)], 1, 2, max_tokens=256)  # sizes the slabs
    before = _available(model)
    rerank_ids(model, [(prefix, docs)], 1, 2, max_tokens=256)
    assert _available(model) == before
    with pytest.raises(ValueError, match="query 0 document 1: a prefix of 64 tokens and a document of 300 tokens"):
        rerank_ids(model, [(prefix, [docs[0], [1] * 300])], 1, 2, max_tokens=256)
    with pytest.raises(ValueError, match="query 1 document 0 holds a token id"):
        rerank_ids(model, [(prefix, docs), ([1], [[V]])], 1, 2, max_tokens=256)
    with pytest.raises(ValueError, match="is empty"):
        rerank_ids(model, [(prefix, [[]])], 1, 2, max_tokens=256)
    with pytest.raises(ValueError, match="must differ"):
        rerank_ids(model, [(prefix, docs)], 3, 3)
    with pytest.raises(ValueError, match="outside"):
        rerank_ids(model, [(prefix, docs)], V, 3)
    assert _available(model) == before
    calls = {"n": 0}
    real = ext.paged_attention_prefixed_segments

    def failing(*a, **k):
        calls["n"] += 1
        if calls["n"] == 3:  # the second pass's first layer: the first pass returned its pages already
            raise ValueError("injected")
        return real(*a, **k)

    monkeypatch.setattr(rerank_mod.ext, "paged_attention_prefixed_segments", failing)
    with pytest.raises(ValueError, match="injected"):
        rerank_ids(model, [(prefix, docs)], 1, 2, max_tokens=256)
    assert _available(model) == before


def test_checkpoint_scores_the_same_bits(tmp_path):
    ns = synthetic_qwen3("tiny-d128", seed=5, device="cpu", realistic=True, tie_word_embeddings=False)
    save_checkpoint(ns, tmp_path / "m")
    a = Qwen3ModelWeek3(synthetic_qwen3("tiny-d128", seed=5, device=DEV, realistic=True, tie_word_embeddings=False), page_size=128)
    b = Qwen3ModelWeek3(load_checkpoint(tmp_path / "m", device=DEV), page_size=128)
    prefix, *docs = _ids(a.vocab_size, [20, 9, 70], seed=6)
    assert torch.equal(rerank_ids(a, [(prefix, docs)], 3, 4, max_tokens=256)[0], rerank_ids(b, [(prefix, docs)], 3, 4, max_tokens=256)[0])


def test_cli_rerank_prints_scores(capsys):
    from tiny_llm_b200 import cli

    assert cli.main(["rerank", "--synthetic", "tiny-d128", "--prefix-ids", "5,17,3", "--document-ids", "9,2;4,8,1;7",
                     "--true-id", "10", "--false-id", "11"]) == 0
    lines = [l for l in capsys.readouterr().out.splitlines() if l.startswith("[")]
    assert len(lines) == 3
    for line in lines:
        assert 0.0 <= float(line.rsplit(": ", 1)[1]) <= 1.0
