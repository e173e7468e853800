"""Beam search on the GPU: ``tl_beam_select`` against the plain-loop rule (``beam_ref.py``) bit for bit, eagerly and
under graph replay; a whole step (``tl_logprobs`` + ``tl_beam_select``) on planted logits at every dtype; greedy
equality with one beam; the protocol on the graph path against the rule applied to the engine's own logits rows; the
beam step graph against the plain decode graph; forks, teacher-forced scores with a negative control, and the pages."""

import importlib.util
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, beam_search_ids, greedy_generate_ids, score_ids
from tiny_llm_b200 import generate as gen
from tiny_llm_b200 import paged_kv_cache as pkv
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.kv_cache import BatchingKvCache
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_beam_ref", "beam_ref.py")
LP = _load("tiny_llm_b200_logprobs_ref", "logprobs_ref.py")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


# ------------------------------------------------------------------ the kernel --
def _case(g, rows, W, E, V=40):
    """Top-N lists on a coarse grid (exact ties within and across rows), with -inf / -1 tails and NaN entries."""
    N = W + E
    lp = -(g.integers(0, 6, (rows, N)).astype(np.float32) * np.float32(0.25))
    lp.sort(axis=1)
    lp = lp[:, ::-1].copy()
    ids = np.stack([g.permutation(V)[:N] for _ in range(rows)]).astype(np.int32)
    for r in range(rows):
        cut = int(g.integers(0, N + 1)) if g.random() < 0.3 else N
        lp[r, cut:], ids[r, cut:] = -np.inf, -1
        if g.random() < 0.1:
            lp[r, int(g.integers(0, N))] = np.nan
    cum = -(g.integers(0, 8, rows).astype(np.float32) * np.float32(0.25))
    if rows > 1 and g.random() < 0.2:
        cum[int(g.integers(0, rows))] = -np.inf
    eos = [int(t) for t in g.permutation(V)[:E]]
    return lp, ids, cum, eos


def _kernel(dev, lp, ids, cum, W, eos):
    cum_d = torch.full((W,), 7.0, device=dev)
    cum_d[: len(cum)] = torch.from_numpy(cum)
    out = torch.full((ext.BEAM_RESULT_WORDS,), -5, dtype=torch.int32, device=dev)
    ext.beam_select(torch.from_numpy(lp).to(dev), torch.from_numpy(ids).to(dev), cum_d, W, eos, out)
    return out.cpu().numpy(), cum_d.cpu().numpy()


def _check(words, cum_after, lp, ids, cum, W, eos):
    live, fin = R.select(lp, ids, cum, W, eos)
    got_live, got_fin = gen.unpack_beam_result(words)
    assert got_live == [(p, t, float(s)) for p, t, s in live]
    assert got_fin == [(p, t, float(s), q) for p, t, s, q in fin]
    np.testing.assert_array_equal(cum_after, R.new_cum(live, W))


@pytest.mark.parametrize("W", range(1, 9))
@pytest.mark.parametrize("E", range(0, 5))
def test_select_equals_the_rule(dev, W, E):
    g = np.random.default_rng(100 * W + E)
    for rows in range(1, W + 1):
        for _ in range(6):
            lp, ids, cum, eos = _case(g, rows, W, E)
            words, cum_after = _kernel(dev, lp, ids, cum, W, eos)
            _check(words, cum_after, lp, ids, cum, W, eos)


def test_select_under_graph_replay(dev):
    W, eos = 4, [3, 11]
    N = W + len(eos)
    lp_d = torch.zeros((W, N), device=dev)
    ids_d = torch.zeros((W, N), dtype=torch.int32, device=dev)
    cum_d = torch.zeros(W, device=dev)
    out = torch.zeros(ext.BEAM_RESULT_WORDS, dtype=torch.int32, device=dev)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ext.beam_select(lp_d, ids_d, cum_d, W, eos, out)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        ext.beam_select(lp_d, ids_d, cum_d, W, eos, out)
    g = np.random.default_rng(5)
    for _ in range(20):
        lp, ids, cum, _ = _case(g, W, W, len(eos))
        ids[ids == eos[0]] = 99
        ids[0, 1] = eos[0]
        lp_d.copy_(torch.from_numpy(lp))
        ids_d.copy_(torch.from_numpy(ids))
        cum_d.copy_(torch.from_numpy(cum))
        graph.replay()
        torch.cuda.synchronize()
        _check(out.cpu().numpy(), cum_d.cpu().numpy(), lp, ids, cum, W, eos)


# ------------------------------------------------------------------ a whole step --
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("V", [151936, 4097, 4095, 37])
def test_a_whole_step_on_planted_logits(dev, dtype, V):
    """Each row's top entries are planted on a grid of 0.5 (exact in every dtype) over a background far below them;
    candidates either tie exactly or differ by at least 0.5 - far above the fp32 bound of ``tl_logprobs`` - so the
    selection is the rule's on the float64 log-probabilities."""
    W, eos = 4, [1, 2]
    N = W + len(eos)
    g = np.random.default_rng(V)
    x = np.full((W, V), -30.0, dtype=np.float32)
    for r in range(W):
        cols = g.permutation(V)[:N]
        x[r, cols] = -(g.integers(0, 4, N) * 0.5)
        x[r, 1] = -0.5 if r % 2 else -1.0
    logits = torch.from_numpy(x).to(dtype).to(dev)
    cum = np.array([0.0, -0.5, -0.5, -1.0], dtype=np.float32)
    _, _, _, ids, top = ext.logprobs(logits, None, None, N)
    cum_d = torch.from_numpy(cum).to(dev)
    out = torch.zeros(ext.BEAM_RESULT_WORDS, dtype=torch.int32, device=dev)
    ext.beam_select(top, ids, cum_d, W, eos, out)
    live, fin = gen.unpack_beam_result(out.cpu().numpy())
    _, _, _, ref_ids, ref_lp = LP.logprobs(logits.float().cpu().numpy(), None, None, N)
    np.testing.assert_array_equal(ids.cpu().numpy(), ref_ids)
    want_live, want_fin = R.select(ref_lp, ref_ids, cum, W, eos)
    assert [(p, t) for p, t, _ in live] == [(p, t) for p, t, _ in want_live]
    assert [(p, t, q) for p, t, _, q in fin] == [(p, t, q) for p, t, _, q in want_fin]
    bound = 1e-5
    assert all(abs(a[2] - b[2]) <= bound for a, b in zip(live, want_live))


# ------------------------------------------------------------------ end to end --
MODELS = {
    "d128": ("tiny-d128", dict(seed=5, realistic=True, max_position_embeddings=4096)),
    "4b": ("qwen3-4b", dict(seed=1, num_hidden_layers=2, vocab_size=4096)),
    "moe": ("tiny-moe-d128", dict(seed=0, realistic=True, max_position_embeddings=4096)),
}
_NS: dict = {}


def _model(key, dev, window=2048):
    if key not in _NS:
        name, kw = MODELS[key]
        _NS[key] = synthetic_qwen3(name, device=dev, **kw)
    m = Qwen3ModelWeek3(_NS[key], page_size=128)
    m.prefill_graph_len = 0
    m.set_max_context(window)
    return m


def _pools_whole(model):
    for pool in model.page_pools:
        assert not pool.used_page_ids and not pool.extra_refs, "every page is back in its pool"


def _prompt(seed, V, n):
    return torch.randint(0, V, (n,), generator=torch.Generator().manual_seed(seed)).tolist()


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("graph", [True, False])
def test_one_beam_with_early_stopping_is_greedy(dev, key, graph):
    model = _model(key, dev)
    if not graph:
        model.use_decode_graph = False
    prompt = _prompt(1, model.vocab_size, 150)
    want = greedy_generate_ids(model, prompt, 40, device=dev)
    (h,) = beam_search_ids(model, prompt, 40, num_beams=1, early_stopping=True, device=dev)
    assert h.ids == want
    eos = want[17]
    want_eos = greedy_generate_ids(model, prompt, 40, eos_token_id=eos, device=dev)
    (h,) = beam_search_ids(model, prompt, 40, num_beams=1, early_stopping=True, eos_token_ids=(eos,), device=dev)
    assert h.ids == want_eos and h.finished == (len(want_eos) < 40)
    assert gen._beam_graph_applies(model, dev, len(prompt) + 40) == graph
    _pools_whole(model)


def _recording(monkeypatch):
    """Every step's logits rows: the prompt's last row, then the engine's W rows after each beam step."""
    rows = []
    first, step = gen._BeamRunner.first, DecodeEngine.beam_step

    def rec_first(self, row):
        rows.append(row.clone())
        return first(self, row)

    def rec_step(self, *a, **k):
        out = step(self, *a, **k)
        rows.append(self.logits.clone())
        return out

    monkeypatch.setattr(gen._BeamRunner, "first", rec_first)
    monkeypatch.setattr(DecodeEngine, "beam_step", rec_step)
    return rows


@pytest.mark.parametrize("key", ["d128", "4b", "moe"])
@pytest.mark.parametrize("W, eos, kw", [(4, (), {}), (8, (7, 9), dict(length_penalty=0.5)), (3, (5,), dict(early_stopping=True))])
def test_the_graph_protocol_follows_the_rule_on_its_own_rows(dev, monkeypatch, key, W, eos, kw):
    model = _model(key, dev)
    prompt = _prompt(2, model.vocab_size, 200)
    eos = tuple(range(3)) + eos if key == "d128" else eos  # frequent EOS ids on the small vocabulary
    eos = eos[:4]
    model.decode_engine(W)  # the reservation first: the search itself then moves no slab
    versions = [p.slab_version for p in model.page_pools]
    rows = _recording(monkeypatch)
    got = beam_search_ids(model, prompt, 24, num_beams=W, eos_token_ids=eos, num_return_sequences=W, device=dev, **kw)
    assert [p.slab_version for p in model.page_pools] == versions, "no fork grew a slab"
    N = W + len(eos)
    it = iter(rows)

    def tops(beams):
        r = next(it)[: len(beams)].contiguous()
        _, _, _, ids, top = ext.logprobs(r, None, None, N)
        return top.cpu().numpy(), ids.cpu().numpy()

    want = R.search(tops, 24, W, eos=eos, num_return_sequences=W, **kw)
    assert [(h.ids, h.sum_logprob, h.score, h.finished) for h in got] == [(list(i), float(s), sc, f) for i, s, sc, f in want]
    _pools_whole(model)


def test_the_beam_step_graph_equals_the_decode_graph_and_eager_launches(dev):
    model = _model("d128", dev)
    W, eos = 4, (3,)
    engine = model.decode_engine(W)
    prompts = [_prompt(10 + b, model.vocab_size, 100 + 37 * b) for b in range(W)]

    def prefilled():
        slots = [BatchingKvCache(W) for _ in range(model.num_hidden_layers)]
        for b, p in enumerate(prompts):
            cache = model.create_kv_cache()
            model(torch.tensor([p], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
            for layer, c in enumerate(cache):
                slots[layer].kv_caches[b] = c
        return slots

    tokens = [5, 6, 7, 8]
    offsets = [len(p) for p in prompts]
    a, b = prefilled(), prefilled()
    plain, _ = engine.step(tokens, offsets, a)
    plain = plain.view(W, -1).clone()
    cum = torch.tensor([0.0, -1.0, -1.5, -2.0], device=dev)
    engine.beam_buffers(eos)
    engine.beam_cum.copy_(cum)
    result = engine.beam_step(tokens, offsets, b, eos).clone()
    torch.cuda.synchronize()
    assert torch.equal(engine.logits, plain)
    _, _, _, ids, top = ext.logprobs(plain, None, None, W + len(eos))
    out = torch.zeros_like(result)
    ext.beam_select(top, ids, cum, W, eos, out)
    assert torch.equal(out, result) and torch.equal(cum, engine.beam_cum)
    assert engine.kernels_per_beam_step > 0
    print(f"kernels per step {engine.kernels_per_step}, per beam step {engine.kernels_per_beam_step}")
    for slots in (a, b):
        for layer in slots:
            for c in layer.kv_caches:
                c.release()
    _pools_whole(model)


@pytest.mark.parametrize("n", [200, 256])
def test_a_fork_copies_exactly(dev, n):
    model = _model("d128", dev)
    model.decode_engine(4)
    cache = model.create_kv_cache()
    model(torch.tensor([_prompt(3, model.vocab_size, n)], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1)
    (kids,) = pkv.fork([(cache, 3)])
    torch.cuda.synchronize()
    for kid in kids:
        for c, p in zip(kid, cache):
            assert c.page_ids[: n // 128] == p.page_ids[: n // 128]
            assert all(torch.equal(x, y) for x, y in zip(c.gather_dense(), p.gather_dense()))
    for caches in (cache, *kids):
        for c in caches:
            c.release()
    _pools_whole(model)


def _parity_bound(model, prompt, dev):
    """Per-token |decode lp - teacher-forced lp| seen on greedy's own tokens, times 4: the decode and prefill paths
    round differently, and a hypothesis's sum is compared against its teacher-forced score within L times this."""
    ids, entries = greedy_generate_ids(model, prompt, 24, device=dev, logprobs=0)
    forced = score_ids(model, prompt + ids, device=dev).entries[len(prompt) - 1 :]
    return 4 * max(abs(a.logprob - b.logprob) for a, b in zip(entries, forced)) + 1e-4


def _score_errors(model, prompt, hyps, eos, dev):
    bad = []
    for h in hyps:
        ids = h.ids + ([eos] if h.finished else [])
        forced = score_ids(model, prompt + ids, device=dev).entries[len(prompt) - 1 :]
        bad.append(abs(sum(e.logprob for e in forced) - h.sum_logprob) / len(ids))
    return bad


def test_every_hypothesis_scores_as_reported_and_a_corrupted_fork_does_not(dev, monkeypatch):
    model = _model("d128", dev)
    prompt = _prompt(4, model.vocab_size, 200)
    bound = _parity_bound(model, prompt, dev)
    eos = 0
    hyps = beam_search_ids(model, prompt, 24, num_beams=4, num_return_sequences=4, eos_token_ids=(eos,), device=dev)
    assert max(_score_errors(model, prompt, hyps, eos, dev)) <= bound
    _pools_whole(model)

    fork = pkv.fork

    def corrupted(requests):
        made = fork(requests)
        for (caches, _), kids in zip(requests, made):
            for kid in kids:
                for c in kid:  # the tail's slots get another live page's data: wrong keys at a valid address
                    pool = c.pool
                    pool._key_pages[c.page_ids[-1]].copy_(pool._key_pages[c.page_ids[0]])
                    pool._value_pages[c.page_ids[-1]].copy_(pool._value_pages[c.page_ids[0]])
        return made

    monkeypatch.setattr(pkv, "fork", corrupted)
    hyps = beam_search_ids(model, prompt, 24, num_beams=4, num_return_sequences=4, eos_token_ids=(eos,), device=dev)
    assert max(_score_errors(model, prompt, hyps, eos, dev)) > bound
    _pools_whole(model)


def test_pages_and_slabs_after_searches(dev, monkeypatch):
    model = _model("d128", dev)
    model.decode_engine(8)
    versions = [p.slab_version for p in model.page_pools]
    raised = []
    check = pkv.TinyKvPagedPool.check_write

    def watched(self, page_id, start):
        try:
            check(self, page_id, start)
        except RuntimeError:
            raised.append(page_id)
            raise

    monkeypatch.setattr(pkv.TinyKvPagedPool, "check_write", watched)
    for W in (2, 5, 8):
        for n in (127, 128, 300):
            beam_search_ids(model, _prompt(W + n, model.vocab_size, n), 140, num_beams=W, device=dev)
            _pools_whole(model)
    assert not raised and [p.slab_version for p in model.page_pools] == versions
