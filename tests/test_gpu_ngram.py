"""Prompt lookup on the GPU: ``tl_ngram_propose`` against the plain-loop proposer (``ngram_ref.py``) exactly, at
histories up to 131,072 tokens, for every (n_min, n_max) and k, with planted matches, appends, any grid and graph
replay; the one-hot rows at every dtype; ``tl_speculative_sample`` with one-hot drafts against the float64 rule; and
``prompt_lookup_generate_ids`` against ``greedy_generate_ids`` on the graph and generic runners."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import stats

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids, prompt_lookup_generate_ids
from tiny_llm_b200 import generate as gen
from tiny_llm_b200.sampler import SamplingParams, sampling_tensors
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


NR = _load("tiny_llm_b200_ngram_ref", "ngram_ref.py")
SR = _load("tiny_llm_b200_spec_sample_ref", "spec_sample_ref.py")

pytestmark = pytest.mark.gpu
TILE = ext.NGRAM_TILE


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


class Call:
    """One history buffer with its state and output, as a request keeps them."""

    def __init__(self, dev, capacity, k, onehot=None):
        self.history = torch.full((capacity,), -7, dtype=torch.int32, device=dev)
        self.state = torch.zeros(ext.NGRAM_STATE_WORDS, dtype=torch.int32, device=dev)
        self.out = torch.empty(2 + k, dtype=torch.int32, device=dev)
        self.k, self.onehot = k, onehot

    def __call__(self, length, appended, n_min, n_max, grid=0):
        ext.ngram_propose(self.history, length, appended, self.k, n_min, n_max, self.out, self.state, self.onehot, grid=grid)
        o = self.out.tolist()
        return o[0], o[1], o[2:] if o[0] else []


def _propose(dev, s, k, n_min, n_max, appended=0, grid=0):
    """The kernel on history s: the first len(s) - appended ids uploaded, the rest appended by argument."""
    call = Call(dev, max(len(s), 1) + 8, k)
    head = len(s) - appended
    if head:
        call.history[:head].copy_(torch.as_tensor(s[:head], dtype=torch.int32))
    got = call(head, s[head:], n_min, n_max, grid)
    assert call.history[: len(s)].tolist() == list(s), "the appended ids are written behind the history"
    assert call.state.tolist() == [0, 0, 0] + [0] * (ext.NGRAM_STATE_WORDS - 3), "the reduction leaves its state zeroed"
    out = call.out.tolist()
    assert out[1] == (got[1] if got[0] else -1) and (got[0] or out[2:] == [-1] * k)
    return got


def _want(s, k, n_min, n_max):
    return (NR.propose if len(s) <= 300 else NR.propose_np)(s, k, n_min, n_max)


PAIRS = [(a, b) for b in range(1, 9) for a in range(1, b + 1)]
LENGTHS = [1, 2, 3, 5, 8, 9, 17, 100, TILE - 1, TILE, TILE + 1, TILE + 2, 2 * TILE + 3, 8192, 32768, 131072]


@pytest.mark.parametrize("alphabet", [3, 151936])
@pytest.mark.parametrize("L", LENGTHS)
def test_kernel_equals_the_reference_on_random_histories(dev, alphabet, L):
    g = torch.Generator().manual_seed(L * 7 + alphabet)
    s = torch.randint(0, alphabet, (L,), generator=g).tolist()
    pairs = PAIRS if L <= 2 * TILE + 3 else PAIRS[:: 5]
    for i, (n_min, n_max) in enumerate(pairs):
        k = 1 + i % 7
        appended = i % 9 if L > 8 else i % (L + 1)
        assert _propose(dev, s, k, n_min, n_max, appended) == _want(s, k, n_min, n_max), (L, alphabet, n_min, n_max, k)


def test_every_ngram_range_and_k_on_one_history(dev):
    g = torch.Generator().manual_seed(11)
    s = torch.randint(0, 5, (3000,), generator=g).tolist()
    for n_min, n_max in PAIRS:
        for k in range(1, 8):
            assert _propose(dev, s, k, n_min, n_max) == _want(s, k, n_min, n_max), (n_min, n_max, k)


def _planted(L, e, n, seed):
    """Distinct ids (no natural match) with s[e-n+1..e] copied to the end: c(e) = n at the planted e."""
    s = (torch.randperm(10 * L + 100, generator=torch.Generator().manual_seed(seed))[:L] + 1).tolist()
    s[L - n :] = s[e - n + 1 : e + 1]
    return s


@pytest.mark.parametrize("L", [300, 3 * TILE + 5, 131072])
def test_planted_matches_at_the_ends_and_on_tile_boundaries(dev, L):
    ends = [0, 1, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, L - 10]
    for i, e in enumerate(x for x in ends if 0 <= x <= L - 10):
        n = min(e + 1, 1 + i % 8)
        s = _planted(L, e, n, seed=i)
        k = 1 + i % 7
        for n_min, n_max in ((1, 8), (n, n), (1, n)):
            got = _propose(dev, s, k, n_min, n_max, appended=i % 9)
            assert got == _want(s, k, n_min, n_max) and got[:2] == (n, e), (L, e, n)
    # e = L - 2: the run `a a ... a` overlapping the suffix, and a match spanning a tile boundary's halo
    s = _planted(L, 5, 1, seed=99)
    s[L - 4 :] = [s[L - 5]] * 4
    assert _propose(dev, s, 3, 1, 8) == _want(s, 3, 1, 8) and _propose(dev, s, 3, 1, 8)[1] == L - 2
    if L > 2 * TILE:
        e = 2 * TILE + 2  # its 8-token match starts in the previous tile
        s = _planted(L, e, 8, seed=7)
        assert _propose(dev, s, 7, 8, 8)[:2] == (8, e)


@pytest.mark.parametrize("L", [50, 5 * TILE + 17, 131072])
def test_the_result_does_not_depend_on_the_grid(dev, L):
    g = torch.Generator().manual_seed(L)
    s = torch.randint(0, 4, (L,), generator=g).tolist()
    want = _want(s, 5, 2, 6)
    for grid in (0, 1, 2, 3, 7, 132, 1000):
        assert _propose(dev, s, 5, 2, 6, appended=3, grid=grid) == want, grid


def test_appends_by_argument_equal_a_history_uploaded_in_one_piece(dev):
    g = torch.Generator().manual_seed(3)
    s = torch.randint(0, 6, (5000,), generator=g).tolist()
    one = Call(dev, 5008, 4)
    one.history[:5000].copy_(torch.as_tensor(s, dtype=torch.int32))
    step = Call(dev, 5008, 4)
    step.history[:100].copy_(torch.as_tensor(s[:100], dtype=torch.int32))
    length, i = 100, 0
    while length < 5000:
        n = min(1 + i % 8, 5000 - length)
        got = step(length, s[length : length + n], 2, 3)
        length += n
        i += 1
        assert got == one(length, [], 2, 3) == _want(s[:length], 4, 2, 3), length
    assert torch.equal(step.history[:5000], one.history[:5000])


def test_the_call_replays_identically_under_a_cuda_graph(dev):
    g = torch.Generator().manual_seed(5)
    L = 40000
    s = torch.randint(0, 3, (L,), generator=g).tolist()
    V = 1000
    onehot = torch.full((6, V), float("-inf"), dtype=torch.bfloat16, device=dev)
    call = Call(dev, L + 8, 6, onehot)
    call.history[: L - 5].copy_(torch.as_tensor(s[: L - 5], dtype=torch.int32))
    want = call(L - 5, [t % V for t in s[L - 5 :]], 2, 5)
    eager_out, eager_rows = call.out.clone(), onehot.clone()
    graph = torch.cuda.CUDAGraph()
    stream = torch.cuda.Stream(dev)
    stream.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            ext.ngram_propose(call.history, L - 5, [t % V for t in s[L - 5 :]], 6, 2, 5, call.out, call.state, onehot)
    torch.cuda.current_stream(dev).wait_stream(stream)
    for _ in range(3):
        call.out.fill_(-9)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(call.out, eager_out) and torch.equal(onehot, eager_rows)
    assert want == _want(s, 6, 2, 5)


# ------------------------------------------------------------------ one-hot rows --
@pytest.mark.parametrize("dtype,V", [(torch.float32, 1000), (torch.float16, 4097), (torch.bfloat16, 4097), (torch.bfloat16, 151936)])
def test_onehot_rows_hold_exactly_the_current_proposals(dev, dtype, V):
    k = 5
    onehot = torch.full((k, V), float("-inf"), dtype=dtype, device=dev)
    call = Call(dev, 4096, k, onehot)
    g = torch.Generator().manual_seed(V)
    s = torch.randint(0, V, (200,), generator=g).tolist()
    call.history[:200].copy_(torch.as_tensor(s, dtype=torch.int32))
    length, matched, unmatched = 200, 0, 0
    for i in range(40):
        # alternately a token that recurs (a match) and a fresh one (none)
        tok = s[int(torch.randint(0, len(s) - 1, (1,), generator=g))] if i % 3 else int(torch.randint(0, V, (1,), generator=g))
        s.append(tok)
        c, e, p = call(length, [tok], 1, 2)
        length += 1
        assert (c, e, p) == _want(s, k, 1, 2)
        want = torch.full((k, V), float("-inf"), dtype=torch.float32)
        for t, v in enumerate(p):
            want[t, v] = 0.0
        assert torch.equal(onehot.float().cpu(), want), f"call {i}: the rows are not exactly the current proposals"
        matched += bool(c)
        unmatched += not c
    assert matched and unmatched


# ------------------------------------------------------------------ the sampled rule with one-hot drafts --
REL, GAP = 2e-5, 1e-3  # as test_gpu_spec_sample.py: decisions may differ from float64 only this close to a flip


def _onehot(d, V, dtype):
    y = torch.full((len(d), V), float("-inf"))
    y[torch.arange(len(d)), torch.as_tensor(d)] = 0.0
    return y.to(dtype)


@pytest.mark.parametrize("dtype,V", [(torch.float32, 1000), (torch.bfloat16, 4097), (torch.bfloat16, 151936)], ids=str)
@pytest.mark.parametrize("params", [(1.0, 0, 0.0), (0.7, 0, 0.0), (0.8, 50, 0.9), (1.3, 20, 0.95)], ids=str)
def test_one_hot_drafts_follow_the_float64_rule(dev, dtype, V, params):
    temp, top_k, top_p = params
    g = torch.Generator().manual_seed(V + int(temp * 10))
    decisions = exceptions = accepted = 0
    for trial in range(6):
        k = 1 + trial
        x = (torch.randn(k + 1, V, generator=g) * (1 + trial % 3)).to(dtype)
        # proposals: the target's argmax, a likely token, or an arbitrary one
        d = [int(x[j].float().argmax()) if j % 3 == 0 else int(torch.topk(x[j].float(), 5).indices[j % 5]) if j % 3 == 1
             else int(torch.randint(0, V, (1,), generator=g)) for j in range(k)]
        for j in range(0, k, 2):  # make every other proposal likely under p, so that both outcomes occur
            x[j, d[j]] = x[j].float().max() + 2
        y = _onehot(d, V, dtype)
        sp = SamplingParams(temp, top_k=top_k or None, top_p=top_p or None, seed=100 + trial)
        per = sampling_tensors([sp] * (k + 1), dev)
        pos = torch.arange(30, 31 + k, dtype=torch.int32, device=dev)
        out = ext.speculative_sample(x.to(dev), y.to(dev), torch.tensor(d, dtype=torch.int32, device=dev), *per, pos).tolist()
        xs, ys = x.double().numpy(), y.double().numpy()
        for j in range(k):
            want = SR.rule_row(xs[j], ys[j], d[j], temp, top_k, top_p, sp.seed, 30 + j)
            q = SR.row_dist(ys[j], temp, top_k, top_p)
            assert q[d[j]] == 1.0, "the one-hot row is the point mass at its proposal"
            decisions += 1
            accepted += want.accepted
            if out[j] != want.token:
                p = SR.row_dist(xs[j], temp, top_k, top_p)
                assert want.margin <= REL * max(p[d[j]], 1.0) or want.residual_gap <= GAP, (j, out[j], want)
                exceptions += 1
    assert exceptions <= max(1, decisions // 50) and 0 < accepted < decisions


def test_one_hot_drafts_give_the_target_distribution_over_60000_rows(dev):
    x = torch.tensor([1.2, 0.3, -0.5, 2.0, 0.9, -1.1, 0.0, 1.5])
    rows, temp, top_k, top_p = 60_000, 0.9, 7, 0.97
    T = rows + 1
    g = torch.Generator().manual_seed(0)
    p = SR.row_dist(x.double().numpy(), temp, top_k, top_p)
    d = torch.multinomial(torch.full((8,), 1.0), rows, replacement=True, generator=g)  # proposals far from p
    X = x.repeat(T, 1).to(dev)
    Y = _onehot(d.tolist(), 8, torch.float32).to(dev)
    temperature = torch.full((T,), temp, device=dev)
    tk = torch.full((T,), top_k, dtype=torch.int32, device=dev)
    tp = torch.full((T,), top_p, device=dev)
    seed = torch.arange(T, dtype=torch.int64, device=dev)
    pos = torch.full((T,), 11, dtype=torch.int32, device=dev)
    out = ext.speculative_sample(X, Y, d.to(torch.int32).to(dev), temperature, tk, tp, seed, pos)[:rows].cpu().numpy()
    counts = np.bincount(out, minlength=8).astype(np.float64)
    assert counts[p == 0].sum() == 0
    live = p > 0
    assert stats.chisquare(counts[live], rows * p[live]).pvalue > 1e-3
    # the acceptance rate is p_d averaged over the proposals
    acc = (out == d.numpy()).mean()
    assert abs(acc - p[d.numpy()].mean()) < 0.02


# ------------------------------------------------------------------ end to end --
MODELS = {
    "d128": ("tiny-d128", dict(seed=5, realistic=True, max_position_embeddings=8192)),
    "4b": ("qwen3-4b", dict(seed=1, num_hidden_layers=2, vocab_size=4096)),
}
_NS: dict = {}


def _model(key, dev):
    if key not in _NS:
        name, kw = MODELS[key]
        _NS[key] = synthetic_qwen3(name, device=dev, **kw)
    m = Qwen3ModelWeek3(_NS[key], page_size=128)
    m.prefill_graph_len = 0
    return m


def _pools_whole(model):
    for pool in model.page_pools:
        assert not pool.used_page_ids, "every page is back in its pool"


def _repeating_prompt(seed, V, n=96):
    g = torch.Generator().manual_seed(seed)
    passage = torch.randint(0, V, (n // 3,), generator=g).tolist()
    return passage + torch.randint(0, V, (5,), generator=g).tolist() + passage + passage[: n // 6]


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("k", [1, 4, 7])
def test_prompt_lookup_equals_greedy(dev, key, k):
    model = _model(key, dev)
    total_accepted = 0
    for seed in range(3):
        prompt = _repeating_prompt(seed, model.vocab_size)
        want = greedy_generate_ids(model, prompt, 160, device=dev)
        got, st = prompt_lookup_generate_ids(model, prompt, 160, proposal_length=k, device=dev)
        assert got == want, (key, k, seed)
        assert all(p in (0, k) and a <= p for p, a in st) and any(p for p, _ in st)
        total_accepted += sum(a for _, a in st)
        _pools_whole(model)
    assert total_accepted > 0, "prompts that repeat a passage accept proposals"
    assert model.verify_engine(k + 1).captures == 1 and model.decode_engine(1).captures <= 1


def test_a_pinned_prompt_accepts_proposals(dev):
    model = _model("d128", dev)
    prompt = _repeating_prompt(0, model.vocab_size)
    got, st = prompt_lookup_generate_ids(model, prompt, 200, proposal_length=4, device=dev)
    assert got == greedy_generate_ids(model, prompt, 200, device=dev)
    assert sum(a for _, a in st) > 0
    print(f"pinned: {len(st)} rounds, {sum(1 for p, _ in st if p)} matched, {sum(a for _, a in st)}/{sum(p for p, _ in st)} accepted")


def test_yarn_history_past_8192_tokens_equals_greedy(dev):
    yarn = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 4096}
    ns = synthetic_qwen3("tiny-d128", seed=3, device=dev, realistic=True, max_position_embeddings=16384, rope_scaling=yarn)
    model = Qwen3ModelWeek3(ns, page_size=128)
    model.prefill_graph_len = 0
    model.set_max_context(16384)
    g = torch.Generator().manual_seed(1)
    passage = torch.randint(0, model.vocab_size, (700,), generator=g).tolist()
    prompt = (passage * 12)[:8300]
    want = greedy_generate_ids(model, prompt, 48, device=dev)
    got, st = prompt_lookup_generate_ids(model, prompt, 48, proposal_length=4, device=dev)
    assert got == want and len(prompt) + len(got) > 8192
    assert model._verify_engines and any(p for p, _ in st)
    _pools_whole(model)


def test_moe_runs_the_generic_runner_to_greedys_ids(dev):
    ns = synthetic_qwen3("tiny-moe-d128", device=dev, seed=0, realistic=True, max_position_embeddings=512)
    model = Qwen3ModelWeek3(ns, page_size=128)
    model.prefill_graph_len = 0
    assert not gen._graph_runner_applies(model, None, dev, 4)
    prompt = _repeating_prompt(2, model.vocab_size, n=60)
    got, st = prompt_lookup_generate_ids(model, prompt, 40, proposal_length=4, ngram=(1, 3), device=dev)
    want = greedy_generate_ids(model, prompt, 40, device=dev)
    # the generic runner's multi-row pass is the operator path, which does not round like the decode step: its ids
    # are greedy's up to the first near-tie, and always its first token
    assert len(got) == 40 and got[0] == want[0] and st and any(p for p, _ in st)
    _pools_whole(model)


def test_each_sampled_round_equals_the_float64_rule_in_situ(dev, monkeypatch):
    model = _model("d128", dev)
    params = SamplingParams(1.0, top_p=0.95, seed=4)
    rounds = []
    original = gen._GraphRunner.verify

    def recording(self, token, proposals, offset, cache):
        rows = self._draft_rows.clone()
        out = original(self, token, proposals, offset, cache)
        k = int(proposals.numel())
        rounds.append((rows, self.model.verify_engine(k + 1).logits.clone(), proposals.clone(), out[0], offset))
        return out

    monkeypatch.setattr(gen._GraphRunner, "verify", recording)
    prompt = _repeating_prompt(4, model.vocab_size)
    got, st = prompt_lookup_generate_ids(model, prompt, 80, proposal_length=4, ngram=(1, 3), device=dev, sampling=params)
    assert len(got) == 80 and rounds
    rejected = exceptions = 0
    for rows, logits, d, out, offset in rounds:
        x, y, d = logits.double().cpu().numpy(), rows.double().cpu().numpy(), d.tolist()
        for j in range(len(d)):
            assert (y[j] == 0).sum() == 1 and y[j][d[j]] == 0, "the draft row is the one-hot row of its proposal"
            want = SR.rule_row(x[j], y[j], d[j], 1.0, 0, 0.95, params.seed, offset + j + 1)
            if out[j] != want.token:
                p = SR.row_dist(x[j], 1.0, 0, 0.95)
                assert want.margin <= REL * max(p[d[j]], 1.0) or want.residual_gap <= GAP
                exceptions += 1
            if not want.accepted:
                rejected += 1
                break
    assert rejected > 0 and exceptions <= 1
    _pools_whole(model)
    assert len(model.verify_engine(5)._graph_spec) == 1, "one sampled verify graph: the one-hot buffer does not move"


def test_a_matched_round_is_one_launch_and_one_replay_without_token_uploads(dev, monkeypatch):
    model = _model("d128", dev)
    k = 4
    engine = model.verify_engine(k + 1)
    prompt = _repeating_prompt(1, model.vocab_size)
    prompt_lookup_generate_ids(model, prompt, 100, proposal_length=k, device=dev)  # captures the graphs
    seen = []
    propose, verify = gen._GraphRunner.propose, gen._GraphRunner.verify

    def counting_propose(self, committed, token):
        self._before = (ext.launch_count(), engine.graph_replays, engine.h2d_bytes)
        out = propose(self, committed, token)
        self._matched = out is not None
        if out is not None:
            assert ext.launch_count() - self._before[0] == 1, "one proposer launch"
        return out

    def counting_verify(self, token, proposals, offset, cache):
        out = verify(self, token, proposals, offset, cache)
        seen.append((ext.launch_count() - self._before[0], engine.graph_replays - self._before[1], engine.h2d_bytes - self._before[2]))
        return out

    monkeypatch.setattr(gen._GraphRunner, "propose", counting_propose)
    monkeypatch.setattr(gen._GraphRunner, "verify", counting_verify)
    got, st = prompt_lookup_generate_ids(model, prompt, 100, proposal_length=k, device=dev)
    assert got == greedy_generate_ids(model, prompt, 100, device=dev)
    assert seen and len(seen) == sum(1 for p, _ in st if p)
    T = k + 1
    for launches, replays, h2d in seen:
        # the proposer's launch, the verify graph's replay, and only the verify pass's own metadata upload (tokens |
        # offsets | context_lens, T int32 each, the proposals' slots overwritten device to device; block tables too
        # when the cache gained a page)
        assert (launches, replays) == (1, 1) and h2d in (3 * T * 4, engine._meta_len * 4)
