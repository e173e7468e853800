"""Speculative sampling on the GPU: ``tl_speculative_sample`` against the float64 rule (``spec_sample_ref.py``), its
bonus row against ``tl_sample`` bit for bit, row independence and graph replay, the output distribution over 60,000
rows, and sampled ``speculative_generate_ids`` on the graph and generic runners."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import stats

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids, speculative_generate_ids
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


R = _load("tiny_llm_b200_spec_sample_ref", "spec_sample_ref.py")

pytestmark = pytest.mark.gpu

# The kernel's p and q are fixed-point sums of fp32 exp terms: each term is within ~1e-5 relative of the float64 value
# (fp32 rounding of (x - m) / T and of expf, for exponents down to -87), each sum within 2^-40 per term.  A decision
# may differ from the float64 rule only where that error can flip it: |u q_d - p_d| within REL of max(p_d, q_d), or a
# residual whose top two float64 scores are within GAP.
REL = 2e-5
GAP = 1e-3


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def _row(kind, V, g):
    if kind == "random":
        return torch.randn(V, generator=g) * 2
    if kind == "peaked":
        x = torch.randn(V, generator=g)
        x[torch.randint(0, V, (3,), generator=g)] += 12
        return x
    if kind == "tied":
        return torch.randint(-3, 3, (V,), generator=g).float()
    x = torch.randn(V, generator=g)  # non-finite
    x[int(torch.randint(0, V, (1,), generator=g))] = float("inf")
    x[int(torch.randint(0, V, (1,), generator=g))] = float("nan")
    return x


def _launch(dev, x, y, params, n0, proposals=None):
    """One launch over target rows x [T, V], draft rows y [T - 1, V] (proposals drawn by tl_sample from y unless
    given), positions n0 + j."""
    T = x.shape[0]
    per = sampling_tensors([params] * T, dev)
    pos = torch.arange(n0, n0 + T, dtype=torch.int32, device=dev)
    if proposals is None:
        proposals = ext.sample(y, *[t[: T - 1] for t in per], pos[: T - 1]) if T > 1 else torch.zeros(0, dtype=torch.int32, device=dev)
    out = ext.speculative_sample(x, y, proposals, *per, pos)
    return out, proposals, per, pos


CASES = [(torch.float32, 1000), (torch.bfloat16, 4097), (torch.bfloat16, 151936)]
PARAMS = [(t, k, p) for t in (0.0, 0.7, 1.3) for k in (0, 50) for p in (0.0, 0.9)]


@pytest.mark.parametrize("dtype,V", CASES, ids=lambda v: str(v))
def test_kernel_against_the_float64_rule(dev, dtype, V):
    g = torch.Generator().manual_seed(V)
    decisions = exceptions = 0
    for i, (temp, top_k, top_p) in enumerate(PARAMS):
        for kind in ("random", "peaked", "tied", "nonfinite"):
            k = 1 + (i + len(kind)) % 7
            x = torch.stack([_row(kind, V, g) for _ in range(k + 1)]).to(dtype)
            # the draft rows: the target's perturbed, so that both acceptance and rejection occur
            y = (x[:k].float() + torch.randn(k, V, generator=g) * 0.7).to(dtype)
            params = SamplingParams(temp, top_k=top_k or None, top_p=top_p or None, seed=1000 + i)
            out, d, _, _ = _launch(dev, x.to(dev), y.to(dev), params, 17)
            out, d = out.tolist(), d.tolist()
            xs, ys = x.double().numpy(), y.double().numpy()
            for j in range(k):
                want = R.rule_row(xs[j], ys[j], d[j], temp, top_k, top_p, params.seed, 17 + j)
                decisions += 1
                if out[j] != want.token:
                    p = R.row_dist(xs[j], temp, top_k, top_p)
                    q = R.row_dist(ys[j], temp, top_k, top_p)
                    near = want.margin <= REL * max(p[d[j]], q[d[j]]) or want.residual_gap <= GAP
                    assert near, f"{kind} {params} row {j}: kernel {out[j]}, rule {want.token} ({want})"
                    exceptions += 1
    assert exceptions <= max(1, decisions // 50), f"{exceptions} near-boundary decisions of {decisions}"
    print(f"{dtype} V={V}: {decisions} decisions, {exceptions} within the error bound")


@pytest.mark.parametrize("dtype,V", CASES, ids=lambda v: str(v))
def test_identical_rows_accept_every_drawn_proposal_and_the_bonus_row_is_tl_sample(dev, dtype, V):
    g = torch.Generator().manual_seed(3 * V)
    for i, (temp, top_k, top_p) in enumerate(PARAMS):
        for kind in ("random", "peaked", "tied", "nonfinite"):
            x = torch.stack([_row(kind, V, g) for _ in range(8)]).to(dtype).to(dev)
            params = SamplingParams(temp, top_k=top_k or None, top_p=top_p or None, seed=7 + i)
            out, d, per, pos = _launch(dev, x, x[:7].contiguous(), params, 40)
            assert torch.equal(out[:7], d), f"{kind} {params}: a proposal drawn from p itself was rejected"
            bonus = ext.sample(x[7:], *[t[7:] for t in per], pos[7:])
            assert int(out[7]) == int(bonus[0])


def test_rows_are_independent_of_their_index_and_replay_under_a_graph(dev):
    V, k = 4097, 7
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(k + 1, V, generator=g) * 2).to(torch.bfloat16).to(dev)
    y = (x[:k].float().cpu() + torch.randn(k, V, generator=g)).to(torch.bfloat16).to(dev)
    params = SamplingParams(1.0, top_k=200, top_p=0.95, seed=5)
    full, d, per, pos = _launch(dev, x, y, params, 100)
    for j in range(k):  # row j alone, as row 0 of a two-row launch at its own position
        xx = torch.stack([x[j], x[k]])
        out, _, _, _ = _launch(dev, xx, y[j : j + 1].contiguous(), params, 100 + j, proposals=d[j : j + 1].contiguous())
        assert int(out[0]) == int(full[j])
    out = torch.empty_like(full)
    ext.speculative_sample(x, y, d, *per, pos, out=out)  # warm-up outside the capture
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ext.speculative_sample(x, y, d, *per, pos, out=out)
    out.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, full)


def test_output_distribution_over_60000_rows_passes_a_chi_square_test(dev):
    x = torch.tensor([1.2, 0.3, -0.5, 2.0, 0.9, -1.1, 0.0, 1.5])
    y = torch.tensor([0.1, 1.4, 0.8, 1.9, -0.3, 0.5, 1.1, -0.8])
    rows, temp, top_k, top_p = 60_000, 0.9, 7, 0.97
    X = x.repeat(rows + 1, 1).to(dev)
    Y = y.repeat(rows, 1).to(dev)
    T = rows + 1
    temperature = torch.full((T,), temp, device=dev)
    tk = torch.full((T,), top_k, dtype=torch.int32, device=dev)
    tp = torch.full((T,), top_p, device=dev)
    seed = torch.arange(T, dtype=torch.int64, device=dev)
    pos = torch.full((T,), 11, dtype=torch.int32, device=dev)
    d = ext.sample(Y, temperature[:rows], tk[:rows], tp[:rows], seed[:rows], pos[:rows])
    out = ext.speculative_sample(X, Y, d, temperature, tk, tp, seed, pos)[:rows].cpu().numpy()
    p = R.row_dist(x.double().numpy(), temp, top_k, top_p)
    counts = np.bincount(out, minlength=8).astype(np.float64)
    assert counts[p == 0].sum() == 0
    live = p > 0
    assert stats.chisquare(counts[live], rows * p[live]).pvalue > 1e-3
    # the proposals alone are far from p: the test sees the rule's correction, not the draft's draws
    dc = np.bincount(d.cpu().numpy(), minlength=8) / rows
    assert np.abs(dc - p).max() > 0.05


def test_vocabularies_above_the_staging_limit_are_refused_before_a_launch(dev):
    V = ext.SPECULATIVE_SAMPLE_MAX_VOCAB + 8
    x = torch.zeros(2, V, device=dev)
    per = sampling_tensors([SamplingParams(1.0)] * 2, dev)
    with pytest.raises(RuntimeError, match="exceeds"):
        ext.speculative_sample(x, x[:1], torch.zeros(1, dtype=torch.int32, device=dev), *per, torch.zeros(2, dtype=torch.int32, device=dev))


# ------------------------------------------------------------------ end to end --
D128 = ("tiny-d128", dict(seed=5, realistic=True, max_position_embeddings=8192))
_NS: dict = {}


def _model(dev, seed=5, name="tiny-d128"):
    if (name, seed) not in _NS:
        _NS[(name, seed)] = synthetic_qwen3(name, device=dev, **{**D128[1], "seed": seed})
    m = Qwen3ModelWeek3(_NS[(name, seed)], page_size=128)
    m.prefill_graph_len = 0
    return m


PROMPT = [5, 17, 3, 250, 9, 44, 100]
SAMPLINGS = [SamplingParams(0.7, top_p=0.9, seed=3), SamplingParams(1.0, seed=11), SamplingParams(1.3, top_k=20, top_p=0.95, seed=2)]


def _pools_whole(*models):
    for m in models:
        for pool in m.page_pools:
            assert not pool.used_page_ids, "every page is back in its pool"


@pytest.fixture(scope="module")
def target(dev):
    return _model(dev)


@pytest.mark.parametrize("k", [1, 4, 7])
@pytest.mark.parametrize("si", range(len(SAMPLINGS)))
def test_same_weights_draft_accepts_everything_and_equals_sampled_generate(dev, target, k, si):
    params = SAMPLINGS[si]
    draft = _model(dev)
    want = greedy_generate_ids(target, PROMPT, 120, device=dev, sampling=params)
    got, st = speculative_generate_ids(draft, target, PROMPT, 120, proposal_length=k, device=dev, sampling=params)
    assert got == want
    assert sum(a for _, a in st) == sum(p for p, _ in st) > 0
    _pools_whole(target, draft)
    assert target.verify_engine(k + 1).captures == 1 and draft.decode_engine(1).captures == 1
    assert target.decode_engine(1).captures <= 1
    # the sampled verify graph issues no more launches than the greedy one (one kernel in place of argmax's two passes)
    assert target.verify_engine(k + 1).kernels_per_sampled_verify <= target.verify_engine(k + 1).kernels_per_step


def test_each_round_equals_the_float64_rule_in_situ(dev, target, monkeypatch):
    draft = _model(dev, seed=11)
    params = SamplingParams(1.0, top_p=0.95, seed=4)
    rounds = []
    original = gen._GraphRunner.verify

    def recording(self, token, proposals, offset, cache):
        rows = self._draft_rows.clone()
        out = original(self, token, proposals, offset, cache)
        k = int(proposals.numel())
        logits = self.model.verify_engine(k + 1).logits.clone()
        rounds.append((rows, logits, proposals.clone(), out[0], offset))
        return out

    monkeypatch.setattr(gen._GraphRunner, "verify", recording)
    got, st = speculative_generate_ids(draft, target, PROMPT, 60, proposal_length=4, device=dev, sampling=params)
    assert len(got) == 60 and rounds
    accepted = rejected = exceptions = 0
    for rows, logits, d, out, offset in rounds:
        x, y, d = logits.double().cpu().numpy(), rows.double().cpu().numpy(), d.tolist()
        for j in range(len(d)):
            want = R.rule_row(x[j], y[j], d[j], 1.0, 0, 0.95, params.seed, offset + j + 1)
            if out[j] != want.token:
                p, q = R.row_dist(x[j], 1.0, 0, 0.95), R.row_dist(y[j], 1.0, 0, 0.95)
                assert want.margin <= REL * max(p[d[j]], q[d[j]]) or want.residual_gap <= GAP
                exceptions += 1
            accepted += want.accepted
            rejected += not want.accepted
            if not want.accepted:
                break  # rows past the first rejection are discarded
    assert rejected > 0 and exceptions <= 1
    _pools_whole(target, draft)


@pytest.mark.parametrize("kind", ["k8", "moe"])
def test_generic_runner_samples_to_completion(dev, kind):
    if kind == "moe":
        ns = synthetic_qwen3("tiny-moe-d128", device=dev, seed=0, realistic=True, max_position_embeddings=512)
        target = Qwen3ModelWeek3(ns, page_size=128)
        draft = _model(dev, seed=11)
        k = 4
    else:
        target, draft, k = _model(dev), _model(dev, seed=11), 8
    assert not gen._graph_runner_applies(target, draft, dev, k)
    params = SamplingParams(0.8, top_k=40, seed=9)
    got, st = speculative_generate_ids(draft, target, PROMPT, 40, proposal_length=k, device=dev, sampling=params)
    # every round checks both caches' offsets (the protocol raises otherwise)
    assert len(got) == 40 and all(p <= k for p, _ in st) and st
    first = greedy_generate_ids(target, PROMPT, 1, device=dev, sampling=params)
    assert got[0] == first[0]  # the target's first token is tl_sample's draw on the prefill's last row
    _pools_whole(target, draft)
