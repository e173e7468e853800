"""Parallel sampling on the H100: ``tl_shared_prefix_attention`` against the float64 paged reference on each row's
full table (G = 2, 4, 8; groups of 1..16 slots beside ungrouped and idle slots; shared runs of 0, 1 and many pages;
1 and many private tokens; 128 to 16K shared tokens), exact needles in shared and private pages, row independence,
and ``parallel_sample_ids`` on the decode engine: ungrouped runs against separately prefilled caches and
``greedy_generate_ids``, grouped runs against teacher-forced scores with a corrupted-page negative control, and the
pages afterwards."""

import importlib.util
import math
import sys
import zlib
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, greedy_generate_ids, parallel_sample_ids, score_ids
from tiny_llm_b200 import engine as eng
from tiny_llm_b200 import generate as gen
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


AR = _load("tiny_llm_b200_attention_ref", "attention_ref.py")
plan = _load("tiny_llm_b200_engine_plan", "engine_plan.py")

pytestmark = pytest.mark.gpu
PAGE, D = 64, 128


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def _layout(g, groups, lone, idle, shared_pages, private, max_pages):
    """Block tables / context lengths of the slots: each group's slots share their first pages, then own private ones.
    groups: counts; lone: ungrouped slots; idle: slots with context 0.  Returns (tables, lens, descriptors, B, P)."""
    B = sum(groups) + lone + idle
    tables = torch.full((B, max_pages), -1, dtype=torch.int32)
    lens = torch.zeros(B, dtype=torch.int32)
    desc = []
    nxt = 0
    b = 0
    for count in groups:
        shared = list(range(nxt, nxt + shared_pages))
        nxt += shared_pages
        for s in range(count):
            ctx = shared_pages * PAGE + int(g.integers(1, private + 1))
            own = -(-ctx // PAGE) - shared_pages
            tables[b, :shared_pages] = torch.tensor(shared, dtype=torch.int32) if shared else tables[b, :0]
            tables[b, shared_pages : shared_pages + own] = torch.arange(nxt, nxt + own, dtype=torch.int32)
            nxt += own
            lens[b] = ctx
            b += 1
        desc.append((b - count, count, shared_pages))
    for _ in range(lone):
        ctx = int(g.integers(1, shared_pages * PAGE + private + 1))
        own = -(-ctx // PAGE)
        tables[b, :own] = torch.arange(nxt, nxt + own, dtype=torch.int32)
        nxt += own
        lens[b] = ctx
        b += 1
    perm = torch.from_numpy(g.permutation(nxt + 1)).to(torch.int32)  # shuffled physical pages
    tables = torch.where(tables >= 0, perm[tables.clamp(min=0).long()], tables)
    return tables, lens, desc, B, nxt + 1


def _run(dev, q, kp, vp, tables, lens, desc, Hq, Hkv, scale):
    groups = torch.tensor(desc or [(0, 0, 0)], dtype=torch.int32).view(-1, 3)
    return ext.shared_prefix_attention(q.to(dev), kp.to(dev), vp.to(dev), tables.to(dev), lens.to(dev), groups.to(dev), groups.contiguous(),
                                       scale, Hkv, Hq)


CASES = [  # (G, groups, lone, idle, shared_pages, private tokens)
    (2, [1], 0, 0, 2, 1), (2, [16, 3], 1, 1, 3, 70), (4, [2], 1, 0, 1, 1), (4, [8], 0, 1, 4, 130), (4, [3, 8, 1], 2, 1, 2, 64),
    (8, [16], 0, 0, 2, 5), (8, [2, 3], 1, 1, 0, 200), (8, [8], 1, 0, 5, 64), (4, [16, 16], 0, 0, 1, 1),
]


@pytest.mark.parametrize("case", CASES, ids=[str(i) for i in range(len(CASES))])
def test_kernel_matches_float64_reference(dev, case):
    import numpy as np

    G, groups, lone, idle, shared_pages, private = case
    g = np.random.default_rng(zlib.crc32(repr(case).encode()))
    Hkv = 2
    Hq = G * Hkv
    max_pages = shared_pages + -(-private // PAGE) + 2
    tables, lens, desc, B, P = _layout(g, groups, lone, idle, shared_pages, private, max_pages)
    q = torch.randn(B * Hq, 1, D).to(torch.bfloat16)
    kp = torch.randn(P, Hkv, PAGE, D).to(torch.bfloat16)
    vp = torch.randn(P, Hkv, PAGE, D).to(torch.bfloat16)
    scale = 1 / math.sqrt(D)
    got = _run(dev, q, kp, vp, tables, lens, desc, Hq, Hkv, scale).cpu()
    ref, A, smax, nvis = AR.paged_reference(q, kp, vp, tables, lens, scale, True, Hkv, Hq)
    AR.assert_within(got, ref, AR.error_bound(ref, A, smax, nvis, D, torch.bfloat16, True), f"case {case}")
    idle_rows = (lens == 0).repeat_interleave(Hq)
    assert torch.equal(got[idle_rows], torch.zeros_like(got[idle_rows]))


@pytest.mark.parametrize("shared_tokens", [128, 1024, 4096, 16384])
def test_split_counts_over_long_shared_runs(dev, shared_tokens):
    import numpy as np

    g = np.random.default_rng(shared_tokens)
    shared_pages = shared_tokens // PAGE
    Hkv, Hq = 8, 32
    tables, lens, desc, B, P = _layout(g, [8], 0, 0, shared_pages, 100, shared_pages + 4)
    q = torch.randn(B * Hq, 1, D).to(torch.bfloat16)
    kp = (0.5 * torch.randn(P, Hkv, PAGE, D)).to(torch.bfloat16)
    vp = torch.randn(P, Hkv, PAGE, D).to(torch.bfloat16)
    scale = 1 / math.sqrt(D)
    got = _run(dev, q, kp, vp, tables, lens, desc, Hq, Hkv, scale).cpu()
    ref, A, smax, nvis = AR.paged_reference(q, kp, vp, tables, lens, scale, True, Hkv, Hq)
    AR.assert_within(got, ref, AR.error_bound(ref, A, smax, nvis, D, torch.bfloat16, True), f"{shared_tokens} shared tokens")


def _needle_setup(g, G=4):
    Hkv = 2
    Hq = G * Hkv
    tables, lens, desc, B, P = _layout(g, [4, 3], 1, 0, 2, 90, 6)
    q = torch.zeros(B * Hq, 1, D, dtype=torch.bfloat16)
    q[:, 0, 0] = 8.0  # every query looks along dimension 0
    kp = torch.zeros(P, Hkv, PAGE, D, dtype=torch.bfloat16)
    vp = torch.zeros(P, Hkv, PAGE, D, dtype=torch.bfloat16)
    return Hq, Hkv, tables, lens, desc, B, P, q, kp, vp


def test_needle_in_a_shared_page_reaches_every_row_of_its_group(dev):
    import numpy as np

    Hq, Hkv, tables, lens, desc, B, P, q, kp, vp = _needle_setup(np.random.default_rng(1))
    page = int(tables[0, 1])
    kp[page, :, 17, 0] = 100.0  # dominates every row that sees it
    vp[page, :, 17, 5] = 1.0
    got = _run(dev, q, kp, vp, tables, lens, desc, Hq, Hkv, 1.0).cpu().view(B, Hq, D)
    for b in range(B):
        want = 1.0 if b < 4 else 0.0
        assert torch.all(got[b, :, 5].float() == want), f"slot {b}"


def test_needle_in_a_private_page_stays_in_its_sample(dev):
    import numpy as np

    Hq, Hkv, tables, lens, desc, B, P, q, kp, vp = _needle_setup(np.random.default_rng(2))
    k = 2  # sample 2 of group 0
    last = int(lens[k]) - 1  # its last key, in a private page
    page, slot = int(tables[k, last // PAGE]), last % PAGE
    kp[page, :, slot, 0] = 100.0
    vp[page, :, slot, 7] = 1.0
    got = _run(dev, q, kp, vp, tables, lens, desc, Hq, Hkv, 1.0).cpu().view(B, Hq, D)
    for b in range(B):
        assert torch.all(got[b, :, 7].float() == (1.0 if b == k else 0.0)), f"slot {b}"


def test_row_independence(dev):
    """A row's bits do not depend on the group's other queries or on count, at a fixed layout of groups."""
    import numpy as np

    g = np.random.default_rng(3)
    G, Hkv = 4, 2
    Hq = G * Hkv
    tables, lens, desc, B, P = _layout(g, [8], 1, 0, 3, 50, 6)
    q = torch.randn(B * Hq, 1, D).to(torch.bfloat16)
    kp = torch.randn(P, Hkv, PAGE, D).to(torch.bfloat16)
    vp = torch.randn(P, Hkv, PAGE, D).to(torch.bfloat16)
    base = _run(dev, q, kp, vp, tables, lens, desc, Hq, Hkv, 0.1).cpu().view(B, Hq, D)
    q2 = q.clone().view(B, Hq, D)
    q2[1:8] = torch.randn(7, Hq, D).to(torch.bfloat16)
    other = _run(dev, q2.view(-1, 1, D), kp, vp, tables, lens, desc, Hq, Hkv, 0.1).cpu().view(B, Hq, D)
    assert torch.equal(base[0], other[0]) and torch.equal(base[8], other[8])
    fewer = _run(dev, q, kp, vp, tables, lens, [(0, 5, 3)], Hq, Hkv, 0.1).cpu().view(B, Hq, D)
    assert torch.equal(base[:5], fewer[:5])


# ------------------------------------------------------------------ the engine --
MODELS = {
    "d128": ("tiny-d128", dict(seed=5, realistic=True, max_position_embeddings=8192)),
    "4b": ("qwen3-4b", dict(seed=1, num_hidden_layers=2, vocab_size=4096)),
}
_NS: dict = {}


def _model(key, dev, window=4096):
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


@pytest.fixture
def rule_on(monkeypatch):
    monkeypatch.setattr(eng, "SHARED_PREFIX_MIN_COUNT", 1)
    monkeypatch.setattr(eng, "SHARED_PREFIX_MIN_TOKENS", 1)


@pytest.fixture
def rule_off(monkeypatch):
    monkeypatch.setattr(eng, "shared_prefix_attention_applies", lambda *a: False)


@pytest.mark.parametrize("key", list(MODELS))
def test_single_sample_equals_greedy_generate(dev, key, rule_off):
    m = _model(key, dev)
    prompt = _prompt(1, m.vocab_size, 150)
    s = SamplingParams(0.8, top_k=50, seed=7)
    got = parallel_sample_ids(m, [prompt], 1, s, 20)[0][0]
    assert got.ids == greedy_generate_ids(m, prompt, 20, sampling=s, device=dev)
    _pools_whole(m)


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("P, n", [(1, 4), (2, 6)])  # B = 4 (matvec stack) and B = 12 (swap-AB stack)
def test_ungrouped_samples_equal_separate_prefills(dev, key, P, n, rule_off):
    """With the rule off, sample j equals slot j of an n-slot run over separately prefilled, unforked caches."""
    m = _model(key, dev)
    prompts = [_prompt(10 + i, m.vocab_size, 140 + 60 * i) for i in range(P)]
    s = SamplingParams(0.9, seed=11)
    got = parallel_sample_ids(m, prompts, n, s, 12)
    from dataclasses import replace

    for i, prompt in enumerate(prompts):
        for j in range(n):
            want = greedy_generate_ids(m, prompt, 12, sampling=replace(s, seed=gen.sample_seed(11, j)), device=dev)
            assert got[i][j].ids == want, (i, j)
    _pools_whole(m)


def _worst_gap(m, prompt, samples):
    """Largest |reported - teacher-forced| log-probability over the samples' ids (``score_ids`` entry k scores id k + 1)."""
    worst = 0.0
    for s in samples:
        tf = [e.logprob for e in score_ids(m, prompt + s.ids, device=m.embedding.weight.scales.device).entries[len(prompt) - 1 :]]
        assert len(tf) == len(s.ids) == len(s.logprobs)
        worst = max([worst] + [abs(e.logprob - t) for e, t in zip(s.logprobs, tf)])
    return worst


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("P, n, length", [(1, 4, 700), (2, 8, 300)])
def test_grouped_logprobs_match_teacher_forcing(dev, key, P, n, length, rule_on):
    m = _model(key, dev)
    prompts = [_prompt(20 + i, m.vocab_size, length + 37 * i) for i in range(P)]
    engine = m.decode_engine(P * n, m.decode_graph_max_seq_len)
    before = [pool._key_pages.data_ptr() for pool in m.page_pools]
    got = parallel_sample_ids(m, prompts, n, SamplingParams(1.0, seed=3), 10, logprobs=0)
    assert engine._graph_grp, "the grouped twin ran"
    page = m.page_size
    want = [(i * n, n, (length + 37 * i) // page) for i in range(P)]
    assert engine._grp_host[:P].tolist() == [list(d) for d in want], "the last round's descriptors share the prompt pages"
    assert [pool._key_pages.data_ptr() for pool in m.page_pools] == before, "no slab was reallocated"
    # bf16 activations: the decode step and the chunked teacher-forced pass round differently; 0.15 nats bounds it
    worst = max(_worst_gap(m, prompt, got[i]) for i, prompt in enumerate(prompts))
    assert worst < 0.15, f"grouped log-probabilities differ from teacher forcing by {worst}"
    _pools_whole(m)


def test_corrupted_shared_page_fails_the_teacher_forced_check(dev, rule_on, monkeypatch):
    """Negative control of the teacher-forced check: with the prompt's shared K pages scaled after the fork, what the
    samples report no longer matches a rescoring over intact pages.  (That the grouped step reads the shared pages
    through the grouped kernel is shown bit for bit by ``test_grouped_step_graph_equals_its_launch_plan``.)"""
    m = _model("4b", dev)
    prompt = _prompt(31, m.vocab_size, 700)
    from tiny_llm_b200 import paged_kv_cache as pkv

    real_fork = pkv.fork

    def corrupting_fork(requests):
        out = real_fork(requests)
        for caches, _ in requests:
            for layer, c in enumerate(caches):
                pool = m.page_pools[layer]
                for pid in c.page_ids[:2]:
                    pool._key_pages[pid].mul_(-3.0)
        return out

    monkeypatch.setattr(pkv, "fork", corrupting_fork)
    got = parallel_sample_ids(m, [prompt], 4, SamplingParams(1.0, seed=3), 8, logprobs=0)[0]
    monkeypatch.setattr(pkv, "fork", real_fork)
    assert _worst_gap(m, prompt, got) >= 0.15
    _pools_whole(m)


class GroupedPlan(plan.Plan):
    """``engine_plan.Plan``'s unfused decode step with ``tl_shared_prefix_attention`` over ``descriptors`` in place of
    ``tl_paged_attention``: the launches of the grouped twin, issued eagerly."""

    def __init__(self, model, descriptors):
        super().__init__(model)
        dev = model.embedding.weight.scales.device
        self.groups_host = torch.tensor(descriptors, dtype=torch.int32).view(-1, 3).contiguous()
        self.groups = self.groups_host.to(dev)

    def _paged(self, name, layer, q, kp, vp, table, ctx, L, token_major=False):
        out = ext.shared_prefix_attention(q, kp, vp, table, ctx, self.groups, self.groups_host, self.scale, self.Hkv, self.Hq)
        self._rec(name, layer, dict(q=q, table=table, ctx=ctx, L=L), out)
        return out


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("P, n", [(1, 4), (2, 6)])  # B = 4 (matvec stack) and B = 12 (swap-AB stack)
def test_grouped_step_graph_equals_its_launch_plan(dev, key, P, n, rule_on):
    """One replay of the grouped twin equals its launches issued eagerly over the same descriptors, bit for bit (logits
    and every slab), the device descriptors it read share the prompt pages, and at the Qwen3-4B width its logits differ
    in bits from the plain step's launches at the same state: the graph attends each group's shared pages through the
    grouped kernel, with the call's descriptors."""
    from tiny_llm_b200 import paged_kv_cache as pkv
    from tiny_llm_b200.kv_cache import BatchingKvCache

    m = _model(key, dev)
    page = m.page_size
    prompts = [_prompt(40 + i, m.vocab_size, 300 + 70 * i) for i in range(P)]
    B = P * n
    engine = m.decode_engine(B, m.decode_graph_max_seq_len)
    slots = []
    for prompt in prompts:
        cache = m.create_kv_cache()
        m(torch.as_tensor(prompt, dtype=torch.int32, device=dev)[None], 0, cache, logits_to_keep=1)
        slots += [cache] + pkv.fork([(cache, n - 1)])[0]
    batch = [BatchingKvCache(B) for _ in range(len(slots[0]))]
    for layer, bc in enumerate(batch):
        bc.kv_caches = [c[layer] for c in slots]
    tokens = [(13 * b + 5) % m.vocab_size for b in range(B)]
    offsets = [len(prompts[b // n]) for b in range(B)]
    descriptors = [(i * n, n, len(prompts[i]) // page) for i in range(P)]
    assert all(d[2] > 0 for d in descriptors)
    before = [(p._key_pages.clone(), p._value_pages.clone()) for p in m.page_pools]
    try:
        engine.decode_on_device(tokens, offsets, batch, 1, sampling=SamplingParams(1.0, seed=1), groups=[(i * n, n) for i in range(P)])
        assert engine._grp_host[:P].tolist() == [list(d) for d in descriptors]
        assert engine._grp_dev[:P].tolist() == [list(d) for d in descriptors], "the descriptors the replay read"
        got = engine.logits.clone()
        meta = plan.decode_metadata(batch, tokens, engine.max_pages, steps=1)
        assert meta.offsets == offsets
        pages = [(k.clone(), v.clone()) for k, v in before]
        want, _ = GroupedPlan(m, descriptors + [(0, 0, 0)] * (B - P)).decode(meta, pages, attention_fused=False)
        assert torch.equal(got, want), "grouped graph against its eager launches"
        for i, (pool, (kp, vp)) in enumerate(zip(m.page_pools, pages)):
            assert torch.equal(pool._key_pages, kp) and torch.equal(pool._value_pages, vp), f"layer {i} slabs"
        if key == "4b":  # at tiny-d128's 2 x 4 heads the two sum orders can round to the same bf16 outputs everywhere
            plain_pages = [(k.clone(), v.clone()) for k, v in before]
            plain, _ = plan.Plan(m).decode(meta, plain_pages, attention_fused=False)
            assert not torch.equal(got, plain), "the grouped step must not be the plain step's bits"
    finally:
        for c in slots:
            gen._release_kv_cache(c)
    _pools_whole(m)


def test_existing_graph_kinds_keep_their_launch_counts(dev, rule_on):
    m = _model("4b", dev)
    prompt = _prompt(5, m.vocab_size, 300)
    engine = m.decode_engine(4, m.decode_graph_max_seq_len)
    greedy_generate_ids(m, prompt, 2, device=dev)
    parallel_sample_ids(m, [prompt], 4, SamplingParams(1.0, seed=1), 4)
    assert engine._graph_grp and engine._graph_sample is None, "the call replayed the grouped twin"
    engine._ensure_sample_graph()  # captured after the grouped twin, beside it
    counts = (engine.kernels_per_step, engine.kernels_per_sampled_step)
    fresh = eng.DecodeEngine(m, 4, m.decode_graph_max_seq_len, engine.device)
    fresh.reserve_pools()
    fresh._ensure_graph()
    fresh._ensure_sample_graph()
    assert (fresh.kernels_per_step, fresh.kernels_per_sampled_step) == counts
    _pools_whole(m)
