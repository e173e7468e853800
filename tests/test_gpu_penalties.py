"""``tl_sample_penalized`` on the H100: every draw against the penalised reference (``penalties_ref``: the penalties
and the min-p threshold restated in fp32, the draw in float64), exact probes, the all-off form against ``tl_sample``,
the token-state update (eager and under graph replay), row independence, and the penalised paths of the engine,
``generate`` and the batcher."""

import importlib.util
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as ref
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, batch_generate, greedy_generate_ids
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.sampler import penalty_tensors, sample_tokens, sampling_tensors, token_state_row
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load_penalties_ref():
    """The helper next to this file, by path: `tests` is no package of this project."""
    name = "tiny_llm_b200_penalties_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("penalties_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


pref = _load_penalties_ref()


def launch(logits, params, positions, state):
    """``ext.sample_penalized`` over the parameters of ``params`` (updates ``state``) -> host int32 tokens."""
    dev = logits.device
    pos = torch.as_tensor(positions, dtype=torch.int32).to(dev)
    return ext.sample_penalized(logits, *sampling_tensors(params, dev), pos, *penalty_tensors(params, dev), state).cpu()


def random_state(rows, V, logits, g):
    """Prompt bits on ~5 % of the tokens, counts 1..5 on ~8 %, and both on a share of each row's top 32 tokens (where
    a penalty changes the draw)."""
    s = torch.zeros(rows, V, dtype=torch.int32)
    s |= torch.where(torch.rand(rows, V, generator=g) < 0.05, 1 << 30, 0).to(torch.int32)
    s += torch.where(torch.rand(rows, V, generator=g) < 0.08, torch.randint(1, 6, (rows, V), generator=g), 0).to(torch.int32)
    top = torch.topk(logits.float().nan_to_num(0.0), min(32, V), dim=1).indices
    hit = torch.rand(top.shape, generator=g) < 0.5
    s.scatter_(1, top, torch.where(hit, (1 << 30) + torch.randint(0, 3, top.shape, generator=g), s.gather(1, top)).to(torch.int32))
    return s


def _tol_accept(x3, T, k, p, mp, seed, pos, got):
    """As test_gpu_sampling's bound, on the penalised row: the kernel's token must be in the loose keep set (top_p + eps)
    and its perturbed score within the fp32 rounding of the best score of the strict keep set (top_p - eps).  min-p and
    top-k are exact (both are comparisons of fp32 values)."""
    x = x3.astype(np.float64)
    ok = ~np.isnan(x)
    V = len(x)
    base = pref.keep_set(x3, k, None, mp, T)
    strict, loose = base.copy(), base.copy()
    if 0 < p < 1:
        M, S = ref.mass_above(x)
        R = float(x[ok].max() - x[ok & np.isfinite(x)].min())
        eps = 2 * (2.0**-22 + R * 2.0**-24) + 2 * V * 2.0**-40 / S
        strict &= M < p - eps
        loose &= M < p + eps
    g = ref.gumbel(V, seed, pos)
    score = x / T + g
    m = x[ok].max()
    d = 2.0**-21 * (1 + np.abs(g) + (np.abs(x) + abs(m)) / T)  # the kernel scores (x - m) / T + g
    if not loose[got]:
        return False
    if not strict.any():
        return True
    best = int(np.argmax(np.where(strict, score, -np.inf)))
    return score[got] + d[got] + d[best] >= score[best]


KP = [(None, None), (50, None), (None, 0.9), (20, 0.5)]


@pytest.mark.parametrize("V,dtype,full", [(1000, torch.float32, True), (4097, torch.bfloat16, True), (151936, torch.bfloat16, False)])
def test_every_draw_equals_the_reference(cuda_device, V, dtype, full):
    g = torch.Generator().manual_seed(V)
    params, positions = [], []
    for T in (0.0, 0.7, 1.3):
        for r in (1.0, 0.8, 1.3):
            for pres in (0.0, 0.5, -0.5):
                for f in (0.0, 0.3):
                    for mp in (0.0, 0.05, 0.3):
                        for j in range(len(KP)) if full else [len(params) % len(KP)]:
                            k, p = KP[j]
                            i = len(params)
                            params.append(SamplingParams(T, k, p, (i * 2654435761) % (1 << 64), r, pres, f, mp))
                            positions.append(1 + 97 * i)
    n = len(params)
    logits = (torch.randn(n, V, generator=g) * torch.tensor([1.0, 3.0, 6.0]).repeat(n)[:n, None]).to(dtype)
    state0 = random_state(n, V, logits, g)
    state = state0.to(cuda_device)
    got = launch(logits.to(cuda_device), params, positions, state).numpy()
    x32 = logits.float().numpy()
    f32 = [t.numpy() for t in sampling_tensors(params, "cpu") + penalty_tensors(params, "cpu")]
    exact = ambiguous = 0
    for i, sp in enumerate(params):
        temp, top_p, rep, pres, freq, mp = (float(f32[j][i]) for j in (0, 2, 4, 5, 6, 7))
        want = pref.sample_row(x32[i], state0[i].numpy(), sp.temperature, sp.top_k, top_p, sp.seed, positions[i], rep, pres, freq, mp)
        if got[i] == want:
            exact += 1
            continue
        x3 = pref.penalize(x32[i], state0[i].numpy(), rep, pres, freq)
        assert sp.temperature > 0 and _tol_accept(x3, sp.temperature, sp.top_k, top_p, mp, sp.seed, positions[i], int(got[i])), (i, sp)
        ambiguous += 1
    print(f"V {V}: {exact} exact, {ambiguous} within the fp32 bound of {n} draws")
    assert ambiguous <= max(1, n // 100)
    want_state = state0.clone()
    want_state[torch.arange(n), torch.from_numpy(got).long()] += 1
    assert torch.equal(state.cpu(), want_state)


def test_exact_probes(cuda_device):
    V = 4097
    dev = cuda_device
    # greedy: the maximum is a prompt token; r = 1.3 moves it below the runner-up
    x = torch.zeros(1, V)
    x[0, 100], x[0, 200] = 5.0, 4.0
    s = torch.zeros(1, V, dtype=torch.int32)
    s[0, 100] = 1 << 30
    assert int(launch(x.to(dev), [SamplingParams(0.0)], [9], s.clone().to(dev))[0]) == 100
    assert int(launch(x.to(dev), [SamplingParams(0.0, repetition_penalty=1.3)], [9], s.clone().to(dev))[0]) == 200
    # min_p = 1 keeps only the maximum's ties: both ties appear over seeds, nothing else
    y = torch.randn(1, V) * 0.01
    y[0, [7, 3000]] = 2.0
    draws = {int(launch(y.to(dev), [SamplingParams(1.0, seed=i, min_p=1.0)], [5], torch.zeros(1, V, dtype=torch.int32, device=dev))[0])
             for i in range(64)}
    assert draws == {7, 3000}
    # rows whose maximum is not finite take the argmax of the penalised row
    rows = torch.randn(4, V)
    rows[0, [10, 20]] = math.inf
    rows[1] = -math.inf
    rows[2, ::3] = math.nan
    rows[2, 50] = math.inf
    rows[3] = math.nan
    st = torch.zeros(4, V, dtype=torch.int32)
    st[0, 10] = 2  # inf stays inf under every penalty
    params = [SamplingParams(0.8, seed=1, repetition_penalty=1.5, presence_penalty=1.0, frequency_penalty=0.5)] * 4
    got = launch(rows.to(dev), params, [3] * 4, st.clone().to(dev))
    for i in range(4):
        assert int(got[i]) == ref.greedy(pref.penalize(rows[i].numpy(), st[i].numpy(), 1.5, 1.0, 0.5).astype(np.float64))


def test_all_off_equals_sample_and_state_update(cuda_device):
    V = 151936
    g = torch.Generator().manual_seed(11)
    n = 48
    logits = (torch.randn(n, V, generator=g) * 3).to(torch.bfloat16).to(cuda_device)
    params = [SamplingParams((0.0, 0.7, 1.3)[i % 3], KP[i % 4][0], KP[i % 4][1], seed=500 + i) for i in range(n)]
    positions = [0 if i % 5 == 0 else 3 + i for i in range(n)]
    state0 = random_state(n, V, logits.cpu(), g).to(cuda_device)
    state = state0.clone()
    got = launch(logits, params, positions, state)
    pos = torch.tensor(positions, dtype=torch.int32, device=cuda_device)
    assert torch.equal(got, ext.sample(logits, *sampling_tensors(params, cuda_device), pos).cpu())
    diff = (state - state0).cpu()
    live = torch.tensor([p > 0 for p in positions])
    assert torch.equal(diff[~live], torch.zeros_like(diff[~live]))
    want = torch.zeros_like(diff)
    want[live, got[live].long()] = 1
    assert torch.equal(diff, want) and torch.equal(state0.cpu() & (1 << 30), state.cpu() & (1 << 30))
    # under graph capture and replay: the same update per replay
    pp = [SamplingParams(0.9, seed=i, repetition_penalty=1.2, presence_penalty=0.4, frequency_penalty=0.2, min_p=0.05) for i in range(n)]
    args = [*sampling_tensors(pp, cuda_device), pos, *penalty_tensors(pp, cuda_device)]
    st = state0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ext.sample_penalized(logits, *args[:4], torch.zeros_like(pos), *args[5:], st)  # warm-up at position 0: counts nothing
    torch.cuda.current_stream().wait_stream(side)
    assert torch.equal(st, state0)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ext.sample_penalized(logits, *args, st)
    assert torch.equal(st, state0)  # capture runs nothing
    eager_state = state0.clone()
    for _ in range(3):
        before = st.clone()
        graph.replay()
        want_tok = ext.sample_penalized(logits, *args, eager_state)
        assert torch.equal(out, want_tok)
        d = (st - before).cpu()
        w = torch.zeros_like(d)
        w[live, out.cpu()[live].long()] = 1
        assert torch.equal(d, w) and torch.equal(st, eager_state)


def test_row_independence(cuda_device):
    V = 151936
    g = torch.Generator().manual_seed(4)
    logits = (torch.randn(64, V, generator=g) * 2).to(torch.bfloat16).to(cuda_device)
    params = [SamplingParams((0.0, 0.7, 1.0, 1.3)[i % 4], (None, 40)[i % 2], (None, 0.9, 0.5)[i % 3], 1000 + i, (1.0, 1.3)[i % 2],
                             (0.0, 0.5, -0.5)[i % 3], (0.0, 0.3)[(i // 2) % 2], (0.0, 0.05, 0.3)[(i // 3) % 3]) for i in range(64)]
    positions = [i * 7 + 3 for i in range(64)]
    state0 = random_state(64, V, logits.cpu(), g).to(cuda_device)
    st = state0.clone()
    a = launch(logits, params, positions, st)
    for i in (0, 1, 5, 37, 63):
        one = state0[i : i + 1].clone()
        assert int(launch(logits[i : i + 1].contiguous(), [params[i]], [positions[i]], one)[0]) == int(a[i])
        assert torch.equal(one[0], st[i])
        j = (i * 13 + 17) % 64
        moved, mst = logits.clone(), state0.clone()
        moved[j], mst[j] = logits[i], state0[i]
        mp, mpos = list(params), list(positions)
        mp[j], mpos[j] = params[i], positions[i]
        assert int(launch(moved, mp, mpos, mst)[j]) == int(a[i]) and torch.equal(mst[j], st[i])


# ------------------------------------------------------------------- engine --
def _model(dev, seed=5):
    ns = synthetic_qwen3("tiny-d128", seed=seed, realistic=True, max_position_embeddings=8192, device=dev)
    return Qwen3ModelWeek3(ns, page_size=64)


def _admit(model, B, msl, lens):
    if B == 1:
        cache = model.create_kv_cache()
        for c in cache:
            c.append_slots(lens[0])
        return cache
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b, n in lens.items():
        cache = model.create_kv_cache()
        for c, t in zip(cache, tables):
            c.append_slots(n)
            t.add_request(c, b)
    return tables


def _fill_slabs(model, seed):
    gen = torch.Generator(device=model.page_pools[0]._key_pages.device).manual_seed(seed)
    for pool in model.page_pools:
        for slab in (pool._key_pages, pool._value_pages):
            slab.copy_(torch.randn(slab.shape, generator=gen, device=slab.device, dtype=torch.float32).to(slab.dtype))


@pytest.mark.parametrize("B,lens,logprobs", [(1, {0: 40}, None), (16, {0: 40, 3: 9, 9: 70, 15: 20}, None),
                                             (32, {0: 30, 2: 65, 5: 12, 11: 90}, None), (16, {0: 40, 3: 9, 9: 70, 15: 20}, 5)])
def test_decode_on_device_penalised_equals_steps_plus_eager(cuda_device, B, lens, logprobs):
    steps, msl = 24, 256
    slots = sorted(lens)
    params = [None] * B
    kinds = [SamplingParams(0.0, repetition_penalty=1.4, frequency_penalty=0.5),  # greedy + penalty
             SamplingParams(0.9, top_p=0.95, presence_penalty=1.0, frequency_penalty=0.3, min_p=0.02),  # sampled + penalty
             SamplingParams(1.1, top_k=30),  # plain sampled
             SamplingParams(0.0)]  # greedy
    for n, b in enumerate(slots):
        p = kinds[n % 4] if B > 1 else kinds[1]
        params[b] = SamplingParams(p.temperature, p.top_k, p.top_p, 77 + b, p.repetition_penalty, p.presence_penalty, p.frequency_penalty,
                                   p.min_p)
    g = torch.Generator().manual_seed(B)
    history = [(torch.randint(0, 512, (lens[b],), generator=g).tolist(), torch.randint(0, 512, (3,), generator=g).tolist()) if b in lens
               else None for b in range(B)]
    runs, counts, lps = {}, {}, {}
    for mode in ("graph", "eager"):
        model = _model(cuda_device)
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, lens)
        _fill_slabs(model, B)
        tokens = [(17 * b + 3) if b in lens else 0 for b in range(B)]
        offsets = [lens.get(b, 0) for b in range(B)]
        if mode == "graph":
            res = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params, logprobs=logprobs, history=history)
            if logprobs is None:
                runs[mode] = res.cpu()
                assert engine.kernels_per_penalized_step == engine.kernels_per_step - 1  # the same single launch as tl_sample
                assert engine._graph_sample is None
            else:
                runs[mode], lp = res[0].cpu(), res[1][0].cpu()
                lps[mode] = lp
            counts[mode] = engine.token_counts.cpu()
        else:
            temperature, top_k, top_p, seed = sampling_tensors(params, cuda_device)
            pen = penalty_tensors(params, cuda_device)
            state = torch.stack([token_state_row(*h, model.vocab_size) if h is not None else torch.zeros(model.vocab_size, dtype=torch.int32)
                                 for h in history]).to(cuda_device)
            out, lp_rows = [], []
            for _ in range(steps):
                logits, _ = engine.step(tokens, offsets, caches)
                logits = logits.view(B, -1)
                pos = torch.tensor([o + 1 if b in lens else 0 for b, o in enumerate(offsets)], dtype=torch.int32, device=cuda_device)
                nxt = ext.sample_penalized(logits, temperature, top_k, top_p, seed, pos, *pen, state)
                if logprobs is not None:
                    lp_rows.append(ext.logprobs(logits, nxt, max_n=logprobs)[1].cpu())
                nxt = nxt.cpu()
                out.append([int(nxt[b]) if b in lens else -1 for b in range(B)])
                tokens = [int(nxt[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
            runs[mode] = torch.tensor(out, dtype=torch.int32)
            counts[mode] = state.cpu()
            if logprobs is not None:
                lps[mode] = torch.stack(lp_rows)
            if B > 16:
                assert engine.variant_replays[16] == steps
    assert torch.equal(runs["graph"], runs["eager"])
    live = torch.tensor([b in lens for b in range(B)])
    assert torch.equal(counts["graph"][live], counts["eager"][live])
    if logprobs is not None:
        assert torch.equal(lps["graph"][:, live], lps["eager"][:, live])


def test_plain_sampled_run_allocates_no_counts(cuda_device):
    model = _model(cuda_device)
    B, msl, lens = 16, 256, {0: 40, 3: 9}
    engine = DecodeEngine(model, B, msl, cuda_device)
    engine.reserve_pools()
    caches = _admit(model, B, msl, lens)
    tokens = [5 if b in lens else 0 for b in range(B)]
    offsets = [lens.get(b, 0) for b in range(B)]
    engine.decode_on_device(tokens, offsets, caches, 4, sampling=SamplingParams(0.8, seed=3))
    assert engine.token_counts is None and engine._graph_pen is None
    offsets = [o + 4 if b in lens else 0 for b, o in enumerate(offsets)]
    engine.decode_on_device(tokens, offsets, caches, 4, sampling=SamplingParams(0.8, seed=3, presence_penalty=0.5))
    assert engine.kernels_per_penalized_step == engine.kernels_per_sampled_step == engine.kernels_per_step - 1


def test_generate_penalised_equals_prefill_plus_decode_on_device(cuda_device):
    model = _model(cuda_device, seed=7)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11, 5, 5]
    p = SamplingParams(0.9, top_k=40, top_p=0.95, seed=12345, repetition_penalty=1.3, presence_penalty=0.7, frequency_penalty=0.4, min_p=0.05)
    n = 20
    greedy_generate_ids(model, prompt, 2, device=cuda_device, sampling=p)
    got = greedy_generate_ids(model, prompt, n, device=cuda_device, sampling=p)
    cache = model.create_kv_cache()
    try:
        logits = model(torch.tensor([prompt], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        state = token_state_row(prompt, [], model.vocab_size, device=cuda_device)[None]
        first = int(sample_tokens(logits[:, -1, :], [p], [len(prompt)], state)[0])
        engine = model.decode_engine(1, model._graph_limit(cache))
        log = engine.decode_on_device([first], [len(prompt)], cache, n - 1, sampling=p, history=[(prompt, [first])])
        want = [first] + log[:, 0].tolist()
    finally:
        for c in cache:
            c.release()
    assert got == want
    assert got != greedy_generate_ids(model, prompt, n, device=cuda_device, sampling=SamplingParams(0.9, 40, 0.95, 12345))


def test_batcher_penalised_tokens_do_not_depend_on_queue_order(cuda_device):
    ns = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, device=cuda_device)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, 500, (int(n),), generator=g).tolist() for n in torch.randint(3, 40, (20,), generator=g)]
    params = [SamplingParams((0.0, 0.8)[i % 2], (None, 50)[i % 3 == 0], None, i, repetition_penalty=1.3 if i % 4 else 1.0,
                             presence_penalty=(2.0, 0.8)[i % 2], frequency_penalty=0.3, min_p=(0.0, 0.05)[i % 2]) for i in range(len(prompts))]
    params[5] = SamplingParams(0.8, seed=5)  # plain sampled and plain greedy requests in the same batches
    params[10] = SamplingParams(0.0)
    budgets = [8 + (i % 7) for i in range(len(prompts))]

    def run(order):
        model = Qwen3ModelWeek3(ns, page_size=64)
        out, lp = batch_generate(model, None, [prompts[i] for i in order], max_seq_len=128, batch_size=16, prefill_step=32, verbose=False,
                                 device=cuda_device, max_new_tokens=[budgets[i] for i in order], sampling=[params[i] for i in order],
                                 logprobs=3)
        return {order[j]: text for j, text in out}, {order[j]: v for j, v in lp.items()}

    fwd, lp_f = run(list(range(len(prompts))))
    bwd, lp_b = run(list(reversed(range(len(prompts)))))
    assert fwd == bwd
    assert lp_f == lp_b
    for i, entries in lp_f.items():
        assert [e.token for e in entries] == [int(t) for t in fwd[i].split()][: len(entries)]
    # a token chosen greedily on the penalised row reports its raw rank: somewhere that rank is not 1
    assert any(e.rank > 1 for i in lp_f if params[i].temperature == 0 and params[i].penalized for e in lp_f[i])
