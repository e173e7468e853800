"""``tl_sample`` on the H100: greedy rows against ``tl_argmax``, every draw against the float64 reference
(``oracle/sampling.py``), determinism and row independence, and the sampled paths of the engine, ``generate`` and the
batcher."""

import math

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as ref
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, batch_generate, greedy_generate_ids
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.sampler import sample_tokens, sampling_tensors
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu
VOCABS = [7, 1000, 4097, 151936]


def launch(logits, params, positions):
    return sample_tokens(logits, params, positions).cpu()


def special_rows(V, g):
    rows = [torch.randn(V, generator=g) * 3]
    tie = torch.randn(V, generator=g)
    tie[[V // 3, V - 1, 0]] = 9.0  # first maximum wins
    rows.append(tie)
    rows.append(torch.full((V,), -math.inf))
    pinf = torch.randn(V, generator=g)
    pinf[V // 2] = math.inf
    pinf[V - 1] = math.inf
    rows.append(pinf)
    ninf = torch.randn(V, generator=g)
    ninf[::2] = -math.inf
    rows.append(ninf)
    nan = torch.randn(V, generator=g)
    nan[::3] = math.nan
    rows.append(nan)
    rows.append(torch.full((V,), math.nan))
    return torch.stack(rows)


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_greedy_rows_equal_argmax(cuda_device, V, dtype):
    g = torch.Generator().manual_seed(V)
    logits = torch.cat([special_rows(V, g), torch.randn(16, V, generator=g) * 4]).to(dtype).to(cuda_device)
    n = logits.shape[0]
    params = [SamplingParams(0.0, top_k=(i % 3) * 5, top_p=0.5 * (i % 2), seed=i) for i in range(n)]
    got = launch(logits, params, list(range(n)))
    assert torch.equal(got, ext.argmax(logits).cpu())
    # a sampled row whose maximum is not finite (or no entry is a number) also returns argmax's token
    idx = [2, 3, 6]
    got = launch(logits[idx].contiguous(), [SamplingParams(0.8, seed=1)] * 3, [5, 5, 5])
    assert torch.equal(got, ext.argmax(logits[idx].contiguous()).cpu())


def _tol_accept(x, T, k, p, seed, pos, got):
    """A draw that differs from the float64 reference passes only when the fp32 operation chain of the kernel could
    have produced it: (a) the perturbed scores x_i / T + g_i are rounded at x / T, at each logf and at the sum, so each is
    within d_i = 2^-21 (1 + |g_i| + |x_i / T|) of the float64 value; (b) the mass above an entry is a quotient of sums
    of e_j = expf(x_j - m) (error <= 2^-22 + |x_j - m| 2^-24 relative) in 2^-40 fixed point, so M_i is within
    eps = 2 (2^-22 + R 2^-24) + 2 V 2^-40 / S of its float64 value (R: the row's finite range).  The kernel's token must
    be in the loose keep set (top_p + eps) and its score within d_got + d_best of the best score of the strict keep set
    (top_p - eps)."""
    ok = ~np.isnan(x)
    V = len(x)
    base = ref.keep_set(x, k, None)
    strict, loose = base.copy(), base.copy()
    if 0 < p < 1:
        M, S = ref.mass_above(x)
        R = float(x[ok].max() - x[ok & np.isfinite(x)].min())
        eps = 2 * (2.0**-22 + R * 2.0**-24) + 2 * V * 2.0**-40 / S
        strict &= M < p - eps
        loose &= M < p + eps
    g = ref.gumbel(V, seed, pos)
    score = x / T + g
    d = 2.0**-21 * (1 + np.abs(g) + np.abs(x / T))
    if not loose[got]:
        return False
    if not strict.any():
        return True
    best = int(np.argmax(np.where(strict, score, -np.inf)))
    return score[got] + d[got] + d[best] >= score[best]


TEMPS = [0.25, 0.7, 1.0, 1.5]
TOPPS = [None, 0.05, 0.5, 0.9, 0.999]


@pytest.mark.parametrize("V,dtype,per", [(1000, torch.float32, 6), (4097, torch.bfloat16, 8), (151936, torch.bfloat16, 1)])
def test_every_draw_equals_the_float64_reference(cuda_device, V, dtype, per):
    g = torch.Generator().manual_seed(V + per)
    params, positions, rows = [], [], []
    for T in TEMPS:
        for k in (None, 1, 2, 50, V - 1):
            for p in TOPPS:
                for r in range(per):
                    i = len(rows)
                    rows.append(torch.randn(V, generator=g) * (1.0, 3.0, 8.0)[i % 3])
                    params.append(SamplingParams(T, top_k=k, top_p=p, seed=(i * 2654435761) % (1 << 64)))
                    positions.append(17 + 131 * i)
    logits = torch.stack(rows).to(dtype).to(cuda_device)
    got = launch(logits, params, positions).numpy()
    x64 = logits.float().cpu().double().numpy()
    p32 = sampling_tensors(params, "cpu")[2].double().numpy()  # the fp32 top_p the kernel compares against
    exact = ambiguous = 0
    for i, sp in enumerate(params):
        p = float(p32[i])
        want = ref.sample_row(x64[i], sp.temperature, sp.top_k, p, sp.seed, positions[i])
        if got[i] == want:
            exact += 1
            continue
        assert _tol_accept(x64[i], sp.temperature, sp.top_k, p, sp.seed, positions[i], int(got[i])), (i, sp, int(got[i]), want)
        ambiguous += 1
    print(f"V {V}: {exact} exact, {ambiguous} within the fp32 bound of {len(params)} draws")
    assert ambiguous <= max(1, len(params) // 100)


def test_determinism_and_row_independence(cuda_device):
    V = 151936
    g = torch.Generator().manual_seed(3)
    logits = (torch.randn(64, V, generator=g) * 2).to(torch.bfloat16).to(cuda_device)
    params = [SamplingParams((0.0, 0.7, 1.0, 1.3)[i % 4], top_k=(None, 40)[i % 2], top_p=(None, 0.9, 0.5)[i % 3], seed=1000 + i)
              for i in range(64)]
    positions = [i * 7 + 3 for i in range(64)]
    a, b = launch(logits, params, positions), launch(logits, params, positions)
    assert torch.equal(a, b)
    for i in (0, 1, 5, 37, 63):
        alone = launch(logits[i : i + 1].contiguous(), [params[i]], [positions[i]])
        assert int(alone[0]) == int(a[i])
        for j in (0, 17, 63):  # the same row at another index of a 64-row launch
            moved = logits.clone()
            moved[j] = logits[i]
            mp, mpos = list(params), list(positions)
            mp[j], mpos[j] = params[i], positions[i]
            assert int(launch(moved, mp, mpos)[j]) == int(a[i])


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


@pytest.mark.parametrize("B,lens", [(1, {0: 40}), (16, {0: 40, 3: 9, 9: 70, 15: 20}), (32, {0: 30, 2: 65, 5: 12, 11: 90})])
def test_decode_on_device_sampled_equals_steps_plus_eager_sample(cuda_device, B, lens):
    steps, msl = 24, 256
    slots = sorted(lens)
    params = [None] * B
    for n, b in enumerate(slots):
        # odd occupied slots greedy, the others sampled
        params[b] = SamplingParams(0.0) if n % 2 else SamplingParams(0.8 if n % 4 == 0 else 1.2, top_k=30 if n % 4 == 2 else None,
                                                                     top_p=0.9, seed=77 + b)
    runs = {}
    for mode in ("graph", "eager", "greedy"):
        model = _model(cuda_device)
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, lens)
        _fill_slabs(model, B)
        tokens = [(17 * b + 3) if b in lens else 0 for b in range(B)]
        offsets = [lens.get(b, 0) for b in range(B)]
        if mode == "graph":
            log = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params).cpu()
            greedy_kernels = engine.kernels_per_step
            assert engine.kernels_per_sampled_step == greedy_kernels - 1  # tl_sample is one launch, tl_argmax two
            runs[mode] = log
        elif mode == "greedy":
            runs[mode] = engine.decode_on_device(tokens, offsets, caches, steps).cpu()
            assert engine.kernels_per_step == greedy_kernels and engine._graph_sample is None
        else:
            temperature, top_k, top_p, seed = sampling_tensors(params, cuda_device)
            out = []
            for _ in range(steps):
                logits, _ = engine.step(tokens, offsets, caches)
                pos = torch.tensor([o + 1 if b in lens else 0 for b, o in enumerate(offsets)], dtype=torch.int32, device=cuda_device)
                nxt = ext.sample(logits.view(B, -1), temperature, top_k, top_p, seed, pos).cpu()
                out.append([int(nxt[b]) if b in lens else -1 for b in range(B)])
                tokens = [int(nxt[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
            runs[mode] = torch.tensor(out, dtype=torch.int32)
            if B > 16:
                assert engine.variant_replays[16] == steps  # the eager loop ran the 16-row variant, the graph the full width
    assert torch.equal(runs["graph"], runs["eager"])
    for b in slots:
        if params[b].temperature == 0:
            assert torch.equal(runs["graph"][:, b], runs["greedy"][:, b])
    sampled = [b for b in slots if params[b].temperature > 0]
    assert any(not torch.equal(runs["graph"][:, b], runs["greedy"][:, b]) for b in sampled)


def test_generate_sampled_equals_prefill_plus_decode_on_device(cuda_device):
    model = _model(cuda_device, seed=7)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11]
    p = SamplingParams(0.9, top_k=40, top_p=0.95, seed=12345)
    n = 20
    greedy_generate_ids(model, prompt, 2, device=cuda_device, sampling=p)  # both runs below then find the graph engines built
    got = greedy_generate_ids(model, prompt, n, device=cuda_device, sampling=p)
    cache = model.create_kv_cache()
    try:
        logits = model(torch.tensor([prompt], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        first = int(sample_tokens(logits[:, -1, :], [p], [len(prompt)])[0])
        engine = model.decode_engine(1, model._graph_limit(cache))
        log = engine.decode_on_device([first], [len(prompt)], cache, n - 1, sampling=p)
        want = [first] + log[:, 0].tolist()
    finally:
        for c in cache:
            c.release()
    assert got == want
    assert got != greedy_generate_ids(model, prompt, n, device=cuda_device)


def test_batcher_sampled_tokens_do_not_depend_on_queue_order(cuda_device):
    ns = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, device=cuda_device)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, 500, (int(n),), generator=g).tolist() for n in torch.randint(3, 40, (20,), generator=g)]
    params = [SamplingParams(0.0) if i % 5 == 0 else SamplingParams(0.8, top_k=(None, 50)[i % 2], top_p=(None, 0.9)[i % 3 == 0], seed=i)
              for i in range(len(prompts))]
    budgets = [8 + (i % 7) for i in range(len(prompts))]

    def run(order):
        model = Qwen3ModelWeek3(ns, page_size=64)
        out = batch_generate(model, None, [prompts[i] for i in order], max_seq_len=128, batch_size=16, prefill_step=32, verbose=False,
                             device=cuda_device, max_new_tokens=[budgets[i] for i in order], sampling=[params[i] for i in order])
        return {order[j]: text for j, text in out}

    forward = run(list(range(len(prompts))))
    backward = run(list(reversed(range(len(prompts)))))
    assert forward == backward
