"""``tl_logprobs`` on the H100: every output against the float64 reference (``tests/logprobs_ref.py``) within the bound
derived from the kernel's rounding points, exact probes, determinism, and the log-probability paths of the engine,
the batcher and prompt scoring.

Which test catches which plausible defect:
* ties broken to the higher id: the flat rows and the ties straddling the N-th place (ids compared exactly);
* the rank counted with ``>=``: every rank is compared exactly, on rows with ties at the target;
* the last slice's tail dropped: the boundary rows put the maximum, the target and list members on the last entries;
* ``S`` accumulated in fp32 in thread order: the absorption rows (maximum 0 at id 0, every other entry -17 or -17.5).
  Their masses, about 4e-8 each, fall below half an ulp of the running sum of the thread that holds the maximum, so an
  fp32 sum in the kernel's thread order drops them; at V = 4097 and 151,936 its ``lse`` is 3-5x the bound, while the
  fixed-point sum stays within it (``test_logprobs_host.py`` replays both sums on the host).  Random rows do not separate
  the two: an fp32 sum stays inside the bound there, and it is as deterministic as the fixed-point one.
"""

import importlib.util
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle.model import ReferenceCpuModel, greedy_decode
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, score_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.sampler import sampling_tensors
from tiny_llm_b200.synthetic import synthetic_qwen3, to_device


def _load_logprobs_ref():
    name = "tiny_llm_b200_logprobs_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("logprobs_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


ref = _load_logprobs_ref()
pytestmark = pytest.mark.gpu
MAX_N = 20


def slice_bounds(V):
    """The first id of every CTA slice after the first (sample_plan's rule)."""
    c = min(-(-V // 4096), 8)
    s = -(-(-(-V // c)) // 8) * 8
    return [k * s for k in range(1, c) if k * s < V]


def rows_for(V, dtype, g):
    rows, targets = [], []

    def add(x, t):
        rows.append(x)
        targets.append(t)

    for scale in (1.0, 3.0, 8.0):
        add(torch.randn(V, generator=g) * scale, int(torch.randint(0, V, (1,), generator=g)))
    peaked = torch.randn(V, generator=g)
    peaked[V // 3] = peaked.max() + 50
    add(peaked, V // 3)
    add(peaked.clone(), 0)
    add(torch.zeros(V), V - 1)  # flat: lp = -log V, ids 0..N-1
    tie = torch.randn(V, generator=g)
    top = tie.max()
    for j, i in enumerate((V - 1, 5, V // 2, 2, V // 4, 7, V - 3, 1, V // 5)):
        tie[i] = top + (1.0 if j < 3 else 0.5)  # 3 above, then 6 tied entries across the 5th..20th places
    add(tie, 7)
    tie2 = tie.clone()
    tie2[[11, 12]] = top + 0.5  # a different tie count
    add(tie2, V // 5)
    if dtype == torch.float32:
        add((torch.rand(V, generator=g) * 2 - 1) * 1e4, 3)
    special = torch.randn(V, generator=g)
    special[::5] = -math.inf
    special[1::7] = math.nan
    add(special, 5)  # a -inf target
    add(special.clone(), 1)  # a NaN target
    few = torch.full((V,), -math.inf)
    few[[2, V - 1]] = 1.0
    few[V // 2] = math.nan
    add(few, 2)  # fewer finite entries than the list
    for level in (-17.0, -17.5):  # absorption rows: see the module docstring
        absorb = torch.full((V,), level)
        absorb[0] = 0.0
        add(absorb, 1)
    pinf = torch.randn(V, generator=g)
    pinf[[4, V - 2]] = math.inf
    add(pinf, 4)
    add(torch.full((V,), -math.inf), 0)
    add(torch.full((V,), math.nan), 0)
    for b in slice_bounds(V) + [V]:  # targets and list members on every slice boundary, the last entry included
        x = torch.randn(V, generator=g)
        x[b - 1] = x.max() + 2.0
        if b < V:
            x[b] = x[b - 1]
        add(x, b - 1)
        add(x.clone(), b if b < V else -1)
    return torch.stack(rows).to(dtype), targets


def check(logits, targets, top_n):
    """Launch ``tl_logprobs`` and hold every output to the reference and its bound."""
    dev = logits.device
    t = torch.tensor(targets, dtype=torch.int32, device=dev)
    tn = torch.tensor(top_n, dtype=torch.int32, device=dev)
    lse, lp, rank, ids, top = (a.cpu() for a in ext.logprobs(logits, t, tn, MAX_N))
    x64 = logits.float().cpu().double().numpy()
    worst = 0.0
    for r in range(x64.shape[0]):
        x = x64[r]
        n = max(0, min(MAX_N, top_n[r]))
        lse_r, lp_r, rank_r, ids_r, lps_r = ref.row(x, targets[r], n)
        assert int(rank[r]) == rank_r, r
        assert ids[r, :n].tolist() == ids_r.tolist() and (ids[r, n:] == -1).all(), r
        assert (top[r, n:] == -math.inf).all()
        if 0 <= targets[r] < x.shape[0] and targets[r] in ids[r].tolist():  # the same expression, the same bits
            j = ids[r].tolist().index(targets[r])
            assert top[r, j].view(torch.int32) == lp[r].view(torch.int32), r
        ok = ~np.isnan(x)
        if not ok.any() or not np.isfinite(x[ok].max()):
            assert (math.isnan(lse_r) and math.isnan(float(lse[r]))) or float(lse[r]) == lse_r, r
            assert math.isnan(float(lp[r])), r
            listed = ids_r >= 0
            assert torch.isnan(top[r, :n][torch.from_numpy(listed)]).all(), r
            assert (top[r, :n][torch.from_numpy(~listed)] == -math.inf).all(), r
            continue
        lp_b, lse_b = ref.bound(x)
        assert abs(float(lse[r]) - lse_r) <= lse_b, (r, float(lse[r]), lse_r, lse_b)
        worst = max(worst, abs(float(lse[r]) - lse_r) / lse_b)
        if math.isnan(lp_r):
            assert math.isnan(float(lp[r])), r
        elif lp_r == -math.inf:
            assert float(lp[r]) == -math.inf, r
        else:
            t_r = targets[r]
            assert abs(float(lp[r]) - lp_r) <= lp_b[t_r], (r, float(lp[r]), lp_r, lp_b[t_r])
        for j in range(n):
            i, want = int(ids_r[j]), float(lps_r[j])
            if i < 0:
                continue
            if want == -math.inf:
                assert float(top[r, j]) == -math.inf
            else:
                assert abs(float(top[r, j]) - want) <= lp_b[i], (r, j, float(top[r, j]), want, lp_b[i])
    return worst


@pytest.mark.parametrize("V,dtype", [(1000, torch.float32), (4097, torch.bfloat16), (151936, torch.bfloat16), (32000, torch.float16)])
def test_every_output_against_the_float64_reference(cuda_device, V, dtype):
    g = torch.Generator().manual_seed(V)
    logits, targets = rows_for(V, dtype, g)
    R = logits.shape[0]
    top_n = [(MAX_N, 5, 1, 0, 20, 3)[r % 6] for r in range(R)]
    worst = check(logits.to(cuda_device), targets, top_n)
    print(f"V {V} {dtype}: {R} rows, largest lse error {worst:.3f} of its bound")
    # without targets and top_n arrays: every row lists max_n entries, targets -1
    lse, lp, rank, ids, top = ext.logprobs(logits[:4].contiguous().to(cuda_device), max_n=3)
    assert torch.isnan(lp).all() and (rank == 0).all() and (ids >= 0).all()
    lse0 = ext.logprobs(logits[:4].contiguous().to(cuda_device))[0]
    assert torch.equal(lse0, lse)


@pytest.mark.parametrize("V", [1000, 151936])
def test_exact_probes_power_of_two_maxima(cuda_device, V):
    rows = []
    J = min(11, int(math.log2(V)) + 1)
    for j in range(J):
        x = torch.full((V,), -math.inf)
        x[torch.randperm(V, generator=torch.Generator().manual_seed(j))[: 2**j]] = 2.5
        rows.append(x)
    logits = torch.stack(rows).to(cuda_device)
    tgt = [int(torch.nonzero(rows[j] == 2.5)[0]) for j in range(J)]
    lse, lp, rank, ids, top = (a.cpu() for a in ext.logprobs(logits, torch.tensor(tgt, dtype=torch.int32, device=cuda_device), None, 1))
    for j in range(J):
        want = -j * math.log(2)
        ulp = float(np.spacing(np.float32(abs(want)))) if j else 0.0
        assert abs(float(lp[j]) - want) <= ulp, (j, float(lp[j]), want)
        assert int(rank[j]) == 1 and int(ids[j, 0]) == min(int(i) for i in torch.nonzero(rows[j] == 2.5))


def test_log_rows_outside_the_capacity_write_nothing(cuda_device):
    V, R, cap, N = 4097, 3, 4, 5
    logits = torch.randn(R, V, device=cuda_device)
    t = torch.arange(R, dtype=torch.int32, device=cuda_device)
    full = ext.logprobs(logits, t, None, N)
    # the logs are the first `cap` blocks of larger buffers: a launch past the end must leave the sentinel block alone
    big = (torch.full((cap + 1, R), 7.0, device=cuda_device), torch.full((cap + 1, R), 7.0, device=cuda_device),
           torch.full((cap + 1, R), 7, dtype=torch.int32, device=cuda_device),
           torch.full((cap + 1, R, N), 7, dtype=torch.int32, device=cuda_device), torch.full((cap + 1, R, N), 7.0, device=cuda_device))
    log = tuple(b[:cap] for b in big)
    for at in (cap, cap + 5, -1):
        ext.logprobs(logits, t, None, N, out=log, out_index=torch.tensor([at], dtype=torch.int32, device=cuda_device))
    torch.cuda.synchronize()
    for b in big:
        assert (b == 7).all()
    ext.logprobs(logits, t, None, N, out=log, out_index=torch.tensor([cap - 1], dtype=torch.int32, device=cuda_device))
    for b, f in zip(big, full):
        assert torch.equal(b[cap - 1].view(torch.int32), f.view(torch.int32)) and (b[cap] == 7).all() and (b[: cap - 1] == 7).all()


def test_determinism_row_independence_and_graph_capture(cuda_device):
    V = 151936
    g = torch.Generator().manual_seed(11)
    logits = (torch.randn(64, V, generator=g) * 3).to(torch.bfloat16).to(cuda_device)
    t = torch.randint(0, V, (64,), generator=g, dtype=torch.int32).to(cuda_device)
    tn = torch.tensor([(0, 5, 20)[i % 3] for i in range(64)], dtype=torch.int32, device=cuda_device)
    full = ext.logprobs(logits, t, tn, MAX_N)
    again = ext.logprobs(logits, t, tn, MAX_N)
    for a, b in zip(full, again):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    for i in (0, 1, 31, 63):
        alone = ext.logprobs(logits[i : i + 1].contiguous(), t[i : i + 1].contiguous(), tn[i : i + 1].contiguous(), MAX_N)
        for a, b in zip(alone, full):
            assert torch.equal(a[0].view(torch.int32), b[i].view(torch.int32)), i
        for j in (0, 17, 63):
            moved, mt, mn = logits.clone(), t.clone(), tn.clone()
            moved[j], mt[j], mn[j] = logits[i], t[i], tn[i]
            out = ext.logprobs(moved, mt, mn, MAX_N)
            for a, b in zip(out, full):
                assert torch.equal(a[j].view(torch.int32), b[i].view(torch.int32)), (i, j)
    # graph capture: the same bits, logging at the device-side index
    cap = 3
    log = (torch.zeros(cap, 64, device=cuda_device), torch.zeros(cap, 64, device=cuda_device),
           torch.zeros(cap, 64, dtype=torch.int32, device=cuda_device), torch.zeros(cap, 64, MAX_N, dtype=torch.int32, device=cuda_device),
           torch.zeros(cap, 64, MAX_N, device=cuda_device))
    index = torch.full((1,), 2, dtype=torch.int32, device=cuda_device)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ext.logprobs(logits, t, tn, MAX_N, out=log, out_index=index)
        s.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            ext.logprobs(logits, t, tn, MAX_N, out=log, out_index=index)
    torch.cuda.current_stream().wait_stream(s)
    for a in log:
        a.zero_()
    index.fill_(1)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(log, full):
        assert torch.equal(a[1].view(torch.int32), b.view(torch.int32))
        assert not a[2].any() and not a[0].any()


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


@pytest.mark.parametrize("sampled", [False, True])
@pytest.mark.parametrize("B,lens", [(1, {0: 40}), (16, {0: 40, 3: 9, 9: 70, 15: 20}), (32, {0: 30, 2: 65, 5: 12, 11: 90})])
def test_decode_on_device_logprobs_equal_steps_plus_eager_logprobs(cuda_device, B, lens, sampled):
    steps, msl, N = 12, 256, 5
    slots = sorted(lens)
    params = None
    if sampled:
        params = [None] * B
        for n, b in enumerate(slots):
            params[b] = SamplingParams(0.0) if n % 2 else SamplingParams(0.9, top_k=30 if n % 4 == 2 else None, top_p=0.9, seed=31 + b)
    runs = {}
    for mode in ("plain", "graph", "eager"):
        model = _model(cuda_device)
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, lens)
        _fill_slabs(model, B)
        tokens = [(17 * b + 3) if b in lens else 0 for b in range(B)]
        offsets = [lens.get(b, 0) for b in range(B)]
        if mode == "plain":
            runs[mode] = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params).cpu()
            kernels, upload = engine.kernels_per_step, engine.upload_bytes_per_step()
        elif mode == "graph":
            log, (lp, rank, ids, top) = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params, logprobs=N)
            runs[mode] = (log.cpu(), lp.cpu(), rank.cpu(), ids.cpu(), top.cpu())
            assert engine.kernels_per_step == kernels and engine.upload_bytes_per_step() == upload
            assert engine.kernels_per_logprobs_step == kernels + (0 if sampled else 1)  # tl_sample is one launch, tl_argmax two
        else:
            out = [[], [], [], [], []]
            samp = None if params is None else sampling_tensors(params, cuda_device)
            for _ in range(steps):
                logits, nxt = engine.step(tokens, offsets, caches)
                logits = logits.view(B, -1)
                if samp is not None:
                    pos = torch.tensor([o + 1 if b in lens else 0 for b, o in enumerate(offsets)], dtype=torch.int32, device=cuda_device)
                    nxt = ext.sample(logits, *samp, pos)
                _, lp, rank, ids, top = ext.logprobs(logits, nxt.to(torch.int32).contiguous(), None, N)
                host = nxt.cpu()
                for k, v in enumerate((host, lp, rank, ids, top)):
                    out[k].append(v.cpu())
                tokens = [int(host[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
            runs[mode] = tuple(torch.stack(v) for v in out)
    graph, eager = runs["graph"], runs["eager"]
    occupied = torch.tensor(slots)
    assert torch.equal(graph[0], runs["plain"])  # logging changes no token
    assert torch.equal(graph[0][:, occupied], eager[0][:, occupied].to(torch.int32))
    for a, b in zip(graph[1:], eager[1:]):
        assert torch.equal(a[:, occupied].view(torch.int32), b[:, occupied].view(torch.int32))
    assert (graph[2][:, occupied] >= 1).all()


def test_logprobs_graph_after_a_run_that_filled_the_token_log(cuda_device):
    """A run of ``log_capacity`` steps leaves the step counter at the end of the logs; capturing the logprobs graph
    afterwards (first use, then again for a new N) must log from row 0 and equal eager steps bit for bit."""
    cap, msl, first = 8, 256, {0: 40}
    runs = {}
    for mode in ("graph", "eager"):
        model = _model(cuda_device)
        engine = DecodeEngine(model, 1, msl, cuda_device, log_capacity=cap)
        engine.reserve_pools()
        caches = _admit(model, 1, msl, first)
        _fill_slabs(model, 1)
        log = engine.decode_on_device([3], [40], caches, cap)  # the counter ends at cap
        token, offset = int(log[-1, 0]), 40 + cap
        out = []
        for n in (3, 5):
            if mode == "graph":
                log, (lp, rank, ids, top) = engine.decode_on_device([token], [offset], caches, 4, logprobs=n)
                out.append((log.cpu(), lp.cpu(), rank.cpu(), ids.cpu(), top.cpu()))
                token = int(log[-1, 0])
                log = engine.decode_on_device([token], [offset + 4], caches, cap)  # fill the log again before the re-capture
            else:
                rows = []
                for _ in range(4):
                    logits, nxt = engine.step([token], [offset], caches)
                    _, lp, rank, ids, top = ext.logprobs(logits.view(1, -1), nxt.to(torch.int32).contiguous(), None, n)
                    rows.append(tuple(v.cpu() for v in (nxt.to(torch.int32), lp, rank, ids, top)))
                    token, offset = int(nxt[0]), offset + 1
                out.append(tuple(torch.stack(v) for v in zip(*rows)))
                log = engine.decode_on_device([token], [offset], caches, cap)
            token, offset = int(log[-1, 0]), offset + 4 + cap if mode == "graph" else offset + cap
        runs[mode] = out
    for g, e in zip(runs["graph"], runs["eager"]):
        for a, b in zip(g, e):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_batcher_entries_do_not_depend_on_queue_order(cuda_device):
    ns = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, device=cuda_device)
    g = torch.Generator().manual_seed(1)
    prompts = [torch.randint(1, 500, (int(n),), generator=g).tolist() for n in torch.randint(3, 40, (20,), generator=g)]
    budgets = [6 + (i % 5) for i in range(len(prompts))]
    for sampling in (None, [SamplingParams(0.8, top_k=(None, 50)[i % 2], seed=i) for i in range(len(prompts))]):

        def run(order):
            model = Qwen3ModelWeek3(ns, page_size=64)
            b = ContinuousBatcher(model, None, [prompts[i] for i in order], max_seq_len=128, batch_size=16, prefill_step=32, verbose=False,
                                  device=cuda_device, max_new_tokens=[budgets[i] for i in order],
                                  sampling=None if sampling is None else [sampling[i] for i in order], logprobs=4)
            out = dict(b.run())
            return {order[j]: (out[j], b.logprobs[j]) for j in range(len(order))}

        forward = run(list(range(len(prompts))))
        backward = run(list(reversed(range(len(prompts)))))
        assert forward == backward
        for text, entries in forward.values():
            assert [e.token for e in entries] == [int(t) for t in text.split()]


# ------------------------------------------------------------------- scoring --
def _chunk_logits(model, ids, chunk, dev):
    cache = model.create_kv_cache()
    try:
        out = []
        for start in range(0, len(ids), chunk):
            piece = torch.tensor([ids[start : start + chunk]], dtype=torch.int32, device=dev)
            out.append(model(piece, start, cache, logits_to_keep=None)[0].float().cpu())
        return torch.cat(out)
    finally:
        for c in cache:
            c.release()


@pytest.mark.parametrize("config,chunk", [("tiny-d128", 7), ("qwen3-0.6b", 64)])
def test_score_ids_against_float64_log_softmax(cuda_device, config, chunk):
    ns = synthetic_qwen3(config, seed=0, realistic=config.startswith("tiny"), max_position_embeddings=1024, device=cuda_device)
    model = Qwen3ModelWeek3(ns, page_size=64)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(1, min(1000, model.vocab_size), (150,), generator=g).tolist()
    result = score_ids(model, ids, chunk=chunk, top_n=3)
    logits = _chunk_logits(model, ids, chunk, cuda_device).double().numpy()  # the same chunking computes the same logits
    assert [e.token for e in result.entries] == ids[1:]
    for p, e in enumerate(result.entries):
        x = logits[p]
        want = float(torch.log_softmax(torch.from_numpy(x), -1)[ids[p + 1]])
        assert abs(e.logprob - want) <= ref.bound(x)[0][ids[p + 1]], p
        assert e.rank == 1 + int((x > x[ids[p + 1]]).sum())
    assert result.nll == pytest.approx(-sum(e.logprob for e in result.entries))
    assert [i for i, _ in result.next_top] == ref.row(logits[-1], -1, 3)[3].tolist()


def test_score_ids_tracks_the_reference_cpu_model(cuda_device):
    kwargs = dict(seed=0, realistic=True, max_position_embeddings=512)
    cpu = synthetic_qwen3("tiny-d128", **kwargs)
    gpu = to_device(synthetic_qwen3("tiny-d128", **kwargs), cuda_device)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11, 8, 1, 77, 402, 65, 9, 33, 210]
    tokens, lp = greedy_decode(ReferenceCpuModel(cpu), prompt, 10, return_logprobs=True)
    result = score_ids(Qwen3ModelWeek3(gpu, page_size=64), list(prompt) + list(tokens), chunk=8)
    for i, (tok, lp_ref) in enumerate(zip(tokens, lp)):
        e = result.entries[len(prompt) - 1 + i]
        assert e.token == tok
        assert abs(e.logprob - float(lp_ref[tok])) <= 0.25, i  # DESIGN section 2's whole-model tolerance
