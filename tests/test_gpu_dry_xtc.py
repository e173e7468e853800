"""DRY and XTC on the H100 (DESIGN.md section 24): ``tl_dry_penalty`` bit for bit against the restatement
(``dry_xtc_ref``), its history append and its no-ops; the XTC draws of ``tl_sample_penalized`` and
``tl_sample_constrained`` against the float64 oracle; and both samplers through ``greedy_generate_ids``, the batcher
and ``decode_on_device``."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


dref = _load("tiny_llm_b200_dry_xtc_ref", "dry_xtc_ref.py")
from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, batch_generate, greedy_generate_ids
from tiny_llm_b200.dry import DryRows
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.logit_controls import control_rows
from tiny_llm_b200.sampler import penalty_tensors, sample_tokens, sampling_tensors, token_state_row, xtc_tensors
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _same_bits(a, b) -> bool:
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    both_nan = np.isnan(a) & np.isnan(b)
    return bool(np.all(both_nan | (a.view(np.int32) == b.view(np.int32))))


def _history(kind: str, n: int, rng: np.random.Generator, V: int) -> list:
    if kind == "random":
        return rng.integers(0, V, n).tolist()
    if kind == "periodic":
        period = rng.integers(0, V, int(rng.integers(2, 40))).tolist()
        return (period * (n // len(period) + 1))[:n]
    if kind == "run":
        return [int(rng.integers(0, V))] * n
    h = rng.integers(0, 12, n).tolist()  # a small alphabet: many short matches
    return h


@pytest.mark.parametrize("V,dtype", [(1000, torch.float32), (4097, torch.bfloat16), (151936, torch.bfloat16), (151936, torch.float32)])
def test_dry_penalty_bit_exact(cuda_device, V, dtype):
    rng = np.random.default_rng(V)
    cases = [("random", 1024, {}), ("periodic", 8192, {}), ("run", 300, {}), ("small", 2000, dict(dry_sequence_breakers=(3, 7))),
             ("periodic", 32768, dict(dry_penalty_last_n=5000)), ("small", 600, dict(dry_allowed_length=1, dry_base=3.0)),
             ("periodic", 4000, dict(dry_multiplier=1e30, dry_base=10.0)), ("small", 50, dict(dry_penalty_last_n=7)),
             ("random", 5, {}), ("run", 2, dict(dry_allowed_length=1))]
    R = len(cases) + 3
    cap = 32768
    tab = DryRows(R, cap, cuda_device)
    hists, params, pos, toks = [], [], [], []
    for r, (kind, n, kw) in enumerate(cases):
        h = _history(kind, n, rng, V)
        p = SamplingParams(0.7, **{"dry_multiplier": 0.8, **kw})
        if kw.get("dry_sequence_breakers") and r % 2:
            h[-1] = 3  # the input token is a breaker: nothing is penalised
        tab.set_row(r, p, h)
        hists.append(h), params.append(p), pos.append(n), toks.append(h[-1])
    # a DRY-off row, a DRY row at position 0, a row past its capacity: all left alone
    off = _history("periodic", 500, rng, V)
    tab.history[R - 3, :499] = torch.tensor(off[:-1], dtype=torch.int32)
    hists.append(off), params.append(None), pos.append(500), toks.append(off[-1])
    tab.set_row(R - 2, SamplingParams(0.7, dry_multiplier=0.8), [1, 1, 1, 1])
    hists.append(None), params.append(None), pos.append(0), toks.append(1)
    tab.set_row(R - 1, SamplingParams(0.7, dry_multiplier=0.8), [1, 1, 1, 1])
    hists.append(None), params.append(None), pos.append(cap + 1), toks.append(1)
    raw = (torch.randn(R, V, generator=torch.Generator().manual_seed(V)) * 4).to(dtype)
    raw[0, 5] = float("nan")
    raw[1, :64] = float("inf")
    zero = torch.zeros((R, ext.CONTROL_ROW_WORDS), dtype=torch.int64, device=cuda_device)
    x = ext.logit_controls(raw.to(cuda_device), zero, torch.zeros(R, dtype=torch.int32, device=cuda_device),
                           torch.zeros(R, dtype=torch.int32, device=cuda_device), torch.full((R, ext.CONTROL_TAIL), -1, dtype=torch.int32,
                                                                                              device=cuda_device))
    before = x.cpu().numpy().copy()
    hist_before = tab.history.cpu().clone()
    ext.dry_penalty(x, tab.table, torch.tensor(pos, dtype=torch.int32, device=cuda_device), torch.tensor(toks, dtype=torch.int32, device=cuda_device),
                    tab.history, tab.scratch)
    got = x.cpu().numpy()
    hist_after = tab.history.cpu()
    for r in range(R):
        p = params[r]
        if p is None:
            assert _same_bits(got[r], before[r]), r
            assert torch.equal(hist_after[r], hist_before[r]), r
            continue
        want = dref.dry_penalize(before[r], hists[r], p.dry_multiplier, p.dry_base, p.dry_allowed_length, p.dry_penalty_last_n,
                                 p.dry_sequence_breakers)
        assert _same_bits(got[r], want), (r, np.flatnonzero(~((got[r] == want) | (np.isnan(got[r]) & np.isnan(want))))[:8])
        n = pos[r]
        assert hist_after[r, n - 1] == toks[r] and torch.equal(hist_after[r, : n - 1], hist_before[r, : n - 1])
    assert any(not _same_bits(got[r], before[r]) for r in range(len(cases)))


def _xtc_grid():
    out = []
    for th in (0.05, 0.1, 0.3):
        for q in (0.5, 1.0):
            for T, k, tp, mp, pen in ((1.0, 0, 0.0, 0.0, False), (0.7, 50, 0.0, 0.0, False), (1.3, 0, 0.9, 0.0, False),
                                      (0.9, 0, 0.0, 0.02, True), (0.6, 20, 0.95, 0.05, True)):
                out.append((th, q, T, k, tp, mp, pen))
    return out


def _peaked(R, V, g):
    """Rows with a handful of likely tokens, so that XTC's top choices exist at every threshold of the grid."""
    x = torch.randn(R, V, generator=g) * 1.5
    for r in range(R):
        top = torch.randperm(V, generator=g)[:6]
        x[r, top] += torch.linspace(7.0, 5.0, 6) + torch.rand(6, generator=g)
    return x


@pytest.mark.parametrize("V,dtype", [(4097, torch.float32), (151936, torch.bfloat16)])
def test_xtc_draws_equal_the_oracle(cuda_device, V, dtype):
    g = torch.Generator().manual_seed(V)
    R = 64
    near = total = 0
    for j, (th, q, T, k, tp, mp, pen) in enumerate(_xtc_grid()):
        x = _peaked(R, V, g).to(dtype)
        params = [SamplingParams(T, top_k=k or None, top_p=tp or None, seed=1000 * j + r, min_p=mp, xtc_threshold=th, xtc_probability=q,
                                 repetition_penalty=1.2 if pen else 1.0, presence_penalty=0.5 if pen else 0.0) for r in range(R)]
        state = torch.stack([token_state_row(torch.randint(0, V, (20,), generator=g).tolist(), torch.randint(0, V, (5,), generator=g).tolist(), V)
                             for _ in range(R)])
        positions = list(range(3, 3 + R))
        temp, top_k, top_p, seed = sampling_tensors(params, cuda_device)
        got = ext.sample_penalized(x.to(cuda_device), temp, top_k, top_p, seed, torch.tensor(positions, dtype=torch.int32, device=cuda_device),
                                   *penalty_tensors(params, cuda_device), state.to(cuda_device), xtc_threshold=xtc_tensors(params, cuda_device)[0],
                                   xtc_probability=xtc_tensors(params, cuda_device)[1]).cpu()
        xf = x.float().numpy()
        for r in range(R):
            p = params[r]
            want, close = dref.xtc_sample_row(xf[r], state[r].numpy(), T, k, tp, p.seed, positions[r], p.repetition_penalty,
                                               p.presence_penalty, 0.0, mp, th, q)
            total += 1
            if close:
                near += 1
                continue
            assert int(got[r]) == want, (j, r)
    print(f"XTC draws V={V}: {total} compared, {near} within 2^-20 of the threshold (not compared)")
    assert near < total // 20


def test_xtc_edges(cuda_device):
    V, R = 4097, 64
    g = torch.Generator().manual_seed(1)
    x = _peaked(R, V, g).to(cuda_device)
    pos = torch.arange(1, R + 1, dtype=torch.int32, device=cuda_device)
    state = torch.zeros((R, V), dtype=torch.int32, device=cuda_device)

    def draw(params, rows=x, st=state, p=pos):
        t, k, tp, s = sampling_tensors(params, cuda_device)
        th, q = xtc_tensors(params, cuda_device)
        return ext.sample_penalized(rows, t, k, tp, s, p, *penalty_tensors(params, cuda_device), st.clone(), xtc_threshold=th,
                                    xtc_probability=q).cpu()

    base = [SamplingParams(0.8, seed=r) for r in range(R)]
    t, k, tp, s = sampling_tensors(base, cuda_device)
    plain = ext.sample(x, t, k, tp, s, pos).cpu()
    # q = 0: today's draw
    assert torch.equal(draw([SamplingParams(0.8, seed=r, xtc_probability=0.0) for r in range(R)]), plain)
    # q = 1: every draw excludes its top choices but the least likely
    q1 = [SamplingParams(0.8, seed=r, xtc_probability=1.0, xtc_threshold=0.05) for r in range(R)]
    got = draw(q1)
    xs = x.cpu().numpy()
    for r in range(R):
        keep = np.ones(V, bool)
        keep2, _ = dref.xtc_keep(xs[r], keep, 0.8, 0.05, 1.0, r, r + 1)
        assert keep2[int(got[r])]
        assert (~keep2).sum() >= 1 or keep2.all()
    # temperature 0 is unchanged
    greedy = [SamplingParams(0.0, xtc_probability=1.0, xtc_threshold=0.01) for _ in range(R)]
    assert torch.equal(draw(greedy), torch.argmax(x, -1).int().cpu())
    # rows are independent of their index and of the row count
    alone = torch.cat([draw([q1[r]], x[r : r + 1], state[r : r + 1], pos[r : r + 1]) for r in (0, 17, 63)])
    assert torch.equal(alone, got[[0, 17, 63]])


def test_xtc_constrained_sees_allowed_entries_only(cuda_device):
    V, R, S = 4097, 16, 3
    g = torch.Generator().manual_seed(2)
    x = _peaked(R, V, g)
    words = (V + 31) // 32
    allowed = np.zeros((R, V), bool)
    for r in range(R):
        top = torch.topk(x[r], 6).indices.numpy()
        allowed[r] = np.random.default_rng(r).random(V) < 0.5
        allowed[r, top[:2]] = False  # the two most likely tokens are disallowed: XTC must not count them
        allowed[r, top[2:]] = True
    masks = np.zeros((R, S + 1, words), dtype=np.uint32)
    for r in range(R):
        bits = np.zeros(words * 32, bool)
        bits[:V] = allowed[r]
        masks[r, :S] = np.packbits(bits, bitorder="little").view("<u4")
    masks_d = torch.from_numpy(masks.view(np.int32)).to(cuda_device)
    dfa = torch.zeros((S, 256), dtype=torch.int32, device=cuda_device)
    offsets = torch.arange(V + 1, dtype=torch.int32, device=cuda_device)
    data = torch.zeros(V, dtype=torch.uint8, device=cuda_device)
    row_bytes = (S + 1) * words * 4
    desc = torch.tensor([[masks_d.data_ptr() + r * row_bytes, dfa.data_ptr(), offsets.data_ptr(), data.data_ptr(), S] for r in range(R)],
                        dtype=torch.int64, device=cuda_device)
    params = [SamplingParams(0.9, seed=r, xtc_probability=1.0, xtc_threshold=0.08) for r in range(R)]
    t, k, tp, s = sampling_tensors(params, cuda_device)
    th, q = xtc_tensors(params, cuda_device)
    state = torch.zeros((R, V), dtype=torch.int32, device=cuda_device)
    pos = torch.full((R,), 0, dtype=torch.int32, device=cuda_device)  # position 0: the states stay as they are
    got = ext.sample_constrained(x.to(cuda_device), t, k, tp, s, pos, desc, *penalty_tensors(params, cuda_device), state, xtc_threshold=th,
                                 xtc_probability=q).cpu()
    near = 0
    for r in range(R):
        want, close = dref.xtc_sample_row(x[r].numpy(), np.zeros(V, np.int64), 0.9, 0, 0.0, r, 0, threshold=0.08, probability=1.0,
                                          allowed=allowed[r])
        near += close
        if not close:
            assert int(got[r]) == want, r
        assert allowed[r, int(got[r])]
    assert near < R // 2


# ------------------------------------------------------------------------------------------------ models --
def _model(dev, seed=5):
    ns = synthetic_qwen3("tiny-d128", seed=seed, realistic=True, max_position_embeddings=8192, device=dev)
    return Qwen3ModelWeek3(ns, page_size=64)


def test_generate_equals_a_host_loop(cuda_device):
    model = _model(cuda_device, seed=7)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11, 5, 17, 3, 250]
    n = 24
    for p in (SamplingParams(0.0, dry_multiplier=2.0, dry_allowed_length=1),
              SamplingParams(0.9, seed=4, dry_multiplier=0.8, dry_sequence_breakers=(5,), xtc_probability=0.7, xtc_threshold=0.05),
              SamplingParams(0.8, seed=2, xtc_probability=1.0, xtc_threshold=0.02, min_p=0.01)):
        got = greedy_generate_ids(model, prompt, n, device=cuda_device, sampling=p)
        cache = model.create_kv_cache()
        want, hist = [], list(prompt)
        state = token_state_row(prompt, [], model.vocab_size)
        try:
            feed, offset = prompt, 0
            for _ in range(n):
                logits = model(torch.tensor([feed], dtype=torch.int32, device=cuda_device), offset, cache, logits_to_keep=1)[0, -1].float().cpu()
                x = logits.numpy()
                if p.dry:
                    x = dref.dry_penalize(x, hist, p.dry_multiplier, p.dry_base, p.dry_allowed_length, p.dry_penalty_last_n,
                                          p.dry_sequence_breakers)
                t, _ = dref.xtc_sample_row(x, state.numpy(), p.temperature, 0, 0.0, p.seed, len(hist), min_p=p.min_p,
                                           threshold=p.xtc_threshold, probability=p.xtc_probability)
                want.append(t)
                state[t] += 1
                offset += len(feed)
                feed = [t]
                hist.append(t)
        finally:
            for c in cache:
                c.release()
        assert got == want, p
    plain = greedy_generate_ids(model, [3] * 6, n, device=cuda_device, sampling=SamplingParams(0.0))
    dry = greedy_generate_ids(model, [3] * 6, n, device=cuda_device, sampling=SamplingParams(0.0, dry_multiplier=5.0, dry_allowed_length=1))
    assert dry != plain


def test_batcher_request_equals_alone_in_two_orders(cuda_device):
    import dataclasses

    ns = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, device=cuda_device)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, 60, (int(n),), generator=g).tolist() for n in torch.randint(3, 40, (10,), generator=g)]
    kinds = [lambda i: SamplingParams(0.8, seed=i, dry_multiplier=1.0, dry_allowed_length=1, xtc_probability=0.5),
             lambda i: SamplingParams(0.0, dry_multiplier=0.8, dry_sequence_breakers=(7, 9), presence_penalty=0.3),
             lambda i: SamplingParams(0.9, seed=i, xtc_probability=1.0, xtc_threshold=0.05),
             lambda i: SamplingParams(0.7, seed=i, logit_bias={40: 2.0})]
    params = [kinds[i % 4](i) for i in range(len(prompts))]
    plain = [dataclasses.replace(p, dry_multiplier=0.0, xtc_probability=0.0) for p in params]
    budget, B = 12, 4

    def serve(idx, per):
        out = batch_generate(Qwen3ModelWeek3(ns, page_size=64), None, [prompts[i] for i in idx], max_seq_len=128, batch_size=B,
                             prefill_step=16, verbose=False, device=cuda_device, max_new_tokens=[budget] * len(idx),
                             sampling=[per[i] for i in idx])
        return {idx[j]: [int(t) for t in text.split()] for j, text in out}

    orders = (list(range(len(prompts))), list(reversed(range(len(prompts)))))
    # The batcher's logits for a request can depend on what else is served beside it, with or without these samplers:
    # a request is checked in an order where its plain twin (DRY and XTC off) gets the ids it gets alone.
    checked = 0
    for order in orders:
        got, twin = serve(order, params), serve(order, plain)
        for i in order:
            if twin[i] != serve([i], plain)[i]:
                continue
            assert got[i] == serve([i], params)[i], (order[0], i)
            checked += 1
    print(f"batcher: {checked} of {2 * len(prompts)} (request, order) pairs checked")
    assert checked >= len(prompts)


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


@pytest.mark.parametrize("B,lens,logprobs", [(1, {0: 40}, None), (16, {0: 40, 3: 9, 9: 70, 15: 20}, None), (16, {0: 40, 3: 9, 9: 70, 15: 20}, 4),
                                             (32, {0: 30, 2: 65, 5: 12, 11: 90}, None), (32, {0: 30, 2: 65, 5: 12, 11: 90}, 3)])
def test_decode_on_device_equals_steps_plus_eager(cuda_device, B, lens, logprobs):
    steps, msl = 20, 256
    slots = sorted(lens)
    g = torch.Generator().manual_seed(B)
    # a slot at offset L has L ids in its cache and is fed the last of its L + 1 history ids
    history = [(torch.randint(0, 40, (lens[b] - 2,), generator=g).tolist(), torch.randint(0, 40, (3,), generator=g).tolist()) if b in lens
               else None for b in range(B)]
    kinds = [lambda b: SamplingParams(0.0, dry_multiplier=1.5, dry_allowed_length=1, dry_sequence_breakers=(3,)),
             lambda b: SamplingParams(0.9, top_p=0.95, seed=b, dry_multiplier=0.8, xtc_probability=0.6, xtc_threshold=0.05, presence_penalty=0.2),
             lambda b: SamplingParams(1.1, top_k=30, seed=b, xtc_probability=1.0, xtc_threshold=0.02),
             lambda b: SamplingParams(0.7, seed=b, dry_multiplier=0.5, dry_penalty_last_n=16, logit_bias={17: 2.0})]
    params = [None] * B
    for n, b in enumerate(slots):
        params[b] = kinds[n % 4 if B > 1 else 1](b)
    runs, lps, final = {}, {}, {}
    for mode in ("graph", "eager"):
        model = _model(cuda_device)
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, lens)
        _fill_slabs(model, B)
        tokens = [history[b][1][-1] if b in lens else 0 for b in range(B)]
        offsets = [lens.get(b, 0) for b in range(B)]
        if mode == "graph":
            res = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params, logprobs=logprobs, history=history)
            runs[mode] = (res if logprobs is None else res[0]).cpu()
            if logprobs is not None:
                lps[mode] = res[1][0].cpu()
            assert engine.kernels_per_controlled_step >= engine.kernels_per_step + 1
            final[mode] = engine._ctl_tab.dry.history.cpu()
        else:
            hist = [None if h is None else (list(h[0]), list(h[1])) for h in history]
            state = torch.stack([token_state_row(*h, model.vocab_size) if h is not None else torch.zeros(model.vocab_size, dtype=torch.int32)
                                 for h in hist]).to(cuda_device)
            out, lp_rows = [], []
            for _ in range(steps):
                logits, _ = engine.step(tokens, offsets, caches)
                logits = logits.view(B, -1)
                pos = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
                table, _ = control_rows(params, model.vocab_size, cuda_device, (), hist, history_capacity=msl)
                nxt = sample_tokens(logits, params, pos, state, controls=table, tokens=tokens)
                if logprobs is not None:
                    lp_rows.append(ext.logprobs(logits, nxt, max_n=logprobs)[1].cpu())
                nxt = nxt.cpu()
                out.append([int(nxt[b]) if b in lens else -1 for b in range(B)])
                tokens = [int(nxt[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
                for b in lens:
                    hist[b][1].append(tokens[b])
            runs[mode] = torch.tensor(out, dtype=torch.int32)
            if logprobs is not None:
                lps[mode] = torch.stack(lp_rows)
            final[mode] = hist
    assert torch.equal(runs["graph"], runs["eager"])
    live = torch.tensor([b in lens for b in range(B)])
    if logprobs is not None:
        assert torch.equal(lps["graph"][:, live], lps["eager"][:, live])
    for b in lens:
        if params[b].dry:  # the device history holds every id up to the last step's input token
            h = final["eager"][b][0] + final["eager"][b][1]
            assert final["graph"][b, : len(h) - 1].tolist() == h[:-1], b


def test_without_either_sampler_nothing_changes(cuda_device):
    model = _model(cuda_device)
    B, msl = 4, 128
    engine = DecodeEngine(model, B, msl, cuda_device)
    engine.reserve_pools()
    caches = _admit(model, B, msl, {0: 10, 1: 12})
    engine.decode_on_device([1, 2, 0, 0], [10, 12, 0, 0], caches, 4, sampling=SamplingParams(0.8, presence_penalty=0.5))
    assert engine._graph_pen is not None and engine._graph_pen_xtc is None
    engine.decode_on_device([1, 2, 0, 0], [14, 16, 0, 0], caches, 4, sampling=SamplingParams(0.8, logit_bias={3: 1.0}),
                            history=[([1] * 14, [1]), ([2] * 16, [2]), None, None])
    assert engine._ctl_tab.dry is None and all(len(k) == 2 for k in engine._graph_ctl)
