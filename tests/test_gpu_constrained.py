"""Regex-constrained generation on the H100: ``tl_constraint_token_masks`` bit for bit against the host references
(shared- and global-memory tables, V = 512 and 151,936), ``tl_sample_constrained`` against ``oracle/sampling.py`` and
the unconstrained kernels on rows with disallowed entries set to -inf, the on-device state advance against the host
walk, and the same constrained request through ``greedy_generate_ids``, the batcher and ``decode_on_device``."""

import importlib.util
import re
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as ref
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, greedy_generate_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.constrained import TokenConstraint, TokenVocabulary, descriptor_state, token_masks_reference
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.sampler import penalty_tensors, sample_tokens, sampling_tensors
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load_constrained_ref():
    name = "tiny_llm_b200_constrained_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("constrained_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


cref = _load_constrained_ref()


# ------------------------------------------------------------------------------------------- token masks --
@pytest.mark.parametrize("V,patterns", [
    (512, [r"[0-9]{4}-[0-9]{2}-[0-9]{2}", r"(ab|cd)*e?", r"é+ж?[α-ω]", r"[^a-c\n]{1,3}", r"[a-z0-9]{250}", r".{0,20}!"]),
    (151936, [r"\d+(\.\d{1,3})?", r"\w+@\w+\.(com|org)", r"(?:yes|no|maybe)", r"[a-z ]{1,40}\.", r"[a-f0-9]{200}"]),
])
def test_token_masks_equal_the_reference(cuda_device, V, patterns):
    vocab = TokenVocabulary.synthetic(V, seed=3)
    sizes = []
    for pattern in patterns:
        c = TokenConstraint.compile(pattern, vocab, device=cuda_device)
        want_m, want_r = token_masks_reference(c.dfa, vocab)
        got_m = c.masks.cpu().numpy().view(np.uint32)
        got_r = c.reach.cpu().numpy().view(np.uint32)
        np.testing.assert_array_equal(got_m, want_m, err_msg=pattern)
        np.testing.assert_array_equal(got_r, want_r, err_msg=pattern)
        sizes.append(c.dfa.num_states)
    assert min(sizes) <= 192 < max(sizes)  # tables in shared memory and in global memory


def test_token_masks_of_a_small_vocabulary_equal_the_per_token_walk(cuda_device):
    vocab = TokenVocabulary.synthetic(128, seed=1)
    for pattern in (r"[0-9]{4}-[0-9]{2}-[0-9]{2}", r"\s*\S+\s*"):
        c = TokenConstraint.compile(pattern, vocab, device=cuda_device)
        m, r = cref.token_masks_walk(c.dfa, vocab)
        np.testing.assert_array_equal(c.masks.cpu().numpy().view(np.uint32), m)
        np.testing.assert_array_equal(c.reach.cpu().numpy().view(np.uint32), r)


def test_dead_end_vocabulary_raises(cuda_device):
    vocab = TokenVocabulary.synthetic(128, seed=1)  # ASCII bytes and a few two-byte letters: no way to spell '中'
    with pytest.raises(ValueError, match="cannot continue the text"):
        TokenConstraint.compile("a中", vocab, device=cuda_device)


# ---------------------------------------------------------------------------------------- the draw itself --
def _rows(V, rows, dtype, g, dev):
    x = torch.randn(rows, V, generator=g) * 3
    return x.to(dtype).to(dev)


def _masked(x, allowed):
    """``x`` with disallowed entries -inf (float32)."""
    return torch.where(allowed, x.float(), torch.full_like(x.float(), float("-inf")))


def _states(c, rows, g):
    """A random reachable state per row (random walks of allowed tokens from the start)."""
    masks = c.masks.cpu().numpy().view(np.uint32)
    out = []
    for _ in range(rows):
        s = 0
        for _ in range(int(torch.randint(0, 6, (1,), generator=g))):
            ok = np.flatnonzero(cref.allowed_bits(masks, s, c.vocab_size))
            t = int(ok[int(torch.randint(0, len(ok), (1,), generator=g))])
            s = c.walk(s, [t])
        out.append(s)
    return out


def _descriptors(cs, states, dev):
    return torch.stack([c.descriptor(s) if c is not None else torch.zeros(5, dtype=torch.int64, device=dev) for c, s in zip(cs, states)])


PARAMS = [SamplingParams(0.0), SamplingParams(0.8, seed=11), SamplingParams(1.0, top_k=5, seed=12), SamplingParams(0.7, top_p=0.9, seed=13),
          SamplingParams(1.2, top_k=50, top_p=0.8, seed=14), SamplingParams(0.9, seed=15, min_p=0.1, presence_penalty=0.5)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("V", [512, 151936])
def test_constrained_draw_equals_the_unconstrained_kernel_and_oracle_on_the_masked_row(cuda_device, dtype, V):
    g = torch.Generator().manual_seed(V + len(str(dtype)))
    vocab = TokenVocabulary.synthetic(V, seed=2)
    c = TokenConstraint.compile(r"[a-z]{2,8}( [a-z]{2,8}){0,3}\.|\d{1,4}", vocab, device=cuda_device)
    rows = 24
    x = _rows(V, rows, dtype, g, cuda_device)
    states = _states(c, rows, g)
    masks = c.masks.cpu().numpy().view(np.uint32)
    allowed = torch.from_numpy(np.stack([cref.allowed_bits(masks, s, V) for s in states])).to(cuda_device)
    params = [PARAMS[r % len(PARAMS)] for r in range(rows)]
    params = [SamplingParams(p.temperature, p.top_k, p.top_p, p.seed + r, p.repetition_penalty, p.presence_penalty, p.frequency_penalty,
                             p.min_p, constraint=c) for r, p in enumerate(params)]
    positions = list(range(1, rows + 1))
    state = torch.zeros(rows, V, dtype=torch.int32, device=cuda_device)
    state[:, :64] = 1  # a few drawn tokens for the penalised rows
    desc = _descriptors([c] * rows, states, cuda_device)
    got = sample_tokens(x, params, positions, state.clone(), desc).cpu()
    # the unconstrained kernel on the -inf-masked row (its penalised form for the penalised rows)
    xm = _masked(x, allowed).to(dtype)
    plain = [SamplingParams(p.temperature, p.top_k, p.top_p, p.seed, p.repetition_penalty, p.presence_penalty, p.frequency_penalty, p.min_p)
             for p in params]
    want = sample_tokens(xm, plain, positions, state.clone()).cpu()
    assert torch.equal(got, want)
    assert allowed.cpu()[torch.arange(rows), got.long()].all()
    # and oracle/sampling.py on the same masked rows, for the rows without penalties
    for r, p in enumerate(plain):
        if not p.penalized:
            assert int(got[r]) == ref.sample_row(xm[r].float().cpu().numpy(), p.temperature, p.top_k, p.top_p, p.seed, positions[r]), r
    # the states advanced along the drawn tokens, on the device
    assert descriptor_state(desc).cpu().tolist() == [c.walk(s, [int(t)]) for s, t in zip(states, got)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_all_allowed_mask_is_bit_identical_to_sample_and_sample_penalized(cuda_device, dtype):
    V, rows = 151936, 16
    c = TokenConstraint.compile(".*", TokenVocabulary([b"a"] * (V - 1) + [None], [V - 1]), device=cuda_device)
    assert bool((c.masks[0] == -1).all())  # every token allowed in the start state ("a"* and EOS)
    g = torch.Generator().manual_seed(1)
    x = _rows(V, rows, dtype, g, cuda_device)
    positions = torch.arange(1, rows + 1, dtype=torch.int32, device=cuda_device)
    for params in ([SamplingParams(0.9, 40, 0.95, seed=r) for r in range(rows)], [PARAMS[r % len(PARAMS)] for r in range(rows)]):
        t = sampling_tensors(params, cuda_device)
        pen = penalty_tensors(params, cuda_device)
        state = torch.randint(0, 3, (rows, V), dtype=torch.int32, device=cuda_device)
        a = ext.sample(x, *t, positions)
        b = ext.sample_constrained(x, *t, positions, torch.stack([c.descriptor()] * rows))
        assert torch.equal(a, b)
        st1, st2 = state.clone(), state.clone()
        a = ext.sample_penalized(x, *t, positions, *pen, st1)
        b = ext.sample_constrained(x, *t, positions, torch.stack([c.descriptor()] * rows), *pen, st2)
        assert torch.equal(a, b) and torch.equal(st1, st2)


def test_mixed_launch_and_rows_without_finite_allowed_entries(cuda_device):
    V, rows = 4097, 12
    vocab = TokenVocabulary.synthetic(V, seed=5)
    c = TokenConstraint.compile(r"\d{3}", vocab, device=cuda_device)
    g = torch.Generator().manual_seed(2)
    x = _rows(V, rows, torch.float32, g, cuda_device)
    masks = c.masks.cpu().numpy().view(np.uint32)
    allowed0 = cref.allowed_bits(masks, 0, V)
    ids = np.flatnonzero(allowed0)
    x[1, torch.from_numpy(ids).to(cuda_device)] = float("-inf")  # no finite allowed entry: the lowest allowed id
    x[3, torch.from_numpy(ids).to(cuda_device)] = float("nan")  # every allowed entry NaN: the lowest allowed id
    x[5, torch.from_numpy(ids[3:]).to(cuda_device)] = float("-inf")
    x[5, torch.from_numpy(ids[:3]).to(cuda_device)] = float("nan")  # NaN then -inf: the first allowed -inf
    x[7, int(ids[5])] = float("inf")
    params = [SamplingParams(0.0 if r % 4 == 0 else 0.8, seed=r, constraint=c if r % 2 else None) for r in range(rows)]
    positions = [0 if r == 9 else r + 1 for r in range(rows)]
    desc = _descriptors([p.constraint for p in params], [0] * rows, cuda_device)
    got = sample_tokens(x, params, positions, None, desc).cpu()
    plain = [SamplingParams(p.temperature, seed=p.seed) for p in params]
    free = sample_tokens(x, plain, positions).cpu()
    for r in range(rows):
        if r % 2 == 0:  # unconstrained rows: tl_sample's token
            assert int(got[r]) == int(free[r])
    assert int(got[1]) == int(ids[0]) and int(got[3]) == int(ids[0]) and int(got[5]) == int(ids[3]) and int(got[7]) == int(ids[5])
    for r in (9, 11):
        assert allowed0[int(got[r])]
    st = descriptor_state(desc).cpu().tolist()
    for r in range(rows):
        if r % 2 == 0:
            assert st[r] == 0 and bool((desc[r] == 0).all())
        elif r == 9:
            assert st[r] == 0  # position 0: no advance
        else:
            assert st[r] == c.walk(0, [int(got[r])])


def test_eos_moves_to_the_terminal_state_which_allows_only_eos(cuda_device):
    V = 512
    vocab = TokenVocabulary.synthetic(V)
    c = TokenConstraint.compile("ok", vocab, device=cuda_device)
    eos = vocab.eos_ids[0]
    s_ok = c.walk(0, [ord("o"), ord("k")])
    x = torch.zeros(3, V, device=cuda_device)
    x[:, eos] = -5.0  # EOS is unlikely but the only allowed token
    desc = _descriptors([c] * 3, [s_ok, c.terminal_state, c.terminal_state], cuda_device)
    got = sample_tokens(x, [SamplingParams(0.0, constraint=c)] * 3, [4, 5, 6], None, desc).cpu().tolist()
    assert got == [eos] * 3
    assert descriptor_state(desc).cpu().tolist() == [c.terminal_state] * 3


# -------------------------------------------------------------------------------------- end to end --
PATTERN = r"(ab|[0-9]{1,3}-){1,3}\.|x[a-z ]{0,6}y"  # at most 13 bytes: every request reaches EOS within 24 tokens


def _model(dev, seed=5):
    ns = synthetic_qwen3("tiny-d128", seed=seed, realistic=True, max_position_embeddings=8192, device=dev)
    return Qwen3ModelWeek3(ns, page_size=64)


def _check_output(c, ids, eos, finished):
    text = b"".join(c.vocabulary.tokens[t] for t in ids)
    if finished:
        assert re.fullmatch(PATTERN, text.decode(), re.ASCII), text
    else:
        assert c.dfa.walk(0, text) >= 0, text


def test_generate_batcher_and_decode_on_device_give_the_same_constrained_tokens(cuda_device):
    model = _model(cuda_device)
    vocab = TokenVocabulary.synthetic(model.vocab_size)
    eos = vocab.eos_ids[0]
    c = TokenConstraint.compile(PATTERN, vocab, device=cuda_device)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, 500, (int(n),), generator=g).tolist() for n in (5, 17, 9, 30, 3, 12)]
    params = [SamplingParams((0.0, 0.9, 1.3)[i % 3], top_k=(None, 40)[i % 2], seed=100 + i, constraint=c) for i in range(len(prompts))]
    n = 24
    gen = {}
    for i, (p, s) in enumerate(zip(prompts, params)):
        ids = greedy_generate_ids(model, p, n, eos_token_id=eos, device=cuda_device, sampling=s)
        gen[i] = ids
        _check_output(c, ids, eos, finished=len(ids) < n)
    assert all(len(v) < n for v in gen.values())
    # the batcher, two batch sizes and queue orders, with unconstrained requests mixed in
    for batch_size, order in ((4, list(range(len(prompts)))), (3, list(reversed(range(len(prompts)))))):
        queue = [prompts[i] for i in order] + [[7, 8, 9]]
        samp = [params[i] for i in order] + [SamplingParams(0.8, seed=1)]
        b = ContinuousBatcher(model, None, queue, max_seq_len=128, batch_size=batch_size, prefill_step=8, verbose=False, eos_token_id=eos,
                              device=cuda_device, max_new_tokens=[n] * len(queue), sampling=samp)
        res = dict(b.run())
        for j, i in enumerate(order):
            got = [int(t) for t in res[j].split()]
            assert got == gen[i], (batch_size, i)
    # decode_on_device from the prompt's first token, with history for the state
    for i in (0, 1, 3):
        p, s = prompts[i], params[i]
        cache = model.create_kv_cache()
        try:
            logits = model(torch.tensor([p], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
            desc = c.descriptor()[None]
            first = int(sample_tokens(logits[:, -1, :], [s], [len(p)], None, desc)[0])
            engine = model.decode_engine(1, model._graph_limit(cache))
            log = engine.decode_on_device([first], [len(p)], cache, n - 1, sampling=s, history=[(p, [first])])
            want = [first] + log[:, 0].tolist()
        finally:
            for cc in cache:
                cc.release()
        got = gen[i]
        assert want[: len(got)] == got
        if len(got) < n:  # past EOS the device loop keeps emitting EOS
            assert set(want[len(got):]) == {eos}


def _admit(model, B, msl, lens):
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b, n in lens.items():
        cache = model.create_kv_cache()
        for cc, t in zip(cache, tables):
            cc.append_slots(n)
            t.add_request(cc, b)
    return tables


@pytest.mark.parametrize("penalized,logprobs", [(False, None), (True, None), (False, 3)])
def test_decode_on_device_constrained_equals_eager_steps(cuda_device, penalized, logprobs):
    B, msl, steps = 16, 256, 12
    lens = {0: 40, 3: 9, 9: 70, 15: 20}
    vocab = TokenVocabulary.synthetic(512)
    runs, lps = {}, {}
    for mode in ("graph", "eager"):
        model = _model(cuda_device)
        c = TokenConstraint.compile(PATTERN, vocab, device=cuda_device)
        extra = dict(presence_penalty=0.8, frequency_penalty=0.2) if penalized else {}
        params = [None] * B
        for n, b in enumerate(sorted(lens)):
            params[b] = SamplingParams((0.0, 0.9)[n % 2], seed=50 + b, constraint=c if n != 2 else None, **extra)
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, lens)
        tokens = [ord("a") if b in lens else 0 for b in range(B)]
        offsets = [lens.get(b, 0) for b in range(B)]
        history = [([1, 2], [ord("a")]) if b in lens else None for b in range(B)]
        if mode == "graph":
            base = engine.decode_on_device(tokens, offsets, caches, 2)  # the unconstrained graphs first
            k_step, k_sampled, h2d = engine.kernels_per_step, engine.kernels_per_sampled_step, engine.h2d_bytes
            offsets = [o + 2 if b in lens else 0 for b, o in enumerate(offsets)]
            tokens = [int(t) if b in lens else 0 for b, t in enumerate(base[-1].tolist())]
            for b in lens:
                history[b] = ([1, 2], [ord("a")])
            res = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params, logprobs=logprobs, history=history)
            out = res if logprobs is None else res[0]
            runs[mode] = out.cpu()
            if logprobs is not None:
                lps[mode] = res[1][0].cpu()
            assert engine.kernels_per_step == k_step and engine.kernels_per_sampled_step == k_sampled
            assert engine.kernels_per_constrained_step == k_step - 1 + (logprobs is not None)  # one launch instead of argmax
            before = engine.h2d_bytes - h2d
            offsets = [o + steps if b in lens else 0 for b, o in enumerate(offsets)]
            h0 = engine.h2d_bytes
            engine.decode_on_device(tokens, offsets, caches, 1)  # unconstrained again: the same upload as before
            assert engine.h2d_bytes - h0 <= before
        else:
            # replay the graph mode's warm-up: two greedy steps first
            for _ in range(2):
                logits, nxt = engine.step(tokens, offsets, caches)
                nxt = nxt.cpu()
                tokens = [int(nxt[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
            desc = _descriptors([None if p is None else p.constraint for p in params],
                                [c.walk(0, [ord("a")]) for _ in range(B)], cuda_device)
            state = None
            if penalized:
                from tiny_llm_b200.sampler import token_state_row

                state = torch.stack([token_state_row([1, 2], [ord("a")], 512) if b in lens else torch.zeros(512, dtype=torch.int32)
                                     for b in range(B)]).to(cuda_device)
            out, lp_rows = [], []
            for _ in range(steps):
                logits, _ = engine.step(tokens, offsets, caches)
                logits = logits.view(B, -1)
                pos = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
                nxt = sample_tokens(logits, params, pos, state, desc)
                if logprobs is not None:
                    lp_rows.append(ext.logprobs(logits, nxt, max_n=logprobs)[1].cpu())
                nxt = nxt.cpu()
                out.append([int(nxt[b]) if b in lens else -1 for b in range(B)])
                tokens = [int(nxt[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
            runs[mode] = torch.tensor(out, dtype=torch.int32)
            if logprobs is not None:
                lps[mode] = torch.stack(lp_rows)
    live = torch.tensor([b in lens for b in range(B)])
    assert torch.equal(runs["graph"][:, live], runs["eager"][:, live])
    if logprobs is not None:
        assert torch.equal(lps["graph"][:, live], lps["eager"][:, live])
