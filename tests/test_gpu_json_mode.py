"""JSON mode on the H100 (DESIGN.md section 20): ``tl_json_token_masks`` bit for bit against the reference language at
V = 151,936 and on an adversarial vocabulary, ``tl_json_advance`` against the host walk, a JSON row's draw against the
unconstrained kernels on the -inf-masked row (with regex, penalised and plain rows in the same launch), and the same
JSON requests through ``greedy_generate_ids``, the batcher, ``decode_on_device`` (eager and graph) and
``parallel_sample_ids``, equal to a host loop under the reference's mask."""

import importlib.util
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, greedy_generate_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.constrained import TokenConstraint, TokenVocabulary, descriptor_values
from tiny_llm_b200.generate import parallel_sample_ids
from tiny_llm_b200.json_mode import ConstraintRows, JsonConstraint, JsonWalker
from tiny_llm_b200.sampler import penalty_tensors, sample_tokens, sampling_tensors, token_state_row
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load(name: str, file: str):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


jref = _load("tiny_llm_b200_json_ref", "json_ref.py")
host = _load("tiny_llm_b200_json_mode_host", "test_json_mode_host.py")

# prefixes that end in every kind of state: inside strings, escapes, \u, multi-byte characters, numbers and literals,
# at both caps, after the top-level close
TEXTS = [b"", b" " * 32, b"{", b'{"', b'{"k', b'{"k\\', b'{"k\\u0', b'{"k\\u00e', b'{"\xc3', b'{"\xe0', b'{"\xe0\xa0', b'{"\xf0\x9f',
         b'{"\xf0\x9f\x98', b'{"k"', b'{"k":', b'{"k": ', b'{"k":-', b'{"k":0', b'{"k":12', b'{"k":1.', b'{"k":1.5', b'{"k":1e',
         b'{"k":1e+', b'{"k":1E-7', b'{"k":t', b'{"k":fal', b'{"k":nul', b'{"k":true', b'{"k":[', b'{"k":[1,', b'{"k":[1 ',
         b'{"k":{', b'{"k":{}', b'{"k":"v"', b'{"k":"v",', b'{"k":' + b" " * 32, b'{"a":' + b"[" * 63, b'{"a":' + b"[" * 63 + b"0",
         b"{}", b"{} ", b"{}" + b"\n" * 32, b'{"k":"v"}']


def _walker(text: bytes) -> JsonWalker:
    w = JsonWalker()
    assert w.walk(text), text
    return w


def _table(c, walkers, vocab_size, dev):
    tab = ConstraintRows(len(walkers), vocab_size, dev, json=True)
    for r, w in enumerate(walkers):
        tab.set_row(r, c, w)
    return tab


@pytest.mark.parametrize("rows", [1, 8, 64])
def test_masks_equal_the_reference_on_an_adversarial_vocabulary(cuda_device, rows):
    vocab = host.adversarial_vocabulary()
    c = JsonConstraint(vocab, device=cuda_device)
    texts = [TEXTS[(r * 7) % len(TEXTS)] for r in range(rows)]
    walkers = [_walker(t) for t in texts]
    terminal = [r % 5 == 4 and jref.classify(t) == "complete" for r, t in enumerate(texts)]
    for w, term in zip(walkers, terminal):
        w.terminal = term
    tab = _table(c, walkers, vocab.size, cuda_device)
    tab.json_masks[:, 0].fill_(-1)  # terminal rows keep this
    tab.before_draw()
    got = tab.json_masks[:, 0].cpu().numpy()
    for r, t in enumerate(texts):
        want = np.full(got.shape[1], -1, dtype=np.int32) if terminal[r] else jref.pack(jref.allowed(t, vocab.tokens, vocab.eos_ids))
        assert np.array_equal(got[r], want), (r, t)
    assert np.array_equal(tab.json_masks[:, 1].cpu().numpy(), np.stack([c.eos_row.cpu().numpy()] * rows))


def test_masks_equal_the_reference_at_full_vocabulary(cuda_device):
    V = 151_936
    vocab = TokenVocabulary.synthetic(V)
    c = JsonConstraint(vocab, device=cuda_device)
    walkers = [_walker(t) for t in TEXTS]
    tab = _table(c, walkers, V, cuda_device)
    tab.before_draw()
    got = tab.json_masks[:, 0].cpu().numpy()
    rng = np.random.default_rng(0)
    for r, t in enumerate(TEXTS):
        want = jref.pack(c.allowed(walkers[r]))  # the host walker, which the host tests hold to the reference
        assert np.array_equal(got[r], want), t
        bits = np.unpackbits(got[r].view(np.uint8), bitorder="little")[:V].astype(bool)
        for i in rng.choice(V, 300, replace=False):  # and a sample of tokens straight against the reference
            tok = vocab.tokens[i]
            expect = (i in vocab.eos_ids and jref.classify(t) == "complete") if tok is None else jref.viable(t + tok)
            assert bits[i] == expect, (t, tok)


def test_advance_equals_the_host_walk_and_skips_position_zero(cuda_device):
    vocab = host.adversarial_vocabulary()
    c = JsonConstraint(vocab, device=cuda_device)
    rng = np.random.default_rng(1)
    walkers = [_walker(t) for t in TEXTS]
    tab = _table(c, walkers, vocab.size, cuda_device)
    tokens, positions = [], []
    for r, w in enumerate(walkers):
        allowed = np.flatnonzero(c.allowed(w))
        tokens.append(int(rng.choice(allowed)))
        positions.append(0 if r % 4 == 3 else 10 + r)
    before = tab.json_states.clone()
    tab.after_draw(torch.tensor(tokens, dtype=torch.int32, device=cuda_device), torch.tensor(positions, dtype=torch.int32, device=cuda_device))
    got = tab.json_states.cpu().tolist()
    for r, w in enumerate(walkers):
        if positions[r] == 0:
            assert got[r] == before[r].tolist()
        else:
            assert got[r] == list(c.walk([tokens[r]], w).words()), (TEXTS[r], vocab.tokens[tokens[r]])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_json_draw_equals_the_unconstrained_kernel_on_the_masked_row(cuda_device, dtype):
    V = 151_936
    vocab = TokenVocabulary.synthetic(V)
    c = JsonConstraint(vocab, device=cuda_device)
    rc = TokenConstraint.compile(r"[a-z ]+", vocab, device=cuda_device)
    g = torch.Generator(device="cpu").manual_seed(3)
    texts = [b"", b'{"k', b'{"k":', b'{"k":[1', b"{}", b'{"a":1,']
    rows = 2 * len(texts)
    x = (torch.randn(rows, V, generator=g) * 3).to(dtype).to(cuda_device)
    x[:, vocab.eos_ids[0]] = 6.0  # EOS likely, allowed only after the close
    kinds = ["json", "regex", "json", "plain", "json", "pen"] * 2
    params, walkers = [], []
    for r, k in enumerate(kinds):
        extra = dict(presence_penalty=0.5, repetition_penalty=1.3) if r % 3 == 2 or k == "pen" else {}
        cons = c if k == "json" else rc if k == "regex" else None
        params.append(SamplingParams((0.0, 0.8, 1.2)[r % 3], top_k=(None, 50)[r % 2], seed=9 + r, constraint=cons, **extra))
        walkers.append(_walker(texts[r % len(texts)]) if k == "json" else None)
    pos = [5 + r for r in range(rows)]
    state = torch.stack([token_state_row([1, 2, 3], [7, 7], V) for _ in range(rows)]).to(cuda_device)
    tab = ConstraintRows(rows, V, cuda_device, json=True)
    for r, p in enumerate(params):
        tab.set_row(r, p.constraint, walkers[r])
    st = state.clone()
    got = sample_tokens(x, params, pos, st, tab).cpu()
    # each JSON row alone equals the unconstrained kernel on its -inf-masked row
    masks = tab.json_masks[:, 0].cpu().numpy()
    for r, k in enumerate(kinds):
        if k != "json":
            continue
        allowed = np.unpackbits(masks[r].view(np.uint8), bitorder="little")[:V].astype(bool)
        assert np.array_equal(allowed, c.allowed(walkers[r]))
        row = x[r : r + 1].clone()
        row[0, torch.from_numpy(~allowed).to(cuda_device)] = float("-inf")
        t = sampling_tensors([params[r]], cuda_device)
        p_ = torch.tensor([pos[r]], dtype=torch.int32, device=cuda_device)
        s1 = state[r : r + 1].clone()
        want = ext.sample_penalized(row, *t, p_, *penalty_tensors([params[r]], cuda_device), s1) if params[r].penalized else ext.sample(row, *t, p_)
        assert int(got[r]) == int(want[0]), r
        assert allowed[int(got[r])]
    # the other rows draw and advance exactly as in the launch without JSON rows
    keep = [r for r, k in enumerate(kinds) if k != "json"]
    desc = torch.stack([torch.tensor(descriptor_values(params[r].constraint), dtype=torch.int64) for r in keep]).to(cuda_device)
    st2 = state[keep].clone()
    alone = sample_tokens(x[keep], [params[r] for r in keep], [pos[r] for r in keep], st2, desc).cpu()
    assert torch.equal(got[keep], alone)
    assert torch.equal(tab.descriptors[keep, 4].cpu(), desc[:, 4].cpu())
    assert torch.equal(st[keep], st2)


# -------------------------------------------------------------------------------------- end to end --
def _model(dev, seed=5):
    ns = synthetic_qwen3("tiny-d128", seed=seed, realistic=True, max_position_embeddings=8192, device=dev)
    return Qwen3ModelWeek3(ns, page_size=64)


def _check_output(vocab, ids, finished):
    text = b"".join(vocab.tokens[t] for t in ids)
    if finished:
        assert isinstance(json.loads(text.decode("utf-8", "strict")), dict) and jref.caps_hold(text), text
    else:
        assert jref.viable(text), text


def _host_loop(model, prompt, n, sampling, vocab, dev):
    """greedy_generate_ids under the reference's mask: the model's logits row, disallowed entries -inf, then the
    unconstrained kernel of the request's parameters."""
    cache = model.create_kv_cache()
    eos = vocab.eos_ids[0]
    out, text = [], b""
    state = token_state_row(prompt, [], model.vocab_size, device=dev)[None] if sampling.penalized else None
    plain = SamplingParams(sampling.temperature, top_k=sampling.top_k, top_p=sampling.top_p, seed=sampling.seed,
                           repetition_penalty=sampling.repetition_penalty, presence_penalty=sampling.presence_penalty,
                           frequency_penalty=sampling.frequency_penalty, min_p=sampling.min_p)
    try:
        tokens, offset = torch.tensor(prompt, dtype=torch.int32, device=dev), 0
        while len(out) < n:
            logits = model(tokens[None], offset, cache, logits_to_keep=1)[:, -1, :].clone()
            allowed = torch.from_numpy(jref.allowed(text, vocab.tokens, vocab.eos_ids)).to(dev)
            logits[0, ~allowed] = float("-inf")
            tok = int(sample_tokens(logits, [plain], [offset + tokens.numel()], state)[0])
            if tok == eos:
                break
            out.append(tok)
            text += vocab.tokens[tok]
            offset += tokens.numel()
            tokens = torch.tensor([tok], dtype=torch.int32, device=dev)
    finally:
        for cc in cache:
            cc.release()
    return out


N_NEW = 24
_RUNS: dict = {}


def _setup(dev):
    """The model, vocabulary, constraints, prompts and parameters of the end-to-end tests, with each request's
    greedy_generate_ids ids (checked against the host loop under the reference's mask once)."""
    if "model" not in _RUNS:
        model = _model(dev)
        vocab = TokenVocabulary.synthetic(model.vocab_size)
        c = JsonConstraint(vocab, device=dev)
        g = torch.Generator().manual_seed(0)
        prompts = [torch.randint(1, 500, (int(k),), generator=g).tolist() for k in (5, 17, 9, 30)]
        params = [SamplingParams(0.0, constraint=c), SamplingParams(0.9, top_k=40, seed=101, constraint=c),
                  SamplingParams(1.3, seed=102, presence_penalty=0.7, constraint=c), SamplingParams(0.0, repetition_penalty=1.4, constraint=c)]
        gen = [greedy_generate_ids(model, p, N_NEW, eos_token_id=vocab.eos_ids[0], device=dev, sampling=s) for p, s in zip(prompts, params)]
        _RUNS.update(model=model, vocab=vocab, c=c, prompts=prompts, params=params, gen=gen)
    return _RUNS


def test_generate_equals_the_host_loop_under_the_reference_mask(cuda_device):
    r = _setup(cuda_device)
    for i, (p, s) in enumerate(zip(r["prompts"], r["params"])):
        ids = r["gen"][i]
        _check_output(r["vocab"], ids, finished=len(ids) < N_NEW)
        assert ids == _host_loop(r["model"], p, N_NEW, s, r["vocab"], cuda_device), i
    ids, entries = greedy_generate_ids(r["model"], r["prompts"][1], N_NEW, eos_token_id=r["vocab"].eos_ids[0], device=cuda_device,
                                       sampling=r["params"][1], logprobs=2)
    assert ids == r["gen"][1] and [e.token for e in entries] == ids


def test_batcher_with_regex_and_plain_requests_mixed_in(cuda_device):
    r = _setup(cuda_device)
    model, vocab, prompts, params, gen = r["model"], r["vocab"], r["prompts"], r["params"], r["gen"]
    eos = vocab.eos_ids[0]
    rc = TokenConstraint.compile(r"[a-z ]{1,12}\.", vocab, device=cuda_device)
    # prefill_step 32 prefills every prompt in one chunk, as greedy_generate_ids does: a chunked prefill rounds the
    # logits differently, which moves greedy picks between near-equal continuation bytes
    for batch_size, order in ((3, [0, 1, 2, 3]), (2, [3, 2, 1, 0])):
        queue = [prompts[i] for i in order] + [[7, 8, 9], [4, 5]]
        samp = [params[i] for i in order] + [SamplingParams(0.8, seed=1, constraint=rc), SamplingParams(0.8, seed=1)]
        b = ContinuousBatcher(model, None, queue, max_seq_len=128, batch_size=batch_size, prefill_step=32, verbose=False, eos_token_id=eos,
                              device=cuda_device, max_new_tokens=[N_NEW] * len(queue), sampling=samp)
        res = dict(b.run())
        for j, i in enumerate(order):
            assert [int(t) for t in res[j].split()] == gen[i], (batch_size, i)
        regex_alone = greedy_generate_ids(model, [7, 8, 9], N_NEW, eos_token_id=eos, device=cuda_device, sampling=samp[-2])
        assert [int(t) for t in res[len(order)].split()] == regex_alone


def test_decode_on_device_from_history(cuda_device):
    r = _setup(cuda_device)
    model, eos = r["model"], r["vocab"].eos_ids[0]
    for i in range(4):
        p, s = r["prompts"][i], r["params"][i]
        cache = model.create_kv_cache()
        try:
            logits = model(torch.tensor([p], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
            tab = ConstraintRows.build([s], model.vocab_size, cuda_device)
            st = token_state_row(p, [], model.vocab_size, device=cuda_device)[None] if s.penalized else None
            first = int(sample_tokens(logits[:, -1, :], [s], [len(p)], st, tab)[0])
            engine = model.decode_engine(1, model._graph_limit(cache))
            log = engine.decode_on_device([first], [len(p)], cache, N_NEW - 1, sampling=s, history=[(p, [first])])
            want = [first] + log[:, 0].tolist()
            assert engine.kernels_per_json_step == engine.kernels_per_step - 1 + 2  # masks and advance instead of argmax
        finally:
            for cc in cache:
                cc.release()
        got = r["gen"][i]
        assert want[: len(got)] == got, i
        if len(got) < N_NEW:
            assert set(want[len(got):]) == {eos}


def test_parallel_samples_equal_their_generate_runs(cuda_device):
    from dataclasses import replace

    from tiny_llm_b200.generate import sample_seed

    r = _setup(cuda_device)
    model, eos, p, s = r["model"], r["vocab"].eos_ids[0], r["prompts"][1], r["params"][1]
    samples = parallel_sample_ids(model, [p], 3, s, N_NEW, eos_token_ids=(eos,), device=cuda_device)[0]
    for j, smp in enumerate(samples):
        want = greedy_generate_ids(model, p, N_NEW, eos_token_id=eos, device=cuda_device, sampling=replace(s, seed=sample_seed(s.seed, j)))
        assert smp.ids == want, j


def test_decode_engine_history_refuses_ids_outside_the_language(cuda_device):
    model = _model(cuda_device)
    vocab = TokenVocabulary.synthetic(model.vocab_size)
    c = JsonConstraint(vocab, device=cuda_device)
    cache = model.create_kv_cache()
    try:
        model(torch.tensor([[1, 2, 3]], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        engine = model.decode_engine(1, model._graph_limit(cache))
        with pytest.raises(ValueError, match="leave the constraint's language"):
            engine.decode_on_device([ord("x")], [3], cache, 2, sampling=SamplingParams(0.0, constraint=c), history=[([1, 2, 3], [ord("x")])])
        with pytest.raises(ValueError, match="keep_logits takes plain sampling"):
            engine.decode_on_device([ord("{")], [3], cache, 2, sampling=SamplingParams(0.5, constraint=c), keep_logits=True)
    finally:
        for cc in cache:
            cc.release()
