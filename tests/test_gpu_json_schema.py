"""JSON Schema structured outputs on the H100 (DESIGN.md section 21): ``tl_schema_token_masks`` bit for bit against the
host walker at V = 151,936 with regex, JSON, two schemas and plain rows in one launch, and against the independent
reference on an adversarial vocabulary; ``tl_schema_advance`` against the host walk; the schema masks under
``{"type": "object"}`` against JSON mode's; and the same schema requests through ``greedy_generate_ids``, the batcher,
``decode_on_device`` and ``parallel_sample_ids``, equal to a host loop under the reference's mask."""

import importlib.util
import json
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, greedy_generate_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.constrained import TokenConstraint, TokenVocabulary
from tiny_llm_b200.generate import parallel_sample_ids
from tiny_llm_b200.json_mode import ConstraintRows, JsonConstraint, JsonWalker
from tiny_llm_b200.json_schema import SCHEMA_MAX_DEPTH, SCHEMA_MAX_ITEMS, JsonSchemaConstraint
from tiny_llm_b200.sampler import sample_tokens, token_state_row
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load(name: str, file: str):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


sref = _load("tiny_llm_b200_json_schema_ref", "json_schema_ref.py")
shost = _load("tiny_llm_b200_json_schema_host", "test_json_schema_host.py")
jhost = _load("tiny_llm_b200_json_mode_host", "test_json_mode_host.py")

PERSON = {
    "type": "object",
    "properties": {
        "name": {"type": "string"},
        "age": {"type": "integer"},
        "email": {"type": "string", "pattern": "^[a-z]{1,12}@[a-z]{1,8}\\.com$"},
        "status": {"enum": ["active", "away", 7, 75, None]},
        "score": {"type": "number"},
        "nick": {"type": ["string", "null"]},
        "tags": {"type": "array", "items": {"type": "string"}, "maxItems": 4},
        "grid": {"type": "array", "items": {"type": "integer"}, "minItems": SCHEMA_MAX_ITEMS, "maxItems": SCHEMA_MAX_ITEMS},
        "address": {"type": "object", "properties": {"street": {"type": "string"}, "zip": {"type": "integer"}}, "required": ["street"]},
        "comments": {"type": "array", "items": {"$ref": "#/$defs/comment"}},
        "extra": {},
    },
    "required": ["name", "age"],
    "$defs": {"comment": {"type": "object", "properties": {"text": {"type": "string"}, "replies": {"type": "array", "items": {"$ref": "#/$defs/comment"}}},
                          "required": ["text"]}},
}
ANY = {"type": "object", "properties": {"x": {}}}
DEEP = b'{"x":' + b"[" * SCHEMA_MAX_DEPTH
# prefixes that end in every kind of state: before the object, keys, inside strings, escapes, \u, multi-byte characters,
# numbers, enum prefixes, patterns, the item cap, recursion, after the close
PERSON_TEXTS = [b"", b" " * 32, b"{", b'{"', b'{"na', b'{"name":"', b'{"name":"a\\', b'{"name":"a\\u00', b'{"name":"\xc3', b'{"name":"\xe0\xa0',
                b'{"name":"x",', b'{"name":"x","age":', b'{"name":"x","age":-', b'{"name":"x","age":12', b'{"name":"x","age":1,"status":"a',
                b'{"name":"x","age":1,"status":7', b'{"name":"x","age":1,"email":"ab@c', b'{"name":"x","age":1,"score":1.5e',
                b'{"name":"x","age":1,"nick":n', b'{"name":"x","age":1,"tags":["a","b","c","d"',
                b'{"name":"x","age":1,"grid":[' + b"0," * (SCHEMA_MAX_ITEMS - 1), b'{"name":"x","age":1,"grid":[' + b"0," * (SCHEMA_MAX_ITEMS - 1) + b"5",
                b'{"name":"x","age":1,"comments":[{"text":"a","replies":[{"text":"b","replies":[',
                b'{"name":"x","age":1,"extra":{"k":[1,{"z":', b'{"name":"x","age":1}', b'{"name":"x","age":1} ']
ANY_TEXTS = [b'{"x":', DEEP, b'{"x":' + b"[" * (SCHEMA_MAX_DEPTH - 1), b'{"x":' + b"[" * (SCHEMA_MAX_DEPTH - 1) + b"0", b'{"x":[{"a":tr', b'{"x":1}']


def _walker(c, text):
    w = c.start()
    assert w.walk(text), text
    return w


def _bits(row, V):
    return np.unpackbits(np.asarray(row).view(np.uint8), bitorder="little")[:V].astype(bool)


def test_masks_mixed_launch_at_full_vocabulary(cuda_device):
    V = 151_936
    vocab = TokenVocabulary.synthetic(V)
    person = JsonSchemaConstraint(PERSON, vocab, device=cuda_device)
    anyc = JsonSchemaConstraint(ANY, vocab, device=cuda_device)
    jc = JsonConstraint(vocab, device=cuda_device)
    rc = TokenConstraint.compile(r"[a-z ]+", vocab, device=cuda_device)
    cases = [(person, t) for t in PERSON_TEXTS] + [(anyc, t) for t in ANY_TEXTS] + [(jc, b'{"k":'), (jc, b'{"k":"a'), (rc, None), (None, None)]
    want: dict = {}
    for rows in (1, 7, 64):
        picks = [cases[(r * 5 + rows) % len(cases)] for r in range(rows)]
        tab = ConstraintRows(rows, V, cuda_device, json=True, schema=True)
        walkers = []
        for r, (c, t) in enumerate(picks):
            w = None if c is None or c is rc else _walker(c, t) if isinstance(c, JsonSchemaConstraint) else JsonWalker()
            if c is jc:
                assert w.walk(t)
            if isinstance(c, JsonSchemaConstraint) and r % 9 == 8 and w.complete:
                w.terminal = True
            walkers.append(w)
            tab.set_row(r, c, w)
        desc = tab.descriptors.clone()
        tab.json_masks[:, 0].fill_(-1)  # rows that are not written keep this
        tab.before_draw()
        got = tab.json_masks[:, 0].cpu().numpy()
        for r, ((c, t), w) in enumerate(zip(picks, walkers)):
            if c is None or c is rc or w.terminal:
                assert (got[r] == -1).all(), r
                continue
            key = (id(c), t)
            if key not in want:
                want[key] = c.allowed(w)
            assert np.array_equal(_bits(got[r], V), want[key]), (rows, r, t)
        assert torch.equal(tab.descriptors, desc)
    # a sample of tokens straight against the reference
    rng = np.random.default_rng(0)
    for t in PERSON_TEXTS[::5]:
        allowed = want[(id(person), t)]
        complete = sref.check(PERSON, t)[1]
        for i in rng.choice(V, 200, replace=False):
            tok = vocab.tokens[i]
            expect = (i in vocab.eos_ids and complete) if tok is None else sref.check(PERSON, t + tok)[0]
            assert allowed[i] == expect, (t, tok)


@pytest.mark.parametrize("rows", [1, 8, 64])
def test_masks_equal_the_reference_on_an_adversarial_vocabulary(cuda_device, rows):
    vocab = jhost.adversarial_vocabulary()
    cons = {"person": JsonSchemaConstraint(PERSON, vocab, device=cuda_device), "any": JsonSchemaConstraint(ANY, vocab, device=cuda_device)}
    schemas = {"person": PERSON, "any": ANY}
    cases = [("person", t) for t in PERSON_TEXTS] + [("any", t) for t in ANY_TEXTS]
    picks = [cases[(r * 3) % len(cases)] for r in range(rows)]
    tab = ConstraintRows(rows, vocab.size, cuda_device, json=False, schema=True)
    for r, (k, t) in enumerate(picks):
        tab.set_row(r, cons[k], _walker(cons[k], t))
    tab.before_draw()
    got = tab.json_masks[:, 0].cpu().numpy()
    eos = set(vocab.eos_ids)
    want: dict = {}
    for r, (k, t) in enumerate(picks):
        if (k, t) not in want:
            complete = sref.check(schemas[k], t)[1]
            want[(k, t)] = np.array([(i in eos and complete) if tok is None else sref.check(schemas[k], t + tok)[0]
                                     for i, tok in enumerate(vocab.tokens)])
        assert np.array_equal(_bits(got[r], vocab.size), want[(k, t)]), (k, t)


def test_advance_equals_the_host_walk_and_skips_position_zero(cuda_device):
    vocab = jhost.adversarial_vocabulary()
    person = JsonSchemaConstraint(PERSON, vocab, device=cuda_device)
    anyc = JsonSchemaConstraint(ANY, vocab, device=cuda_device)
    cases = [(person, t) for t in PERSON_TEXTS] + [(anyc, t) for t in ANY_TEXTS]
    rng = np.random.default_rng(1)
    tab = ConstraintRows(len(cases), vocab.size, cuda_device, json=False, schema=True)
    walkers, tokens, positions = [], [], []
    for r, (c, t) in enumerate(cases):
        w = _walker(c, t)
        walkers.append(w)
        tab.set_row(r, c, w)
        tokens.append(int(rng.choice(np.flatnonzero(c.allowed(w)))))
        positions.append(0 if r % 4 == 3 else 10 + r)
    before = tab.schema_states.clone()
    tab.after_draw(torch.tensor(tokens, dtype=torch.int32, device=cuda_device), torch.tensor(positions, dtype=torch.int32, device=cuda_device))
    got = tab.schema_states.cpu().tolist()
    for r, ((c, t), w) in enumerate(zip(cases, walkers)):
        if positions[r] == 0:
            assert got[r] == before[r].tolist()
        else:
            assert got[r] == list(c.words(c.walk([tokens[r]], w))), (t, vocab.tokens[tokens[r]])


def test_any_object_schema_masks_equal_json_mode(cuda_device):
    vocab = jhost.adversarial_vocabulary()
    sc = JsonSchemaConstraint({"type": "object"}, vocab, device=cuda_device)
    jc = JsonConstraint(vocab, device=cuda_device)
    push = max(t.count(b"[") + t.count(b"{") for t in vocab.tokens if t is not None)
    rng = np.random.default_rng(2)
    compared = 0
    for walk in range(6):
        text, jw, sw = b"", JsonWalker(), sc.start()
        for _ in range(60):
            if jw.depth + push < SCHEMA_MAX_DEPTH:  # below the schema's depth cap for every token
                tab = ConstraintRows(2, vocab.size, cuda_device, json=True, schema=True)
                tab.set_row(0, jc, jw)
                tab.set_row(1, sc, sw)
                tab.before_draw()
                m = tab.json_masks[:, 0].cpu().numpy()
                assert np.array_equal(m[0], m[1]), text
                compared += 1
            allowed = np.flatnonzero(jc.allowed(jw) & sc.allowed(sw))
            t = int(rng.choice(allowed))
            if t in vocab.eos_ids:
                break
            assert jw.walk(vocab.tokens[t]) and sw.walk(vocab.tokens[t])
            text += vocab.tokens[t]
    assert compared > 100


# -------------------------------------------------------------------------------------- end to end --
SMALL = {"type": "object", "properties": {"id": {"type": "integer"}, "tag": {"enum": ["a", "bb", 3]}, "kids": {"type": "array", "maxItems": 2,
                                                                                                             "items": {"$ref": "#"}}},
         "required": ["id"]}


def _model(dev, seed=5):
    ns = synthetic_qwen3("tiny-d128", seed=seed, realistic=True, max_position_embeddings=8192, device=dev)
    return Qwen3ModelWeek3(ns, page_size=64)


def _check_output(vocab, ids, finished):
    text = b"".join(vocab.tokens[t] for t in ids)
    if finished:
        v = shost._parse(text)
        assert v is not None and shost._valid(v, SMALL, SMALL), text
    else:
        assert sref.check(SMALL, text)[0], text


def _ref_mask(text, vocab):
    complete = sref.check(SMALL, text)[1]
    eos = set(vocab.eos_ids)
    return np.array([(i in eos and complete) if t is None else sref.check(SMALL, text + t)[0] for i, t in enumerate(vocab.tokens)])


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
            allowed = torch.from_numpy(_ref_mask(text, vocab)).to(dev)
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
    if "model" not in _RUNS:
        model = _model(dev)
        vocab = TokenVocabulary.synthetic(model.vocab_size)
        c = JsonSchemaConstraint(SMALL, vocab, device=dev)
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


def test_batcher_with_json_regex_and_plain_requests_mixed_in(cuda_device):
    r = _setup(cuda_device)
    model, vocab, prompts, params, gen = r["model"], r["vocab"], r["prompts"], r["params"], r["gen"]
    eos = vocab.eos_ids[0]
    rc = TokenConstraint.compile(r"[a-z ]{1,12}\.", vocab, device=cuda_device)
    jc = JsonConstraint(vocab, device=cuda_device)
    for batch_size, order in ((3, [0, 1, 2, 3]), (2, [3, 2, 1, 0])):
        queue = [prompts[i] for i in order] + [[7, 8, 9], [4, 5], [6, 6]]
        samp = [params[i] for i in order] + [SamplingParams(0.8, seed=1, constraint=rc), SamplingParams(0.8, seed=1),
                                             SamplingParams(0.0, constraint=jc)]
        b = ContinuousBatcher(model, None, queue, max_seq_len=128, batch_size=batch_size, prefill_step=32, verbose=False, eos_token_id=eos,
                              device=cuda_device, max_new_tokens=[N_NEW] * len(queue), sampling=samp)
        res = dict(b.run())
        for j, i in enumerate(order):
            assert [int(t) for t in res[j].split()] == gen[i], (batch_size, i)
        for k, prompt in ((len(order), [7, 8, 9]), (len(order) + 2, [6, 6])):
            alone = greedy_generate_ids(model, prompt, N_NEW, eos_token_id=eos, device=cuda_device, sampling=samp[k])
            assert [int(t) for t in res[k].split()] == alone


def test_decode_on_device_from_history_and_launch_counts(cuda_device):
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
            assert engine.kernels_per_schema_step == engine.kernels_per_step - 1 + 2  # masks and advance instead of argmax
        finally:
            for cc in cache:
                cc.release()
        got = r["gen"][i]
        assert want[: len(got)] == got, i
        if len(got) < N_NEW:
            assert set(want[len(got):]) == {eos}


def test_existing_graph_kinds_keep_their_launch_counts(cuda_device):
    r = _setup(cuda_device)
    model, vocab = r["model"], r["vocab"]
    rc = TokenConstraint.compile(r"[a-z ]+", vocab, device=cuda_device)
    jc = JsonConstraint(vocab, device=cuda_device)
    cache = model.create_kv_cache()
    try:
        model(torch.tensor([[1, 2, 3]], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        engine = model.decode_engine(1, model._graph_limit(cache))
        engine.decode_on_device([ord("a")], [3], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=rc))
        engine.decode_on_device([ord("{")], [5], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=jc))
        counts = (engine.kernels_per_constrained_step, engine.kernels_per_json_step)
        engine.decode_on_device([ord("{")], [7], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=r["c"]))
        assert (engine.kernels_per_constrained_step, engine.kernels_per_json_step) == counts
        assert counts[1] == counts[0] + 2 == engine.kernels_per_step + 1  # the draw, then masks and advance around it
        assert engine.kernels_per_schema_step == engine.kernels_per_json_step
    finally:
        for cc in cache:
            cc.release()


def test_parallel_samples_equal_their_generate_runs(cuda_device):
    from dataclasses import replace

    from tiny_llm_b200.generate import sample_seed

    r = _setup(cuda_device)
    model, eos, p, s = r["model"], r["vocab"].eos_ids[0], r["prompts"][1], r["params"][1]
    samples = parallel_sample_ids(model, [p], 3, s, N_NEW, eos_token_ids=(eos,), device=cuda_device)[0]
    for j, smp in enumerate(samples):
        want = greedy_generate_ids(model, p, N_NEW, eos_token_id=eos, device=cuda_device, sampling=replace(s, seed=sample_seed(s.seed, j)))
        assert smp.ids == want, j
        _check_output(r["vocab"], smp.ids, finished=len(smp.ids) < N_NEW)


def test_finished_texts_validate_with_jsonschema(cuda_device):
    jsonschema = pytest.importorskip("jsonschema")
    r = _setup(cuda_device)
    for ids in r["gen"]:
        if len(ids) < N_NEW:
            jsonschema.validate(json.loads(b"".join(r["vocab"].tokens[t] for t in ids)), SMALL)
