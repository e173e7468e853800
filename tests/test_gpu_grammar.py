"""Grammar-constrained generation on the H100 (DESIGN.md section 23): ``tl_grammar_token_masks`` bit for bit against
the host walker at V = 151,936 with grammar (one blob staged in shared memory, one read through L1), schema, JSON,
regex and plain rows in one launch, at the depth and parse caps; ``tl_grammar_advance`` against the host walk; a
grammar past the parse cap; and grammar requests through ``greedy_generate_ids``, the batcher, ``decode_on_device`` and
``parallel_sample_ids``, equal to a host loop under the Earley reference's mask."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, greedy_generate_ids
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.constrained import TokenConstraint, TokenVocabulary
from tiny_llm_b200.generate import parallel_sample_ids
from tiny_llm_b200.grammar import GRAMMAR_MAX_DEPTH, GRAMMAR_MAX_PARSES, GRAMMAR_SMEM_BYTES, GrammarConstraint, GrammarWalker
from tiny_llm_b200.json_mode import ConstraintRows, JsonConstraint, JsonWalker
from tiny_llm_b200.json_schema import JsonSchemaConstraint
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


gref = _load("tiny_llm_b200_grammar_ref", "grammar_ref.py")
ghost = _load("tiny_llm_b200_grammar_host", "test_grammar_host.py")

EXPR, NESTING = ghost.EXPR, ghost.NESTING
_WORDS = [a + b for a in ("al", "be", "ga", "de", "ep", "ze", "th", "io", "ka", "la", "mu", "nu", "xi", "pi", "rh", "si")
          for b in ("pha", "ta", "mma", "lta", "silon", "na", "ron", "ga", "vo", "que")]
BIG = ('root ::= list\nlist ::= "[" ws item (ws "," ws item)* ws "]"\nitem ::= word | list | num\nws ::= [ \\t\\n]{0,3}\n'
       'num ::= "-"? [0-9]{1,8} ("." [0-9]{1,6})?\nword ::= "\\"" (' + " | ".join(f'"{w}"' for w in _WORDS) + ') "\\""')
EIGHT = ('root ::= "ab" tail\ntail ::= ' + " | ".join(f"r{k}" for k in range(1, 9)) + "\n"
         + "\n".join(f'r{k} ::= "x" r{k} "{k}" | "z"' for k in range(1, 9)))
CAP = ('root ::= "ab" tail\ntail ::= ' + " | ".join(f"r{k}" for k in range(1, 10)) + "\n"
       + "\n".join(f'r{k} ::= "x" r{k} "{k}" | "z"' for k in range(1, 10)))


def _bits(row, V):
    return np.unpackbits(np.asarray(row).view(np.uint8), bitorder="little")[:V].astype(bool)


def _walker(c, text):
    w = c.start()
    assert w.walk(text), text
    return w


def test_masks_mixed_launch_at_full_vocabulary(cuda_device):
    V = 151_936
    vocab = TokenVocabulary.synthetic(V)
    expr = GrammarConstraint(EXPR, vocab, device=cuda_device)
    big = GrammarConstraint(BIG, vocab, device=cuda_device)
    nest = GrammarConstraint(NESTING, vocab, device=cuda_device)
    eight = GrammarConstraint(EIGHT, vocab, device=cuda_device)
    assert expr.compiled.blob.size <= GRAMMAR_SMEM_BYTES < big.compiled.blob.size  # one staged, one read through L1
    sc = JsonSchemaConstraint({"type": "object", "properties": {"k": {"type": "integer"}}}, vocab, device=cuda_device)
    jc = JsonConstraint(vocab, device=cuda_device)
    rc = TokenConstraint.compile(r"[a-z ]+", vocab, device=cuda_device)
    cases = ([(expr, t) for t in (b"", b"(", b"((1+", b"12", b"(1)+(2")]
             + [(big, t) for t in (b"", b"[", b'["al', b"[1.5, [", b'[["gamma"],\t-')]
             + [(nest, b"(" * (GRAMMAR_MAX_DEPTH - 1)), (nest, b"([" * 15), (nest, b"(" * (GRAMMAR_MAX_DEPTH - 1) + b"x))")]
             + [(eight, b"abxx"), (eight, b"abxxz"), (eight, b"ab")]
             + [(sc, b'{"k":'), (jc, b'{"k":"a'), (rc, None), (None, None)])
    want: dict = {}
    seen_parses = 0
    for rows in (1, 9, 64):
        picks = [cases[(r * 7 + rows) % len(cases)] for r in range(rows)]
        tab = ConstraintRows(rows, V, cuda_device, json=True, schema=True, grammar=True)
        walkers = []
        for r, (c, t) in enumerate(picks):
            w = None
            if isinstance(c, (GrammarConstraint, JsonSchemaConstraint)):
                w = _walker(c, t)
                if isinstance(c, GrammarConstraint):
                    seen_parses = max(seen_parses, len(w.parses))
                if r % 11 == 10 and w.complete:
                    w.terminal = True
            elif c is jc:
                w = JsonWalker()
                assert w.walk(t)
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
    assert seen_parses == GRAMMAR_MAX_PARSES
    # the walker's masks straight against the reference, on a sample of tokens
    rng = np.random.default_rng(0)
    for c, text, g in ((expr, b"((1+", EXPR), (big, b'["al', BIG), (eight, b"abxx", EIGHT)):
        ref = gref.Earley(g)
        allowed = want[(id(c), text)]
        complete = ref.check(text)[1]
        for i in rng.choice(V, 150, replace=False):
            tok = vocab.tokens[i]
            expect = (i in vocab.eos_ids and complete) if tok is None else ref.check(text + tok)[0]
            assert allowed[i] == expect, (text, tok)


def test_advance_equals_the_host_walk(cuda_device):
    vocab = TokenVocabulary.synthetic(3000)
    cons = {g: GrammarConstraint(g, vocab, device=cuda_device) for g in (EXPR, BIG, NESTING, EIGHT)}
    cases = [(EXPR, b""), (EXPR, b"(1+"), (EXPR, b"12"), (BIG, b"[1"), (BIG, b'["de'), (NESTING, b"(" * (GRAMMAR_MAX_DEPTH - 2)),
             (NESTING, b"([x"), (EIGHT, b"abx"), (EIGHT, b"abxx"), (EXPR, b"(1)")]
    rng = np.random.default_rng(1)
    eos = vocab.eos_ids[0]
    tab = ConstraintRows(len(cases), vocab.size, cuda_device, json=False, grammar=True)
    walkers, tokens, positions = [], [], []
    for r, (g, t) in enumerate(cases):
        c = cons[g]
        w = _walker(c, t)
        walkers.append(w)
        tab.set_row(r, c, w)
        allowed = np.flatnonzero(c.allowed(w))
        tokens.append(eos if r == len(cases) - 1 else int(rng.choice(allowed[allowed != eos])))
        positions.append(0 if r % 4 == 3 else 10 + r)
    before = tab.grammar_states.clone()
    tab.after_draw(torch.tensor(tokens, dtype=torch.int32, device=cuda_device), torch.tensor(positions, dtype=torch.int32, device=cuda_device))
    got = tab.grammar_states.cpu().tolist()
    for r, ((g, t), w) in enumerate(zip(cases, walkers)):
        if positions[r] == 0:
            assert got[r] == before[r].tolist()
        else:
            c = cons[g]
            after = c.walk([tokens[r]], w)
            assert got[r] == list(c.words(after)), (t, vocab.tokens[tokens[r]])
    assert GrammarWalker(cons[EXPR].compiled, got[-1]).terminal


def test_a_grammar_past_the_parse_cap_allows_only_reference_tokens_and_raises(cuda_device):
    vocab = TokenVocabulary.synthetic(512)
    c = GrammarConstraint(CAP, vocab, device=cuda_device)
    ref = gref.Earley(CAP)
    tab = ConstraintRows(2, vocab.size, cuda_device, json=False, grammar=True)
    tab.set_row(0, c)
    tab.set_row(1, c, _walker(c, b"ab"))
    tab.before_draw()
    got = tab.json_masks[:, 0].cpu().numpy()
    start = _bits(got[0], vocab.size)
    assert start.any()
    for i in np.flatnonzero(start):
        assert ref.check(vocab.tokens[i])[0]
    assert not _bits(got[1], vocab.size).any()  # every continuation keeps nine parses
    assert ref.check(b"abx")[0] and ref.check(b"abz")[1]
    tokens = torch.tensor([ord("a"), 0], dtype=torch.int32, device=cuda_device)  # row 1: the draw's fallback, lowest id
    with pytest.raises(ValueError, match=f"GRAMMAR_MAX_PARSES = {GRAMMAR_MAX_PARSES}"):
        tab.after_draw(tokens, torch.tensor([1, 1], dtype=torch.int32, device=cuda_device))
    assert tab.walkers()[1].failed and not tab.walkers()[0].failed
    model = _model(cuda_device)
    ids = [vocab.tokens.index(b"a"), vocab.tokens.index(b"b")]
    with pytest.raises(ValueError, match="GRAMMAR_MAX_PARSES"):
        greedy_generate_ids(model, [5, 17, 3], 8, eos_token_id=vocab.eos_ids[0], device=cuda_device,
                            sampling=SamplingParams(0.0, constraint=c))
    cache = model.create_kv_cache()
    try:
        p = [5, 17, 3]
        model(torch.tensor([p + ids[:1]], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        engine = model.decode_engine(1, model._graph_limit(cache))
        with pytest.raises(ValueError, match="GRAMMAR_MAX_PARSES"):
            engine.decode_on_device([ids[1]], [len(p) + 1], cache, 3, sampling=SamplingParams(0.0, constraint=c), history=[(p, ids)])
    finally:
        for cc in cache:
            cc.release()


# -------------------------------------------------------------------------------------- end to end --
SMALL = '''root ::= expr
expr ::= term | term ws "+" ws expr
term ::= [0-9]{1,3} | "(" expr ")"
ws   ::= " "?'''


def _model(dev, seed=5):
    ns = synthetic_qwen3("tiny-d128", seed=seed, realistic=True, max_position_embeddings=8192, device=dev)
    return Qwen3ModelWeek3(ns, page_size=64)


def _ref_mask(ref, text, vocab):
    """The reference's allowed tokens after ``text``: each token's bytes fed to the Earley sets, sharing prefixes."""
    sets = ref.initial()
    for b in text:
        sets = ref.feed(sets, b)
    out = np.zeros(vocab.size, dtype=bool)
    out[vocab.eos_ids] = ref.complete(sets)
    order = sorted((t, i) for i, t in enumerate(vocab.tokens) if t is not None)
    prev, stack = b"", [sets]
    for tok, i in order:
        lcp = 0
        while lcp < min(len(tok), len(prev)) and tok[lcp] == prev[lcp]:
            lcp += 1
        del stack[lcp + 1 :]
        for j in range(lcp, len(tok)):
            s = stack[j]
            stack.append(s if not s[-1] else ref.feed(s, tok[j]))
        prev = tok
        out[i] = bool(stack[len(tok)][-1])
    return out


def _check_output(vocab, ids, finished):
    text = b"".join(vocab.tokens[t] for t in ids)
    viable, complete = gref.Earley(SMALL).check(text)
    assert viable and (complete or not finished), text


def _host_loop(model, prompt, n, sampling, vocab, dev):
    """greedy_generate_ids under the reference's mask: the model's logits row, disallowed entries -inf, then the
    unconstrained kernel of the request's parameters."""
    cache = model.create_kv_cache()
    eos = vocab.eos_ids[0]
    ref = gref.Earley(SMALL)
    out, text = [], b""
    state = token_state_row(prompt, [], model.vocab_size, device=dev)[None] if sampling.penalized else None
    plain = SamplingParams(sampling.temperature, top_k=sampling.top_k, top_p=sampling.top_p, seed=sampling.seed,
                           repetition_penalty=sampling.repetition_penalty, presence_penalty=sampling.presence_penalty,
                           frequency_penalty=sampling.frequency_penalty, min_p=sampling.min_p)
    try:
        tokens, offset = torch.tensor(prompt, dtype=torch.int32, device=dev), 0
        while len(out) < n:
            logits = model(tokens[None], offset, cache, logits_to_keep=1)[:, -1, :].clone()
            allowed = torch.from_numpy(_ref_mask(ref, text, vocab)).to(dev)
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
        c = GrammarConstraint(SMALL, vocab, device=dev)
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


def test_batcher_with_schema_json_regex_and_plain_requests_mixed_in(cuda_device):
    r = _setup(cuda_device)
    model, vocab, prompts, params, gen = r["model"], r["vocab"], r["prompts"], r["params"], r["gen"]
    eos = vocab.eos_ids[0]
    rc = TokenConstraint.compile(r"[a-z ]{1,12}\.", vocab, device=cuda_device)
    jc = JsonConstraint(vocab, device=cuda_device)
    sc = JsonSchemaConstraint({"type": "object", "properties": {"k": {"type": "integer"}}}, vocab, device=cuda_device)
    for batch_size, order in ((3, [0, 1, 2, 3]), (2, [3, 2, 1, 0])):
        queue = [prompts[i] for i in order] + [[7, 8, 9], [4, 5], [6, 6], [3, 1]]
        samp = [params[i] for i in order] + [SamplingParams(0.8, seed=1, constraint=rc), SamplingParams(0.8, seed=1),
                                             SamplingParams(0.0, constraint=jc), SamplingParams(0.7, seed=4, constraint=sc)]
        b = ContinuousBatcher(model, None, queue, max_seq_len=128, batch_size=batch_size, prefill_step=32, verbose=False, eos_token_id=eos,
                              device=cuda_device, max_new_tokens=[N_NEW] * len(queue), sampling=samp)
        res = dict(b.run())
        for j, i in enumerate(order):
            assert [int(t) for t in res[j].split()] == gen[i], (batch_size, i)
        for k, prompt in ((len(order), [7, 8, 9]), (len(order) + 2, [6, 6]), (len(order) + 3, [3, 1])):
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
            assert engine.kernels_per_grammar_step == engine.kernels_per_step - 1 + 2  # masks and advance instead of argmax
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
    sc = JsonSchemaConstraint({"type": "object"}, vocab, device=cuda_device)
    cache = model.create_kv_cache()
    try:
        model(torch.tensor([[1, 2, 3]], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        engine = model.decode_engine(1, model._graph_limit(cache))
        engine.decode_on_device([ord("a")], [3], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=rc))
        engine.decode_on_device([ord("{")], [5], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=jc))
        engine.decode_on_device([ord("{")], [7], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=sc))
        counts = (engine.kernels_per_step, engine.kernels_per_constrained_step, engine.kernels_per_json_step, engine.kernels_per_schema_step)
        engine.decode_on_device([ord("1")], [9], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=r["c"]))
        assert (engine.kernels_per_step, engine.kernels_per_constrained_step, engine.kernels_per_json_step,
                engine.kernels_per_schema_step) == counts
        assert counts[1] + 2 == counts[2] == counts[3] == counts[0] + 1
        assert engine.kernels_per_grammar_step == counts[3]
        engine.decode_on_device([ord("a")], [11], cache, 2, sampling=SamplingParams(0.5, seed=1, constraint=rc))
        assert engine.kernels_per_constrained_step == counts[1]
    finally:
        for cc in cache:
            cc.release()


def test_decode_on_device_runs_schema_and_json_slots_beside_grammar_slots(cuda_device):
    r = _setup(cuda_device)
    model, vocab = r["model"], r["vocab"]
    eos = vocab.eos_ids[0]
    jc = JsonConstraint(vocab, device=cuda_device)
    sc = JsonSchemaConstraint({"type": "object", "properties": {"k": {"type": "integer"}}}, vocab, device=cuda_device)
    slots = [(r["prompts"][0], r["params"][0]), ([6, 6], SamplingParams(0.0, constraint=jc)), ([3, 1], SamplingParams(0.7, seed=4, constraint=sc)),
             (r["prompts"][1], r["params"][1])]
    want = [greedy_generate_ids(model, p, N_NEW, eos_token_id=eos, device=cuda_device, sampling=s) for p, s in slots]
    B, msl = len(slots), 256
    caches, firsts = [], []
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    try:
        for b, (p, s) in enumerate(slots):
            cache = model.create_kv_cache()
            caches.append(cache)
            logits = model(torch.tensor([p], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
            st = token_state_row(p, [], model.vocab_size, device=cuda_device)[None] if s.penalized else None
            firsts.append(int(sample_tokens(logits[:, -1, :], [s], [len(p)], st, ConstraintRows.build([s], model.vocab_size, cuda_device))[0]))
            for c, t in zip(cache, tables):
                t.add_request(c, b)
        engine = model.decode_engine(B, msl)
        log = engine.decode_on_device(firsts, [len(p) for p, _ in slots], tables, N_NEW - 1, sampling=[s for _, s in slots],
                                      history=[(p, [f]) for (p, _), f in zip(slots, firsts)])
        assert engine.kernels_per_grammar_step == engine.kernels_per_step - 1 + 6  # three masks launches and three advances
        for b, w in enumerate(want):
            got = [firsts[b]] + log[:, b].tolist()
            assert got[: len(w)] == w, b
    finally:
        for cache in caches:
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


def test_other_paths_refuse_grammar_rows(cuda_device):
    r = _setup(cuda_device)
    model, s = r["model"], SamplingParams(0.7, seed=1, constraint=r["c"])
    cache = model.create_kv_cache()
    try:
        model(torch.tensor([[1, 2, 3]], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)
        engine = model.decode_engine(1, model._graph_limit(cache))
        with pytest.raises(ValueError, match="keep_logits takes plain sampling: no grammar constraint"):
            engine.decode_on_device([4], [3], cache, 2, sampling=s, keep_logits=True)
    finally:
        for cc in cache:
            cc.release()
    with pytest.raises(ValueError, match="the sampled verify pass takes no grammar constraint"):
        model.verify_engine(3).verify(4, [5, 6], 3, None, sampling=s, draft_logits=torch.zeros(2, model.vocab_size, device=cuda_device))
