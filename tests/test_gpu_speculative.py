"""Speculative decoding on the GPU: the R-row fused decode attention against R single-row launches, the verify graph
against T successive decode steps, and ``speculative_generate_ids`` against ``greedy_generate_ids``, all bit for bit."""

import copy
import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3, greedy_generate_ids, speculative_generate_ids
from tiny_llm_b200.synthetic import synthetic_qwen3

from tiny_llm_b200.paged_kv_cache import TinyKvPagedCache


def _load(name, file):
    """A helper next to this file, by path: `tests` is no package of this project."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


ar = _load("tiny_llm_b200_attention_ref", "attention_ref.py")

pytestmark = pytest.mark.gpu
BF16 = torch.bfloat16


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


# ------------------------------------------------------------------ kernel: R rows per request --
def _attention_case(dev, G, R, ctx0, max_context, idle, seed, Hkv=2, page=16):
    """Two requests (the first idle when ``idle``) of R rows; row j of a live request at position ctx0 + j."""
    D, Hq, B = 128, G * Hkv, 2
    g = torch.Generator(device=dev).manual_seed(seed)
    mp = (max_context + page - 1) // page
    P = B * mp + 3
    kp = torch.randn(P, Hkv, page, D, device=dev, generator=g).to(BF16)
    vp = torch.randn(P, Hkv, page, D, device=dev, generator=g).to(BF16)
    perm = torch.randperm(P, device=dev, generator=g)[: B * mp].to(torch.int32)
    table = perm.view(B, mp).contiguous()
    qkv = (torch.randn(B * R, (Hq + 2 * Hkv) * D, device=dev, generator=g) * 2).to(BF16)
    qn = (1 + 0.3 * torch.randn(D, device=dev, generator=g)).to(BF16)
    kn = (1 + 0.3 * torch.randn(D, device=dev, generator=g)).to(BF16)
    pos = torch.tensor([[0 if (idle and b == 0) else ctx0 + j for j in range(R)] for b in range(B)], dtype=torch.int32, device=dev)
    ctx = pos + 1
    if idle:
        ctx[0] = 0
    return dict(qkv=qkv, qn=qn, kn=kn, pos=pos, ctx=ctx, table=table, kp=kp, vp=vp, Hq=Hq, Hkv=Hkv, B=B, max_context=max_context)


def _run(c, qkv, pos, ctx, table, kp, vp, R):
    freq = ext.rope_inv_freq_table(128, 1e6, qkv.device)
    return ext.decode_attention_fused(qkv, c["qn"], c["kn"], pos.reshape(-1).contiguous(), table, ctx.reshape(-1).contiguous(), freq, kp, vp,
                                      c["Hq"], c["Hkv"], 1e-6, 128 ** -0.5, c["max_context"], rows_per_request=R)


CASES = {  # name: (ctx0, max_context)
    "round": (37, 200),
    "page": (12, 200),           # rows cross the 16-token page at 16
    "256-round": (251, 600),     # rows cross the 256-token staging round
    "split": (1021, 8192),       # nsplit > 1; rows cross the split boundary at 1024 (and a round and a page)
}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("R", [1, 2, 3, 4, 5, 6, 7, 8])
def test_r_rows_equal_r_single_row_launches(dev, case, G, R):
    ctx0, max_context = CASES[case]
    for idle in (False, True):
        c = _attention_case(dev, G, R, ctx0, max_context, idle, seed=G * 100 + R + (7 if idle else 0))
        kp_seq, vp_seq = c["kp"].clone(), c["vp"].clone()
        rows = []
        for j in range(R):
            qkv_j = c["qkv"].view(c["B"], R, -1)[:, j].contiguous()
            rows.append(_run(c, qkv_j, c["pos"][:, j], c["ctx"][:, j], c["table"], kp_seq, vp_seq, 1))
        want = torch.stack(rows, 1).reshape(c["B"] * R, -1)
        kp, vp = c["kp"].clone(), c["vp"].clone()
        before = ext.launch_count()
        got = _run(c, c["qkv"], c["pos"], c["ctx"], c["table"], kp, vp, R)
        launches = ext.launch_count() - before
        torch.cuda.synchronize()
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), f"{case} G={G} R={R} idle={idle}: outputs differ"
        assert torch.equal(kp.view(torch.int16), kp_seq.view(torch.int16)) and torch.equal(vp.view(torch.int16), vp_seq.view(torch.int16))
        assert launches == (2 if max_context > 512 else 1)  # splits of >= 512 tokens: a merge launch beyond one
        if idle:
            assert not got[:R].float().abs().any(), "an idle request sees no keys"


def test_r_rows_see_exactly_their_causal_prefix(dev):
    """Needles: V rows are one-hot at the new tokens' positions, so row j's output is nonzero in the columns of rows
    <= j only."""
    G, R, ctx0 = 2, 6, 40
    c = _attention_case(dev, G, R, ctx0, 200, False, seed=3)
    D, Hq, Hkv = 128, c["Hq"], c["Hkv"]
    qkv = c["qkv"].clone().view(c["B"] * R, Hq + 2 * Hkv, D)
    qkv[:, Hq:Hq + Hkv] = 0                         # equal keys: every visible row weighs the same
    qkv[:, Hq + Hkv:] = 0
    for j in range(R):
        qkv.view(c["B"], R, Hq + 2 * Hkv, D)[:, j, Hq + Hkv:, j] = 1.0   # row j's V: one-hot in column j
    vp = torch.zeros_like(c["vp"])                  # older V rows: zero
    out = _run(c, qkv.view(c["B"] * R, -1).contiguous(), c["pos"], c["ctx"], c["table"], c["kp"].clone(), vp, R)
    out = out.view(c["B"], R, Hq, D).float()
    for j in range(R):
        seen = (out[:, j, :, :R] != 0).all(dim=(0, 1))
        assert seen[: j + 1].all() and not seen[j + 1 :].any(), f"row {j} sees {seen.tolist()}"


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("ctx0,max_context,page", [(20, 256, 16), (1021, 8192, 64)])
def test_r_rows_against_float64(dev, G, ctx0, max_context, page):
    """Every row of an R = 8 launch against the float64 paged reference over exactly its causal prefix.  The k part of
    qkv repeats the q row and k_norm = q_norm, so each row's appended key is, bit for bit, the q it used (read back
    from the cache).  At a short context the references that see one key more (the next row's) or one key less (its
    own) must be out of bounds: the check separates row j from its neighbours."""
    R, Hkv, D, B, eps, scale = 8, 2, 128, 2, 1e-6, 128 ** -0.5
    Hq = G * Hkv
    g = torch.Generator().manual_seed(ctx0 + G)
    max_pages = (max_context + page - 1) // page
    kp, vp, bt, _, _ = ar.paged_inputs(g, [ctx0 + R] * B, page, Hkv, D, BF16, max_pages=max_pages, key_rms=1.0)
    kp, vp, bt = kp.to(dev), vp.to(dev), bt.to(dev)
    pos = (ctx0 + torch.arange(R, dtype=torch.int32)).repeat(B).to(dev)
    q_raw = torch.randn(B, R, Hkv, D, generator=g).to(BF16)
    v_new = torch.randn(B, R, Hkv, D, generator=g).to(BF16)
    qkv = torch.cat([q_raw.repeat_interleave(G, dim=2), q_raw, v_new], dim=2).reshape(B * R, (Hq + 2 * Hkv) * D).contiguous().to(dev)
    w = torch.full((D,), 0.53).to(BF16).to(dev)  # |q| ~ 6: a row's score against its own key ~ 3 nats
    freq = ext.rope_inv_freq_table(D, 1e6, dev)
    got = ext.decode_attention_fused(qkv, w, w, pos, bt, pos + 1, freq, kp, vp, Hq, Hkv, eps, scale, max_context, rows_per_request=R)
    torch.cuda.synchronize()
    got = got.view(B, R, Hq * D)
    for j in range(R):
        cur = ctx0 + j
        pid = bt[:, cur // page].long()
        q = kp[pid, :, cur % page].repeat_interleave(G, dim=1).reshape(B * Hq, 1, D)
        cl = torch.full((B,), cur + 1, dtype=torch.int32, device=dev)
        got_j = got[:, j].reshape(B * Hq, 1, D)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, bt, cl, scale, True, Hkv, Hq)
        ar.assert_within(got_j, ref, ar.error_bound(ref, A, smax, nvis, D, BF16, p_rounded=False), f"G={G} ctx0={ctx0} row {j}")
        if ctx0 < 100:
            for delta in (-1, 1):
                ref_d, A_d, smax_d, nvis_d = ar.paged_reference(q, kp, vp, bt, cl, scale, True, Hkv, Hq, ctx_delta=delta)
                tol_d = ar.error_bound(ref_d, A_d, smax_d, nvis_d, D, BF16, p_rounded=False)
                assert bool(((got_j.to(torch.float64) - ref_d).abs() > tol_d).any()), f"row {j} is within the bound of context {delta:+d}"


# ------------------------------------------------------------------ engine: verify step == T decode steps --
MODELS = {
    "d128": ("tiny-d128", dict(seed=5, realistic=True, max_position_embeddings=8192)),
    "4b": ("qwen3-4b", dict(seed=1, num_hidden_layers=2, vocab_size=4096)),
    "0.6b": ("qwen3-0.6b", dict(seed=2, num_hidden_layers=2, vocab_size=4096)),
}
_NS: dict = {}


def _model(key, dev):
    if key not in _NS:
        name, kw = MODELS[key]
        _NS[key] = synthetic_qwen3(name, device=dev, **kw)
    return Qwen3ModelWeek3(_NS[key], page_size=128)


def _prefilled(model, prompt, seed):
    """Reserve (as the B = 1 decode engine does), randomise every slab, prefill through model(...)."""
    model.decode_engine(1)
    g = torch.Generator(device=model.page_pools[0]._key_pages.device).manual_seed(seed)
    for pool in model.page_pools:
        pool._key_pages.normal_(generator=g)
        pool._value_pages.normal_(generator=g)
    cache = model.create_kv_cache()
    model(prompt[None], 0, cache, logits_to_keep=1)
    return cache


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("ctx0", [126, 4093])
@pytest.mark.parametrize("T", [2, 5, 8])
def test_verify_step_equals_t_decode_steps(dev, key, ctx0, T):
    a, b = _model(key, dev), _model(key, dev)
    for m in (a, b):
        m.prefill_graph_len = 0
    V = a.vocab_size
    g = torch.Generator(device=dev).manual_seed(ctx0 + T)
    prompt = torch.randint(0, V, (ctx0,), device=dev, generator=g, dtype=torch.int32)
    toks = torch.randint(0, V, (T,), generator=torch.Generator().manual_seed(T)).tolist()
    ca, cb = _prefilled(a, prompt, 9), _prefilled(b, prompt, 9)
    dec = a.decode_engine(1)
    want_logits, want_next = [], []
    for j in range(T):
        logits, nxt = dec.step([toks[j]], [ctx0 + j], ca)
        want_logits.append(logits[0, 0].clone())
        want_next.append(int(nxt[0]))
    ver = b.verify_engine(T)
    logits, nxt = ver.verify(toks[0], torch.tensor(toks[1:], dtype=torch.int32, device=dev), ctx0, cb)
    torch.cuda.synchronize()
    assert torch.equal(logits.view(torch.int16), torch.stack(want_logits).view(torch.int16))
    assert nxt.tolist() == want_next
    for i, (pa, pb) in enumerate(zip(a.page_pools, b.page_pools)):
        assert torch.equal(pa._key_pages.view(torch.int16), pb._key_pages.view(torch.int16)), f"layer {i} K"
        assert torch.equal(pa._value_pages.view(torch.int16), pb._value_pages.view(torch.int16)), f"layer {i} V"
    assert ca[0].offset == cb[0].offset == ctx0 + T
    # one verify replay issues the launches of one decode step (whose count includes the token-advance kernel)
    assert ver.kernels_per_step == dec.kernels_per_step - 1
    assert ver.captures == 1 and ver.max_seq_len == dec.max_seq_len
    for c in (ca, cb):
        for layer in c:
            layer.release()


# ------------------------------------------------------------------ end to end --
@pytest.fixture(scope="module")
def target(dev):
    m = _model("d128", dev)
    m.prefill_graph_len = 0  # greedy and speculative runs prefill the prompt through the same path
    return m


def _draft(kind, dev):
    if kind == "same":
        m = _model("d128", dev)
    else:
        name, kw = MODELS["d128"]
        m = Qwen3ModelWeek3(synthetic_qwen3(name, device=dev, **{**kw, "seed": 11}), page_size=128)
    m.prefill_graph_len = 0
    return m


PROMPT = [5, 17, 3, 250, 9, 44, 100]


def _pools_whole(*models):
    for m in models:
        for pool in m.page_pools:
            assert not pool.used_page_ids, "every page is back in its pool"


@pytest.mark.parametrize("kind", ["same", "other"])
@pytest.mark.parametrize("k", [1, 4, 7, 8])
def test_speculative_equals_greedy(dev, target, kind, k):
    draft = _draft(kind, dev)
    want = greedy_generate_ids(target, PROMPT, 200, device=dev)
    got, stats = speculative_generate_ids(draft, target, PROMPT, 200, proposal_length=k, device=dev)
    # every round checks both caches' offsets (the protocol raises otherwise), on the generic path (k = 8) too
    if k == 8:  # the generic path: its multi-row pass is the operator path, which does not round like the decode step
        assert len(got) == 200 and got[0] == want[0] and all(p <= 8 for p, _ in stats)
    else:
        assert got == want
    proposed, accepted = sum(p for p, _ in stats), sum(a for _, a in stats)
    if kind == "same" and k <= 7:
        assert accepted == proposed, "the target's own weights: every proposal is accepted"
    _pools_whole(target, draft)
    if k <= 7:
        assert target.verify_engine(k + 1).captures == 1 and draft.decode_engine(1).captures == 1
        assert target.decode_engine(1).captures <= 1


def test_eos_inside_an_accepted_run_and_as_a_bonus(dev, target):
    draft = _draft("same", dev)
    k = 4
    want = greedy_generate_ids(target, PROMPT, 120, device=dev)
    for residue in (2, 0):  # index 5 r + 2: inside a round's accepted run; 5 r + 5: a round's bonus token
        idx = next(i for i in range(5, 120) if i % (k + 1) == residue and want[i] not in want[:i])
        eos = want[idx]
        got, _ = speculative_generate_ids(draft, target, PROMPT, 200, proposal_length=k, eos_token_ids=(eos,), device=dev)
        assert got == greedy_generate_ids(target, PROMPT, 200, eos_token_id=eos, device=dev) == want[:idx]
    _pools_whole(target, draft)


def test_perturbed_draft_hits_every_mismatch_index_and_frees_pages(dev, monkeypatch):
    """A draft whose final norm weight is perturbed disagrees now and then.  Among a few fixed perturbations one run
    must reach a mismatch at proposal 1, at a middle proposal, at the last proposal and a full acceptance, and a
    rewind that gives a page back (16-token pages); every run equals greedy."""
    _model("d128", dev)
    ns = _NS["d128"]
    target = Qwen3ModelWeek3(ns, page_size=16)
    target.prefill_graph_len = 0
    freed = []
    original = TinyKvPagedCache.rewind

    def rewind(self, n):
        before = len(self.page_ids)
        out = original(self, n)
        freed.append(before - len(self.page_ids))
        return out

    monkeypatch.setattr(TinyKvPagedCache, "rewind", rewind)
    k = 4
    want = greedy_generate_ids(target, PROMPT, 200, device=dev)
    covered = None
    for i, s in enumerate((0.05, 0.1, 0.2, 0.4, 0.8)):
        ns2 = copy.deepcopy(ns)
        g = torch.Generator(device=dev).manual_seed(100 + i)
        w = ns2.model.norm.weight
        ns2.model.norm.weight = (w.float() * (1 + s * torch.randn(w.shape, device=dev, generator=g))).to(w.dtype)
        draft = Qwen3ModelWeek3(ns2, page_size=16)
        draft.prefill_graph_len = 0
        freed.clear()
        got, stats = speculative_generate_ids(draft, target, PROMPT, 200, proposal_length=k, device=dev)
        assert got == want
        _pools_whole(target, draft)
        kinds = {"first": any(a == 0 and p == k for p, a in stats), "middle": any(0 < a < k - 1 for _, a in stats),
                 "last": any(a == k - 1 for _, a in stats), "full": any(a == k for _, a in stats), "page freed": any(f > 0 for f in freed)}
        if all(kinds.values()):
            covered = s
            break
    assert covered is not None, f"no perturbation reached every case: {kinds}"


def test_generation_past_the_graph_length_equals_greedy(dev):
    """Past ``decode_graph_max_seq_len`` the engines cannot hold the request: rounds stop before it and the run ends
    target-only through model(...), as greedy does."""
    _model("d128", dev)
    models = []
    for ns in (_NS["d128"], _NS["d128"]):
        m = Qwen3ModelWeek3(ns, page_size=16)
        m.prefill_graph_len = 0
        m.decode_graph_max_seq_len = 256
        models.append(m)
    target, draft = models
    prompt = torch.randint(0, 512, (200,), generator=torch.Generator().manual_seed(4)).tolist()
    want = greedy_generate_ids(target, prompt, 120, device=dev)
    got, stats = speculative_generate_ids(draft, target, prompt, 120, proposal_length=4, device=dev)
    assert got == want and len(got) == 120 and stats
    _pools_whole(target, draft)
    long_prompt = torch.randint(0, 512, (300,), generator=torch.Generator().manual_seed(5)).tolist()
    got, stats = speculative_generate_ids(draft, target, long_prompt, 20, proposal_length=4, device=dev)
    assert got == greedy_generate_ids(target, long_prompt, 20, device=dev) and stats == []
    _pools_whole(target, draft)
