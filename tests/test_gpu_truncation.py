"""Top-n-sigma, locally typical sampling and Mirostat 2.0 on the H100 (DESIGN.md section 25): the draws and mu updates
of ``tl_sample_penalized_trunc`` and ``tl_sample_constrained_trunc`` against the float64 restatement
(``truncation_ref``) at every dtype and cluster size, planted boundary probes, row independence, graph replay, the
all-off equivalence with the existing entries, and the samplers through ``greedy_generate_ids``, the batcher,
``parallel_sample_ids`` and ``decode_on_device``."""

import dataclasses
import importlib.util
import math
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


tref = _load("tiny_llm_b200_truncation_ref", "truncation_ref.py")
kref = _load("tiny_llm_b200_keep_set_ref", "keep_set_ref.py")
from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams, batch_generate, greedy_generate_ids
from tiny_llm_b200.engine import DecodeEngine
from tiny_llm_b200.generate import parallel_sample_ids
from tiny_llm_b200.sampler import (mirostat_start, penalty_tensors, sample_tokens, sampling_tensors, token_state_row, truncation_tensors,
                                   xtc_tensors)
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu

VOCABS = [1, 7, 4096, 4097, 8193, 12289, 16385, 20481, 24577, 28673, 151936, 409600]
TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
COUNTS: dict = {}


def _count(key, n_rows, near, wrong):
    c = COUNTS.setdefault(key, [0, 0, 0])
    c[0] += n_rows
    c[1] += near
    c[2] += wrong


# --------------------------------------------------------------------------------------------- launches --
def _masks(allowed, dev):
    """One-state descriptors whose mask is each row's ``allowed`` (state 0, a DFA that stays at 0)."""
    R, V = allowed.shape
    words = (V + 31) // 32
    masks = np.zeros((R, 2, words), dtype=np.uint32)
    for r in range(R):
        bits = np.zeros(words * 32, bool)
        bits[:V] = allowed[r]
        masks[r, 0] = np.packbits(bits, bitorder="little").view("<u4")
    masks_d = torch.from_numpy(masks.view(np.int32)).to(dev)
    dfa = torch.zeros((1, 256), dtype=torch.int32, device=dev)
    offsets = torch.arange(V + 1, dtype=torch.int32, device=dev)
    data = torch.zeros(V, dtype=torch.uint8, device=dev)
    row_bytes = 2 * words * 4
    desc = torch.tensor([[masks_d.data_ptr() + r * row_bytes, dfa.data_ptr(), offsets.data_ptr(), data.data_ptr(), 1] for r in range(R)],
                        dtype=torch.int64, device=dev)
    return desc, (masks_d, dfa, offsets, data)


def draw(x, params, positions, state, mu, allowed=None, dev="cuda"):
    """One truncation launch over the rows ``x`` (a device tensor) -> (tokens, mu') on the host."""
    t, k, tp, s = sampling_tensors(params, dev)
    pos = torch.tensor(positions, dtype=torch.int32, device=dev)
    trunc = dict(zip(("typical_p", "top_n_sigma", "mirostat_tau", "mirostat_eta"), truncation_tensors(params, dev)))
    th, q = xtc_tensors(params, dev)
    mu_d = torch.tensor(mu, dtype=torch.float32, device=dev)
    pen = (*penalty_tensors(params, dev), state)
    if allowed is None:
        got = ext.sample_penalized(x, t, k, tp, s, pos, *pen, xtc_threshold=th, xtc_probability=q, mirostat_mu=mu_d, **trunc)
    else:
        desc, keep = _masks(allowed, dev)
        got = ext.sample_constrained(x, t, k, tp, s, pos, desc, *pen, xtc_threshold=th, xtc_probability=q, mirostat_mu=mu_d, **trunc)
        torch.cuda.synchronize()
        del keep
    return got.cpu().numpy(), mu_d.cpu().numpy()


def _grid(V, rounds):
    temps = (0.6, 1.0, 1.7)
    extras = [{}, dict(top_k=50), dict(top_p=0.9), dict(min_p=0.05), dict(repetition_penalty=1.3, presence_penalty=0.5, frequency_penalty=0.3),
              dict(xtc_probability=1.0, xtc_threshold=0.05)]
    rows = []
    for r in range(rounds):
        combos = [(tp, ns) for tp in (0.2, 0.5, 0.9, 0.99) for ns in (0.0, 0.5, 1.0, 3.0)]
        for j, (tp, ns) in enumerate(combos):
            rows.append((SamplingParams(temps[(j + r) % 3], seed=1000 * r + j, typical_p=tp, top_n_sigma=ns, **extras[(j + r) % 6]), None))
        mir = [(tau, eta) for tau in (1.0, 3.0, 5.0, 8.0) for eta in (0.05, 0.1, 1.0)]
        for j, (tau, eta) in enumerate(mir):
            pen = dict(repetition_penalty=1.2) if (j + r) % 4 == 0 else {}
            p = SamplingParams(temps[(j + r) % 3], seed=500 + 1000 * r + j, mirostat=2, mirostat_tau=tau, mirostat_eta=eta, **pen)
            rows.append((p, mirostat_start(p) - 0.37 * ((j + r) % 5)))
    return rows


def _rows(R, V, dtype, g):
    x = (torch.randn(R, V, generator=g) * 2.5).to(TORCH[dtype])
    if V > 16:
        x[torch.rand(R, V, generator=g) < 0.01] = -float("inf")
    return x


def _state(R, V, rng):
    st = np.zeros((R, V), np.int32)
    st[rng.random((R, V)) < 0.05] |= 1 << 30
    c = rng.random((R, V)) < 0.03
    st[c] += rng.integers(1, 4, size=int(c.sum())).astype(np.int32)
    return st


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("dtype", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("form", ["penalized", "constrained"])
def test_draw_sweep_equals_the_reference(cuda_device, V, dtype, form):
    g = torch.Generator().manual_seed(V * 7 + len(dtype))
    rng = np.random.default_rng(V + len(form))
    grid = _grid(V, 1 if V >= 151936 else 2)
    R = len(grid)
    x = _rows(R, V, dtype, g)
    params = [p for p, _ in grid]
    mu = [0.0 if m is None else m for _, m in grid]
    positions = rng.integers(1, 5000, size=R).tolist()
    st = _state(R, V, rng)
    allowed = None
    if form == "constrained":
        allowed = rng.random((R, V)) < 0.7
        allowed[np.arange(R), rng.integers(0, V, size=R)] = True
    tokens, mu2 = draw(x.to(cuda_device), params, positions, torch.from_numpy(st).to(cuda_device), mu,
                       None if allowed is None else allowed, cuda_device)
    xf = x.float().numpy()
    near = wrong = mu_checked = 0
    for r, p in enumerate(params):
        want, want_mu, close = tref.sample_row(xf[r], st[r], p.temperature, p.top_k or 0, p.top_p or 0.0, p.seed, positions[r],
                                               p.repetition_penalty, p.presence_penalty, p.frequency_penalty, p.min_p, p.xtc_threshold,
                                               p.xtc_probability, p.typical_p, p.top_n_sigma, p.mirostat_tau if p.mirostat else 0.0,
                                               p.mirostat_eta, mu[r], None if allowed is None else allowed[r])
        if allowed is not None:
            assert allowed[r, tokens[r]], (r, p)
        if close:
            near += 1
            continue
        ok = int(tokens[r]) == want
        if ok and p.mirostat:
            ok = tref.mu_close(float(mu2[r]), want_mu, p.mirostat_eta)
            mu_checked += 1
        wrong += not ok
        assert ok, (r, p, int(tokens[r]), want, float(mu2[r]), want_mu)
    _count((form, dtype), R, near, wrong)
    print(f"{form} {dtype} V={V}: {R} draws, {near} in the band, {mu_checked} mu checked, {wrong} mismatches outside it")


def test_print_counts():
    for k, (n, near, wrong) in sorted(COUNTS.items()):
        print(f"draw sweep {k}: {n} draws, {near} with a boundary in the band, {wrong} mismatches outside it")


# ------------------------------------------------------------------------------------------------ probes --
def _settle(x, T, keep, target, margin=0.25, start=1, tries=1 << 14, seed=77):
    """A position at which ``target``'s float64 score beats every other live entry by ``margin`` and the best kept
    entry other than the target beats the rest of the kept ones by ``margin``: the draw shows whether target is kept."""
    live = np.flatnonzero(np.isfinite(x))
    for pos in range(start, start + tries):
        sc = x[live] / T + kref.gumbel_at(live, seed, pos)
        o = np.argsort(-sc)
        if live[o[0]] != target or (len(o) > 1 and sc[o[0]] - sc[o[1]] < margin):
            continue
        others = [j for j in o if keep[live[j]] and live[j] != target]
        if len(others) > 1 and sc[others[0]] - sc[others[1]] < margin:
            continue
        return pos, (target if keep[target] else (int(live[others[0]]) if others else target))
    raise AssertionError("no position settles the probe")


def _probe(dev, V, vals, idx, T, target, dtype="f32", **kw):
    """Plant ``vals`` at ``idx`` (every other entry -inf) and draw with ``kw``; returns (token, expected, keep)."""
    x = np.full(V, -np.inf, np.float32)
    x[idx] = vals
    p = SamplingParams(T, seed=77, **{k: v for k, v in kw.items() if k != "mu"})
    mu = kw.get("mu", mirostat_start(p) if p.mirostat else 0.0)
    st = np.zeros(V, np.int32)
    x3 = x.astype(np.float32)
    if p.mirostat:
        keep, _, _ = tref.mirostat_keep(x3, T, mu)
    else:
        keep = tref.penalties_ref.keep_set(x3, 0, 0.0, 0.0, T)
        keep, _ = tref.nsigma_keep(x3, keep, p.top_n_sigma)
        keep, _ = tref.typical_keep(x3, keep, p.typical_p)
    pos, want = _settle(x.astype(np.float64), T, keep, target)
    xt = torch.from_numpy(x).to(TORCH[dtype]).to(dev)[None]
    tok, _ = draw(xt, [p], [pos], torch.zeros((1, V), dtype=torch.int32, device=dev), [mu], None, dev)
    ref_tok, _, _ = tref.sample_row(x, st, T, 0, 0.0, 77, pos, typical_p=p.typical_p, top_n_sigma=p.top_n_sigma,
                                    mirostat_tau=p.mirostat_tau if p.mirostat else 0.0, mirostat_eta=p.mirostat_eta, mu=mu)
    assert ref_tok == want
    return int(tok[0]), want, keep


@pytest.mark.parametrize("V", [8, 4097, 151936])
def test_planted_probes(cuda_device, V):
    spots = sorted({0, V - 1, min(kref.plan(V)[1] - 1, V - 1), (kref.plan(V)[0] - 1) * kref.plan(V)[1], V // 2, V // 3})[:6]
    if len(spots) < 5:
        spots = list(range(5))
    a, b, c, d, e = spots[:5]
    # typical, tied d at the boundary: b and c share a logit, so both stay or both go
    vals = [0.0, -1.0, -1.0, -3.0, -5.0]
    x = np.full(V, -np.inf)
    x[[a, b, c, d, e]] = vals
    _, dist = tref.typical_distances(x.astype(np.float32), np.isfinite(x))
    _, keep_all = tref.typical_keep(x.astype(np.float32), np.isfinite(x), 0.999)
    p_, dd = tref.typical_distances(x.astype(np.float32), np.isfinite(x))
    order = np.argsort(dd[[a, b, c, d, e]])
    mass_below_tie = sum(p_[i] for i in (a, b, c, d, e) if dd[i] < dd[b])
    for tp, inside in ((mass_below_tie + 1e-3, True), (max(mass_below_tie - 1e-3, 1e-3), False)):
        if not inside and mass_below_tie < 2e-3:
            continue
        got, want, keep = _probe(cuda_device, V, vals, [a, b, c, d, e], 1.0, c, typical_p=tp)
        assert keep[b] == keep[c] == inside
        assert got == want, ("typical tie", tp)
    # top-n-sigma: two finite entries 0 and -2 (mean -1, sigma 1): n = 2 puts the bound on -2, n one ulp below 2 one
    # fp32 ulp above it
    for n, inside in ((2.0, True), (float(np.nextafter(np.float32(2.0), np.float32(0.0))), False)):
        got, want, keep = _probe(cuda_device, V, [0.0, -2.0], [a, b], 1.0, b, top_n_sigma=n)
        assert bool(keep[b]) == inside
        assert got == want, ("top-n-sigma", n)
    # one finite entry: sigma 0, the maximum's ties stay
    got, want, _ = _probe(cuda_device, V, [1.5], [c], 0.8, c, top_n_sigma=1.0)
    assert got == want == c
    got, want, _ = _probe(cuda_device, V, [1.5], [c], 0.8, c, typical_p=0.3)
    assert got == want == c
    # Mirostat: four ties at the maximum (p = 1/4 each, -log2 p = 2) and mu = 2 keeps them all; mu so low that only
    # the maximum survives
    got, want, keep = _probe(cuda_device, V, [0.0, 0.0, 0.0, 0.0, -3.0], [a, b, c, d, e], 1.0, d, mirostat=2, mu=2.0)
    assert keep[[a, b, c, d]].all() and got == want == d
    got, want, keep = _probe(cuda_device, V, [0.0, -0.5, -1.0, -2.0], [a, b, c, d], 1.0, c, mirostat=2, mu=0.01)
    assert keep.sum() == 1 and got == want == a


def test_nan_and_inf_entries(cuda_device):
    V = 4097
    x = (torch.randn(4, V, generator=torch.Generator().manual_seed(3)) * 2).float()
    x[:, ::7] = float("nan")
    x[:, 3::11] = -float("inf")
    params = [SamplingParams(1.0, seed=1, typical_p=0.5), SamplingParams(0.8, seed=2, top_n_sigma=1.0),
              SamplingParams(1.2, seed=3, mirostat=2, mirostat_tau=3.0), SamplingParams(0.7, seed=4, typical_p=0.9, top_n_sigma=2.0)]
    mu = [0.0, 0.0, 6.0, 0.0]
    tok, mu2 = draw(x.to(cuda_device), params, [9, 9, 9, 9], torch.zeros((4, V), dtype=torch.int32, device=cuda_device), mu)
    for r, p in enumerate(params):
        assert math.isfinite(float(x[r, tok[r]]))
        want, wmu, near = tref.sample_row(x[r].numpy(), np.zeros(V, np.int32), p.temperature, 0, 0.0, p.seed, 9, typical_p=p.typical_p,
                                          top_n_sigma=p.top_n_sigma, mirostat_tau=p.mirostat_tau if p.mirostat else 0.0,
                                          mirostat_eta=p.mirostat_eta, mu=mu[r])
        if not near:
            assert tok[r] == want
            if p.mirostat:
                assert tref.mu_close(float(mu2[r]), wmu, p.mirostat_eta)


def test_greedy_and_position_zero_leave_mu(cuda_device):
    V = 4097
    x = torch.randn(2, V, generator=torch.Generator().manual_seed(4)).to(cuda_device)
    p0 = SamplingParams(0.0, mirostat=2, mirostat_tau=3.0)
    p1 = SamplingParams(0.9, seed=3, mirostat=2, mirostat_tau=3.0)
    st = torch.zeros((2, V), dtype=torch.int32, device=cuda_device)
    tok, mu2 = draw(x, [p0, p1], [5, 0], st, [4.5, 4.5])
    assert mu2.tolist() == [4.5, 4.5]
    assert tok[0] == int(torch.argmax(x[0]))


# ------------------------------------------------------------------------------------- mu, rows, replay --
@pytest.mark.parametrize("V", [4097, 151936])
def test_mu_teacher_forced(cuda_device, V):
    g = torch.Generator().manual_seed(V)
    worst = near = checked = 0
    for tau, eta in ((1.0, 0.05), (3.0, 0.1), (5.0, 1.0), (8.0, 0.1)):
        p = SamplingParams(1.0, seed=int(tau * 10), mirostat=2, mirostat_tau=tau, mirostat_eta=eta)
        mu = mirostat_start(p)
        for step in range(24):
            x = torch.randn(1, V, generator=g) * 3
            tok, mu2 = draw(x.to(cuda_device), [p], [step + 1], torch.zeros((1, V), dtype=torch.int32, device=cuda_device), [mu])
            want, wmu, close = tref.sample_row(x[0].numpy(), np.zeros(V, np.int32), 1.0, 0, 0.0, p.seed, step + 1, mirostat_tau=tau,
                                               mirostat_eta=eta, mu=mu)
            if close:
                near += 1
            else:
                assert tok[0] == want
                assert tref.mu_close(float(mu2[0]), wmu, eta), (float(mu2[0]), wmu)
                worst = max(worst, abs(float(mu2[0]) - wmu))
                checked += 1
            mu = float(mu2[0])  # the kernel's own mu feeds the next step
    print(f"mu teacher-forced V={V}: {checked} steps checked, {near} in the band, worst |mu' - ref| = {worst:.3g}")


def _mixed(R):
    out = []
    for r in range(R):
        k = r % 4
        out.append([SamplingParams(0.9, seed=r, typical_p=0.7), SamplingParams(1.1, seed=r, top_n_sigma=1.5, top_k=40),
                    SamplingParams(0.8, seed=r, mirostat=2, mirostat_tau=4.0, mirostat_eta=0.2), SamplingParams(0.7, seed=r, presence_penalty=0.4)][k])
    return out


def test_row_alone_equals_row_in_a_launch(cuda_device):
    V, R = 151936, 64
    x = (torch.randn(R, V, generator=torch.Generator().manual_seed(9)) * 2.5).to(torch.bfloat16).to(cuda_device)
    params = _mixed(R)
    mu = [mirostat_start(p) if p.mirostat else 0.0 for p in params]
    st = torch.zeros((R, V), dtype=torch.int32, device=cuda_device)
    tok, mu2 = draw(x, params, list(range(1, R + 1)), st.clone(), mu)
    for r in (0, 1, 2, 3, 17, 38, 63):
        t1, m1 = draw(x[r : r + 1].contiguous(), [params[r]], [r + 1], st[r : r + 1].clone(), [mu[r]])
        assert t1[0] == tok[r] and m1[0] == mu2[r], r


def test_replay_equals_eager(cuda_device):
    V, R = 32000, 8
    x = (torch.randn(R, V, generator=torch.Generator().manual_seed(5)) * 2).to(cuda_device)
    params = _mixed(R)
    t, k, tp, s = sampling_tensors(params, cuda_device)
    pen = penalty_tensors(params, cuda_device)
    th, q = xtc_tensors(params, cuda_device)
    trunc = dict(zip(("typical_p", "top_n_sigma", "mirostat_tau", "mirostat_eta"), truncation_tensors(params, cuda_device)))
    pos = torch.arange(1, R + 1, dtype=torch.int32, device=cuda_device)
    mu0 = torch.tensor([mirostat_start(p) if p.mirostat else 0.0 for p in params], device=cuda_device)

    def run(state, mu):
        return ext.sample_penalized(x, t, k, tp, s, pos, *pen, state, xtc_threshold=th, xtc_probability=q, mirostat_mu=mu, **trunc)

    st_e, mu_e = torch.zeros((R, V), dtype=torch.int32, device=cuda_device), mu0.clone()
    eager = [run(st_e, mu_e).clone() for _ in range(3)]
    st_g, mu_g = torch.zeros((R, V), dtype=torch.int32, device=cuda_device), mu0.clone()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        run(torch.zeros_like(st_g), mu0.clone())  # warm-up outside the graph
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run(st_g, mu_g)
    got = []
    for _ in range(3):
        graph.replay()
        got.append(out.clone())
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, got))
    assert torch.equal(mu_e, mu_g) and torch.equal(st_e, st_g)


@pytest.mark.parametrize("V", [7, 4097, 151936])
def test_all_off_equals_the_existing_entries(cuda_device, V):
    R = 12
    x = (torch.randn(R, V, generator=torch.Generator().manual_seed(V)) * 2).to(torch.bfloat16).to(cuda_device)
    params = [SamplingParams(0.9, seed=r, top_k=[0, 20][r % 2], top_p=[None, 0.9][r % 3 == 0], presence_penalty=[0.0, 0.3][r % 2],
                             xtc_probability=[0.0, 0.5][r % 4 == 1]) for r in range(R)]
    t, k, tp, s = sampling_tensors(params, cuda_device)
    pen = penalty_tensors(params, cuda_device)
    th, q = xtc_tensors(params, cuda_device)
    trunc = dict(zip(("typical_p", "top_n_sigma", "mirostat_tau", "mirostat_eta"), truncation_tensors(params, cuda_device)))
    pos = torch.arange(1, R + 1, dtype=torch.int32, device=cuda_device)
    st = torch.zeros((R, V), dtype=torch.int32, device=cuda_device)
    mu = torch.zeros(R, device=cuda_device)
    a = ext.sample_penalized(x, t, k, tp, s, pos, *pen, st.clone(), xtc_threshold=th, xtc_probability=q)
    b = ext.sample_penalized(x, t, k, tp, s, pos, *pen, st.clone(), xtc_threshold=th, xtc_probability=q, mirostat_mu=mu, **trunc)
    assert torch.equal(a, b)
    desc = torch.zeros((R, 5), dtype=torch.int64, device=cuda_device)
    c = ext.sample_constrained(x, t, k, tp, s, pos, desc, *pen, st.clone(), xtc_threshold=th, xtc_probability=q, mirostat_mu=mu, **trunc)
    assert torch.equal(a, c)
    plain = [SamplingParams(0.9, seed=r, top_k=[0, 20][r % 2]) for r in range(R)]
    t, k, tp, s = sampling_tensors(plain, cuda_device)
    pen = penalty_tensors(plain, cuda_device)
    trunc = dict(zip(("typical_p", "top_n_sigma", "mirostat_tau", "mirostat_eta"), truncation_tensors(plain, cuda_device)))
    assert torch.equal(ext.sample(x, t, k, tp, s, pos), ext.sample_penalized(x, t, k, tp, s, pos, *pen, st.clone(), mirostat_mu=mu, **trunc))
    assert torch.equal(mu, torch.zeros(R, device=cuda_device))


# ---------------------------------------------------------------------------------------------- callers --
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


KINDS = [lambda b: SamplingParams(0.9, seed=b, typical_p=0.8),
         lambda b: SamplingParams(1.1, seed=b, top_n_sigma=1.0, presence_penalty=0.2),
         lambda b: SamplingParams(0.8, seed=b, mirostat=2, mirostat_tau=3.0, mirostat_eta=0.3),
         lambda b: SamplingParams(0.7, seed=b, top_p=0.9),
         lambda b: SamplingParams(0.9, seed=b, repetition_penalty=1.2, typical_p=0.6, top_n_sigma=2.0, xtc_probability=0.5),
         lambda b: None]


@pytest.mark.parametrize("B,lens", [(1, {0: 40}), (16, {0: 40, 3: 9, 9: 70, 15: 20, 6: 33, 12: 5}),
                                    (32, {0: 30, 2: 65, 5: 12, 11: 90, 20: 44, 31: 7})])
def test_decode_on_device_equals_steps_plus_eager(cuda_device, B, lens):
    steps, msl = 20, 256
    slots = sorted(lens)
    g = torch.Generator().manual_seed(B)
    history = [(torch.randint(0, 40, (lens[b] - 2,), generator=g).tolist(), torch.randint(0, 40, (3,), generator=g).tolist()) if b in lens
               else None for b in range(B)]
    params = [None] * B
    for n, b in enumerate(slots):
        params[b] = KINDS[n % len(KINDS) if B > 1 else 2](b)
    start = [1.7 + 0.5 * b if b % 2 else None for b in range(B)]  # half the Mirostat slots start from a given mu
    runs, mus = {}, {}
    for mode in ("graph", "eager"):
        model = _model(cuda_device)
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, lens)
        _fill_slabs(model, B)
        tokens = [history[b][1][-1] if b in lens else 0 for b in range(B)]
        offsets = [lens.get(b, 0) for b in range(B)]
        mu0 = [(start[b] if start[b] is not None else mirostat_start(params[b])) if params[b] is not None and params[b].mirostat else 0.0
               for b in range(B)]
        if mode == "graph":
            runs[mode] = engine.decode_on_device(tokens, offsets, caches, steps, sampling=params, history=history,
                                                 mirostat_mu=start).cpu()
            mus[mode] = engine.mirostat_mu.cpu()
        else:
            state = torch.stack([token_state_row(*history[b], model.vocab_size) if b in lens else torch.zeros(model.vocab_size, dtype=torch.int32)
                                 for b in range(B)]).to(cuda_device)
            mu = torch.tensor(mu0, dtype=torch.float32, device=cuda_device)
            out = []
            for _ in range(steps):
                logits, _ = engine.step(tokens, offsets, caches)
                pos = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
                nxt = sample_tokens(logits.view(B, -1), params, pos, state, mirostat_mu=mu).cpu()
                out.append([int(nxt[b]) if b in lens else -1 for b in range(B)])
                tokens = [int(nxt[b]) if b in lens else 0 for b in range(B)]
                offsets = [o + 1 if b in lens else 0 for b, o in enumerate(offsets)]
            runs[mode] = torch.tensor(out, dtype=torch.int32)
            mus[mode] = mu.cpu()
    live = [b for b in range(B) if b in lens]
    assert torch.equal(runs["graph"][:, live], runs["eager"][:, live])
    miro = [b for b in live if params[b] is not None and params[b].mirostat]
    assert torch.equal(mus["graph"][miro], mus["eager"][miro])


def test_generate_equals_prefill_plus_decode_on_device(cuda_device):
    model = _model(cuda_device, seed=7)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11]
    n = 16
    for p in (SamplingParams(0.9, seed=3, mirostat=2, mirostat_tau=3.0, mirostat_eta=0.2),
              SamplingParams(0.8, seed=4, typical_p=0.7, top_n_sigma=1.5, frequency_penalty=0.2)):
        got = greedy_generate_ids(model, prompt, n, device=cuda_device, sampling=p)
        cache = model.create_kv_cache()
        try:
            logits = model(torch.tensor([prompt], dtype=torch.int32, device=cuda_device), 0, cache, logits_to_keep=1)[:, -1, :]
            state = token_state_row(prompt, [], model.vocab_size, device=cuda_device)[None]
            mu = torch.full((1,), mirostat_start(p), dtype=torch.float32, device=cuda_device)
            first = int(sample_tokens(logits, [p], [len(prompt)], state, mirostat_mu=mu)[0])
            engine = DecodeEngine(model, 1, 256, cuda_device)
            rest = engine.decode_on_device([first], [len(prompt)], cache, n - 1, sampling=p, history=[(prompt, [first])],
                                           mirostat_mu=[float(mu[0])] if p.mirostat else None)
            want = [first] + rest[:, 0].cpu().tolist()
        finally:
            for c in cache:
                c.release()
        assert got == want, p


def test_batcher_in_two_orders(cuda_device):
    ns = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, device=cuda_device)
    g = torch.Generator().manual_seed(0)
    prompts = [torch.randint(1, 60, (int(n),), generator=g).tolist() for n in torch.randint(3, 40, (12,), generator=g)]
    kinds = [lambda i: SamplingParams(0.9, seed=i, mirostat=2, mirostat_tau=4.0),
             lambda i: SamplingParams(0.8, seed=i, typical_p=0.8),
             lambda i: SamplingParams(1.0, seed=i, top_n_sigma=1.0, presence_penalty=0.3),
             lambda i: SamplingParams(0.7, seed=i, top_p=0.9)]
    params = [kinds[i % 4](i) for i in range(len(prompts))]
    plain = [dataclasses.replace(p, mirostat=0, typical_p=1.0, top_n_sigma=0.0) for p in params]
    budget, B = 12, 16

    def serve(idx, per):
        out = batch_generate(Qwen3ModelWeek3(ns, page_size=64), None, [prompts[i] for i in idx], max_seq_len=128, batch_size=B,
                             prefill_step=16, verbose=False, device=cuda_device, max_new_tokens=[budget] * len(idx),
                             sampling=[per[i] for i in idx])
        return {idx[j]: [int(t) for t in text.split()] for j, text in out}

    # as for DRY and XTC: a request is checked in an order where its plain twin gets the ids it gets alone
    checked = 0
    alone = {}
    for order in (list(range(len(prompts))), list(reversed(range(len(prompts))))):
        got, twin = serve(order, params), serve(order, plain)
        for i in order:
            if i not in alone:
                alone[i] = (serve([i], plain)[i], serve([i], params)[i])
            if twin[i] != alone[i][0]:
                continue
            assert got[i] == alone[i][1], (order[0], i)
            checked += 1
    print(f"batcher: {checked} of {2 * len(prompts)} (request, order) pairs checked")
    assert checked >= len(prompts) // 2


def test_parallel_samples_equal_generate(cuda_device, monkeypatch):
    import tiny_llm_b200.engine as eng

    # the set-up of test_gpu_parallel_sample's equality tests: no prefill graph, 128-slot pages, no grouped attention
    monkeypatch.setattr(eng, "shared_prefix_attention_applies", lambda *a: False)
    ns = synthetic_qwen3("tiny-d128", seed=5, realistic=True, max_position_embeddings=8192, device=cuda_device)
    model = Qwen3ModelWeek3(ns, page_size=128)
    model.prefill_graph_len = 0
    model.set_max_context(4096)
    prompt = torch.randint(0, model.vocab_size, (150,), generator=torch.Generator().manual_seed(1)).tolist()
    for p in (SamplingParams(0.9, seed=11), SamplingParams(0.9, seed=11, mirostat=2, mirostat_tau=3.0, mirostat_eta=0.2),
              SamplingParams(0.8, seed=12, typical_p=0.6, top_n_sigma=2.0)):
        got = parallel_sample_ids(model, [prompt], 4, p, 12, device=cuda_device)[0]
        for j, s in enumerate(got):
            want = greedy_generate_ids(model, prompt, 12, device=cuda_device, sampling=dataclasses.replace(p, seed=p.seed + j))
            assert s.ids == want, (p, j)


def test_regex_constrained_mirostat_stays_in_its_language(cuda_device):
    import re

    from tiny_llm_b200.constrained import TokenConstraint, TokenVocabulary

    model = _model(cuda_device, seed=2)
    V = model.vocab_size
    vocab = TokenVocabulary.synthetic(V, seed=5)
    c = TokenConstraint.compile(r"[0-9]{3}-[0-9]{2}", vocab, device=cuda_device)
    for seed in range(3):
        p = SamplingParams(0.9, seed=seed, mirostat=2, mirostat_tau=2.0, constraint=c)
        ids = greedy_generate_ids(model, [5, 17, 3], 12, device=cuda_device, sampling=p)
        text = b"".join(vocab.tokens[t] or b"" for t in ids).decode()
        assert re.fullmatch(r"[0-9]{3}-[0-9]{2}", text) or re.fullmatch(r"[0-9]{0,3}(-[0-9]{0,2})?", text), text


def test_calls_without_the_new_fields_are_unchanged(cuda_device):
    model = _model(cuda_device)
    B, msl = 4, 128
    per = [SamplingParams(0.8, seed=1, presence_penalty=0.5), SamplingParams(0.8, seed=2), None, None]
    counts = []
    for with_trunc in (False, True):
        engine = DecodeEngine(model, B, msl, cuda_device)
        engine.reserve_pools()
        caches = _admit(model, B, msl, {0: 10, 1: 12})
        if with_trunc:  # a truncation call first, then the same plain call
            engine.decode_on_device([1, 2, 0, 0], [10, 12, 0, 0], caches, 2, sampling=[SamplingParams(0.8, typical_p=0.5), per[1], None, None])
            caches = _admit(model, B, msl, {0: 10, 1: 12})
        h0 = engine.h2d_bytes
        engine.decode_on_device([1, 2, 0, 0], [10, 12, 0, 0], caches, 4, sampling=per)
        counts.append((engine.kernels_per_step, engine.kernels_per_penalized_step, engine.h2d_bytes - h0))
        if not with_trunc:
            assert engine._graph_pen_trunc is None and engine.mirostat_mu is None and engine._trunc_dev is None
    assert counts[0][:2] == counts[1][:2]
    print(f"kernels per step {counts[0][0]}, per penalised step {counts[0][1]}, upload bytes {counts[0][2]} / {counts[1][2]}")
