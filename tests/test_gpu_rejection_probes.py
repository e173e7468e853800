"""Speculative sampling's accept / residual rule and XTC's exclusion on the H100, probe by probe
(``tests/rejection_probe_ref.py``): every probe asserts one token with ``==``, with no tolerance and no skipped draw.

* ``tl_speculative_sample``: one launch per (V, dtype) holds every probe row and the bonus row, fp32 / fp16 / bf16 at
  one vocabulary per cluster size and at the 204,800 limit; again from views offset by one element (scalar staging);
  one launch replayed under a CUDA graph.
* XTC: ``ext.sample_penalized`` with every penalty off and on, and ``ext.sample_constrained`` with the penalty state
  (XTC needs it), all with the XTC arrays, at the same vocabularies and 409,600.  The penalised forms must add exactly 1
  to ``state[row, token]`` for position > 0; the constrained form must advance the row's DFA by the drawn token.
"""

import collections
import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


P = _load("tiny_llm_b200_rejection_probe_ref", "rejection_probe_ref.py")
K = P.K
pytestmark = pytest.mark.gpu

TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
DFA_STATES = 3  # state s moves to (s + byte) % 3 on a token's single byte (token id & 0xFF)
_CACHE = {}
SEEN = collections.defaultdict(set)  # class -> {(cluster size, dtype)} compared on the GPU


def _seed_i64(s: int) -> int:
    return s - (1 << 64) if s >= 1 << 63 else s


def _catalogue(kind, V, dtype):
    if (kind, V, dtype) not in _CACHE:
        _CACHE.clear()
        _CACHE[(kind, V, dtype)] = (P.SpecCatalogue if kind == "spec" else P.XtcCatalogue)(V, dtype)
    return _CACHE[(kind, V, dtype)]


def _rows(arrays, dtype, dev, unaligned):
    x = torch.from_numpy(np.stack(arrays)).to(TORCH[dtype])
    if not unaligned:
        return x.to(dev)
    flat = torch.empty(x.numel() + 1, dtype=x.dtype, device=dev)
    view = flat[1:].view(x.shape)  # 2 or 4 bytes off a 16-byte boundary: staging takes the scalar path
    view.copy_(x)
    return view


# ------------------------------------------------------------------------------------- speculative sample --
def _spec_args(cat, dev, unaligned=False):
    rows = cat.probes + [cat.bonus]
    x = _rows([pr.x for pr in rows], cat.dtype, dev, unaligned)
    y = _rows([pr.y for pr in cat.probes], cat.dtype, dev, unaligned)
    d = torch.tensor([pr.d for pr in cat.probes], dtype=torch.int32, device=dev)
    f = lambda vals, dt: torch.tensor(vals, dtype=dt, device=dev)  # noqa: E731
    return (x, y, d, f([pr.T for pr in rows], torch.float32), f([pr.k for pr in rows], torch.int32), f([pr.p for pr in rows], torch.float32),
            f([_seed_i64(pr.seed) for pr in rows], torch.int64), f([pr.pos for pr in rows], torch.int32))


def _spec_wrong(cat, got, label):
    rows = cat.probes + [cat.bonus]
    return [f"{label}: got {g}, {pr}" for g, pr in zip(got, rows) if g != pr.want]


@pytest.mark.parametrize("V", P.SPEC_VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_speculative_sample_probes(cuda_device, dtype, V):
    cat = _catalogue("spec", V, dtype)
    args = _spec_args(cat, cuda_device)
    wrong = _spec_wrong(cat, ext.speculative_sample(*args).cpu().tolist(), "aligned")
    if V % 8 == 0:  # the rows above staged with 16-byte loads; the same rows from unaligned views
        wrong += _spec_wrong(cat, ext.speculative_sample(*_spec_args(cat, cuda_device, True)).cpu().tolist(), "unaligned")
    if (V, dtype) == (12289, "f16"):  # one launch replayed under a CUDA graph
        out = torch.empty(len(cat.probes) + 1, dtype=torch.int32, device=cuda_device)
        ext.speculative_sample(*args, out=out)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ext.speculative_sample(*args, out=out)
        out.fill_(-1)
        graph.replay()
        torch.cuda.synchronize()
        wrong += _spec_wrong(cat, out.cpu().tolist(), "graph replay")
    C = K.plan(V)[0]
    counts = collections.Counter(pr.kind for pr in cat.probes)
    for kind in counts:
        SEEN["spec " + kind].add((C, dtype))
    acc = sum(pr.accepted for pr in cat.probes)
    print(f"speculative V {V} (C {C}) {dtype}: {len(cat.probes)} probes, {acc} accepted, {dict(counts)}")
    assert not wrong, f"{len(wrong)} wrong tokens:\n" + "\n".join(wrong)


# ---------------------------------------------------------------------------------------------------- XTC --
def _constraints(probes, V, dev):
    """One descriptor per probe over a 3-state DFA whose every state allows the probe's tokens, initial state j % 3."""
    words = (V + 31) // 32
    masks = np.zeros((len(probes), DFA_STATES + 1, words), dtype=np.uint32)
    for j, pr in enumerate(probes):
        bits = np.zeros(words * 32, bool)
        bits[:V] = True if pr.allowed is None else pr.allowed
        masks[j, :DFA_STATES] = np.packbits(bits, bitorder="little").view("<u4")
    masks_d = torch.from_numpy(masks.view(np.int32)).to(dev)
    dfa = torch.tensor([[(s + b) % DFA_STATES for b in range(256)] for s in range(DFA_STATES)], dtype=torch.int32, device=dev)
    offsets = torch.arange(V + 1, dtype=torch.int32, device=dev)
    data = (torch.arange(V, dtype=torch.int32) & 0xFF).to(torch.uint8).to(dev)
    states = [j % DFA_STATES for j in range(len(probes))]
    row_bytes = (DFA_STATES + 1) * words * 4
    desc = torch.tensor([[masks_d.data_ptr() + j * row_bytes, dfa.data_ptr(), offsets.data_ptr(), data.data_ptr(), DFA_STATES | (s << 32)]
                         for j, s in enumerate(states)], dtype=torch.int64, device=dev)
    return desc, states, (masks_d, dfa, offsets, data)


def _xtc_run(form, probes, dtype, dev, unaligned=False):
    n, V = len(probes), probes[0].V
    x = _rows([pr.x for pr in probes], dtype, dev, unaligned)
    f = lambda vals, dt: torch.tensor(vals, dtype=dt, device=dev)  # noqa: E731
    base = (f([pr.T for pr in probes], torch.float32), f([pr.k for pr in probes], torch.int32), f([pr.p for pr in probes], torch.float32),
            f([_seed_i64(pr.seed) for pr in probes], torch.int64), f([pr.pos for pr in probes], torch.int32))
    on = form != "penalized off"
    cols = [[pr.r, pr.pres, pr.freq, pr.min_p] if pr.penalized else ([1.3, 0.5, 0.3, 0.0] if on else [1.0, 0.0, 0.0, 0.0]) for pr in probes]
    pen = [f([c[j] for c in cols], torch.float32) for j in range(4)]
    st = np.stack([pr.state if pr.state is not None else np.zeros(V, np.int32) for pr in probes])
    if not on:  # every penalty off: the state is not read, whatever it holds
        st = np.random.default_rng(V).integers(0, 4, (n, V)).astype(np.int32) | np.int32(1 << 30)
    state0 = torch.from_numpy(st).to(dev)
    state = state0.clone()
    xtc = dict(xtc_threshold=f([pr.theta for pr in probes], torch.float32), xtc_probability=f([pr.q for pr in probes], torch.float32))
    desc = None
    if form.startswith("penalized"):
        got = ext.sample_penalized(x, *base, *pen, state, **xtc)
    else:
        desc, s0, _keep = _constraints(probes, V, dev)
        got = ext.sample_constrained(x, *base, desc, *pen, state, **xtc)
    got = got.cpu().tolist()
    wrong = [f"{form}{' (unaligned)' if unaligned else ''}: got {got[j]}, {pr}" for j, pr in enumerate(probes) if got[j] != pr.want]
    tok = torch.tensor(got, dtype=torch.int64)
    live = torch.tensor([pr.pos > 0 for pr in probes])
    dstate = (state - state0).cpu()
    w = torch.zeros_like(dstate)
    w[live, tok[live]] = 1
    assert torch.equal(dstate, w), form
    if desc is not None:
        after = desc.view(torch.int32)[:, 9].cpu().tolist()
        assert after == [(s + (t & 0xFF)) % DFA_STATES if pr.pos > 0 else s for s, t, pr in zip(s0, got, probes)], form
    return wrong


@pytest.mark.parametrize("V", P.XTC_VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_xtc_probes(cuda_device, dtype, V):
    cat = _catalogue("xtc", V, dtype)
    wrong = []
    for form in P.XTC_FORMS:
        wrong += _xtc_run(form, [pr for pr in cat.probes if form in P.xtc_forms_of(pr)], dtype, cuda_device)
    if V % 8 == 0:
        wrong += _xtc_run("penalized on", [pr for pr in cat.probes if "penalized on" in P.xtc_forms_of(pr)], dtype, cuda_device, unaligned=True)
    C = K.plan(V)[0]
    counts = collections.Counter(pr.kind for pr in cat.probes)
    for kind in counts:
        SEEN["xtc " + kind].add((C, dtype))
    print(f"XTC V {V} (C {C}) {dtype}: {len(cat.probes)} probes, {dict(counts)}")
    assert not wrong, f"{len(wrong)} wrong tokens:\n" + "\n".join(wrong)


def test_every_class_reached_every_cluster_size_and_dtype():
    """Runs after the launches above: every probe class was compared at every cluster size it can be built at, in
    every dtype (the classes that need 7 entries start at V = 7, those that need two ranks at C = 2)."""
    if not SEEN:
        pytest.skip("no probe launch ran in this session")
    need = {(C, dt) for C in range(1, 9) for dt in P.DTYPES}
    missing = {}
    for kind, seen in sorted(SEEN.items()):
        want = {(C, dt) for C, dt in need if not (kind == "xtc one member of A per rank" and C == 1)}
        print(f"{kind}: {len(seen)} (cluster size, dtype) pairs")
        if want - seen:
            missing[kind] = sorted(want - seen)
    assert not missing, missing
