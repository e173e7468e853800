"""The keep set of ``sample_kernel`` on the H100, probe by probe (``tests/keep_set_ref.py``): every probe asserts one
token with ``==``, in every kernel form that can run it (``ext.sample``, ``ext.sample_penalized`` with every penalty
off and on, ``ext.sample_constrained`` without and with a state), fp32 / fp16 / bf16, at one vocabulary per cluster
size and at the limits, and from a logits view offset by one element (staging not vectorised).

Which probe catches which defect:
* a threshold kept with ``> tau``: every probe whose target is the boundary entry itself;
* too few radix levels (for bf16, or for penalised rows whose values leave the bf16 grid): the just-outside entries
  one ulp or one key-bucket below x_(k) or v*;
* the k-th count off by one at a bin edge: the top-k boundary probes whose neighbours differ in each key byte;
* a Philox counter without the slice start: the planted winners on the slices of ranks above 0;
* ``x / T`` overflowing for tiny temperatures: the temperature probes (the maximum must win).
The penalised forms must add exactly 1 to ``state[row, token]`` for position > 0 and nothing at position 0; the
constrained forms must advance the row's DFA state by the drawn token."""

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


K = _load("tiny_llm_b200_keep_set_ref", "keep_set_ref.py")
pytestmark = pytest.mark.gpu

# one per cluster size C = 1..8 (sample_plan: C = ceil(V / 4096), at most 8), the 151,936 vocabulary and the limit
VOCABS = [1, 7, 4096, 4097, 8193, 12289, 16385, 20481, 24577, 28673, 151936, 409600]
TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
DFA_STATES = 3  # the probes' DFA: state s moves to (s + byte) % 3 on a token's single byte (token id & 0xFF)


def _seed_i64(s: int) -> int:
    return s - (1 << 64) if s >= 1 << 63 else s


def _constraints(probes, V, dev):
    """One descriptor per probe over a 3-state DFA whose every state allows the probe's tokens, initial state j % 3;
    returns the descriptors, the initial states and the tensors they point into."""
    words = (V + 31) // 32
    masks = np.zeros((len(probes), DFA_STATES + 1, words), dtype=np.uint32)
    for j, pr in enumerate(probes):
        allowed = np.ones(V, bool) if pr.allowed is None else pr.allowed
        bits = np.zeros(words * 32, bool)
        bits[:V] = allowed
        masks[j, :DFA_STATES] = np.packbits(bits, bitorder="little").view("<u4")
    masks_d = torch.from_numpy(masks.view(np.int32)).to(dev)
    dfa = torch.tensor([[(s + b) % DFA_STATES for b in range(256)] for s in range(DFA_STATES)], dtype=torch.int32, device=dev)
    offsets = torch.arange(V + 1, dtype=torch.int32, device=dev)
    data = (torch.arange(V, dtype=torch.int32) & 0xFF).to(torch.uint8).to(dev)
    states = [j % DFA_STATES for j in range(len(probes))]
    row_bytes = (DFA_STATES + 1) * words * 4
    desc = torch.tensor([[masks_d.data_ptr() + j * row_bytes, dfa.data_ptr(), offsets.data_ptr(), data.data_ptr(),
                          DFA_STATES | (s << 32)] for j, s in enumerate(states)], dtype=torch.int64, device=dev)
    return desc, states, (masks_d, dfa, offsets, data)


def _logits(probes, dtype, dev, unaligned):
    x = torch.from_numpy(np.stack([pr.x for pr in probes])).to(TORCH[dtype])
    if not unaligned:
        return x.to(dev)
    flat = torch.empty(x.numel() + 1, dtype=x.dtype, device=dev)
    view = flat[1:].view(x.shape)  # 4 or 2 bytes off a 16-byte boundary: staging takes the scalar path
    view.copy_(x)
    return view


def run(form, probes, dtype, dev, unaligned=False):
    """Launch ``form`` over the probes as one multi-row launch; check the token-state update and the DFA advance of
    every row and return the probes whose token is not the reference's."""
    n, V = len(probes), probes[0].V
    x = _logits(probes, dtype, dev, unaligned)
    temp = torch.tensor([pr.T for pr in probes], dtype=torch.float32, device=dev)
    top_k = torch.tensor([pr.k for pr in probes], dtype=torch.int32, device=dev)
    top_p = torch.tensor([pr.p for pr in probes], dtype=torch.float32, device=dev)
    seed = torch.tensor([_seed_i64(pr.seed) for pr in probes], dtype=torch.int64, device=dev)
    pos = torch.tensor([pr.pos for pr in probes], dtype=torch.int32, device=dev)
    base = (temp, top_k, top_p, seed, pos)
    pen = state0 = None
    if form != "sample" and form != "constrained":
        on = form != "penalized off"
        cols = [[pr.r, pr.pres, pr.freq, pr.min_p] if pr.penalized else ([1.3, 0.5, 0.3, 0.0] if on else [1.0, 0.0, 0.0, 0.0])
                for pr in probes]
        pen = [torch.tensor([c[j] for c in cols], dtype=torch.float32, device=dev) for j in range(4)]
        st = np.stack([pr.state if pr.state is not None else np.zeros(V, np.int32) for pr in probes])
        if not on:  # every penalty off: the state is not read, whatever it holds
            st = np.random.default_rng(V).integers(0, 4, (n, V)).astype(np.int32) | np.int32(1 << 30)
        state0 = torch.from_numpy(st).to(dev)
    state = None if state0 is None else state0.clone()
    desc = None
    if form == "sample":
        got = ext.sample(x, *base)
    elif form.startswith("penalized"):
        got = ext.sample_penalized(x, *base, *pen, state)
    else:
        desc, s0, _keep = _constraints(probes, V, dev)
        got = ext.sample_constrained(x, *base, desc, *(pen or []), *([state] if state is not None else []))
    got = got.cpu().tolist()
    wrong = [f"{form}{' (unaligned)' if unaligned else ''}: got {got[j]}, {pr}" for j, pr in enumerate(probes) if got[j] != pr.want]
    want_tok = torch.tensor(got, dtype=torch.int64)  # the state and the DFA follow the token drawn
    live = torch.tensor([pr.pos > 0 for pr in probes])
    if state is not None:
        d = (state - state0).cpu()
        w = torch.zeros_like(d)
        w[live, want_tok[live]] = 1
        assert torch.equal(d, w), form
    if desc is not None:
        after = desc.view(torch.int32)[:, 9].cpu().tolist()
        assert after == [(s + (t & 0xFF)) % DFA_STATES if pr.pos > 0 else s for s, t, pr in zip(s0, got, probes)], form
    return wrong


_CATALOGUES = {}


def catalogue(V, dtype):
    if (V, dtype) not in _CATALOGUES:
        _CATALOGUES.clear()
        _CATALOGUES[(V, dtype)] = K.Catalogue(V, dtype).probes
    return _CATALOGUES[(V, dtype)]


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("dtype", K.DTYPES)
def test_every_probe_in_every_form(cuda_device, dtype, V):
    probes = catalogue(V, dtype)
    wrong = []
    for form in K.FORMS:
        wrong += run(form, [pr for pr in probes if form in K.forms_of(pr)], dtype, cuda_device)
    if V % 8 == 0:  # vectorised staging above; the same rows from an unaligned view
        for form in ("sample", "penalized on"):
            wrong += run(form, [pr for pr in probes if form in K.forms_of(pr)], dtype, cuda_device, unaligned=True)
    kinds = {pr.kind.split()[0] for pr in probes}
    print(f"V {V} {dtype}: {len(probes)} probes ({sum(pr.inside for pr in probes)} inside), kinds {sorted(kinds)}")
    assert not wrong, f"{len(wrong)} wrong draws:\n" + "\n".join(wrong)


def test_vocab_above_the_limit_is_refused(cuda_device):
    V = 409601
    x = torch.zeros(1, V, dtype=torch.bfloat16, device=cuda_device)
    f = torch.ones(1, dtype=torch.float32, device=cuda_device)
    i = torch.ones(1, dtype=torch.int32, device=cuda_device)
    seed = torch.ones(1, dtype=torch.int64, device=cuda_device)
    state = torch.zeros(1, V, dtype=torch.int32, device=cuda_device)
    desc = torch.zeros(1, 5, dtype=torch.int64, device=cuda_device)
    launches = ext.launch_count()
    for call in (lambda: ext.sample(x, f, i, f, seed, i), lambda: ext.sample_penalized(x, f, i, f, seed, i, f, f, f, f, state),
                 lambda: ext.sample_constrained(x, f, i, f, seed, i, desc), lambda: ext.sample_constrained(x, f, i, f, seed, i, desc, f, f, f, f, state)):
        with pytest.raises(RuntimeError, match="sample: vocab 409601 exceeds 409600"):
            call()
    torch.cuda.synchronize()
    assert ext.launch_count() == launches and torch.equal(state, torch.zeros_like(state))
