"""Top-n-sigma, locally typical sampling and Mirostat 2.0 on the H100, probe by probe (``tests/truncation_probe_ref.py``):
every probe asserts one token with ``==``, with no tolerance and no skipped draw, and every row's mu' exactly or within
the emulated ``expf`` interval.

One launch per (V, dtype, form) holds every probe row of the form, at one vocabulary per cluster size, 151,936, 204,800
and 409,600, in fp32, fp16 and bf16:

* ``ext.sample_penalized`` with every penalty off (the state is junk that must not be read) and on;
* ``ext.sample_constrained`` with the penalty state and a 3-state DFA whose every state allows the probe's tokens.

Non-Mirostat rows carry a sentinel mu and a junk eta that must stay unread.  The penalised forms must add exactly 1 to
``state[row, token]`` for position > 0; the constrained form must advance the row's DFA by the drawn token.  The
"penalized on" launch is repeated from views offset by one element (scalar staging), and one launch is replayed under
a CUDA graph.
"""

import collections
import importlib.util
import sys
import time
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


P = _load("tiny_llm_b200_truncation_probe_ref", "truncation_probe_ref.py")
K = P.K
pytestmark = pytest.mark.gpu

TORCH = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
DFA_STATES = 3  # state s moves to (s + byte) % 3 on a token's single byte (token id & 0xFF)
SEEN = collections.defaultdict(set)  # class -> {(cluster size, dtype)} compared on the GPU
TIMES = {}


def _seed_i64(s: int) -> int:
    return s - (1 << 64) if s >= 1 << 63 else s


def _rows(arrays, dtype, dev, unaligned):
    x = torch.from_numpy(np.stack(arrays)).to(TORCH[dtype])
    if not unaligned:
        return x.to(dev)
    flat = torch.empty(x.numel() + 1, dtype=x.dtype, device=dev)
    view = flat[1:].view(x.shape)  # 2 or 4 bytes off a 16-byte boundary: staging takes the scalar path
    view.copy_(x)
    return view


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


class Launch:
    """The device arrays of one launch over ``probes`` in ``form``."""

    def __init__(self, form, probes, dtype, dev, unaligned=False):
        self.form, self.probes = form, probes
        n, V = len(probes), probes[0].V
        f = lambda vals, dt: torch.tensor(vals, dtype=dt, device=dev)  # noqa: E731
        self.x = _rows([pr.x for pr in probes], dtype, dev, unaligned)
        self.base = (f([pr.T for pr in probes], torch.float32), f([pr.k for pr in probes], torch.int32),
                     f([pr.p for pr in probes], torch.float32), f([_seed_i64(pr.seed) for pr in probes], torch.int64),
                     f([pr.pos for pr in probes], torch.int32))
        on = form != "penalized off"
        cols = [[pr.r, pr.pres, pr.freq, pr.min_p] if pr.penalized else ([1.3, 0.5, 0.3, 0.0] if on else [1.0, 0.0, 0.0, 0.0])
                for pr in probes]
        self.pen = [f([c[j] for c in cols], torch.float32) for j in range(4)]
        st = np.stack([pr.state if pr.state is not None else np.zeros(V, np.int32) for pr in probes])
        if not on:  # every penalty off: the state is not read, whatever it holds
            st = np.random.default_rng(V).integers(0, 4, (n, V)).astype(np.int32) | np.int32(1 << 30)
        self.state0 = torch.from_numpy(st).to(dev)
        self.state = self.state0.clone()
        self.mu0 = f([pr.mu for pr in probes], torch.float32)
        self.mu = self.mu0.clone()
        self.kw = dict(xtc_threshold=f([pr.theta for pr in probes], torch.float32), xtc_probability=f([pr.q for pr in probes], torch.float32),
                       typical_p=f([pr.typical_p for pr in probes], torch.float32), top_n_sigma=f([pr.n_sigma for pr in probes], torch.float32),
                       mirostat_tau=f([pr.tau for pr in probes], torch.float32), mirostat_eta=f([pr.eta for pr in probes], torch.float32))
        self.desc = self.s0 = self._keep = None
        if not form.startswith("penalized"):
            self.desc, self.s0, self._keep = _constraints(probes, V, dev)

    def run(self):
        if self.desc is None:
            return ext.sample_penalized(self.x, *self.base, *self.pen, self.state, mirostat_mu=self.mu, **self.kw)
        return ext.sample_constrained(self.x, *self.base, self.desc, *self.pen, self.state, mirostat_mu=self.mu, **self.kw)

    def check(self, got, label):
        """Tokens, mu', the penalty state and the DFA state after one launch -> the wrong rows."""
        got = got.cpu().tolist()
        mu = self.mu.cpu().numpy()
        wrong = []
        for j, pr in enumerate(self.probes):
            if got[j] != pr.want:
                wrong.append(f"{label}: got {got[j]}, {pr}")
            elif not (pr.mu_lo <= float(mu[j]) <= pr.mu_hi):
                wrong.append(f"{label}: mu' {float(mu[j])!r}, {pr}")
        tok = torch.tensor(got, dtype=torch.int64)
        live = torch.tensor([pr.pos > 0 for pr in self.probes])
        dstate = (self.state - self.state0).cpu()
        w = torch.zeros_like(dstate)
        w[live, tok[live]] = 1
        assert torch.equal(dstate, w), label
        if self.desc is not None:
            after = self.desc.view(torch.int32)[:, 9].cpu().tolist()
            assert after == [(s + (t & 0xFF)) % DFA_STATES if pr.pos > 0 else s for s, t, pr in zip(self.s0, got, self.probes)], label
        return wrong


def _run(form, probes, dtype, dev, unaligned=False):
    L = Launch(form, probes, dtype, dev, unaligned)
    return L.check(L.run(), form + (" (unaligned)" if unaligned else ""))


@pytest.mark.parametrize("V", P.VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_truncation_probes(cuda_device, dtype, V):
    t0 = time.perf_counter()
    cat = P.Catalogue(V, dtype)
    t1 = time.perf_counter()
    wrong = []
    for form in P.FORMS:
        rows = [pr for pr in cat.probes if form in P.forms_of(pr)]
        if rows:
            wrong += _run(form, rows, dtype, cuda_device)
    if V % 8 == 0:
        wrong += _run("penalized on", [pr for pr in cat.probes if "penalized on" in P.forms_of(pr)], dtype, cuda_device, unaligned=True)
    if (V, dtype) == (12289, "bf16"):  # one launch replayed under a CUDA graph
        L = Launch("constrained + state", [pr for pr in cat.probes if "constrained + state" in P.forms_of(pr)], dtype, cuda_device)
        stream = torch.cuda.Stream()
        with torch.cuda.stream(stream):
            L.run()  # warm-up outside the graph
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = L.run()
        L.state.copy_(L.state0)  # the warm-up drew once: back to the starting state, mu and DFA states
        L.mu.copy_(L.mu0)
        L.desc.view(torch.int32)[:, 9] = torch.tensor(L.s0, dtype=torch.int32, device=cuda_device)
        out.fill_(-1)
        graph.replay()
        torch.cuda.synchronize()
        wrong += L.check(out, "graph replay")
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    C = K.plan(V)[0]
    counts = collections.Counter(pr.kind for pr in cat.probes)
    for kind in counts:
        SEEN[kind].add((C, dtype))
    exact = sum(pr.mirostat and pr.pos > 0 and pr.mu_exact for pr in cat.probes)
    TIMES[(V, dtype)] = (t1 - t0, t2 - t1)
    print(f"truncation V {V} (C {C}) {dtype}: {len(cat.probes)} probes, {exact} exact mu', catalogue {t1 - t0:.2f} s, "
          f"launches {t2 - t1:.2f} s")
    assert not wrong, f"{len(wrong)} wrong rows:\n" + "\n".join(wrong)


def test_every_class_reached_every_cluster_size_and_dtype():
    """Runs after the launches above: every probe class was compared at every cluster size it can be built at, in
    every dtype (most classes start at V = 8; Mirostat's ties at V = 4)."""
    if not SEEN:
        pytest.skip("no probe launch ran in this session")
    need = {(C, dt) for C in range(1, 9) for dt in P.DTYPES}
    missing = {}
    for kind, seen in sorted(SEEN.items()):
        print(f"{kind}: {len(seen)} (cluster size, dtype) pairs")
        if need - seen:
            missing[kind] = sorted(need - seen)
    total = sum(a + b for a, b in TIMES.values())
    print(f"{len(TIMES)} (V, dtype) pairs in {total:.1f} s (catalogues {sum(a for a, _ in TIMES.values()):.1f} s)")
    assert not missing, missing
