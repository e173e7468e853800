"""The planted-winner probe builder (``tests/keep_set_ref.py``) on the host: ``gumbel_at`` against
``oracle.sampling.gumbel``, and every probe of a catalogue against the whole-row references, so the tokens the GPU test
asserts are the references' tokens."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest

from oracle import sampling as ref


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


K = _load("tiny_llm_b200_keep_set_ref", "keep_set_ref.py")


@pytest.mark.parametrize("V", [7, 4097, 28673, 151936])
def test_gumbel_at_equals_the_whole_row(V):
    rng = np.random.default_rng(V)
    C, s = K.plan(V)
    idx = sorted({0, V - 1, *[r * s - d for r in range(1, C) for d in (0, 1)], *rng.integers(0, V, 64).tolist()})
    for seed, pos in ((0, 0), (1 << 63 | 12345, 1), (0xFFFFFFFF, (1 << 31) - 1), (0x1234_5678_9ABC_DEF0, 977)):
        full = ref.gumbel(V, seed, pos)
        np.testing.assert_array_equal(K.gumbel_at(idx, seed, pos), full[idx])
    ps = np.array([3, 99, 2**31 - 1])
    many = K.gumbel_at(idx, 42, ps)
    for j, p in enumerate(ps):
        np.testing.assert_array_equal(many[j], ref.gumbel(V, 42, int(p))[idx])


def test_keys_and_level_splits():
    for v in (0.0, -0.0, 1.5, -1.5, 1e-45, -3.4e38, float("inf"), float("-inf")):
        assert K.from_key(K.key(v)) == float(np.float32(v))
    assert K.key(0.0) == K.key(-0.0) and K.key(-1e-45) < K.key(0.0) < K.key(1e-45)
    for dtype, levels in (("f32", (0, 1, 2, 3)), ("f16", (0, 1, 2)), ("bf16", (0, 1))):
        for level in levels:
            for v0 in (1.53125, 300.0) + ((-0.71875,) if dtype == "f32" else ()):  # the catalogue's uses
                a, b = K.split_at_level(v0, level, dtype)
                assert K.next_below(a, dtype) == b


@pytest.mark.parametrize("V", [1, 7, 4097, 12289])
@pytest.mark.parametrize("dtype", K.DTYPES)
def test_every_probe_is_the_references_token(V, dtype):
    probes = K.Catalogue(V, dtype).probes
    assert probes
    for pr in probes:
        want = K.draw(pr)  # penalties_ref.sample_row, or the masked row through oracle.sampling
        assert want == pr.want, pr
        if not pr.penalized and pr.allowed is None:
            assert ref.sample_row(pr.x.astype(np.float64), pr.T, pr.k, pr.p, pr.seed, pr.pos) == pr.want, pr
        if pr.keep is not None:
            assert bool(pr.keep[pr.target]) == pr.inside, pr
            assert pr.inside == (pr.want == pr.target), pr
            assert pr.keep[pr.want], pr
    if V >= 4097:
        kinds = {pr.kind.split()[0] for pr in probes}
        assert {"top-k", "top-p", "k/p", "min-p", "penalised", "mask", "temperature", "pos"} <= kinds
        assert sum(pr.inside for pr in probes) and sum(not pr.inside for pr in probes)


def test_the_penalised_bf16_probe_of_the_issue():
    """The case that motivated the probes: raw 1.53125 and a prompt token 2.0 under repetition 1.3 (1.5384616) share a
    16-bit key bucket; top-k 1 keeps the penalised one alone."""
    p = np.float32(2.0) / np.float32(1.3)
    assert K.key(p) >> 16 == K.key(1.53125) >> 16 and p > 1.53125
    probes = [pr for pr in K.Catalogue(4097, "bf16").probes if pr.kind.startswith("penalised repetition +")]
    assert len(probes) == 4 and {pr.inside for pr in probes} == {True, False}
    for pr in probes:
        st = pr.staged()
        t, other = pr.planted[0], pr.planted[1]
        assert K.key(st[t]) >> 16 == K.key(st[other]) >> 16 and st[other] < st[t]
