"""The float64 sampling reference (``oracle/sampling.py``) on the host: Philox4x32-10 known answers, keep sets against
the in-tree sampler's rule, tied top-k boundaries, and the distribution of seeded draws."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import sampling as ref


def _frontdoor():
    """``test_frontdoor_host.py`` by path: `tests` is no package of this project."""
    name = "tiny_llm_b200_test_frontdoor_host"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("test_frontdoor_host.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


@pytest.mark.parametrize("counter,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(counter, key, want):
    assert tuple(int(w) for w in ref.philox4x32_10(np.array(counter), key)) == want


def test_uniforms_are_exact_in_fp32_and_inside_the_open_interval():
    u = ref.uniforms(4099, seed=(7 << 32) | 11, pos=12345)
    assert np.array_equal(u.astype(np.float32).astype(np.float64), u)
    assert (u > 0).all() and (u < 1).all()
    # seed and position select different streams; the word of entry i is word i % 4 of group i >> 2
    assert not np.array_equal(u, ref.uniforms(4099, seed=11, pos=12345))
    assert not np.array_equal(u, ref.uniforms(4099, seed=(7 << 32) | 11, pos=12346))
    w = ref.philox4x32_10(np.array([2, 12345, 0, 0]), (11, 7))
    assert u[9] == (2.0 * (int(w[1]) >> 9) + 1.0) * 2.0**-24


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("top_k", [None, 1, 2, 5, 39])
@pytest.mark.parametrize("top_p", [None, 0.05, 0.35, 0.6, 0.9, 0.999])
def test_keep_set_equals_the_reference_sampler_rule_on_untied_rows(seed, top_k, top_p):
    logits = torch.randn(40, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * (1 + seed)
    logprobs = (logits - torch.logsumexp(logits, dim=0)).tolist()
    want = _frontdoor().reference_sampler_keep_set(logprobs, top_p, top_k)
    got = set(np.flatnonzero(ref.keep_set(np.array(logprobs), top_k, top_p)).tolist())
    assert got == want


def test_tied_top_k_boundary_keeps_every_tie():
    x = np.array([3.0, 1.0, 2.0, 2.0, 2.0, 0.5, 2.0])
    assert np.flatnonzero(ref.keep_set(x, 2, None)).tolist() == [0, 2, 3, 4, 6]
    assert np.flatnonzero(ref.keep_set(x, 5, None)).tolist() == [0, 2, 3, 4, 6]
    assert np.flatnonzero(ref.keep_set(x, 6, None)).tolist() == [0, 1, 2, 3, 4, 6]
    # ties share the mass strictly above them: all four 2.0 entries are kept or none is
    M, _ = ref.mass_above(x)
    assert len(set(M[[2, 3, 4, 6]].tolist())) == 1
    p0 = float(np.exp(3.0) / np.exp(x).sum())
    assert np.flatnonzero(ref.keep_set(x, None, p0 + 1e-9)).tolist() == [0, 2, 3, 4, 6]
    assert np.flatnonzero(ref.keep_set(x, None, p0)).tolist() == [0]


def test_greedy_rules_and_nan():
    assert ref.sample_row(np.array([1.0, 5.0, 5.0, 2.0]), 0.0, None, None, 0, 0) == 1
    assert ref.sample_row(np.array([np.nan, 1.0, np.nan]), 0.0, None, None, 0, 0) == 1
    assert ref.sample_row(np.array([np.nan, np.nan]), 0.7, None, None, 0, 0) == 0
    assert ref.sample_row(np.array([-np.inf, -np.inf]), 0.7, None, None, 0, 0) == 0
    assert ref.sample_row(np.array([0.0, np.inf, 1.0, np.inf]), 0.7, None, None, 0, 0) == 1
    for pos in range(50):  # NaN is never drawn
        assert ref.sample_row(np.array([0.1, np.nan, 0.2, np.nan]), 1.5, None, None, 3, pos) in (0, 2)


@pytest.mark.parametrize("temperature,top_k,top_p", [(1.0, None, None), (0.7, 4, None), (1.5, None, 0.8), (0.5, 6, 0.9)])
def test_draws_over_positions_follow_the_renormalised_target(temperature, top_k, top_p):
    """200,000 positions of one row under one seed: the token counts against softmax(x / T) on the keep set
    (chi-square, p = 1e-6)."""
    x = np.array([1.2, -0.3, 0.8, 2.0, -1.5, 0.0, 1.9, -0.7, 0.4, 1.1])
    n = 200_000
    keep = ref.keep_set(x, top_k, top_p)
    ctr = np.zeros((n, 3, 4), dtype=np.uint64)
    ctr[:, :, 0] = np.arange(3, dtype=np.uint64)
    ctr[:, :, 1] = np.arange(n, dtype=np.uint64)[:, None]
    words = ref.philox4x32_10(ctr, (1234, 0)).reshape(n, 12)[:, : len(x)].astype(np.uint64)
    u = (2.0 * (words >> np.uint64(9)).astype(np.float64) + 1.0) * 2.0**-24
    score = np.where(keep, x / temperature - np.log(-np.log(u)), -np.inf)
    drawn = score.argmax(axis=1)
    # the vectorised draw is the reference's
    for pos in (0, 1, 777, n - 1):
        assert drawn[pos] == ref.sample_row(x, temperature, top_k, top_p, 1234, pos)
    target = np.where(keep, np.exp((x - x.max()) / temperature), 0.0)
    target /= target.sum()
    counts = np.bincount(drawn, minlength=len(x))
    assert (counts[~keep] == 0).all()
    chi2, pvalue = stats.chisquare(counts[keep], n * target[keep])
    assert pvalue > 1e-6, (chi2, pvalue)
