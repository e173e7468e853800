"""The truncation probe catalogues (``tests/truncation_probe_ref.py``) on the host: every probe's token and mu' are the
kernel rule's under every ``expf`` shift and ``truncation_ref``'s outside its bands, the typical and Mirostat probes
agree with the outside definitions where those coincide, and every defect of the mutation table gets at least one probe
wrong, at every (V, dtype) where it can show."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


P = _load("tiny_llm_b200_truncation_probe_ref", "truncation_probe_ref.py")
K, TR = P.K, P.TR

# Defects that cannot show at a (V, C): the reason is the exemption.  Below V = 8 only the one-entry probes and (from
# V = 4) Mirostat's ties are built.
EXEMPT = {
    "> at the crossing": (lambda V, C: True, "a mass exactly at typical_p S_K needs an exactly known expf other than expf(0)"),
    "mu read from rank 0": (lambda V, C: C < 2, "one CTA: rank 0 holds every entry"),
}
AT_SMALL_V = {"no 2^40 cap", "> at the threshold", "mu read one entry on"}

_CACHE = {}


def _catalogue(V, dtype):
    if (V, dtype) not in _CACHE:
        _CACHE.clear()
        _CACHE[(V, dtype)] = P.Catalogue(V, dtype)
    return _CACHE[(V, dtype)]


def _right(pr, d) -> bool:
    return d.token == pr.want and pr.mu_lo <= d.mu <= pr.mu_hi


@pytest.mark.parametrize("V", P.VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_probes_are_the_rules_tokens(V, dtype):
    cat = _catalogue(V, dtype)
    assert cat.probes
    for pr in cat.probes:
        for shift in P.SHIFTS:
            d = P.trunc_rule(pr, shift=shift)
            assert _right(pr, d), (shift, d.token, d.mu, pr)
        token, mu, near = P.whole_row(pr)
        assert not near and token == pr.want, (token, near, pr)
        if pr.mirostat and pr.pos > 0 and not P._support(pr).point:
            assert TR.mu_close(pr.mu_lo, mu, pr.eta) and TR.mu_close(pr.mu_hi, mu, pr.eta), (mu, pr)
            assert pr.mu_hi - pr.mu_lo <= 2.0**-18 * max(1.0, abs(mu)), pr  # far tighter than the 2^-16 eta band
        else:
            assert mu == pr.mu_lo == pr.mu_hi == float(np.float32(pr.mu)), (mu, pr)


@pytest.mark.parametrize("V", [7, 4097, 28673, 151936])
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_outside_definitions_where_they_coincide(V, dtype):
    """Typical probes over the whole row (no other cut, no mask) keep what ``transformers``' warper keeps; Mirostat
    probes without penalties or masks, at mu >= 0, keep what llama.cpp's loop keeps and give its mu' within the band."""
    cat = _catalogue(V, dtype)
    typ = miro = 0
    for pr in cat.probes:
        s = P._support(pr)
        if s.point or pr.allowed is not None or pr.state is not None:
            continue
        d = P.trunc_rule(pr)
        if 0 < pr.typical_p < 1 and not pr.mirostat and pr.k == 0 and pr.min_p == 0 and pr.n_sigma == 0:
            assert np.array_equal(TR.hf_typical_keep(s.full, pr.typical_p)[s.J], d.keep), pr
            typ += 1
        if pr.mirostat and pr.pos > 0 and pr.mu >= 0:  # below 0 llama.cpp keeps one tie of the maximum, the kernel all
            want = int(np.flatnonzero(s.J == pr.want)[0])  # on the finite entries alone (-log2 0 has no value)

            def pick(idx, q, want=want):
                return int(np.flatnonzero(idx == want)[0])

            token, mu, kept = TR.llama_mirostat_v2(s.x, pr.T, float(np.float32(pr.mu)), float(np.float32(pr.tau)),
                                                     float(np.float32(pr.eta)), pick)
            assert token == want and np.array_equal(s.J[kept], np.sort(s.J[d.keep])), pr
            assert TR.mu_close(pr.mu_lo, mu, pr.eta), (mu, pr)
            miro += 1
    print(f"V {V} {dtype}: {typ} typical and {miro} Mirostat probes against the outside definitions")
    assert V < 8 or (typ and miro)


@pytest.mark.parametrize("V", P.VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_every_truncation_defect_is_caught(V, dtype):
    cat = _catalogue(V, dtype)
    C = K.plan(V)[0]
    report = {}
    for variant in P.VARIANTS:
        exempt = EXEMPT.get(variant)
        if V == 1 or (V < 8 and variant not in AT_SMALL_V) or (exempt and exempt[0](V, C)):
            report[variant] = "exempt" + (f" ({exempt[1]})" if exempt and exempt[0](V, C) else "")
            continue
        alive = all(_right(pr, P.trunc_rule(pr, variant)) for pr in cat.probes)
        report[variant] = "alive" if alive else "killed"
    print(f"V {V} {dtype}: " + ", ".join(f"{v}: {s}" for v, s in report.items()))
    assert not [v for v, s in report.items() if s == "alive"], report
