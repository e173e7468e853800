"""The speculative-sampling and XTC probe catalogues (``tests/rejection_probe_ref.py``) on the host: every probe's token
is the independent whole-row rule's, and every defect of the mutation table gets at least one probe wrong, at every
(V, dtype) where it can show."""

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


P = _load("tiny_llm_b200_rejection_probe_ref", "rejection_probe_ref.py")
K, R, X = P.K, P.R, P.X

# Defects that cannot show at a (V, C): the reason is the exemption.  At V = 1 the one entry is both rows' point mass,
# so only a proposal outside the row (d = -1, d = V) can be decided wrongly; XTC's A has at most one member there.
SPEC_EXEMPT = {
    "p_d, q_d read from rank 0": (lambda V, C: C < 2, "one CTA: rank 0 holds every entry"),
    "residual noise without the slice start": (lambda V, C: C < 2, "one CTA: every slice starts at 0"),
}
XTC_EXEMPT = {
    "A per CTA": (lambda V, C: C < 2, "one CTA holds the whole row"),
    "A's minimum from rank 0": (lambda V, C: C < 2, "one CTA holds the whole row"),
}
SPEC_AT_V1 = {"no q_d > 0 guard"}

_CACHE = {}


def _catalogue(kind, V, dtype):
    if (kind, V, dtype) not in _CACHE:
        _CACHE.clear()
        _CACHE[(kind, V, dtype)] = (P.SpecCatalogue if kind == "spec" else P.XtcCatalogue)(V, dtype)
    return _CACHE[(kind, V, dtype)]


def test_noise_and_uniforms_equal_the_reference_streams():
    V = 4097
    idx = [0, 3, 4, 2055, 2056, 4096]
    for seed, pos in ((0x1234_5678_9ABC_DEF0, 977), (1 << 63 | 5, 1)):
        for stream in (0, 1, 2, 3):
            np.testing.assert_array_equal(P.noise_at(idx, seed, pos, stream), R.residual_gumbel(V, seed, pos, stream)[idx])
        assert P.u_odd_at(seed, [pos], 1)[0] / P.U_ONE == R.accept_uniform(seed, pos)
        assert P.u_odd_at(seed, [pos], 3)[0] / P.U_ONE == X.xtc_uniform(seed, pos)
        np.testing.assert_array_equal(P.noise_at(idx, seed, pos, 0), K.gumbel_at(idx, seed, pos))


@pytest.mark.parametrize("V", P.SPEC_VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_speculative_probes_are_the_rules_tokens(V, dtype):
    cat = _catalogue("spec", V, dtype)
    assert cat.probes and {pr.accepted for pr in cat.probes} == ({False} if V == 1 else {True, False})
    for pr in cat.probes:
        dec = P.spec_rule(pr)
        assert dec.token == pr.want and dec.accepted == pr.accepted, pr
        if pr.exact:  # the rule on the same masses in float64 (no tie is near: u is an odd multiple of 2^-24)
            p = P.row_dist(pr.x, pr.T, pr.k, pr.p, True)
            q = P.row_dist(pr.y, pr.T, pr.k, pr.p, True)
            want = R.decide(p.p, q.p, pr.d, pr.seed, pr.pos, ref.greedy(pr.x))
        else:  # the whole-row float64 rule, REL clear of its acceptance boundary
            want = R.rule_row(pr.x, pr.y, pr.d, pr.T, pr.k, pr.p, pr.seed, pr.pos)
            if 0 <= pr.d < V:
                pd = R.row_dist(pr.x, pr.T, pr.k, pr.p)[pr.d]
                qd = R.row_dist(pr.y, pr.T, pr.k, pr.p)[pr.d]
                assert want.margin >= P.REL * max(pd, qd), pr
        assert want.token == pr.want and want.accepted == pr.accepted, (want, pr)
        assert want.residual_gap >= P.MARGIN, pr
    b = cat.bonus
    assert R.rule([b.x], [], [], [b.T], [b.k], [b.p], [b.seed], [b.pos])[0].token == b.want


@pytest.mark.parametrize("V", P.XTC_VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_xtc_probes_are_the_rules_tokens(V, dtype):
    cat = _catalogue("xtc", V, dtype)
    assert cat.probes
    for pr in cat.probes:
        st = np.zeros(V, np.int32) if pr.state is None else pr.state
        token, near = X.xtc_sample_row(pr.x, st, pr.T, pr.k, pr.p, pr.seed, pr.pos, pr.r, pr.pres, pr.freq, pr.min_p, pr.theta, pr.q,
                                       pr.allowed)
        assert not near and token == pr.want, pr
        assert P.xtc_rule(pr)[0] == pr.want, pr
    if V >= 7:  # the gate: q == u does not fire, q one ulp above u does
        gates = {pr.kind: pr for pr in cat.probes if pr.kind.startswith("gate")}
        assert gates["gate q == u"].q == P._xtc_u(gates["gate q == u"].seed, gates["gate q == u"].pos)
        assert gates["gate q == u"].want == gates["gate q == u"].pre != gates["gate q above u"].want


def _alive(kind, V, dtype, variant):
    cat = _catalogue(kind, V, dtype)
    rule = (lambda pr: P.spec_rule(pr, variant).token) if kind == "spec" else (lambda pr: P.xtc_rule(pr, variant)[0])
    return all(rule(pr) == pr.want for pr in cat.probes)


@pytest.mark.parametrize("V", P.SPEC_VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_every_speculative_defect_is_caught(V, dtype):
    C = K.plan(V)[0]
    report = {}
    for variant in P.SPEC_VARIANTS:
        exempt = SPEC_EXEMPT.get(variant)
        if (V == 1 and variant not in SPEC_AT_V1) or (exempt and exempt[0](V, C)):
            report[variant] = "exempt"
            continue
        report[variant] = "alive" if _alive("spec", V, dtype, variant) else "killed"
    print(f"speculative V {V} {dtype}: " + ", ".join(f"{v}: {s}" for v, s in report.items()))
    assert not [v for v, s in report.items() if s == "alive"], report


@pytest.mark.parametrize("V", P.XTC_VOCABS)
@pytest.mark.parametrize("dtype", P.DTYPES)
def test_every_xtc_defect_is_caught(V, dtype):
    C = K.plan(V)[0]
    report = {}
    for variant in P.XTC_VARIANTS:
        exempt = XTC_EXEMPT.get(variant)
        if V == 1 or (exempt and exempt[0](V, C)):
            report[variant] = "exempt"
            continue
        report[variant] = "alive" if _alive("xtc", V, dtype, variant) else "killed"
    print(f"XTC V {V} {dtype}: " + ", ".join(f"{v}: {s}" for v, s in report.items()))
    assert not [v for v, s in report.items() if s == "alive"], report
