"""DRY and XTC on the host (DESIGN.md section 24): field validation, the contract's restatement against a brute-force
port of text-generation-webui's loop, the DRY row packing, the CLI flags and every refusal."""

import random

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


dref = _load("tiny_llm_b200_dry_xtc_ref", "dry_xtc_ref.py")
from tiny_llm_b200 import dry
from tiny_llm_b200.cli import parse_dry_xtc
from tiny_llm_b200.logit_controls import ControlRows
from tiny_llm_b200.sampler import SamplingParams


@pytest.mark.parametrize("kw, field", [
    (dict(dry_multiplier=-1.0), "dry_multiplier"),
    (dict(dry_multiplier=float("inf")), "dry_multiplier"),
    (dict(dry_multiplier=0.5, dry_base=1.0), "dry_base"),
    (dict(dry_multiplier=0.5, dry_base=float("nan")), "dry_base"),
    (dict(dry_multiplier=0.5, dry_allowed_length=0), "dry_allowed_length"),
    (dict(dry_multiplier=0.5, dry_allowed_length=2.5), "dry_allowed_length"),
    (dict(dry_multiplier=0.5, dry_penalty_last_n=-1), "dry_penalty_last_n"),
    (dict(dry_multiplier=0.5, dry_sequence_breakers="abc"), "dry_sequence_breakers"),
    (dict(dry_multiplier=0.5, dry_sequence_breakers=[-1]), "dry_sequence_breakers"),
    (dict(dry_multiplier=0.5, dry_sequence_breakers=list(range(65))), "dry_sequence_breakers"),
    (dict(xtc_probability=1.5), "xtc_probability"),
    (dict(xtc_probability=-0.1), "xtc_probability"),
    (dict(xtc_probability=0.5, xtc_threshold=0.0), "xtc_threshold"),
    (dict(xtc_probability=0.5, xtc_threshold=1.5), "xtc_threshold"),
])
def test_fields_are_validated_by_name(kw, field):
    with pytest.raises(ValueError, match=field):
        SamplingParams(0.7, **kw)


def test_fields_normalise_and_flag():
    p = SamplingParams(0.7, dry_multiplier=0.8, dry_sequence_breakers=[9, 3, 3], xtc_probability=0.5)
    assert p.dry_sequence_breakers == (3, 9) and hash(p) == hash(SamplingParams(0.7, dry_multiplier=0.8, dry_sequence_breakers=(3, 9),
                                                                                 xtc_probability=0.5))
    assert p.dry and p.controls and p.xtc and p.penalized
    off = SamplingParams(0.7)
    assert not off.dry and not off.xtc and not off.controls and not off.penalized
    assert (off.dry_base, off.dry_allowed_length, off.dry_penalty_last_n, off.xtc_threshold) == (1.75, 2, 0, 0.1)


def _histories(rng: random.Random):
    """Random and adversarial histories: periodic repeats, self-overlapping runs, breakers inside and at the end."""
    out = []
    for _ in range(1500):
        n = rng.randint(1, 120)
        kind = rng.randrange(5)
        if kind == 0:
            h = [rng.randrange(6) for _ in range(n)]
        elif kind == 1:
            period = [rng.randrange(20) for _ in range(rng.randint(1, 6))]
            h = (period * (n // len(period) + 1))[:n]
        elif kind == 2:
            h = [rng.randrange(2)] * n  # "a a a a": matches overlap their suffix
        elif kind == 3:
            h = [rng.randrange(50) for _ in range(n)]
        else:
            period = [rng.randrange(8) for _ in range(rng.randint(2, 5))]
            h = (period * (n // len(period) + 1))[:n]
            for _ in range(rng.randint(0, 3)):
                h[rng.randrange(n)] = rng.randrange(8)
        breakers = rng.sample(range(8), rng.randint(0, 2)) if rng.random() < 0.5 else ()
        if breakers and rng.random() < 0.2:
            h[-1] = breakers[0]
        last_n = rng.choice([0, 0, 1, 2, 5, 17, n, n + 3])
        out.append((h, tuple(breakers), last_n))
    # matches at and past the cap
    out.append(([1, 2] * 100, (), 0))
    out.append(([3] * 150, (), 0))
    out.append(([3] * 150, (), 70))
    return out


def test_restatement_equals_the_brute_force_loop():
    rng = random.Random(7)
    V = 64
    for h, brk, last_n in _histories(rng):
        x = np.asarray([rng.uniform(-8, 8) for _ in range(V)], dtype=np.float32)
        for m, b, a in ((0.8, 1.75, 2), (1.0, 3.0, 1), (2.0, 1.1, 4)):
            want = dref.webui_dry(x, h, m, b, a, last_n, brk)
            got = dref.dry_penalize(x, h, m, b, a, last_n, brk)
            np.testing.assert_array_equal(got, want, err_msg=f"{h} {brk} {last_n} {(m, b, a)}")


def test_cap_and_overflow():
    h = [3] * 200
    lengths = dref.match_lengths(h, ())
    assert lengths == {3: 64}
    P = dry.penalty_table(1.0, 1.75, 2)
    assert P[0] == 1.0 and P[62] == np.float32(1.75**62) and P[62] > 1e15 and not P[63]
    assert np.isinf(dry.penalty_table(1e30, 10.0, 1)[20])
    y = dref.dry_penalize(np.zeros(8, np.float32), h, 1e30, 10.0, 1)
    assert np.isneginf(y[3]) and not np.isinf(y[:3]).any()


def test_row_packing_round_trips():
    p = SamplingParams(0.7, dry_multiplier=0.8, dry_base=2.0, dry_allowed_length=3, dry_penalty_last_n=100, dry_sequence_breakers=(11, 5))
    row = dry.pack_row(p)
    assert row.shape == (dry.ROW_WORDS,) and row.dtype == np.int32
    back = dry.unpack_row(row)
    assert back["flags"] == dry.FLAG_ON and back["dry_allowed_length"] == 3 and back["dry_penalty_last_n"] == 100
    assert back["dry_sequence_breakers"] == (5, 11)
    np.testing.assert_array_equal(back["penalty"], dref.penalty_table(0.8, 2.0, 3))
    assert not dry.pack_row(SamplingParams(0.7)).any() and not dry.pack_row(None).any()


def test_control_rows_carry_the_dry_table():
    p = SamplingParams(0.7, dry_multiplier=0.8)
    tab = ControlRows(2, 100, "cpu", history_capacity=16)
    assert tab.dry is None
    assert tab.set_row(1, p, [4, 5, 6], [7]) == 7
    assert tab.dry is not None and tab.dry.history[1, :4].tolist() == [4, 5, 6, 7] and tab.dry.table[1, 0] == dry.FLAG_ON
    assert tab.descriptors[1].any()  # a DRY-only row is a controlled row that copies its logits
    tab.clear_row(1)
    assert not tab.dry.table[1].any() and not tab.descriptors[1].any()
    with pytest.raises(ValueError, match="history capacity"):
        ControlRows(1, 100, "cpu").set_row(0, p, [1, 2], [])
    with pytest.raises(ValueError, match="exceeds its capacity"):
        ControlRows(1, 100, "cpu", history_capacity=2).set_row(0, p, [1, 2, 3], [])


class _Tok:
    def encode(self, text, add_special_tokens=False):
        return [ord(c) for c in text]


def test_cli_parsing():
    assert parse_dry_xtc() == {}
    got = parse_dry_xtc(0.8, 1.5, 3, 64, "13,198", 0.2, 0.5)
    assert got == dict(dry_multiplier=0.8, dry_base=1.5, dry_allowed_length=3, dry_penalty_last_n=64, dry_sequence_breakers=[13, 198],
                       xtc_probability=0.5, xtc_threshold=0.2)
    got = parse_dry_xtc(0.8, dry_sequence_breakers='["\\n", ":", "ab"]', tokenizer=_Tok())
    assert got["dry_sequence_breakers"] == [ord("\n"), ord(":"), ord("b")]  # the last id of encode("a" + s)
    with pytest.raises(ValueError, match="tokenizer"):
        parse_dry_xtc(0.8, dry_sequence_breakers='["\\n"]')
    with pytest.raises(ValueError, match="dry-sequence-breakers"):
        parse_dry_xtc(0.8, dry_sequence_breakers="1,x")
    SamplingParams(0.7, **parse_dry_xtc(0.8, dry_sequence_breakers='[":"]', tokenizer=_Tok(), xtc_probability=1.0))


def test_cli_flags_exist():
    from tiny_llm_b200 import cli

    src = open(cli.__file__).read()
    for flag in ("--dry-multiplier", "--dry-base", "--dry-allowed-length", "--dry-penalty-last-n", "--dry-sequence-breakers",
                 "--xtc-threshold", "--xtc-probability"):
        assert f'"{flag}"' in src


def test_refusals_name_the_field():
    from tiny_llm_b200 import generate

    p = SamplingParams(0.7, dry_multiplier=0.8)
    q = SamplingParams(0.7, xtc_probability=0.5)
    for sp, field in ((p, "dry_multiplier"), (q, "xtc_probability")):
        with pytest.raises(ValueError, match=field):
            generate._spec_sampling(sp, None)  # speculative decoding and prompt lookup
    with pytest.raises(ValueError, match="dry_multiplier"):
        generate._check_parallel_args(None, [[1, 2]], 2, p, 4, None, None)


def test_dry_refuses_a_constraint():
    from tiny_llm_b200.constrained import TokenConstraint

    c = TokenConstraint.__new__(TokenConstraint)  # the type check only: no device tables needed
    with pytest.raises(ValueError, match="dry_multiplier takes no constraint"):
        SamplingParams(0.7, dry_multiplier=0.8, constraint=c)
