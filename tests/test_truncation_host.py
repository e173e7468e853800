"""Top-n-sigma, locally typical sampling and Mirostat 2.0 on the host (DESIGN.md section 25): field validation and the
Mirostat refusals, every path that refuses the new samplers, the CLI flags, and the float64 restatement
(``truncation_ref``) against ``transformers``' ``TypicalLogitsWarper`` and llama.cpp's Mirostat 2.0 loop."""

import importlib.util
import math
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


tref = _load("tiny_llm_b200_truncation_ref", "truncation_ref.py")
from oracle import sampling as oref
from tiny_llm_b200 import SamplingParams
from tiny_llm_b200.sampler import any_truncation, mirostat_start, truncation_tensors


# ------------------------------------------------------------------------------------------------ fields --
@pytest.mark.parametrize("kw,name", [(dict(typical_p=0.0), "typical_p"), (dict(typical_p=1.01), "typical_p"), (dict(typical_p=float("nan")), "typical_p"),
                                     (dict(typical_p=True), "typical_p"), (dict(top_n_sigma=-0.5), "top_n_sigma"),
                                     (dict(top_n_sigma=float("inf")), "top_n_sigma"), (dict(mirostat=3), "mirostat"),
                                     (dict(mirostat=2.0), "mirostat"), (dict(mirostat=True), "mirostat"),
                                     (dict(mirostat=2, mirostat_tau=0.0), "mirostat_tau"), (dict(mirostat=2, mirostat_tau=-1.0), "mirostat_tau"),
                                     (dict(mirostat=2, mirostat_eta=float("inf")), "mirostat_eta"), (dict(mirostat_eta=0.0), "mirostat_eta")])
def test_fields_are_validated(kw, name):
    with pytest.raises(ValueError, match=name):
        SamplingParams(0.8, **kw)


def test_mirostat_1_is_refused():
    with pytest.raises(ValueError, match="Mirostat 1.0 is not supported; use mirostat=2"):
        SamplingParams(0.8, mirostat=1)


@pytest.mark.parametrize("kw,name", [(dict(top_k=20), "top_k"), (dict(top_p=0.9), "top_p"), (dict(min_p=0.05), "min_p"),
                                     (dict(typical_p=0.9), "typical_p"), (dict(top_n_sigma=1.0), "top_n_sigma"),
                                     (dict(xtc_probability=0.5), "xtc_probability")])
def test_mirostat_refuses_the_other_truncations(kw, name):
    with pytest.raises(ValueError, match=name):
        SamplingParams(0.8, mirostat=2, **kw)


def test_mirostat_combines_with_penalties_and_inert_settings():
    p = SamplingParams(0.8, mirostat=2, top_k=0, top_p=1.0, repetition_penalty=1.2, dry_multiplier=0.5)
    assert p.penalized and p.truncation and p.controls


def test_defaults_are_off_and_penalized_follows():
    p = SamplingParams(0.8)
    assert (p.typical_p, p.top_n_sigma, p.mirostat, p.mirostat_tau, p.mirostat_eta) == (1.0, 0.0, 0, 5.0, 0.1)
    assert not p.truncation and not p.penalized
    for kw in (dict(typical_p=0.9), dict(top_n_sigma=1.0), dict(mirostat=2)):
        q = SamplingParams(0.8, **kw)
        assert q.truncation and q.penalized and hash(q) is not None
    assert not any_truncation([None, p]) and any_truncation([None, SamplingParams(0.8, typical_p=0.5)])


def test_truncation_tensors_and_mu_start():
    ps = [SamplingParams(0.8, typical_p=0.5), None, SamplingParams(0.8, mirostat=2, mirostat_tau=3.0, mirostat_eta=0.2),
          SamplingParams(0.8, top_n_sigma=1.5, mirostat_tau=9.0)]
    tp, ns, tau, eta = (t.tolist() for t in truncation_tensors(ps, "cpu"))
    assert tp == [0.5, 1.0, 1.0, 1.0] and ns == [0.0, 0.0, 0.0, 1.5]
    assert tau == [0.0, 0.0, 3.0, 0.0] and [round(v, 6) for v in eta] == [0.0, 0.0, 0.2, 0.0]
    assert mirostat_start(ps[2]) == 6.0


# -------------------------------------------------------------------------------------------- refusals --
NEW = [(dict(typical_p=0.9), "typical_p"), (dict(top_n_sigma=1.0), "top_n_sigma"), (dict(mirostat=2), "mirostat")]


@pytest.mark.parametrize("kw,name", NEW)
def test_speculative_and_lookup_refuse(kw, name):
    from tiny_llm_b200.generate import _spec_sampling

    with pytest.raises(ValueError, match=name):
        _spec_sampling(SamplingParams(0.8, **kw), None)


@pytest.mark.parametrize("kw,name", NEW)
def test_keep_logits_refuses(kw, name):
    from tiny_llm_b200.engine import DecodeEngine

    # keep_logits is refused before the engine touches the device
    engine = DecodeEngine.__new__(DecodeEngine)
    engine.log_capacity = 8
    engine.B = 1
    with pytest.raises(ValueError, match=name):
        DecodeEngine.decode_on_device(engine, [0], [0], None, 1, sampling=SamplingParams(0.8, **kw), keep_logits=True)


def _parsed(monkeypatch, argv):
    from tiny_llm_b200 import cli

    seen = {}
    for name in ("cmd_generate", "cmd_batch"):
        monkeypatch.setattr(cli, name, lambda args: seen.setdefault("args", args) and 0)
    cli.main(argv)
    return seen["args"]


def test_cli_parses_the_flags(monkeypatch):
    from tiny_llm_b200.cli import _penalties

    a = _parsed(monkeypatch, ["generate", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3", "--sampler-temp", "0.8", "--typical-p", "0.9",
                              "--top-n-sigma", "1.5", "--seed", "3"])
    assert _penalties(a) == dict(typical_p=0.9, top_n_sigma=1.5)
    a = _parsed(monkeypatch, ["batch", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3", "--mirostat", "2", "--mirostat-tau", "4",
                              "--mirostat-eta", "0.2"])
    assert _penalties(a) == dict(mirostat=2, mirostat_tau=4.0, mirostat_eta=0.2)
    a = _parsed(monkeypatch, ["generate", "--synthetic", "tiny-d128", "--prompt-ids", "5,17,3"])
    assert _penalties(a) == {}
    with pytest.raises(SystemExit):
        _parsed(monkeypatch, ["generate", "--synthetic", "tiny-d128", "--mirostat", "1"])


@pytest.mark.parametrize("flags,name", [(["--typical-p", "0.9"], "--typical-p"), (["--top-n-sigma", "1"], "--top-n-sigma"),
                                        (["--mirostat", "2"], "--mirostat")])
@pytest.mark.parametrize("mode", [["--num-beams", "2"], ["--prompt-lookup", "3"], ["--draft-synthetic", "tiny-d128"]])
def test_cli_refuses_beams_and_proposers(flags, name, mode):
    from tiny_llm_b200.cli import main

    with pytest.raises(SystemExit) as e:
        main(["generate", "--synthetic", "tiny-d128", "--device", "cpu", "--prompt-ids", "5,17,3", *mode, *flags])
    assert name in str(e.value)


# ------------------------------------------------------------------------------------------- reference --
def _rows(n, V, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        x = (rng.standard_normal(V) * rng.choice([0.5, 2.0, 5.0])).astype(np.float32)
        if i % 3 == 1:
            x[rng.random(V) < 0.1] = -np.inf
        out.append(x)
    return out


@pytest.mark.parametrize("mass", [0.2, 0.5, 0.9, 0.99])
def test_typical_equals_transformers(mass):
    pytest.importorskip("transformers")
    import torch
    from transformers.generation.logits_process import TypicalLogitsWarper

    warper = TypicalLogitsWarper(mass=mass)
    checked = near = 0
    for x in _rows(60, 300, int(mass * 100)):
        keep, close = tref.typical_keep(x, np.isfinite(x), mass)
        out = warper(None, torch.from_numpy(x.astype(np.float64))[None]).numpy()[0]
        hf = np.isfinite(out) & np.isfinite(x)
        mine_np = tref.hf_typical_keep(x, mass) & np.isfinite(x)
        if close:
            near += 1
            continue
        assert np.array_equal(keep, hf)
        assert np.array_equal(keep, mine_np)
        checked += 1
    assert checked >= 50, (checked, near)


def test_typical_keeps_ties_and_the_smallest_distance():
    x = np.array([0.0, -1.0, -1.0, -3.0, -np.inf], np.float32)
    keep, _ = tref.typical_keep(x, np.isfinite(x), 0.01)
    _, d = tref.typical_distances(x, np.isfinite(x))
    assert keep[np.argmin(d)] and keep.sum() >= 1
    for p in np.linspace(0.05, 0.95, 19):
        keep, _ = tref.typical_keep(x, np.isfinite(x), float(p))
        assert keep[1] == keep[2] and not keep[4]


def test_nsigma_bound():
    x = np.array([0.0, -2.0, -np.inf, np.nan], np.float32)
    assert tref.nsigma_bound(x, 2.0) == -2.0
    keep, _ = tref.nsigma_keep(x, ~np.isnan(x), 2.0)
    assert keep.tolist() == [True, True, False, False]
    keep, _ = tref.nsigma_keep(x, ~np.isnan(x), float(np.nextafter(np.float32(2), np.float32(0))))
    assert keep.tolist() == [True, False, False, False]
    one = np.array([-np.inf, 3.0, 3.0], np.float32)
    keep, _ = tref.nsigma_keep(one, np.ones(3, bool), 5.0)  # sigma 0: the maximum's ties stay
    assert keep.tolist() == [False, True, True]


@pytest.mark.parametrize("T,tau,eta", [(1.0, 3.0, 0.1), (0.7, 5.0, 0.05), (1.3, 1.0, 1.0), (1.0, 8.0, 0.1)])
def test_mirostat_equals_llama_cpp_over_64_steps(T, tau, eta):
    V = 500
    rng = np.random.default_rng(int(tau * 10 + eta * 100))
    mu_mine = mu_llama = float(np.float32(2 * tau))
    for step in range(64):
        x = (rng.standard_normal(V) * 3).astype(np.float32)
        keep, p, near = tref.mirostat_keep(x, T, mu_mine)
        score = np.where(keep, oref.perturbed(x.astype(np.float64), T, 42, step + 1), -np.inf)
        token = int(np.argmax(score))

        def pick(ids, q, token=token):
            return int(np.flatnonzero(ids == token)[0])

        if not near:
            t2, mu2, kept = tref.llama_mirostat_v2(x, T, mu_llama, tau, eta, pick)
            assert np.array_equal(kept, np.flatnonzero(keep)) and t2 == token
            mu_mine = tref.mirostat_update(p, keep, token, mu_mine, tau, eta)
            assert abs(mu_mine - mu2) <= 1e-5 * max(1.0, abs(mu2)), step
            mu_llama = mu_mine  # fp32 state, as the kernel keeps it
        else:
            mu_llama = mu_mine = tref.mirostat_update(p, keep, token, mu_mine, tau, eta)
    assert math.isfinite(mu_mine)


def test_mirostat_keeps_the_maximum_when_mu_is_low():
    x = np.array([1.0, 0.5, -2.0], np.float32)
    keep, _, _ = tref.mirostat_keep(x, 1.0, -3.0)
    assert keep.tolist() == [True, False, False]
    keep, _, _ = tref.mirostat_keep(np.array([0.0, 0.0, 0.0, 0.0], np.float32), 1.0, 2.0)
    assert keep.all()
