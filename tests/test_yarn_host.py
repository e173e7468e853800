"""YaRN RoPE scaling and the graph engines' context window on the host: the frequency table and attention factor against
the literal Qwen3-4B values and the float64 definition (``yarn_ref.py``), config parsing and its round trip through a
checkpoint, refusal of other scaling types, the CLI flags, and the KV-page reservation arithmetic and its refusal."""

import importlib.util
import json
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from tiny_llm_b200 import cli
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.qwen3_week2 import Qwen3ModelWeek2
from tiny_llm_b200.qwen3_week3 import Qwen3ModelWeek3, check_kv_reservation, kv_reservation_bytes, kv_reservation_pages
from tiny_llm_b200.rope_scaling import Yarn, parse_cli, parse_rope_scaling, rope_inv_freq, yarn_correction_range
from tiny_llm_b200.synthetic import make_args, synthetic_qwen3


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


_ref = _load("tiny_llm_b200_yarn_ref", "yarn_ref.py")
yarn_mscale, yarn_table = _ref.yarn_mscale, _ref.yarn_table

QWEN3_YARN = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}


def test_qwen3_4b_literal_values():
    y = parse_rope_scaling(QWEN3_YARN, 40960)
    assert yarn_correction_range(y, 1e6, 128) == (23.0, 40.0)
    table = rope_inv_freq(128, 1e6, y, "cpu").numpy()
    ref, extrap, low, high = yarn_table(1e6, 128, 4.0, 32768)
    assert (low, high) == (23, 40)
    i = np.arange(64)
    plain = rope_inv_freq(128, 1e6, None, "cpu").numpy()
    assert np.array_equal(table[i <= 23], plain[i <= 23])
    assert round(table[24] / plain[24], 5) == 0.95588
    assert np.allclose(table[i >= 40] / plain[i >= 40], 0.25, rtol=1e-15, atol=0)
    np.testing.assert_allclose(table, ref, rtol=1e-14, atol=0)
    assert round(y.mscale, 10) == 1.1386294361 and round(y.mscale**2, 10) == 1.2964769928
    assert y.mscale == yarn_mscale(4.0) and y.window == 131072


def test_table_matches_the_definition_over_a_range_of_configs():
    for theta, D, s, L0 in ((1e6, 128, 4.0, 64), (1e4, 64, 2.0, 4096), (5e5, 128, 8.0, 8192), (1e6, 128, 1.0, 32768)):
        y = parse_rope_scaling({"rope_type": "yarn", "factor": s, "original_max_position_embeddings": L0}, 1)
        got = rope_inv_freq(D, theta, y, "cpu").numpy()
        np.testing.assert_allclose(got, yarn_table(theta, D, s, L0)[0], rtol=1e-14, atol=0)


def test_degenerate_ramp_gets_its_thousandth():
    y = Yarn(4.0, 6, beta_fast=32.0, beta_slow=1.0)  # corr(32) < 0 and -1 < corr(1) < 0 -> low = high = 0
    assert yarn_correction_range(y, 1e6, 128) == (0.0, 0.001)
    assert yarn_table(1e6, 128, 4.0, 6)[2:] == (0, 0.001)
    np.testing.assert_allclose(rope_inv_freq(128, 1e6, y, "cpu").numpy(), yarn_table(1e6, 128, 4.0, 6)[0], rtol=1e-14, atol=0)


def test_explicit_attention_factor_and_betas():
    y = parse_rope_scaling({**QWEN3_YARN, "attention_factor": 1.5, "beta_fast": 16, "beta_slow": 2}, 40960)
    assert y.mscale == 1.5 and (y.beta_fast, y.beta_slow) == (16.0, 2.0)
    assert parse_rope_scaling(y.to_config(), 40960) == y
    assert parse_rope_scaling({"rope_type": "yarn", "factor": 2.0}, 40960).original_max_position_embeddings == 40960


@pytest.mark.parametrize("kind", ["linear", "dynamic", "llama3", "longrope", "su"])
def test_other_scaling_types_are_refused(kind):
    with pytest.raises(ValueError, match="not supported"):
        parse_rope_scaling({"rope_type": kind, "factor": 2.0}, 4096)
    with pytest.raises(ValueError, match="not supported"):
        parse_rope_scaling({"type": kind, "factor": 2.0}, 4096)


@pytest.mark.parametrize("bad", [{"rope_type": "yarn"}, {"rope_type": "yarn", "factor": 0.5}, {"rope_type": "yarn", "factor": float("nan")},
                                 {"rope_type": "yarn", "factor": 2.0, "attention_factor": -1.0}, {"rope_type": "yarn", "factor": 2.0, "beta_fast": 0.5}])
def test_bad_yarn_parameters_are_refused(bad):
    with pytest.raises(ValueError):
        parse_rope_scaling(bad, 4096)


@pytest.mark.parametrize("key", ["mscale", "mscale_all_dim", "truncate", "finetuned"])
def test_yarn_keys_it_does_not_compute_are_refused(key):
    with pytest.raises(ValueError, match="not supported"):
        parse_rope_scaling({**QWEN3_YARN, key: 1.0}, 40960)


def test_no_scaling_forms():
    assert parse_rope_scaling(None, 1) is None and parse_rope_scaling({}, 1) is None and parse_rope_scaling({"rope_type": "default"}, 1) is None


def _tiny_dir(tmp_path, **over):
    ns = synthetic_qwen3("tiny", seed=0, **over)
    save_checkpoint(ns, tmp_path)
    return ns


def test_checkpoint_round_trip_keeps_rope_scaling(tmp_path):
    ns = _tiny_dir(tmp_path, rope_scaling=QWEN3_YARN)
    assert json.loads((tmp_path / "config.json").read_text())["rope_scaling"] == QWEN3_YARN
    back = load_checkpoint(tmp_path)
    assert back.args.rope_scaling == ns.args.rope_scaling == QWEN3_YARN


def test_checkpoint_without_scaling_has_none(tmp_path):
    _tiny_dir(tmp_path)
    assert "rope_scaling" not in json.loads((tmp_path / "config.json").read_text())
    assert getattr(load_checkpoint(tmp_path).args, "rope_scaling", None) is None


@pytest.mark.parametrize("kind", ["linear", "dynamic", "llama3"])
def test_checkpoint_with_another_scaling_type_is_refused(tmp_path, kind):
    _tiny_dir(tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    cfg["rope_scaling"] = {"rope_type": kind, "factor": 4.0}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="not supported"):
        load_checkpoint(tmp_path)


def test_make_args_checks_rope_scaling():
    assert make_args("tiny", rope_scaling=QWEN3_YARN).rope_scaling == QWEN3_YARN
    assert not hasattr(make_args("tiny"), "rope_scaling") and not hasattr(make_args("tiny", rope_scaling=None), "rope_scaling")
    with pytest.raises(ValueError):
        make_args("tiny", rope_scaling={"rope_type": "linear", "factor": 2.0})


def test_week3_model_on_the_host_folds_m_squared_into_the_scale():
    plain = Qwen3ModelWeek3(synthetic_qwen3("tiny", seed=0), page_size=4)
    yarn = Qwen3ModelWeek3(synthetic_qwen3("tiny", seed=0, rope_scaling={"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 64}),
                           page_size=4)
    m = 0.1 * math.log(4.0) + 1
    for a, b in zip(plain.layers_inner, yarn.layers_inner):
        assert a.self_attn.scale == 32**-0.5 and a.self_attn.rope.inv_freq is None
        assert b.self_attn.scale == 32**-0.5 * m * m
        assert b.self_attn.rope.inv_freq is yarn.rope_inv_freq  # one table per model
    assert plain.rope_inv_freq is None and yarn.rope_inv_freq.dtype == torch.float64 and yarn.rope_inv_freq.shape == (16,)


def test_week2_model_refuses_yarn():
    with pytest.raises(ValueError, match="does not implement RoPE scaling"):
        Qwen3ModelWeek2(synthetic_qwen3("tiny", seed=0, rope_scaling=QWEN3_YARN))


def test_cli_rope_scaling_and_max_context_flags(monkeypatch):
    seen = {}
    monkeypatch.setattr(cli, "cmd_generate", lambda args: seen.setdefault("generate", args) and 0)
    monkeypatch.setattr(cli, "cmd_batch", lambda args: seen.setdefault("batch", args) and 0)
    monkeypatch.setattr(cli, "cmd_score", lambda args: seen.setdefault("score", args) and 0)
    for name in ("generate", "batch", "score"):
        ap_args = [name, "--synthetic", "tiny", "--rope-scaling", "yarn:4:32768", "--max-context", "131072"]
        cli.main(ap_args)
    for name in ("generate", "batch", "score"):
        assert seen[name].rope_scaling == QWEN3_YARN and seen[name].max_context == 131072
    assert parse_cli("yarn:2.5") == {"rope_type": "yarn", "factor": 2.5}


@pytest.mark.parametrize("argv", [
    ["generate", "--synthetic", "tiny", "--rope-scaling", "linear:4"],
    ["generate", "--synthetic", "tiny", "--rope-scaling", "yarn"],
    ["generate", "--synthetic", "tiny", "--rope-scaling", "yarn:x"],
    ["generate", "--synthetic", "tiny", "--rope-scaling", "yarn:0.5"],
    ["generate", "--model", "/nonexistent", "--rope-scaling", "yarn:4"],
    ["generate", "--synthetic", "tiny", "--max-context", "0"],
    ["score", "--synthetic", "tiny", "--max-context", "x"],
    ["batch", "--synthetic", "tiny", "--max-context", "256", "--max-seq-len", "512"],
])
def test_cli_refuses_bad_flags(argv):
    with pytest.raises(SystemExit):
        cli.main(argv)


def test_reservation_arithmetic_at_qwen3_4b():
    # (B + 1) * ceil(W / page) + 1 pages per layer; a 128-slot page of 8 KV heads x 128 dims, K and V in bf16, is 512 KiB,
    # 18 MiB across 36 layers
    assert kv_reservation_pages(131072, 128, 1) == 2 * 1024 + 1
    assert kv_reservation_pages(8192, 128, 4) == 5 * 64 + 1
    assert kv_reservation_pages(1000, 128, 1) == 2 * 8 + 1
    per_page = 2 * 8 * 128 * 128 * 2
    assert per_page * 36 == 18 << 20
    need = kv_reservation_bytes(36, 8, 128, 128, 131072, 1)
    assert need == 36 * 2049 * per_page
    assert 36.0 < need / 2**30 < 36.1


def test_reservation_refusal_message():
    check_kv_reservation(100, 100, 8192, 1)
    with pytest.raises(MemoryError, match=r"context window 131072 for 1 slot\(s\) needs 38673580032 bytes \(36\.02 GiB\).*only 1073741824 bytes"):
        check_kv_reservation(kv_reservation_bytes(36, 8, 128, 128, 131072, 1), 1 << 30, 131072, 1)


def test_window_setter_on_the_host():
    model = Qwen3ModelWeek3(synthetic_qwen3("tiny", seed=0), page_size=16)
    assert model.max_context == 8192 == model.decode_graph_max_seq_len
    model.set_max_context(1000)
    assert model.max_context == 1008  # whole pages
    assert Qwen3ModelWeek3(synthetic_qwen3("tiny", seed=0), page_size=16, max_context=131072).decode_graph_max_seq_len == 131072
    with pytest.raises(ValueError):
        model.set_max_context(0)
    assert model.kv_reservation_bytes(1008, 2) == kv_reservation_bytes(2, 2, 32, 16, 1008, 2)
