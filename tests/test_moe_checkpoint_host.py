"""Qwen3-MoE checkpoints on the host: save/load round trips of both router layouts (the model's own quantisation and
mlx_lm's 8-bit group-64 router), every loader refusal, the float64 router reference, and tl_moe_router's argument
refusals in the C entry and the shim (no device needed)."""

import ctypes
import importlib.util
import json
import sys
from pathlib import Path

import pytest
import torch
from safetensors.torch import load_file, save_file

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.moe import _check_router, router_logits
from tiny_llm_b200.quantize import QuantizedWeights, dequantize_weights
from tiny_llm_b200.synthetic import MOE_KEYS, make_args, named_tensors, synthetic_qwen3



def _load(name, file):
    """The helper next to this file, by path: `tests` is no package of this project."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).resolve().parent / file)
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


R = _load("tiny_llm_b200_moe_router_ref", "moe_router_ref.py")
probe_value, router_ref, unpack8 = R.probe_value, R.router_ref, R.unpack8
LAYOUTS = {"g128": {}, "g64": dict(router_bits=8, router_group_size=64)}


def bits_of(t: torch.Tensor) -> torch.Tensor:
    """The tensor's bytes as integers (equal bits compare equal, NaN patterns included)."""
    return t.contiguous().view(torch.uint8)


def assert_same_model(a, b):
    ta, tb = dict(named_tensors(a)), dict(named_tensors(b))
    assert ta.keys() == tb.keys()
    for name in ta:
        assert ta[name].dtype == tb[name].dtype and ta[name].shape == tb[name].shape, name
        assert torch.equal(bits_of(ta[name]), bits_of(tb[name])), name
    assert vars(a.args) == vars(b.args)
    for la, lb in zip(a.model.layers, b.model.layers):
        for name in ("gate", "switch_mlp", "gate_proj"):
            assert hasattr(la.mlp, name) == hasattr(lb.mlp, name)
        if hasattr(la.mlp, "gate"):
            assert (la.mlp.gate.bits, la.mlp.gate.group_size) == (lb.mlp.gate.bits, lb.mlp.gate.group_size)
            for p in ("gate_proj", "up_proj", "down_proj"):
                ea, eb = getattr(la.mlp.switch_mlp, p), getattr(lb.mlp.switch_mlp, p)
                assert (ea.bits, ea.group_size) == (eb.bits, eb.group_size) == (4, 128)


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_tiny_moe_round_trips_bit_exactly(tmp_path, layout):
    m = synthetic_qwen3("tiny-moe-d128", seed=0, realistic=True, **LAYOUTS[layout])
    save_checkpoint(m, tmp_path)
    config = json.loads((tmp_path / "config.json").read_text())
    assert config["model_type"] == "qwen3_moe"
    assert {k: config[k] for k in MOE_KEYS} == {k: getattr(m.args, k) for k in MOE_KEYS}
    # layer 0 is dense (mlp_only_layers = [0]): only layer 1's router is written as an override
    want = {"group_size": 128, "bits": 4}
    if layout == "g64":
        want["model.layers.1.mlp.gate"] = {"group_size": 64, "bits": 8}
    assert config["quantization"] == want
    loaded = load_checkpoint(tmp_path)
    assert_same_model(m, loaded)
    assert loaded.model.layers[1].mlp.gate.weight.shape == (8, 256 * (8 if layout == "g64" else 4) // 32)
    # a second save of the loaded model writes the same files
    save_checkpoint(loaded, tmp_path / "again")
    assert json.loads((tmp_path / "again" / "config.json").read_text()) == config


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_30b_a3b_shaped_model_round_trips(tmp_path, layout):
    """Two sparse layers of the published Qwen3-30B-A3B shape (128 experts of 768, hidden 2048, untied head); the
    tensors are left uninitialised, so the check is on names, shapes, bits and args."""
    m = synthetic_qwen3("qwen3-30b-a3b", empty=True, num_hidden_layers=2, vocab_size=4096, **LAYOUTS[layout])
    save_checkpoint(m, tmp_path)
    config = json.loads((tmp_path / "config.json").read_text())
    assert config["num_experts"] == 128 and config["moe_intermediate_size"] == 768 and config["tie_word_embeddings"] is False
    overrides = {k for k in config["quantization"] if k.startswith("model.")}
    assert overrides == ({"model.layers.0.mlp.gate", "model.layers.1.mlp.gate"} if layout == "g64" else set())
    loaded = load_checkpoint(tmp_path)
    assert_same_model(m, loaded)
    assert loaded.model.layers[1].mlp.switch_mlp.down_proj.weight.shape == (128, 2048, 768 // 8)


def test_loader_fills_the_moe_defaults_of_make_args(tmp_path):
    m = synthetic_qwen3("tiny-moe-d128", seed=0)
    save_checkpoint(m, tmp_path)
    config = json.loads((tmp_path / "config.json").read_text())
    for key in ("num_experts_per_tok", "norm_topk_prob", "decoder_sparse_step"):
        config.pop(key)
    (tmp_path / "config.json").write_text(json.dumps(config))
    args = load_checkpoint(tmp_path).args
    want = make_args({k: config[k] for k in ("hidden_size", "num_hidden_layers", "num_attention_heads", "num_key_value_heads", "head_dim",
                                             "intermediate_size", "vocab_size", "num_experts", "moe_intermediate_size", "mlp_only_layers")})
    for key in MOE_KEYS:
        assert getattr(args, key) == getattr(want, key), key


# ----------------------------------------------------------------------------------------------------- refusals --
def saved(tmp_path, config_edit=None, tensor_edit=None, **kw):
    save_checkpoint(synthetic_qwen3("tiny-moe-d128", seed=0, **kw), tmp_path)
    config = json.loads((tmp_path / "config.json").read_text())
    if config_edit:
        config_edit(config)
    (tmp_path / "config.json").write_text(json.dumps(config))
    if tensor_edit:
        tensors = load_file(str(tmp_path / "model.safetensors"))
        tensor_edit(tensors)
        save_file(tensors, str(tmp_path / "model.safetensors"))
    return tmp_path


def test_wrong_expert_count_is_refused(tmp_path):
    path = saved(tmp_path, config_edit=lambda c: c.update(num_experts=4))
    with pytest.raises(ValueError, match=r"model\.layers\.1\.mlp\.gate\.weight has shape \(8, 32\), expected \(4, 32\)"):
        load_checkpoint(path)


def test_wrong_expert_shape_is_refused(tmp_path):
    path = saved(tmp_path, config_edit=lambda c: c.update(moe_intermediate_size=256))
    with pytest.raises(ValueError, match=r"switch_mlp\.gate_proj\.weight has shape \(8, 128, 32\), expected \(8, 256, 32\)"):
        load_checkpoint(path)


def test_expert_tensor_of_the_wrong_width_is_refused(tmp_path):
    def narrow(t):
        name = "model.layers.1.mlp.switch_mlp.gate_proj.scales"
        t[name] = t[name][:, :, :1].contiguous()

    with pytest.raises(ValueError, match=r"gate_proj\.scales has shape \(8, 128, 1\), expected \(8, 128, 2\)"):
        load_checkpoint(saved(tmp_path, tensor_edit=narrow))


def test_missing_switch_mlp_tensor_is_refused(tmp_path):
    path = saved(tmp_path, tensor_edit=lambda t: t.pop("model.layers.1.mlp.switch_mlp.up_proj.biases"))
    with pytest.raises(KeyError, match=r"model\.layers\.1\.mlp\.switch_mlp\.up_proj\.biases"):
        load_checkpoint(path)


def test_8_bit_experts_are_refused_by_the_loader(tmp_path):
    save_checkpoint(synthetic_qwen3("tiny-moe-d128", seed=0, bits=8), tmp_path)
    with pytest.raises(ValueError, match="8-bit"):
        load_checkpoint(tmp_path)


@pytest.mark.parametrize("key", ["model.layers.1.mlp.switch_mlp.gate_proj", "model.layers.0.mlp.gate", "model.layers.1.self_attn.q_proj",
                                 "model.embed_tokens"])
def test_override_off_a_sparse_router_is_refused(tmp_path, key):
    path = saved(tmp_path, config_edit=lambda c: c["quantization"].update({key: {"group_size": 64, "bits": 8}}))
    with pytest.raises(ValueError, match=f"{key!r}.*mixed per-layer quantisation"):
        load_checkpoint(path)


@pytest.mark.parametrize("bits, group", [(4, 64), (8, 32), (4, 32)])
def test_router_override_other_than_8_bits_group_64_is_refused(tmp_path, bits, group):
    path = saved(tmp_path, config_edit=lambda c: c["quantization"].update({"model.layers.1.mlp.gate": {"group_size": group, "bits": bits}}))
    with pytest.raises(ValueError, match=r"'model\.layers\.1\.mlp\.gate'.*8 bits / group 64"):
        load_checkpoint(path)


def test_router_override_equal_to_the_global_setting_loads(tmp_path):
    path = saved(tmp_path, config_edit=lambda c: c["quantization"].update({"model.layers.1.mlp.gate": {"group_size": 128, "bits": 4}}))
    assert load_checkpoint(path).model.layers[1].mlp.gate.group_size == 128


def test_router_declared_at_group_64_but_stored_at_128_is_refused(tmp_path):
    path = saved(tmp_path, config_edit=lambda c: c["quantization"].update({"model.layers.1.mlp.gate": {"group_size": 64, "bits": 8}}))
    with pytest.raises(ValueError, match=r"model\.layers\.1\.mlp\.gate\.weight has shape \(8, 32\), expected \(8, 64\)"):
        load_checkpoint(path)


def test_global_group_64_stays_refused(tmp_path):
    path = saved(tmp_path, config_edit=lambda c: c["quantization"].update(group_size=64))
    with pytest.raises(ValueError, match="group_size = 64"):
        load_checkpoint(path)


def test_moe_refuses_a_group_64_router_of_another_width():
    w = QuantizedWeights(scales=torch.ones(8, 4), biases=torch.zeros(8, 4), group_size=64, bits=4, weight=torch.zeros(8, 32, dtype=torch.int32))
    with pytest.raises(ValueError, match="group-64 router must have 8-bit codes"):
        _check_router(w)
    _check_router(QuantizedWeights(scales=torch.ones(8, 4), biases=torch.zeros(8, 4), group_size=64, bits=8, weight=torch.zeros(8, 64, dtype=torch.int32)))


def test_router_selection_keeps_the_caller_projection_for_group_128():
    w = QuantizedWeights(scales=torch.ones(8, 2), biases=torch.zeros(8, 2), group_size=128, bits=4, weight=torch.zeros(8, 32, dtype=torch.int32))
    seen = []
    router_logits(torch.zeros(3, 256), w, projection=lambda h, ww: seen.append((h.shape, ww)) or "projected")
    assert seen == [((3, 256), w)]


def test_synthetic_router_layout_leaves_every_other_draw_alone():
    a = synthetic_qwen3("tiny-moe-d128", seed=3)
    b = synthetic_qwen3("tiny-moe-d128", seed=3, router_bits=8, router_group_size=64)
    assert torch.equal(bits_of(a.model.layers[1].mlp.switch_mlp.gate_proj.weight.view(torch.int32)),
                       bits_of(synthetic_qwen3("tiny-moe-d128", seed=3).model.layers[1].mlp.switch_mlp.gate_proj.weight.view(torch.int32)))
    gate = b.model.layers[1].mlp.gate
    assert (gate.bits, gate.group_size, tuple(gate.weight.shape), tuple(gate.scales.shape)) == (8, 64, (8, 64), (8, 4))
    assert a.model.layers[0].mlp.gate_proj.weight.shape == b.model.layers[0].mlp.gate_proj.weight.shape
    with pytest.raises(ValueError, match="router bits"):
        synthetic_qwen3("tiny-moe-d128", router_bits=8, router_group_size=32)


# ------------------------------------------------------------------------------------------- float64 reference --
def test_router_reference_equals_the_dequantised_product():
    g = torch.Generator().manual_seed(0)
    E, H, T = 8, 256, 5
    codes = torch.randint(0, 256, (E, H), generator=g)
    from tiny_llm_b200.synthetic import pack_codes

    w = pack_codes(codes, 8)
    scales = (torch.randn(E, H // 64, generator=g) * 0.01).to(torch.bfloat16)
    biases = (torch.randn(E, H // 64, generator=g) * 0.1).to(torch.bfloat16)
    x = torch.randn(T, H, generator=g).to(torch.bfloat16)
    assert torch.equal(unpack8(w), codes)
    ref, bound = router_ref(x, w, scales, biases)
    dense = dequantize_weights(w, scales.to(torch.float64), biases.to(torch.float64), 64, 8)
    assert torch.allclose(ref, x.to(torch.float64) @ dense.T, rtol=0, atol=1e-12)
    assert bool((bound > 0).all()) and bool((bound < 0.05 * ref.abs().max()).all())


def test_probe_value_rounds_in_fp32_then_to_the_dtype():
    assert probe_value(0.5, 255, -1.0, 2.0, torch.bfloat16) == 253.0  # 0.5 * 255 * 2 - 2, exact
    assert probe_value(0.5, 255, 0.0, 1.5, torch.bfloat16) == 191.0  # 191.25 rounds to bf16's 8 significant bits
    assert probe_value(0.5, 255, 0.0, 1.5, torch.float16) == 191.25


# ---------------------------------------------------------------------------------------------------- refusals --
def test_c_entry_refuses_bad_arguments():
    lib = ctypes.CDLL(str(ext.current_library_path()))
    f = lib.tl_moe_router
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_float] + [ctypes.c_void_p] * 4 + [ctypes.c_int] * 4 + [ctypes.c_void_p]
    p, null = 16, None
    # tl_moe_router(x, norm_weight, eps, w, scales, biases, logits, T, E, H, dtype, stream)
    assert f(p, null, 0.0, p, p, p, p, 4, 128, 2048, 0, null) == -1  # fp32
    assert f(p, null, 0.0, p, p, p, p, -1, 128, 2048, 2, null) == -1  # rows
    assert f(p, null, 0.0, p, p, p, p, (1 << 19) + 1, 128, 2048, 2, null) == -1  # rows past the limit
    assert f(p, null, 0.0, p, p, p, p, 4, 0, 2048, 2, null) == -1  # no experts
    assert f(p, null, 0.0, p, p, p, p, 4, 257, 2048, 2, null) == -1  # too many experts
    assert f(p, null, 0.0, p, p, p, p, 4, 128, 96, 2, null) == -1  # H % 64
    assert f(p, null, 0.0, p, p, p, p, 4, 128, 0, 1, null) == -1
    for i in (0, 3, 4, 5, 6):  # each required pointer null in turn
        args = [p, null, 0.0, p, p, p, p, 4, 128, 2048, 2, null]
        args[i] = null
        assert f(*args) == -1, i
    assert f(8, null, 0.0, p, p, p, p, 4, 128, 2048, 2, null) == -1  # misaligned x
    assert f(p, null, 0.0, 8, p, p, p, 4, 128, 2048, 2, null) == -1  # misaligned codes
    assert f(p, 8, 0.0, p, p, p, p, 4, 128, 2048, 2, null) == -1  # misaligned norm weight
    assert f(null, null, 0.0, null, null, null, null, 0, 128, 2048, 2, null) == 0  # no rows


def test_c_entry_names_the_failed_argument():
    assert "tl_moe_router" in ext.EXPORTED_SYMBOLS
    f = ext._lib.tl_moe_router
    assert f(16, None, 0.0, 16, 16, 16, 16, 4, 128, 96, 2, None) == -1
    assert "multiple of 64" in ext._lib.tl_last_error().decode()


def shim_args(T=4, E=8, H=256, dtype=torch.bfloat16):
    return (torch.zeros(T, H, dtype=dtype), torch.zeros(E, H // 4, dtype=torch.int32), torch.ones(E, H // 64, dtype=dtype),
            torch.zeros(E, H // 64, dtype=dtype))


@pytest.mark.parametrize("case, message", [
    ("fp32", "float16 or bfloat16"),
    ("h96", "multiple of 64"),
    ("g128_weight", r"packed 8-bit codes \[E, H / 4\]"),
    ("e257", "1 to 256 experts"),
    ("scales_g128", r"\[E, H / 64\]"),
    ("scales_dtype", r"\[E, H / 64\] = \[8, 4\] of x's dtype"),
    ("norm_shape", "norm weight must be"),
    ("norm_dtype", "norm weight must be"),
    ("cpu", "GPU-only"),
])
def test_shim_refuses_before_touching_a_device(case, message):
    x, w, s, b = shim_args()
    kw = {}
    if case == "fp32":
        x = x.float()
    elif case == "h96":
        x, w, s, b = shim_args(H=96)
    elif case == "g128_weight":
        w = torch.zeros(8, 256 // 8, dtype=torch.int32)
    elif case == "e257":
        x, w, s, b = shim_args(E=257)
    elif case == "scales_g128":
        s = b = torch.ones(8, 2, dtype=torch.bfloat16)
    elif case == "scales_dtype":
        s = s.half()
    elif case == "norm_shape":
        kw = dict(norm_weight=torch.ones(128, dtype=torch.bfloat16), eps=1e-6)
    elif case == "norm_dtype":
        kw = dict(norm_weight=torch.ones(256, dtype=torch.float16), eps=1e-6)
    with pytest.raises(RuntimeError, match=message):
        ext.moe_router(x, w, s, b, **kw)
