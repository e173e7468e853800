"""8-bit (W8A16) support on the host: packing and the affine quantiser against dequantize_weights, synthetic 8-bit
checkpoints through save/load, the loader's refusals, the shim's bit inference and argument errors, the C siblings in
the header and the shim, the CLI flag and the streamed-bytes count."""

import json
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3
from tiny_llm_b200.checkpoint import load_checkpoint, save_checkpoint
from tiny_llm_b200.quantize import dequantize_weights
from tiny_llm_b200.synthetic import make_args, pack_codes, quantize_affine, quantize_w4, synthetic_qwen3, weight_stream_bytes


def test_pack_codes_round_trips_through_dequantize_weights():
    g = torch.Generator().manual_seed(0)
    codes = torch.randint(0, 256, (8, 256), generator=g)
    codes[0, :4] = torch.tensor([0, 127, 128, 255])
    words = pack_codes(codes, 8)
    assert words.shape == (8, 64) and words.dtype == torch.uint32
    ones = torch.ones(8, 2, dtype=torch.float32)
    assert torch.equal(dequantize_weights(words, ones, torch.zeros_like(ones), 128, 8), codes.to(torch.float32))
    assert (int(words.view(torch.int32)[0, 0]) & 0xFFFFFFFF) == 0xFF80_7F00  # code j of a word in bits 8j..8j+7


def test_affine_quantiser_at_8_bits_decodes_within_half_a_step():
    g = torch.Generator().manual_seed(1)
    w = torch.randn(16, 384, generator=g)
    words, scales, biases = quantize_affine(w, 8)
    assert words.shape == (16, 96) and scales.shape == biases.shape == (16, 3)
    back = dequantize_weights(words, scales.float(), biases.float(), 128, 8)
    step = scales.float().repeat_interleave(128, dim=1)
    assert bool(((back - w).abs() <= 0.5 * step + 1e-2 * w.abs().amax()).all())
    # 8 bits is finer than 4 bits on the same weights
    w4, s4, b4 = quantize_w4(w)
    err4 = (dequantize_weights(w4, s4.float(), b4.float(), 128, 4) - w).abs().mean()
    assert float((back - w).abs().mean()) < float(err4) / 8


def test_four_bit_quantiser_is_unchanged():
    g = torch.Generator().manual_seed(2)
    w = torch.randn(8, 256, generator=g)
    for a, b in zip(quantize_affine(w, 4), quantize_w4(w)):
        assert torch.equal(a.view(torch.int32) if a.dtype == torch.uint32 else a, b.view(torch.int32) if b.dtype == torch.uint32 else b)
    with pytest.raises(ValueError, match="4 or 8"):
        quantize_affine(w, 6)


def test_synthetic_8bit_model_has_8bit_layouts_and_the_default_stays_4bit():
    m8 = synthetic_qwen3("tiny-d128", seed=0, bits=8)
    m4 = synthetic_qwen3("tiny-d128", seed=0)
    q8, q4 = m8.model.layers[0].self_attn.q_proj, m4.model.layers[0].self_attn.q_proj
    assert (q8.bits, q4.bits) == (8, 4)
    assert q8.weight.shape[1] == 2 * q4.weight.shape[1] == 256 // 4
    assert synthetic_qwen3("tiny-d128", seed=0, bits=8, empty=True).model.embed_tokens.weight.shape == (512, 64)
    with pytest.raises(ValueError, match="4 or 8"):
        synthetic_qwen3("tiny", bits=3)


def test_synthetic_8bit_checkpoint_round_trips(tmp_path):
    m = synthetic_qwen3("tiny-d128", seed=0, bits=8, realistic=True)
    save_checkpoint(m, tmp_path)
    assert json.loads((tmp_path / "config.json").read_text())["quantization"] == {"group_size": 128, "bits": 8}
    back = load_checkpoint(tmp_path)
    for a, b in ((m.model.embed_tokens, back.model.embed_tokens), (m.model.layers[1].mlp.down_proj, back.model.layers[1].mlp.down_proj)):
        assert b.bits == 8 and b.group_size == 128
        assert torch.equal(a.weight.view(torch.int32), b.weight.view(torch.int32))
        assert torch.equal(a.scales, b.scales) and torch.equal(a.biases, b.biases)


def _saved(tmp_path, bits=8, **quant):
    m = synthetic_qwen3("tiny", seed=0, bits=bits if bits in (4, 8) else 4)
    save_checkpoint(m, tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    cfg["quantization"] = {"group_size": 128, "bits": bits, **quant}
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    return tmp_path


@pytest.mark.parametrize("bits", [2, 3, 6])
def test_loader_refuses_other_widths(tmp_path, bits):
    with pytest.raises(ValueError, match=f"bits = {bits}"):
        load_checkpoint(_saved(tmp_path, bits))


def test_loader_refuses_group_64(tmp_path):
    with pytest.raises(ValueError, match="group_size = 64"):
        load_checkpoint(_saved(tmp_path, group_size=64))


def test_loader_refuses_per_layer_overrides(tmp_path):
    path = _saved(tmp_path, **{"model.layers.0.mlp.down_proj": {"group_size": 128, "bits": 4}})
    with pytest.raises(ValueError, match="model.layers.0.mlp.down_proj"):
        load_checkpoint(path)
    load_checkpoint(_saved(tmp_path, **{"model.layers.0.mlp.down_proj": {"group_size": 128, "bits": 8}}))  # the same as global


def test_loader_checks_each_linear_against_the_declared_width(tmp_path):
    # a 4-bit checkpoint declared as 8-bit: weight.shape[1] * 32 / 8 != scales.shape[1] * 128
    m = synthetic_qwen3("tiny", seed=0)
    save_checkpoint(m, tmp_path)
    cfg = json.loads((tmp_path / "config.json").read_text())
    cfg["quantization"]["bits"] = 8
    (tmp_path / "config.json").write_text(json.dumps(cfg))
    with pytest.raises(ValueError, match="do not match 8-bit codes"):
        load_checkpoint(tmp_path)


def test_qwen3_moe_at_8_bits_is_refused():
    m = synthetic_qwen3("tiny-moe-d128", seed=0, bits=8)
    with pytest.raises(ValueError, match="8-bit"):
        Qwen3ModelWeek3(m)


def test_weight_stream_bytes_counts_1_03125_bytes_per_weight_at_8_bits():
    args = make_args("qwen3-4b")
    b4, b8 = weight_stream_bytes(args), weight_stream_bytes(args, bits=8)
    assert b4 == weight_stream_bytes(args, bits=4)
    assert b8 * 17 == pytest.approx(b4 * 33, rel=1e-9)


def test_shim_infers_the_code_width_of_fused_weights():
    N = 512
    assert ext.packed_bits(torch.empty(4, N // 8), N) == 4
    assert ext.packed_bits(torch.empty(4, N // 4), N) == 8
    assert ext.packed_bits(torch.empty(4, N * 6 // 32), N) is None
    assert ext.packed_bits(torch.empty(4, N // 2), N) is None


def test_shim_refuses_widths_before_touching_a_device():
    x = torch.zeros(2, 256, dtype=torch.bfloat16)
    s = torch.ones(64, 2, dtype=torch.bfloat16)
    w6 = torch.zeros(64, 256 * 6 // 32, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="4- or 8-bit"):
        ext.quantized_matmul_fused(s, s, w6, x)
    with pytest.raises(RuntimeError, match="4- or 8-bit"):
        ext.quantized_matmul_residual_norm(s, s, w6, x, torch.zeros(2, 64, dtype=torch.bfloat16), torch.ones(64, dtype=torch.bfloat16), 1e-6)
    with pytest.raises(RuntimeError, match="bits must be 4 or 8"):
        ext.quantized_matmul(s, s, 128, 6, x, w6, True)
    with pytest.raises(RuntimeError, match="a must have the same number of columns as b"):
        ext.quantized_matmul(s, s, 128, 8, x, torch.zeros(64, 256 // 8, dtype=torch.int32), True)
    with pytest.raises(RuntimeError, match="4- or 8-bit weights"):
        ext.quantized_embedding(torch.zeros(3, dtype=torch.int32), s, s, w6, 128, 6)


def test_bits_siblings_are_declared_exported_and_bound():
    header = (Path(__file__).resolve().parents[1] / "include" / "tiny_llm_b200.h").read_text()
    siblings = ["tl_quantized_matmul_bits", "tl_quantized_matmul_workspace_bits", "tl_quantized_matmul_route_bits", "tl_quantized_embedding_bits",
                "tl_quantized_matmul_fused_bits", "tl_quantized_matmul_fused_workspace_bits", "tl_quantized_matmul_residual_norm_bits",
                "tl_qkv_project_rope_append_bits", "tl_qkv_project_rope_append_table_bits"]
    for name in siblings:
        assert name in ext.EXPORTED_SYMBOLS
        assert name[: -len("_bits")] in ext.EXPORTED_SYMBOLS
    for name in siblings:
        assert f"{name}(" in header


def test_c_route_refuses_other_widths_without_a_device():
    A = 0
    with pytest.raises(RuntimeError, match="bits must be 4 or 8"):
        ext.quantized_matmul_route(1, 512, 256, 512, ext.PRO_NONE, False, False, torch.bfloat16, A, A, A, A, bits=6)
    assert ext.quantized_matmul_route(3, 512, 256, 512, ext.PRO_NONE, False, False, torch.bfloat16, A, A, A, A, bits=8)[0] == ext.W4_VANILLA


def test_cli_synthetic_bits_flag(monkeypatch):
    from tiny_llm_b200 import cli

    seen = {}

    def fake_generate(args):
        ns, _, _ = cli._load(args, "cpu")
        seen["bits"] = ns.model.layers[0].self_attn.q_proj.bits
        return 0

    monkeypatch.setattr(cli, "cmd_generate", fake_generate)
    assert cli.main(["generate", "--synthetic", "tiny", "--synthetic-bits", "8", "--prompt-ids", "1,2"]) == 0
    assert seen["bits"] == 8
    assert cli.main(["generate", "--synthetic", "tiny", "--prompt-ids", "1,2"]) == 0
    assert seen["bits"] == 4
    with pytest.raises(SystemExit):
        cli.main(["generate", "--synthetic", "tiny", "--synthetic-bits", "6"])
    with pytest.raises(SystemExit):
        cli.main(["generate", "--model", "x", "--synthetic-bits", "8"])


def test_workspace_queries_return_nothing_for_other_widths():
    lib = ext._lib
    bf16 = 2 if not hasattr(ext, "_DTYPE_CODE") else ext._DTYPE_CODE[torch.bfloat16]
    M, N, K = 32, 4096, 1024  # the split-reduction kernel: a workspace at 4 and 8 bits
    for bits in (4, 8):
        assert lib.tl_quantized_matmul_workspace_bits(M, N, K, bf16, bits, 1, 0) > 0
        assert lib.tl_quantized_matmul_fused_workspace_bits(M, N, K, N, ext.PRO_NONE, bf16, bits) > 0
    assert lib.tl_quantized_matmul_workspace_bits(M, N, K, bf16, 4, 1, 0) == lib.tl_quantized_matmul_workspace(M, N, K, bf16, 1, 0)
    for bits in (3, 6, 16):
        assert lib.tl_quantized_matmul_workspace_bits(M, N, K, bf16, bits, 1, 0) == 0
        assert lib.tl_quantized_matmul_fused_workspace_bits(M, N, K, N, ext.PRO_NONE, bf16, bits) == 0
