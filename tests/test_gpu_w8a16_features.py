"""The graph engines and the features built on them, with 8-bit models: the 4-bit identity tests, run unchanged on
8-bit weights.

Each 4-bit test module named below is loaded a second time, under its own name, with its ``synthetic_qwen3`` building
8-bit models (``bits=8``); the tests collected here are that copy's.  They compare every engine and feature against
the operator path (or its own eager launches) bit for bit wherever the 4-bit test does, and against the CPU oracle
within its tolerance.  Covered:
  * the decode graph at 1 to 32 rows (the 8-bit streaming kernel up to 8 rows, the 8-bit split-reduction wgmma kernel
    above, inside captured graphs with the engine's workspace), the device-resident loop and the public model call;
  * the penalised, constrained and logprobs graph kinds, the beam step graph, speculative and prompt-lookup verify, and
    parallel sampling's grouped step graph (one open defect: the verify pass past 4K tokens of context, marked below);
  * the prefill chunk engine and the decode graphs of a YaRN model against ``engine_plan``'s launch plan;
  * LoRA adapters in the decode and prefill engines;
  * ``embed_ids`` against the operator path.
Qwen3-MoE is refused at 8 bits (test_w8a16_host), so the MoE parameters of the 4-bit tests are left out."""

import functools
import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


class _WidthAwareExt:
    """The extension as ``engine_plan.py`` calls it: the plan writes its per-operator projection and route queries for
    4-bit weights, so here the code width of each packed weight is taken from its shape (``ext.packed_bits``)."""

    def __getattr__(self, name):
        return getattr(ext, name)

    @staticmethod
    def quantized_matmul(scales, biases, group_size, bits, a, b, *args, **kwargs):
        return ext.quantized_matmul(scales, biases, group_size, ext.packed_bits(b, a.shape[1]), a, b, *args, **kwargs)

    @staticmethod
    def quantized_matmul_route(M, N, K, lda, prologue, fused, use_simdgroup, dtype, a, b, scales, biases, bits=4):
        width = ext.packed_bits(b, N) if isinstance(b, torch.Tensor) else bits
        return ext.quantized_matmul_route(M, N, K, lda, prologue, fused, use_simdgroup, dtype, a, b, scales, biases, bits=width)


def _w8(stem):
    """A second instance of tests/<stem>.py whose synthetic models are 8-bit (and whose launch plan, if it has one,
    takes 8-bit weights)."""
    module = _load(f"tiny_llm_b200_w8a16_{stem}", f"{stem}.py")
    module.synthetic_qwen3 = functools.partial(synthetic_qwen3, bits=8)
    if hasattr(module, "plan"):  # the plan, and any wrapper the module puts around the extension for it
        plan = _load("tiny_llm_b200_w8a16_engine_plan", "engine_plan.py")
        plan.ext = module.ext = _WidthAwareExt()
        module.plan = plan
    return module


engine = _w8("test_gpu_engine")
penalties = _w8("test_gpu_penalties")
constrained = _w8("test_gpu_constrained")
logprobs = _w8("test_gpu_logprobs")
beam = _w8("test_gpu_beam")
speculative = _w8("test_gpu_speculative")
ngram = _w8("test_gpu_ngram")
long_context = _w8("test_gpu_long_context")
lora = _w8("test_gpu_lora")
parallel = _w8("test_gpu_parallel_sample")
embed = _w8("test_gpu_embed")

# fixtures of the copies (the same definitions in every module that has them)
dev = engine.dev
tiny_gpu = engine.tiny_gpu
target = speculative.target
rule_on, rule_off = parallel.rule_on, parallel.rule_off

# decode graph, device-resident loop, public call, scheduler
test_engine_step_matches_the_operator_path = engine.test_engine_step_matches_the_operator_path
test_device_resident_greedy_loop_equals_host_driven_loop = engine.test_device_resident_greedy_loop_equals_host_driven_loop
test_public_model_call_uses_the_graph_and_matches_operator_path = engine.test_public_model_call_uses_the_graph_and_matches_operator_path
test_scheduler_runs_on_the_graph_path_and_releases_everything = engine.test_scheduler_runs_on_the_graph_path_and_releases_everything

# penalised, constrained and logprobs graph kinds (B up to 32: the 8-bit wgmma kernel in the graphs)
test_decode_on_device_penalised_equals_steps_plus_eager = penalties.test_decode_on_device_penalised_equals_steps_plus_eager
test_generate_penalised_equals_prefill_plus_decode_on_device = penalties.test_generate_penalised_equals_prefill_plus_decode_on_device
test_decode_on_device_constrained_equals_eager_steps = constrained.test_decode_on_device_constrained_equals_eager_steps
test_generate_batcher_and_decode_on_device_give_the_same_constrained_tokens = (
    constrained.test_generate_batcher_and_decode_on_device_give_the_same_constrained_tokens)
test_decode_on_device_logprobs_equal_steps_plus_eager_logprobs = logprobs.test_decode_on_device_logprobs_equal_steps_plus_eager_logprobs
test_score_ids_tracks_the_reference_cpu_model = logprobs.test_score_ids_tracks_the_reference_cpu_model

# beam search
test_the_beam_step_graph_equals_the_decode_graph_and_eager_launches = beam.test_the_beam_step_graph_equals_the_decode_graph_and_eager_launches


@pytest.mark.parametrize("key", ["d128", "4b"])
@pytest.mark.parametrize("graph", [True, False])
def test_one_beam_with_early_stopping_is_greedy(dev, key, graph):
    beam.test_one_beam_with_early_stopping_is_greedy(dev, key, graph)


# speculative and prompt-lookup verify
@pytest.mark.parametrize("key", ["d128", "4b", "0.6b"])
@pytest.mark.parametrize("ctx0", [126, pytest.param(4093, marks=pytest.mark.xfail(strict=False, reason=(
    "open defect at 8 bits: past 4K tokens of context the T-row verify pass can differ from T decode steps in the last "
    "bits (3 of 18 seed / length combinations of the 0.6b shape; 0 of 18 at 4 bits; the 8-bit streaming kernel's rows "
    "are independent of each other, so the difference comes from elsewhere in the verify path)")))])
@pytest.mark.parametrize("T", [2, 5, 8])
def test_verify_step_equals_t_decode_steps(dev, key, ctx0, T):
    speculative.test_verify_step_equals_t_decode_steps(dev, key, ctx0, T)


test_speculative_equals_greedy = speculative.test_speculative_equals_greedy
test_prompt_lookup_equals_greedy = ngram.test_prompt_lookup_equals_greedy

# long context: YaRN decode and prefill-chunk graphs against the launch plan, and the oracle
test_yarn_decode_and_chunk_graphs_equal_the_plan = long_context.test_yarn_decode_and_chunk_graphs_equal_the_plan
test_yarn_model_paths_and_oracle_agree = long_context.test_yarn_model_paths_and_oracle_agree

# LoRA adapters in the decode (1 to 32 rows) and prefill engines
test_decode_engine_matches_the_operator_path = lora.test_decode_engine_matches_the_operator_path
test_decode_on_device_gives_the_tokens_of_step = lora.test_decode_on_device_gives_the_tokens_of_step
test_prefill_engine_matches_the_operator_path = lora.test_prefill_engine_matches_the_operator_path

# parallel sampling
test_single_sample_equals_greedy_generate = parallel.test_single_sample_equals_greedy_generate


@pytest.mark.parametrize("key", ["d128", "4b"])
def test_ungrouped_samples_equal_separate_prefills(dev, key, rule_off):
    """B = 4: the n-slot run and the single-request runs are both on the streaming kernel, whose rows do not depend on
    each other, so the sampled ids must agree.  (The 4-bit test's B = 12 case compares the swap-AB kernel, which rounds
    weights to bf16, with the streaming kernel, which does not: agreement of sampled ids there is not an identity.)"""
    parallel.test_ungrouped_samples_equal_separate_prefills(dev, key, 1, 4, rule_off)


test_grouped_step_graph_equals_its_launch_plan = parallel.test_grouped_step_graph_equals_its_launch_plan

# embeddings
test_embed_ids_matches_operator_path = embed.test_embed_ids_matches_operator_path
test_embed_ids_bits_do_not_depend_on_placement = embed.test_embed_ids_bits_do_not_depend_on_placement


def test_the_copies_build_8bit_models(dev):
    """Every model the tests above build is 8-bit: the copies' constructor is the 8-bit one."""
    for module in (engine, penalties, constrained, logprobs, beam, speculative, ngram, long_context, lora, parallel, embed):
        ns = module.synthetic_qwen3("tiny", seed=0)
        assert ns.model.layers[0].self_attn.q_proj.bits == 8
