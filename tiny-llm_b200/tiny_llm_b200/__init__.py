"""tiny_llm_b200 - tiny-llm's Qwen3 inference operators, models and scheduler
re-hosted on torch tensors over the sm_90a extension.  The public names are
those of ``tiny_llm_ref`` (``src/tiny_llm_ref/__init__.py``)."""

from .attention import *  # noqa: F401,F403
from .attention import paged_attention, scaled_dot_product_attention_grouped, scaled_dot_product_attention_simple, causal_mask
from .basics import linear, silu, softmax
from .batch import ContinuousBatcher, Request, batch_generate
from .checkpoint import load_checkpoint, load_tokenizer, save_checkpoint
from .embed import embed_ids
from .rerank import rerank_ids, split_shared_prefix
from .embedding import Embedding, QuantizedEmbedding
from .generate import (BeamHypothesis, ParallelSample, beam_search_ids, greedy_generate_ids, parallel_sample_ids, prompt_lookup_generate_ids,
                       simple_generate_with_kv_cache, speculative_generate, speculative_generate_ids)
from .kv_cache import BatchingKvCache, TinyKvCache, TinyKvFullCache
from .layer_norm import RMSNorm
from .moe import Moe, grouped_expert_linear, route_topk
from .models import dispatch_model, shortcut_name_to_full_name
from .paged_kv_cache import PagedKvMetadata, TinyKvPagedCache, TinyKvPagedPool
from .positional_encoding import RoPE
from .sampler import SamplingParams, make_sampler
from .logprobs import PromptScore, TokenLogprobs, score_ids, token_logprobs
from .quantize import (
    QuantizedWeights,
    dequantize_linear,
    dequantize_weights,
    quantized_linear,
    quantized_matmul,
    quantized_matmul_vanilla,
    quantized_matvec_custom,
)
from .qwen3_week2 import WEEK2_CHECKPOINTS, Qwen3ModelWeek2
from .qwen3_week3 import Qwen3ModelWeek3
from .week2_kernels import FastRMSNorm, FastRoPE, decode_attention_custom, scaled_dot_product_attention, swiglu
