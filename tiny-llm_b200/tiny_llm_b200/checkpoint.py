"""Checkpoint front door: MLX 4-bit safetensors -> the ``mlx_model`` duck type.

The reference loads ``Qwen/Qwen3-*-MLX-4bit`` with ``mlx_lm.load``
(``main.py:96-98``, ``batch-main.py:62-64``) and hands the
resulting object to ``dispatch_model``; the models only look at ``.args`` and at
``weight / scales / biases / group_size / bits`` of every quantised layer
(``src/tiny_llm_ref/qwen3_week3.py:225-313``).  An MLX 4-bit
checkpoint directory is ``config.json`` + ``model*.safetensors`` whose tensors
are named ``model.layers.{i}.self_attn.q_proj.{weight,scales,biases}`` ... with
``weight`` packed uint32 ``[out, in/8]`` in exactly the nibble order
``dequantize_weights`` decodes (quantize.py:103-121), so loading is a rename into
``SimpleNamespace``s: no tensor is transformed.  Embedding checkpoints (Qwen3-Embedding) save the bare ``Qwen3Model``:
the same tensors without the ``model.`` prefix and without ``lm_head``; they load too.

``save_checkpoint`` writes the same layout (used by the tests to round-trip a
synthetic model, and handy for producing fixtures); there is no network here, so
real weights have to be placed on disk by the user.
"""

from __future__ import annotations

import json
from pathlib import Path
from types import SimpleNamespace

import torch

from .rope_scaling import parse_rope_scaling
from .synthetic import named_tensors

ARG_KEYS = ("num_hidden_layers", "hidden_size", "vocab_size", "num_attention_heads", "num_key_value_heads", "head_dim",
            "intermediate_size", "rms_norm_eps", "max_position_embeddings", "rope_theta", "tie_word_embeddings")
_LINEARS = {"self_attn": ("q_proj", "k_proj", "v_proj", "o_proj"), "mlp": ("gate_proj", "up_proj", "down_proj")}


def _read_tensors(path: Path) -> dict:
    from safetensors import safe_open

    files = sorted(path.glob("*.safetensors"))
    if not files:
        raise FileNotFoundError(f"no *.safetensors under {path}")
    tensors = {}
    for file in files:
        with safe_open(str(file), framework="pt", device="cpu") as f:
            for name in f.keys():
                tensors[name] = f.get_tensor(name)
    return tensors


def load_checkpoint(path, device="cpu") -> SimpleNamespace:
    """``mlx_lm.load(path)[0]`` as far as the tiny-llm models look at it."""
    path = Path(path)
    config = json.loads((path / "config.json").read_text())
    quant = config.get("quantization") or config.get("quantization_config") or {}
    group_size, bits = int(quant.get("group_size", 128)), int(quant.get("bits", 4))
    _check_quantization(quant, group_size, bits)
    if "head_dim" not in config:
        config["head_dim"] = config["hidden_size"] // config["num_attention_heads"]
    config.setdefault("tie_word_embeddings", True)
    missing = [k for k in ARG_KEYS if k not in config]
    if missing:
        raise ValueError(f"config.json lacks {missing}")
    args = SimpleNamespace(**{k: config[k] for k in ARG_KEYS})
    # RoPE scaling: static YaRN is applied (rope_scaling.py); any other type raises ValueError here rather than load and
    # compute every position wrongly
    scaling = parse_rope_scaling(config.get("rope_scaling"), args.max_position_embeddings)
    if scaling is not None:
        args.rope_scaling = scaling.to_config()
    tensors = _read_tensors(path)
    # Qwen3Model naming (embedding checkpoints): embed_tokens.*, layers.{i}.*, norm.*, no lm_head
    root = "model." if "model.embed_tokens.weight" in tensors or "embed_tokens.weight" not in tensors else ""
    if not root and "lm_head.weight" not in tensors:
        args.tie_word_embeddings = True  # no head of its own: the model embeds, its logits are the tied embedding's

    def take(name: str) -> torch.Tensor:
        if name not in tensors:
            raise KeyError(f"checkpoint has no tensor {name!r}")
        return tensors[name].to(device)

    def linear(prefix: str) -> SimpleNamespace:
        weight = take(prefix + ".weight")
        if weight.dtype == torch.int32:
            weight = weight.view(torch.uint32)
        if weight.dtype != torch.uint32:
            raise ValueError(f"{prefix}.weight is {weight.dtype}: expected packed uint32 (a {bits}-bit MLX checkpoint)")
        scales = take(prefix + ".scales")
        if weight.dim() != 2 or scales.dim() != 2 or weight.shape[1] * 32 // bits != scales.shape[1] * group_size or (weight.shape[1] * 32) % bits:
            raise ValueError(f"{prefix}: packed weight {tuple(weight.shape)} and scales {tuple(scales.shape)} do not match {bits}-bit codes "
                             f"at group {group_size} (weight.shape[1] * 32 / bits must equal scales.shape[1] * {group_size})")
        return SimpleNamespace(weight=weight, scales=scales, biases=take(prefix + ".biases"), group_size=group_size, bits=bits)

    def norm(prefix: str) -> SimpleNamespace:
        return SimpleNamespace(weight=take(prefix + ".weight"))

    layers = []
    for i in range(args.num_hidden_layers):
        base = f"{root}layers.{i}"
        attn = SimpleNamespace(**{n: linear(f"{base}.self_attn.{n}") for n in _LINEARS["self_attn"]},
                               q_norm=norm(f"{base}.self_attn.q_norm"), k_norm=norm(f"{base}.self_attn.k_norm"))
        mlp = SimpleNamespace(**{n: linear(f"{base}.mlp.{n}") for n in _LINEARS["mlp"]})
        layers.append(SimpleNamespace(self_attn=attn, mlp=mlp, input_layernorm=norm(f"{base}.input_layernorm"),
                                      post_attention_layernorm=norm(f"{base}.post_attention_layernorm")))
    model = SimpleNamespace(args=args, model=SimpleNamespace(embed_tokens=linear(f"{root}embed_tokens"), layers=layers, norm=norm(f"{root}norm")))
    if not args.tie_word_embeddings:
        model.lm_head = linear("lm_head")
    return model


def _check_quantization(quant: dict, group_size: int, bits: int) -> None:
    """The projection kernels take MLX affine 4- or 8-bit codes at group 128, one width for the whole model."""
    if bits not in (4, 8):
        raise ValueError(f"quantization.bits = {bits}: only 4- and 8-bit checkpoints are supported")
    if group_size != 128:
        raise ValueError(f"quantization.group_size = {group_size}: only group size 128 is supported (convert with --q-group-size 128)")
    for key, value in quant.items():  # mlx-lm writes per-layer overrides as {"<layer path>": {"group_size", "bits"}}
        if isinstance(value, dict) and (int(value.get("bits", bits)) != bits or int(value.get("group_size", group_size)) != group_size):
            raise ValueError(f"quantization override for {key!r} ({value}) differs from the global {bits} bits / group {group_size}: "
                             "mixed per-layer quantisation is not supported")


def save_checkpoint(model_ns: SimpleNamespace, path) -> None:
    """Write ``model_ns`` in the MLX layout of its width (config.json + model.safetensors)."""
    from safetensors.torch import save_file

    path = Path(path)
    path.mkdir(parents=True, exist_ok=True)
    first = model_ns.model.embed_tokens
    config = {k: getattr(model_ns.args, k) for k in ARG_KEYS}
    scaling = parse_rope_scaling(getattr(model_ns.args, "rope_scaling", None), model_ns.args.max_position_embeddings)
    if scaling is not None:
        config["rope_scaling"] = scaling.to_config()
    config["quantization"] = {"group_size": first.group_size, "bits": first.bits}
    config["model_type"] = "qwen3"
    (path / "config.json").write_text(json.dumps(config, indent=1))
    tensors = {}
    for name, tensor in named_tensors(model_ns):
        if name.startswith("args."):
            continue
        tensors[name] = tensor.detach().cpu().contiguous()
    save_file(tensors, str(path / "model.safetensors"))


def load_tokenizer(path):
    """The Hugging Face tokenizer of the checkpoint directory wrapped with the two attributes the
    generation loops use from mlx_lm's TokenizerWrapper (``detokenizer``, ``_tokenizer``)."""
    from transformers import AutoTokenizer

    return TokenizerWrapper(AutoTokenizer.from_pretrained(str(path)))


class _Detokenizer:
    """mlx_lm's streaming detokenizer interface (reset / add_token / last_segment / text) by full re-decode."""

    def __init__(self, tokenizer):
        self._tokenizer = tokenizer
        self.reset()

    def reset(self) -> None:
        self.tokens: list[int] = []
        self.text = ""
        self.last_segment = ""

    def add_token(self, token: int) -> None:
        self.tokens.append(int(token))
        text = self._tokenizer.decode(self.tokens)
        if text.endswith("�"):  # incomplete UTF-8 sequence: wait for the next token
            self.last_segment = ""
            return
        self.last_segment = text[len(self.text):]
        self.text = text


class TokenizerWrapper:
    def __init__(self, tokenizer):
        self._tokenizer = tokenizer
        self.detokenizer = _Detokenizer(tokenizer)
        self.eos_token_id = tokenizer.eos_token_id

    def encode(self, text, add_special_tokens: bool = False):
        return self._tokenizer.encode(text, add_special_tokens=add_special_tokens)

    def apply_chat_template(self, *a, **k):
        return self._tokenizer.apply_chat_template(*a, **k)

    def __getattr__(self, name):
        return getattr(self._tokenizer, name)
