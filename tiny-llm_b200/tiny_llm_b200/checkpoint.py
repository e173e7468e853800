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

Qwen3-MoE checkpoints (``model_type: "qwen3_moe"``, e.g. Qwen3-30B-A3B) add the MoE config keys; a sparse layer
holds its router as ``mlp.gate.*`` and its experts as 3-D ``mlp.switch_mlp.{gate,up,down}_proj.*`` (``[E, out,
in * bits / 32]``), and its router may carry mlx_lm's 8-bit group-64 quantisation override (``ROUTER_OVERRIDE``).

``save_checkpoint`` writes the same layout (used by the tests to round-trip a
synthetic model, and handy for producing fixtures); there is no network here, so
real weights have to be placed on disk by the user.
"""

from __future__ import annotations

import json
import re
from pathlib import Path
from types import SimpleNamespace

import torch

from .rope_scaling import parse_rope_scaling
from .synthetic import MOE_KEYS, is_sparse_layer, moe_defaults, named_tensors

ARG_KEYS = ("num_hidden_layers", "hidden_size", "vocab_size", "num_attention_heads", "num_key_value_heads", "head_dim",
            "intermediate_size", "rms_norm_eps", "max_position_embeddings", "rope_theta", "tie_word_embeddings")
_LINEARS = {"self_attn": ("q_proj", "k_proj", "v_proj", "o_proj"), "mlp": ("gate_proj", "up_proj", "down_proj")}
ROUTER_OVERRIDE = {"bits": 8, "group_size": 64}  # how mlx_lm quantises qwen3_moe routers (mlp.gate) apart from the model
_ROUTER_KEY = re.compile(r"(?:model\.)?layers\.(\d+)\.mlp\.gate")


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
    if "head_dim" not in config:
        config["head_dim"] = config["hidden_size"] // config["num_attention_heads"]
    config.setdefault("tie_word_embeddings", True)
    missing = [k for k in ARG_KEYS if k not in config]
    if missing:
        raise ValueError(f"config.json lacks {missing}")
    args = SimpleNamespace(**{k: config[k] for k in ARG_KEYS})
    if config.get("num_experts", 0) > 0:  # Qwen3-MoE: the keys Qwen3ModelWeek3 reads, with synthetic.make_args' defaults
        moe = moe_defaults({k: config[k] for k in ("intermediate_size", *MOE_KEYS) if k in config})
        for k in MOE_KEYS:
            setattr(args, k, moe[k])
    routers = _check_quantization(quant, group_size, bits, args)
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

    def packed(prefix: str, width: int) -> torch.Tensor:
        weight = take(prefix + ".weight")
        if weight.dtype == torch.int32:
            weight = weight.view(torch.uint32)
        if weight.dtype != torch.uint32:
            raise ValueError(f"{prefix}.weight is {weight.dtype}: expected packed uint32 (a {width}-bit MLX checkpoint)")
        return weight

    def linear(prefix: str, width: int = bits, group: int = group_size) -> SimpleNamespace:
        weight = packed(prefix, width)
        scales = take(prefix + ".scales")
        if weight.dim() != 2 or scales.dim() != 2 or weight.shape[1] * 32 // width != scales.shape[1] * group or (weight.shape[1] * 32) % width:
            raise ValueError(f"{prefix}: packed weight {tuple(weight.shape)} and scales {tuple(scales.shape)} do not match {width}-bit codes "
                             f"at group {group} (weight.shape[1] * 32 / bits must equal scales.shape[1] * {group})")
        return SimpleNamespace(weight=weight, scales=scales, biases=take(prefix + ".biases"), group_size=group, bits=width)

    def experts(prefix: str, out_dim: int, in_dim: int) -> SimpleNamespace:
        """SwitchLinear layout: weight [E, out, in * bits / 32], scales and biases [E, out, in / group]."""
        weight, scales, biases = packed(prefix, bits), take(prefix + ".scales"), take(prefix + ".biases")
        E = args.num_experts
        for name, tensor, want in (("weight", weight, (E, out_dim, in_dim * bits // 32)), ("scales", scales, (E, out_dim, in_dim // group_size)),
                                   ("biases", biases, (E, out_dim, in_dim // group_size))):
            if tuple(tensor.shape) != want:
                raise ValueError(f"{prefix}.{name} has shape {tuple(tensor.shape)}, expected {want} (num_experts = {E}, "
                                 f"{bits}-bit codes at group {group_size} of a [{out_dim}, {in_dim}] expert)")
        return SimpleNamespace(weight=weight, scales=scales, biases=biases, group_size=group_size, bits=bits)

    def router(prefix: str, index: int) -> SimpleNamespace:
        width, group = routers.get(index, (bits, group_size))
        gate = linear(prefix, width, group)
        want = (args.num_experts, args.hidden_size * width // 32)
        if tuple(gate.weight.shape) != want:
            raise ValueError(f"{prefix}.weight has shape {tuple(gate.weight.shape)}, expected {want} (num_experts = {args.num_experts}, "
                             f"hidden_size = {args.hidden_size}, {width}-bit codes)")
        return gate

    def mlp(base: str, index: int) -> SimpleNamespace:
        if not is_sparse_layer(args, index):
            return SimpleNamespace(**{n: linear(f"{base}.mlp.{n}") for n in _LINEARS["mlp"]})
        H, inter = args.hidden_size, args.moe_intermediate_size
        switch = f"{base}.mlp.switch_mlp"
        return SimpleNamespace(gate=router(f"{base}.mlp.gate", index),
                               switch_mlp=SimpleNamespace(gate_proj=experts(f"{switch}.gate_proj", inter, H), up_proj=experts(f"{switch}.up_proj", inter, H),
                                                          down_proj=experts(f"{switch}.down_proj", H, inter)))

    def norm(prefix: str) -> SimpleNamespace:
        return SimpleNamespace(weight=take(prefix + ".weight"))

    layers = []
    for i in range(args.num_hidden_layers):
        base = f"{root}layers.{i}"
        attn = SimpleNamespace(**{n: linear(f"{base}.self_attn.{n}") for n in _LINEARS["self_attn"]},
                               q_norm=norm(f"{base}.self_attn.q_norm"), k_norm=norm(f"{base}.self_attn.k_norm"))
        layers.append(SimpleNamespace(self_attn=attn, mlp=mlp(base, i), input_layernorm=norm(f"{base}.input_layernorm"),
                                      post_attention_layernorm=norm(f"{base}.post_attention_layernorm")))
    model = SimpleNamespace(args=args, model=SimpleNamespace(embed_tokens=linear(f"{root}embed_tokens"), layers=layers, norm=norm(f"{root}norm")))
    if not args.tie_word_embeddings:
        model.lm_head = linear("lm_head")
    return model


def _check_quantization(quant: dict, group_size: int, bits: int, args) -> dict:
    """The projection kernels take MLX affine 4- or 8-bit codes at group 128, one width for the whole model.  The one
    exception is the router (``mlp.gate``) of a Qwen3-MoE sparse layer, which may be 8 bits at group 64
    (``ROUTER_OVERRIDE``, what mlx_lm gives qwen3_moe routers; ``tl_moe_router`` runs it).  Returns {layer index:
    (bits, group_size)} of those routers."""
    if bits not in (4, 8):
        raise ValueError(f"quantization.bits = {bits}: only 4- and 8-bit checkpoints are supported")
    if group_size != 128:
        raise ValueError(f"quantization.group_size = {group_size}: only group size 128 is supported (convert with --q-group-size 128)")
    moe = getattr(args, "num_experts", 0) > 0
    if moe and bits == 8 and any(is_sparse_layer(args, i) for i in range(args.num_hidden_layers)):
        raise ValueError("Qwen3-MoE with 8-bit weights is not supported (there is no 8-bit grouped expert GEMM); use a 4-bit checkpoint")
    routers = {}
    for key, value in quant.items():  # mlx-lm writes per-layer overrides as {"<layer path>": {"group_size", "bits"}}
        if not isinstance(value, dict):
            continue
        setting = (int(value.get("bits", bits)), int(value.get("group_size", group_size)))
        if setting == (bits, group_size):
            continue
        router = _ROUTER_KEY.fullmatch(key)
        if router is None or not is_sparse_layer(args, int(router.group(1))):
            raise ValueError(f"quantization override for {key!r} ({value}) differs from the global {bits} bits / group {group_size}: "
                             "mixed per-layer quantisation is not supported")
        if setting != (ROUTER_OVERRIDE["bits"], ROUTER_OVERRIDE["group_size"]):
            raise ValueError(f"quantization override for the router {key!r} ({value}): a router must be quantised as the model "
                             f"({bits} bits / group {group_size}) or at 8 bits / group 64")
        routers[int(router.group(1))] = setting
    return routers


def save_checkpoint(model_ns: SimpleNamespace, path) -> None:
    """Write ``model_ns`` in the MLX layout of its width (config.json + model.safetensors)."""
    from safetensors.torch import save_file

    path = Path(path)
    path.mkdir(parents=True, exist_ok=True)
    first = model_ns.model.embed_tokens
    args = model_ns.args
    config = {k: getattr(args, k) for k in ARG_KEYS}
    scaling = parse_rope_scaling(getattr(args, "rope_scaling", None), args.max_position_embeddings)
    if scaling is not None:
        config["rope_scaling"] = scaling.to_config()
    quant = {"group_size": first.group_size, "bits": first.bits}
    moe = getattr(args, "num_experts", 0) > 0
    if moe:
        config.update({k: getattr(args, k) for k in MOE_KEYS})
        for i, layer in enumerate(model_ns.model.layers):
            gate = layer.mlp.gate if is_sparse_layer(args, i) else None
            if gate is not None and (gate.bits, gate.group_size) != (first.bits, first.group_size):
                quant[f"model.layers.{i}.mlp.gate"] = {"group_size": gate.group_size, "bits": gate.bits}
    config["quantization"] = quant
    config["model_type"] = "qwen3_moe" if moe else "qwen3"
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
