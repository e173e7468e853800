"""Multi-LoRA serving: bf16 low-rank adapters over the frozen W4A16 base, chosen per request.

A ``LoraAdapter`` is what a QLoRA fine-tune produces: per targeted projection ``A [r, in]`` and ``B [out, r]`` in bf16
and ``alpha``; the projection's output becomes ``W x + (alpha / r) B A x``.  ``LoraAdapter.load`` / ``save`` read and
write the PEFT layout (``adapter_config.json`` + ``adapter_model.safetensors``).

An ``AdapterSet`` packs up to 32 adapters once per device into the per-site slabs ``tl_lora_apply`` reads
(``include/tiny_llm_b200.h``): per layer the sites q|k|v, o, gate|up and down, each ``A [n, nseg * r_max, N]`` and one
``B [n, K_s, r_max]`` per segment, ranks padded to the set's ``r_max`` with zeros.  A request names its adapter; the rows
of a launch carry the adapter's id (``id_of``), -1 for the base model, so one launch and one captured graph serve any
mix (DESIGN.md section 12).
"""

from __future__ import annotations

import json
import re
from pathlib import Path
from types import SimpleNamespace

import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

PROJECTIONS = ("q", "k", "v", "o", "gate", "up", "down")
SITES = {"qkv": ("q", "k", "v"), "o": ("o",), "gate_up": ("gate", "up"), "down": ("down",)}
MAX_ADAPTERS = ext.LORA_MAX_ADAPTERS
RANKS = ext.LORA_RANKS
_BLOCK = {"q": "self_attn", "k": "self_attn", "v": "self_attn", "o": "self_attn", "gate": "mlp", "up": "mlp", "down": "mlp"}
_KEY = re.compile(r"^base_model\.model\.model\.layers\.(\d+)\.(self_attn|mlp)\.(q|k|v|o|gate|up|down)_proj\.lora_(A|B)\.weight$")


def projection_shapes(args) -> dict:
    """``{projection: (out, in)}`` of one layer of the base model."""
    H, I = args.hidden_size, args.intermediate_size
    q, kv = args.num_attention_heads * args.head_dim, args.num_key_value_heads * args.head_dim
    return {"q": (q, H), "k": (kv, H), "v": (kv, H), "o": (H, q), "gate": (I, H), "up": (I, H), "down": (H, I)}


def _check_rank(rank) -> int:
    if rank not in RANKS:
        raise ValueError(f"LoRA rank must be one of {RANKS}, got {rank}")
    return int(rank)


class LoraAdapter:
    """One adapter: ``tensors[(layer, projection)] = (A [rank, in], B [out, rank])`` in bf16, ``scale = alpha / rank``."""

    def __init__(self, name: str, rank: int, alpha: float, tensors: dict):
        self.name = str(name)
        self.rank = _check_rank(rank)
        self.alpha = float(alpha)
        self.tensors = {}
        for (layer, proj), (A, B) in tensors.items():
            if proj not in PROJECTIONS:
                raise ValueError(f"adapter {name!r}: unknown projection {proj!r}")
            if A.dim() != 2 or B.dim() != 2 or A.shape[0] != self.rank or B.shape[1] != self.rank:
                raise ValueError(f"adapter {name!r}: layer {layer} {proj}_proj has A {tuple(A.shape)} and B {tuple(B.shape)}, "
                                 f"expected [{self.rank}, in] and [out, {self.rank}]")
            self.tensors[(int(layer), proj)] = (A.to(torch.bfloat16).contiguous(), B.to(torch.bfloat16).contiguous())

    @property
    def scale(self) -> float:
        return self.alpha / self.rank

    @property
    def targets(self) -> tuple:
        return tuple(p for p in PROJECTIONS if any(proj == p for _, proj in self.tensors))

    def check_against(self, args) -> None:
        """Refuse tensors that do not fit the base model ``args`` describes."""
        shapes = projection_shapes(args)
        for (layer, proj), (A, B) in self.tensors.items():
            if not 0 <= layer < args.num_hidden_layers:
                raise ValueError(f"adapter {self.name!r}: layer {layer} does not exist (the base has {args.num_hidden_layers})")
            out, inp = shapes[proj]
            if A.shape[1] != inp or B.shape[0] != out:
                raise ValueError(f"adapter {self.name!r}: layer {layer} {proj}_proj is A {tuple(A.shape)}, B {tuple(B.shape)}; "
                                 f"the base projection is [{out}, {inp}]")

    @staticmethod
    def synthetic(model_args, rank: int, targets=PROJECTIONS, seed: int = 0, name: str | None = None, alpha: float | None = None) -> "LoraAdapter":
        """A seeded random adapter for ``model_args`` (there is no trained one without a network): ``A ~ N(0, 1 / in)``,
        ``B ~ N(0, 0.02^2)`` (never zero, unlike a freshly initialised PEFT adapter), ``alpha = 2 * rank``."""
        rank = _check_rank(rank)
        gen = torch.Generator().manual_seed(0x10A0 + seed)
        shapes = projection_shapes(model_args)
        tensors = {}
        for layer in range(model_args.num_hidden_layers):
            for proj in targets:
                out, inp = shapes[proj]
                A = torch.randn(rank, inp, generator=gen) * inp**-0.5
                B = torch.randn(out, rank, generator=gen) * 0.02
                tensors[(layer, proj)] = (A, B)
        return LoraAdapter(name if name is not None else f"synthetic-r{rank}-s{seed}", rank, 2.0 * rank if alpha is None else alpha, tensors)

    @staticmethod
    def load(path, name: str | None = None) -> "LoraAdapter":
        """Read a PEFT adapter directory."""
        from safetensors import safe_open

        path = Path(path)
        config = json.loads((path / "adapter_config.json").read_text())
        label = name if name is not None else path.name
        for flag in ("use_dora", "use_rslora"):
            if config.get(flag):
                raise ValueError(f"adapter {label!r}: {flag} is not supported")
        if config.get("bias", "none") not in ("none", None, False):
            raise ValueError(f"adapter {label!r}: bias = {config['bias']!r} is not supported (only 'none')")
        for key in ("r", "lora_alpha"):
            if key not in config:
                raise ValueError(f"adapter {label!r}: adapter_config.json lacks {key!r}")
        halves: dict = {}
        with safe_open(str(path / "adapter_model.safetensors"), framework="pt", device="cpu") as f:
            for key in f.keys():
                m = _KEY.match(key)
                if m is None:
                    raise ValueError(f"adapter {label!r}: unknown tensor {key!r}")
                halves.setdefault((int(m.group(1)), m.group(3)), {})[m.group(4)] = f.get_tensor(key)
        tensors = {}
        for (layer, proj), ab in halves.items():
            if set(ab) != {"A", "B"}:
                raise ValueError(f"adapter {label!r}: layer {layer} {proj}_proj has lora_{'A' if 'A' in ab else 'B'} only")
            tensors[(layer, proj)] = (ab["A"], ab["B"])
        listed = {t[:-5] if t.endswith("_proj") else t for t in config.get("target_modules", [])}
        found = {proj for _, proj in tensors}
        if listed and not found <= listed:
            raise ValueError(f"adapter {label!r}: tensors for {sorted(found - listed)} but target_modules = {sorted(listed)}")
        return LoraAdapter(label, int(config["r"]), float(config["lora_alpha"]), tensors)

    def save(self, path) -> None:
        """Write the PEFT layout ``load`` reads."""
        from safetensors.torch import save_file

        path = Path(path)
        path.mkdir(parents=True, exist_ok=True)
        config = {"peft_type": "LORA", "r": self.rank, "lora_alpha": self.alpha, "target_modules": [f"{p}_proj" for p in self.targets],
                  "bias": "none", "use_dora": False, "use_rslora": False}
        (path / "adapter_config.json").write_text(json.dumps(config, indent=1))
        out = {}
        for (layer, proj), (A, B) in self.tensors.items():
            base = f"base_model.model.model.layers.{layer}.{_BLOCK[proj]}.{proj}_proj"
            out[f"{base}.lora_A.weight"] = A.cpu().contiguous()
            out[f"{base}.lora_B.weight"] = B.cpu().contiguous()
        save_file(out, str(path / "adapter_model.safetensors"))


class AdapterSet:
    """Up to 32 adapters packed for one base model on one device.  ``sites[layer]`` has ``qkv``, ``o``, ``gate_up`` and
    ``down``: an ``ext.LoraSite``, or None where no adapter of the set targets the site (no launch is issued there)."""

    def __init__(self, model_args, adapters, device="cpu"):
        adapters = list(adapters)
        if not 1 <= len(adapters) <= MAX_ADAPTERS:
            raise ValueError(f"an adapter set holds 1 to {MAX_ADAPTERS} adapters, got {len(adapters)}")
        names = [a.name for a in adapters]
        if len(set(names)) != len(names):
            raise ValueError(f"adapter names must be unique, got {names}")
        for a in adapters:
            a.check_against(model_args)
        self.adapters = adapters
        self.names = names
        self.r_max = max(a.rank for a in adapters)
        self.device = torch.device(device)
        n, r_max = len(adapters), self.r_max
        shapes = projection_shapes(model_args)
        scales = torch.tensor([a.scale for a in adapters], dtype=torch.float32, device=self.device)
        ranks = torch.tensor([a.rank for a in adapters], dtype=torch.int32, device=self.device)
        self.sites = []
        for layer in range(model_args.num_hidden_layers):
            entry = {}
            for site, projs in SITES.items():
                if not any((layer, p) in a.tensors for a in adapters for p in projs):
                    entry[site] = None
                    continue
                N = shapes[projs[0]][1]
                A = torch.zeros((n, len(projs) * r_max, N), dtype=torch.bfloat16)
                Bs = [torch.zeros((n, shapes[p][0], r_max), dtype=torch.bfloat16) for p in projs]
                mask = torch.zeros(n, dtype=torch.int32)
                for i, a in enumerate(adapters):
                    for s, p in enumerate(projs):
                        if (layer, p) in a.tensors:
                            At, Bt = a.tensors[(layer, p)]
                            A[i, s * r_max : s * r_max + a.rank] = At
                            Bs[s][i, :, : a.rank] = Bt
                            mask[i] |= 1 << s
                entry[site] = ext.LoraSite(A.to(self.device), [b.to(self.device) for b in Bs], scales, ranks, mask.to(self.device))
            self.sites.append(SimpleNamespace(**entry))

    def id_of(self, name: str | None) -> int:
        """The adapter's id in this set; None (the base model) is -1."""
        if name is None:
            return -1
        try:
            return self.names.index(name)
        except ValueError:
            raise KeyError(f"no adapter named {name!r} is loaded (loaded: {self.names})") from None

    def row_ids(self, ids, rows_per_id: int = 1) -> torch.Tensor:
        """int32 device tensor with each of ``ids`` repeated for ``rows_per_id`` consecutive rows."""
        return torch.tensor([int(i) for i in ids for _ in range(rows_per_id)], dtype=torch.int32, device=self.device)


def adapter_ids_of(model, adapters, count: int) -> list[int] | None:
    """Per-request adapter ids from ``adapters`` (None, one name for all, or one name or None per request); None when no
    request names an adapter."""
    if adapters is None:
        return None
    names = [adapters] * count if isinstance(adapters, str) else list(adapters)
    if len(names) != count:
        raise ValueError(f"adapters must be one name or a list of {count} (one per prompt)")
    if all(n is None for n in names):
        return None
    loaded = getattr(model, "adapters", None)
    if loaded is None:
        raise ValueError("a request names an adapter but the model has none loaded (Qwen3ModelWeek3.load_adapters)")
    return [loaded.id_of(n) for n in names]
