"""RoPE scaling for long context: static YaRN, the scaling Qwen3 documents for its 131,072-token window.

``config.json`` states it as ``"rope_scaling": {"rope_type": "yarn", "factor": 4.0,
"original_max_position_embeddings": 32768}``.  The project pins the semantics itself (DESIGN.md "Long context"):
with ``half = D / 2`` and ``i = 0 .. half - 1``

    extrap_i = theta^(-i / half),  interp_i = extrap_i / s
    corr(r)  = D * ln(L0 / (2 pi r)) / (2 ln theta)
    low      = max(floor(corr(beta_fast)), 0),  high = min(ceil(corr(beta_slow)), D - 1)   (high += 0.001 if equal)
    ramp_i   = clamp((i - low) / (high - low), 0, 1)
    inv_freq_i = interp_i * ramp_i + extrap_i * (1 - ramp_i)
    m        = attention_factor, or 0.1 ln(s) + 1

The rotated q and k are each scaled by ``m``; the model folds ``m^2`` into the attention scale instead, so the K pages
hold unscaled keys.  The window is ``s * L0``.  Any other ``rope_type`` is refused: it would load and compute wrongly.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import torch

YARN_BETA_FAST = 32.0
YARN_BETA_SLOW = 1.0
_YARN_KEYS = {"rope_type", "type", "factor", "original_max_position_embeddings", "beta_fast", "beta_slow", "attention_factor"}


@dataclass(frozen=True)
class Yarn:
    """Static YaRN parameters (``s``, ``L0``, the two betas and an optional explicit attention factor)."""

    factor: float
    original_max_position_embeddings: int
    beta_fast: float = YARN_BETA_FAST
    beta_slow: float = YARN_BETA_SLOW
    attention_factor: float | None = None

    @property
    def mscale(self) -> float:
        """``m``: the factor q and k are each scaled by."""
        return float(self.attention_factor) if self.attention_factor is not None else 0.1 * math.log(self.factor) + 1.0

    @property
    def window(self) -> int:
        """Positions the scaled model covers: ``s * L0``."""
        return int(self.factor * self.original_max_position_embeddings)

    def to_config(self) -> dict:
        """The ``rope_scaling`` entry of ``config.json``."""
        cfg = {"rope_type": "yarn", "factor": self.factor, "original_max_position_embeddings": self.original_max_position_embeddings}
        if self.beta_fast != YARN_BETA_FAST:
            cfg["beta_fast"] = self.beta_fast
        if self.beta_slow != YARN_BETA_SLOW:
            cfg["beta_slow"] = self.beta_slow
        if self.attention_factor is not None:
            cfg["attention_factor"] = self.attention_factor
        return cfg


def parse_rope_scaling(cfg, max_position_embeddings: int) -> Yarn | None:
    """``config.json``'s ``rope_scaling`` (a dict, a ``Yarn`` or None) as a ``Yarn``, or None for no scaling.
    ``ValueError`` for any other scaling type or for parameters out of range."""
    if cfg is None or isinstance(cfg, Yarn):
        return cfg
    if not isinstance(cfg, dict):
        raise ValueError(f"rope_scaling must be a mapping, got {type(cfg).__name__}")
    if not cfg:
        return None
    kind = cfg.get("rope_type", cfg.get("type"))
    if kind == "default":
        return None
    if kind != "yarn":
        raise ValueError(f"rope_scaling type {kind!r} is not supported (only static 'yarn')")
    unknown = sorted(set(cfg) - _YARN_KEYS)
    if unknown:  # e.g. mscale, mscale_all_dim, truncate: variants this definition does not compute
        raise ValueError(f"rope_scaling: yarn keys {unknown} are not supported (known: {sorted(_YARN_KEYS)})")
    if "factor" not in cfg:
        raise ValueError("rope_scaling: yarn needs a 'factor'")
    factor = float(cfg["factor"])
    original = int(cfg.get("original_max_position_embeddings") or max_position_embeddings)
    beta_fast = float(cfg.get("beta_fast", YARN_BETA_FAST))
    beta_slow = float(cfg.get("beta_slow", YARN_BETA_SLOW))
    attention_factor = cfg.get("attention_factor")
    if not factor >= 1.0 or not math.isfinite(factor):
        raise ValueError(f"rope_scaling: yarn factor must be a finite number >= 1 (got {cfg['factor']!r})")
    if original <= 0:
        raise ValueError(f"rope_scaling: original_max_position_embeddings must be positive (got {original})")
    if not beta_fast > beta_slow > 0:
        raise ValueError(f"rope_scaling: need beta_fast > beta_slow > 0 (got {beta_fast}, {beta_slow})")
    if attention_factor is not None:
        attention_factor = float(attention_factor)
        if not attention_factor > 0 or not math.isfinite(attention_factor):
            raise ValueError(f"rope_scaling: attention_factor must be positive (got {cfg['attention_factor']!r})")
    return Yarn(factor, original, beta_fast, beta_slow, attention_factor)


def parse_cli(spec: str) -> dict:
    """``--rope-scaling yarn:FACTOR[:ORIGINAL]`` as a ``rope_scaling`` config entry."""
    parts = spec.split(":")
    if parts[0] != "yarn" or len(parts) not in (2, 3):
        raise ValueError(f"--rope-scaling expects yarn:FACTOR[:ORIGINAL] (got {spec!r})")
    try:
        cfg = {"rope_type": "yarn", "factor": float(parts[1])}
        if len(parts) == 3:
            cfg["original_max_position_embeddings"] = int(parts[2])
    except ValueError:
        raise ValueError(f"--rope-scaling expects yarn:FACTOR[:ORIGINAL] (got {spec!r})") from None
    parse_rope_scaling(cfg, 1)  # range checks
    return cfg


def yarn_correction_range(yarn: Yarn, theta: float, head_dim: int) -> tuple[float, float]:
    """``(low, high)`` of the ramp; ``high`` already carries the +0.001 of a degenerate range."""

    def corr(r: float) -> float:
        return head_dim * math.log(yarn.original_max_position_embeddings / (2 * math.pi * r)) / (2 * math.log(theta))

    low = max(math.floor(corr(yarn.beta_fast)), 0)
    high = min(math.ceil(corr(yarn.beta_slow)), head_dim - 1)
    if low == high:
        high += 0.001
    return float(low), float(high)


def default_inv_freq(head_dim: int, theta: float, device) -> torch.Tensor:
    """Unscaled float64 ``[head_dim / 2]`` frequencies.  On a GPU they are formed by the RoPE kernels' own expression
    (``ext.rope_default_inv_freq``), so a site given them computes the bits of its ``base`` path."""
    if torch.device(device).type == "cuda":
        from extensions_b200 import tiny_llm_ext_b200 as ext

        return ext.rope_default_inv_freq(head_dim, theta, device)
    half = head_dim // 2
    theta32 = float(torch.tensor(float(theta), dtype=torch.float32))  # the kernels take base as a float
    return torch.exp2(-torch.arange(half, dtype=torch.float64) / half * math.log2(theta32)).to(device)


def rope_inv_freq(head_dim: int, theta: float, scaling: Yarn | None, device) -> torch.Tensor:
    """The model's float64 ``[head_dim / 2]`` RoPE frequency table: ``default_inv_freq``, blended in float64 for YaRN."""
    extrap = default_inv_freq(head_dim, theta, device)
    if scaling is None:
        return extrap
    low, high = yarn_correction_range(scaling, theta, head_dim)
    i = torch.arange(head_dim // 2, dtype=torch.float64, device=extrap.device)
    ramp = ((i - low) / (high - low)).clamp(0.0, 1.0)
    interp = extrap / scaling.factor
    return (interp * ramp + extrap * (1.0 - ramp)).contiguous()
