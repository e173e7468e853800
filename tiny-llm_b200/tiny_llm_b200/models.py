"""Model dispatch (``src/tiny_llm/models.py:8-18``)."""

from __future__ import annotations

from .qwen3_week2 import Qwen3ModelWeek2
from .qwen3_week3 import Qwen3ModelWeek3

# model_names.py:1-8
MODEL_SHORTCUTS = {
    "qwen3-0.6b": "Qwen/Qwen3-0.6B-MLX-4bit",
    "qwen3-1.7b": "Qwen/Qwen3-1.7B-MLX-4bit",
    "qwen3-4b": "Qwen/Qwen3-4B-MLX-4bit",
}


def shortcut_name_to_full_name(name: str) -> str:
    return MODEL_SHORTCUTS.get(name.lower(), name)


def dispatch_model(model_name: str, mlx_model, week: int, **kwargs):
    """Week 2 -> dense-cache model, week 3 -> paged model.  Week 1 (uncached,
    readable-only) is not part of the CUDA hot path; its CPU restatement lives
    in ``oracle/model.py``."""
    full = shortcut_name_to_full_name(model_name)
    if full.startswith("Qwen/Qwen3"):
        if week == 2:
            return Qwen3ModelWeek2(mlx_model, **kwargs)
        if week == 3:
            return Qwen3ModelWeek3(mlx_model, **kwargs)
    raise ValueError(f"{full} for week {week} not supported")
