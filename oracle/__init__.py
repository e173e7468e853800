"""CPU oracle for the tiny-llm Qwen3 W4A16 inference hot path.

THIS PACKAGE IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may import it.  The shipped package
(``tiny-llm_b200/``) never imports ``oracle`` and has no CPU fallback: its
operators raise when the CUDA extension is missing or when handed CPU tensors.

What it restates (all paths relative to the tiny-llm repository):

* ``oracle.ops``      - the arithmetic of every native primitive in
  ``src/extensions_ref/src/*.metal`` with the same rounding points (fp32
  accumulation, one bf16 rounding at the store), plus the builder-time
  validation of ``src/extensions_ref/src/*.cpp``.
* ``oracle.readable`` - the Week-1 readable operators
  (``src/tiny_llm_ref/{basics,layer_norm,positional_encoding,attention}.py``),
  the only part of the reference that can run on a CPU at all.
* ``oracle.model``    - ``Qwen3ModelWeek2(checkpoint="kv-cache")``
  (``src/tiny_llm_ref/qwen3_week2.py``) and the greedy loop of
  ``simple_generate_with_kv_cache`` (``src/tiny_llm_ref/generate.py:49-81``):
  "tiny_llm_ref's own CPU path", used as the reported CPU baseline.
* ``oracle.ext_cpu``  - a CPU stand-in with the exact function surface of the
  ``_ext`` module (``src/extensions_ref/bindings.cpp:14-46``) so that tests can
  drive the product's host logic (page pools, scheduler, models) without a GPU.

Pinning status (see DESIGN.md "Oracle"):

* integer / structural behaviour (page ids, page_lens, block tables, context
  lengths, growth counters, scheduler call traces, validation errors) is pinned
  by the literal known-answer values in the reference's own tests
  (``tests_refsol/test_week_3_day_{1,2,3,4}.py``), transcribed in
  ``tests/golden/reference_literals.json`` and in ``tests/``.
* floating-point operators: MLX (the reference's array runtime and the oracle
  of its float tests) cannot be installed here, and every reference primitive
  throws on CPU, so no reference-produced float output exists.  The float
  restatements are pinned by (a) the in-tree layout spec
  ``quantize.py:103-121`` checked through identity-matrix products, (b) the
  cross-implementation equalities the reference itself asserts (fast==readable
  RMSNorm/RoPE/SwiGLU, decode==grouped attention on the deterministic
  ``sin(arange*0.017+phase)`` fixtures, paged==dense, Week3==Week2) evaluated
  between two independently written restatements (``ops`` vs ``readable``),
  and (c) hand-computed closed-form cases.  Against MLX library outputs
  (``mx.quantized_matmul``, ``mx.fast.rope`` ...) parity is UNPINNED.
"""

from . import ops, readable  # noqa: F401
