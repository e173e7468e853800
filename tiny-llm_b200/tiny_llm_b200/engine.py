"""CUDA-graph decode engine for the Week-3 paged model (CUDA host runtime).

The reference issues ~500 operator calls per generated token from a Python loop
(SURVEY.md section 3.1); at these speeds one W4A16 projection lasts about a
microsecond, so per-call dispatch would leave the GPU idle >90 % of the time.
The engine keeps the operator semantics and removes the dispatch:

* one decode step (embedding -> 36 blocks -> norm -> tied head -> greedy
  argmax) for a fixed number of slots ``B`` is captured once into a CUDA graph
  over static buffers and replayed per step;
* everything the step needs from the scheduler is DATA, not kernel arguments:
  token ids, RoPE offsets, post-append context lengths and the per-layer block
  tables live in one device buffer that is refreshed with a single pinned
  host->device copy; K/V appends and attention read page ids from it;
* the integer page bookkeeping stays on the host in the very same
  ``TinyKvPagedCache`` / ``TinyKvPagedPool`` objects the per-operator path uses
  (``append_token_slot``), so block tables, page ids and counters are identical;
* ``decode_on_device`` runs N greedy steps with no host involvement at all
  (token feedback + position advance by ``tl_decode_advance``, pages allocated
  ahead) - the device-resident number of bench.py.  With ``sampling`` it replays
  a second self-advancing graph that draws each slot's token with the seeded
  ``tl_sample`` kernel instead of ``tl_argmax``, and with a penalised slot a
  third one with ``tl_sample_penalized`` over per-slot token counts kept on the
  device.

Page slabs must not move while a graph is alive: pools are ``reserve()``d up
front and the engine re-captures if a slab pointer changes.
"""

from __future__ import annotations

import gc
from types import SimpleNamespace

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

from .json_mode import ConstraintRows, JsonConstraint
from .json_schema import JsonSchemaConstraint
from .kv_cache import BatchingKvCache
from .moe import Moe, router_logits
from .paged_kv_cache import TinyKvPagedCache

# Decode attention runs as one fused launch while slots x max_seq_len stays within this: beyond it the K/V stream, not
# the launch count, bounds the step.
FUSED_ATTENTION_MAX_SLOT_TOKENS = 16384

# Grouped decode attention (tl_shared_prefix_attention, DESIGN.md section 16) replaces the step's attention for a group
# of COUNT slots sharing SHARED_TOKENS prompt tokens only where tools/parallel_sample_bench.py measured it faster.
SHARED_PREFIX_MIN_COUNT = 2
SHARED_PREFIX_MIN_TOKENS = 1024


def shared_prefix_attention_applies(count: int, shared_tokens: int, model) -> bool:
    """Whether a group of ``count`` slots that share ``shared_tokens`` leading tokens decodes with grouped attention:
    the kernel's conditions (bf16, head_dim 128, pages a multiple of 64 slots, ``count x G <= 128``) and the measured
    rule (DESIGN.md section 16)."""
    attn0 = model.layers_inner[0].self_attn
    G = attn0.num_heads // attn0.num_kv_heads
    if (attn0.head_dim != 128 or model.page_size % 64 != 0 or 128 % G != 0 or count * G > 128
            or model.embedding.weight.scales.dtype != torch.bfloat16):
        return False
    return count >= SHARED_PREFIX_MIN_COUNT and shared_tokens >= SHARED_PREFIX_MIN_TOKENS


def shared_run(tables, first: int, count: int, write_from: int, page_size: int) -> int:
    """Leading pages that slots ``first .. first + count - 1`` share in every layer of ``tables`` ([layers, B,
    max_pages] page ids), stopping before the page holding position ``write_from`` (the first a slot may still write).
    Forks share the same run in every layer; a group whose layers disagree is refused with ``ValueError``."""
    limit = max(write_from, 0) // page_size
    rows = np.asarray(tables)[:, first : first + count, :limit]
    same = (rows == rows[:, :1, :]).all(axis=1) & (rows[:, 0, :] >= 0)  # [layers, limit]
    runs = [int(np.argmin(r)) if not r.all() else limit for r in same]
    if len(set(runs)) != 1:
        raise ValueError(f"slots {first}..{first + count - 1} do not share the same pages in every layer")
    return runs[0]


def _concat_weights(parts):
    """Stack packed projections along the output dimension (one launch instead of
    len(parts)): rows of codes, scales and biases are simply concatenated."""
    first = parts[0]
    return SimpleNamespace(
        weight=torch.cat([p.weight.view(torch.int32) if p.weight.dtype == torch.uint32 else p.weight for p in parts], dim=0).contiguous(),
        scales=torch.cat([p.scales for p in parts], dim=0).contiguous(),
        biases=torch.cat([p.biases for p in parts], dim=0).contiguous(),
        group_size=first.group_size,
        bits=first.bits,
    )


def _interleave_gate_up(gate, up):
    """gate|up rows in blocks of 8 (``ext.interleave_gate_up``): the streaming kernel's
    EPI_SWIGLU_PAIRS epilogue then emits swiglu(gate, up) directly, so the MLP activation never
    makes a round trip through memory as two separate vectors."""
    as_i32 = lambda w: w.view(torch.int32) if w.dtype == torch.uint32 else w
    return SimpleNamespace(
        weight=ext.interleave_gate_up(as_i32(gate.weight), as_i32(up.weight)),
        scales=ext.interleave_gate_up(gate.scales, up.scales),
        biases=ext.interleave_gate_up(gate.biases, up.biases),
        group_size=gate.group_size,
        bits=gate.bits,
    )


def pack_layers(model) -> list:
    """Per layer, the weights of the fused launches: q|k|v and gate|up share their input, so they stream as one launch
    each.  ``Qwen3ModelWeek3.packed_layers`` keeps one such copy per model for all of its engines."""
    return [SimpleNamespace(qkv=_concat_weights([b.self_attn.wq, b.self_attn.wk, b.self_attn.wv]),
                            gate_up=b.mlp.w_gate_up if isinstance(b.mlp, Moe) else _interleave_gate_up(b.mlp.w_gate, b.mlp.w_up))
            for b in model.layers_inner]


def _normed(h, norm):
    return ext.rms_norm(h, norm._weight_as(h.dtype, h.device), norm.eps)


def _proj(h, w):
    return ext.quantized_matmul(w.scales, w.biases, w.group_size, w.bits, h, w.weight, True)


def _moe_mlp(moe, x, h=None, ln2=None, nxt=None):
    """The sparse MLP of one layer (``moe.Moe``) in place of the dense gate|up and down launches: returns the residual
    stream ``x`` plus the expert mixture.  ``h``: the rows already normalised by the post-attention RMSNorm; without it
    (the matvec stack) the router projection takes ``ln2`` as its prologue and the gather applies it to each row.  With
    ``nxt`` (the next RMSNorm) the combine also returns its output, as ``(x, h)``.  Every row is routed, idle slots and
    padding rows included: a row's result depends only on that row."""
    if h is None:
        norm = (ln2._weight_as(x.dtype, x.device), ln2.eps)
        logits = router_logits(x, moe.w_router, norm=norm)
    else:
        norm, logits = None, router_logits(h, moe.w_router, projection=_proj)
    _, ids, scores = ext.moe_topk(logits, moe.num_experts_per_tok, moe.norm_topk_prob)
    return moe.experts(x if h is None else h, ids, scores, residual=x, gather_norm=norm,
                       next_norm=None if nxt is None else (nxt._weight_as(x.dtype, x.device), nxt.eps))


def _swap_ab_layers(model, x, attention):
    """The layer stack for 9 to 128 rows ``x`` (decode slots or prefill tokens); returns the final hidden rows, already
    normalised.  The projections run on the swap-AB wgmma kernel (w4a16_skinny.cu: weights streamed once for all rows),
    which has no prologue, so the first RMSNorm is its own (tiny) launch; after that the residual projections (o, down)
    hand the NEXT RMSNorm's output back together with the residual stream (one launch: the kernel that adds the
    split-reduction planes has the whole row in registers).  The rounding points are those of the operator sequence.
    ``attention(i, block, h)`` runs layer ``i``'s q|k|v projection and attention on the normalised rows ``h`` and
    returns ``[rows, Hq * D]``."""
    layers = list(model.layers_inner)
    packed = model.packed_layers()
    h = _normed(x, layers[0].input_layernorm)
    for i, block in enumerate(layers):
        wo, gate_up = block.self_attn.wo, packed[i].gate_up
        ln2 = block.post_attention_layernorm
        y = attention(i, block, h)
        x, h = ext.quantized_matmul_residual_norm(wo.scales, wo.biases, wo.weight, y, x, ln2._weight_as(x.dtype, x.device), ln2.eps)
        nxt = layers[i + 1].input_layernorm if i + 1 < len(layers) else model.norm
        if isinstance(block.mlp, Moe):
            x, h = _moe_mlp(block.mlp, x, h, nxt=nxt)
            continue
        wd = block.mlp.w_down
        act = ext.quantized_matmul_fused(gate_up.scales, gate_up.biases, gate_up.weight, h, epilogue=ext.EPI_SWIGLU_PAIRS)
        x, h = ext.quantized_matmul_residual_norm(wd.scales, wd.biases, wd.weight, act, x, nxt._weight_as(x.dtype, x.device), nxt.eps)
    return h


def lora_projection_is_fused(rows: int) -> bool:
    """Whether ``_lora_layers`` projects ``rows`` rows through ``quantized_matmul_fused`` (else ``quantized_matmul``)."""
    return rows <= 128


def _lora_layers(model, x, ids, attention):
    """The layer stack of a model with an ``AdapterSet`` (``lora.py``), for any number of rows ``x``; ``ids`` holds one
    adapter id per row (device data: -1 runs the base model) and ``attention(i, block, qkv)`` turns layer ``i``'s q|k|v
    rows into ``[rows, Hq * D]``.  Returns the residual stream before the final norm.

    Every adapter delta has to land on its projection's output before the next operator reads it, so the fused
    prologues and epilogues of the base stacks (RMSNorm into the projection, SwiGLU and the residual out of it) are
    their own launches here: rms_norm, q|k|v, lora, attention, o, lora (+ residual), rms_norm, gate, up, lora, swiglu,
    down, lora (+ residual).  A site no adapter of the set targets issues no lora launch (its residual is ``add``).
    Up to 128 rows the projections are the fused entry's (streaming matvec to 8 rows, swap-AB wgmma split reduction to
    128); beyond, the plain entry's 128-token wgmma tile GEMM, as in the base prefill engine's per-operator branch (the
    fused entry would keep such chunks on the streaming matvec, one pass over the weights per 32 rows).
    The rounding points are those of the operator path with the same ids."""
    packed, sites = model.packed_layers(), model.adapters.sites
    if lora_projection_is_fused(x.shape[0]):
        fused = lambda w, h: ext.quantized_matmul_fused(w.scales, w.biases, w.weight, h)
    else:
        fused = lambda w, h: _proj(h, w)

    def plus_residual(inp, out, site):
        return ext.add(x, out) if site is None else ext.lora_apply(inp, out, ids, site, residual=x)

    for i, block in enumerate(model.layers_inner):
        at, mlp, st = block.self_attn, block.mlp, sites[i]
        h = _normed(x, block.input_layernorm)
        qkv = fused(packed[i].qkv, h)
        if st.qkv is not None:
            ext.lora_apply(h, qkv, ids, st.qkv)
        y = attention(i, block, qkv)
        x = plus_residual(y, fused(at.wo, y), st.o)
        h = _normed(x, block.post_attention_layernorm)
        gate, up = fused(mlp.w_gate, h), fused(mlp.w_up, h)
        if st.gate_up is not None:
            ext.lora_apply(h, [gate, up], ids, st.gate_up)
        act = ext.swiglu(gate, up)
        x = plus_residual(act, fused(mlp.w_down, act), st.down)
    return x


class _GraphEngine:
    """What the decode and prefill engines share: the geometry, one pinned int32 metadata block with its device mirror
    (each engine lays it out as ``header | block tables`` and initialises the tables to -1), the event that keeps the
    pinned block from being rewritten while its upload is still in flight, and graph capture on a side stream.

    Page slabs must not move while a graph is alive, so the graphs are re-captured when a pool's slab version changes.
    The warm-up passes of every capture really run: with the previous step's metadata still on the device they would
    append a stale token's K/V through a stale block table - possibly into a page that has been released and handed to
    another request since (slabs move when a second engine reserves more pages).  So ``_capture`` first sets the device
    metadata to all-idle (``_set_idle``: nothing is appended, attention sees no keys); every replay uploads the real
    block first."""

    def __init__(self, model, max_seq_len: int, device, header_len: int, table_rows: int):
        self.model = model
        self.device = torch.device(device)
        self.page_size = model.page_size
        self.max_pages = (max_seq_len + self.page_size - 1) // self.page_size
        self.max_seq_len = self.max_pages * self.page_size
        self.n_layers = model.num_hidden_layers
        self.lora = model.adapters  # an AdapterSet: this is a LoRA engine (``_lora_layers``, per-row adapter ids as device data)
        attn = model.layers_inner[0].self_attn
        self.Hq, self.Hkv, self.D = attn.num_heads, attn.num_kv_heads, attn.head_dim
        # tables: [layers, table_rows, max_pages]
        self._meta_len = header_len + self.n_layers * table_rows * self.max_pages
        self.meta_host = torch.empty(self._meta_len, dtype=torch.int32, pin_memory=True)
        self.meta_np = self.meta_host.numpy()
        self.meta_np[:header_len] = 0
        self.meta_np[header_len:] = -1
        self.meta_dev = self.meta_host.to(self.device, copy=True)
        self._upload_event = torch.cuda.Event()
        self._upload_pending = False
        self._stream = torch.cuda.Stream(device=self.device)
        self._graph = None
        self._slab_ptrs = None
        self.captures = 0  # graph (re-)captures: 1 + one per move of the page slabs
        self.logits = None

    def reserve_pools(self, pages_per_layer: int) -> None:
        for pool in self.model.page_pools:
            pool.reserve(pages_per_layer, self.Hkv, self.D, dtype=torch.bfloat16, device=self.device)

    def _slabs(self):
        return tuple(p.slab_version for p in self.model.page_pools)  # changes whenever a pool's slabs are (re)allocated

    def _ensure_graph(self) -> None:
        if self._graph is None or self._slab_ptrs != self._slabs():
            self._capture()

    def _capture(self) -> None:
        self.captures += 1
        self._slab_ptrs = self._slabs()
        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self._capture_graphs()
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _graph_of(self, body, pool=None, warmups: int = 2) -> torch.cuda.CUDAGraph:
        """Run ``body`` ``warmups`` times (lazy kernel attribute setup must not happen under capture), then capture it
        on the side stream, into ``pool`` if given.  ``self._launches`` is the number of library launches captured."""
        for _ in range(warmups):
            body()
        self._stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        launched = ext.launch_count()
        # No garbage collection inside the capture: a collected engine frees its pinned metadata block, and the host
        # allocator's event calls on another stream invalidate a global-mode capture.
        gc_was_enabled = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(graph, stream=self._stream, pool=pool):
                body()
        finally:
            if gc_was_enabled:
                gc.enable()
        self._launches = ext.launch_count() - launched
        return graph

    def _host_write_begin(self) -> None:
        """The pinned block is about to be rewritten: the previous upload must have been consumed
        (a caller that keeps sampling on the device never synchronises between steps)."""
        if self._upload_pending:
            self._upload_event.synchronize()
            self._upload_pending = False

    def _alloc_adapter_ids(self, rows: int, key) -> None:
        """A LoRA engine's adapter id per row, in its own pinned block (all -1: the base model), uploaded when it changes;
        ``key`` is what ``_set_adapter_ids`` compares against for that state."""
        self._ad_host = torch.full((rows,), -1, dtype=torch.int32).pin_memory()
        self.adapter_ids = self._ad_host.to(self.device, copy=True)
        self._ad_key = key

    def _set_adapter_ids(self, key) -> int:
        """Upload the rows' ids if they changed: ``key`` is a tuple of one id per row, or one int for all rows.  Returns
        the bytes copied."""
        if key == self._ad_key:
            return 0
        self._host_write_begin()
        self._ad_host.numpy()[:] = key
        self._upload_meta(self.adapter_ids, self._ad_host)
        self._ad_key = key
        return 4 * self._ad_host.numel()

    def _upload_meta(self, dev, host) -> None:
        """Copy the pinned block (or a prefix of it) to its device mirror on the current stream."""
        dev.copy_(host, non_blocking=True)
        self._upload_event.record()
        self._upload_pending = True


class _LockstepGroup:
    """The per-layer cache objects of ONE request plus the number of one-token appends the engine
    has accounted for but not yet written into them (see ``TinyKvPagedCache._lazy``)."""

    __slots__ = ("caches", "pending")

    def __init__(self, caches):
        self.caches = caches
        self.pending = 0

    def settle(self) -> None:
        n = self.pending
        if n:
            self.pending = 0
            for c in self.caches:
                c._page_lens[-1] += n
                c._offset += n


class _SlotRecord:
    """What the engine knows about the request in one decode slot."""

    __slots__ = ("c0", "group", "lockstep", "epoch", "offset", "pages")

    def __init__(self, c0, group, lockstep):
        self.c0, self.group, self.lockstep = c0, group, lockstep
        self.epoch = c0.epoch
        self.offset = c0._offset      # logical context length (settled offset + pending)
        self.pages = len(c0.page_ids)


class DecodeEngine(_GraphEngine):
    """One decode step of ``B`` slots as a CUDA graph (module docstring).  Metadata block:
    ``tokens [N] | offsets [N] | context_lens [N] | block tables [Ly, B, MP]`` with ``N = B * rows_per_request`` query
    rows (``rows_per_request > 1``: ``VerifyEngine``, consecutive tokens of one request per slot).  The fused path uses
    the model's one packed weight copy (``Qwen3ModelWeek3.packed_layers``); B > 8 runs the layer stack shared with the
    prefill engine (``_swap_ab_layers``)."""

    def __init__(self, model, batch_size: int, max_seq_len: int, device, log_capacity: int = 4096, fused: bool = True, *,
                 _row_variants: bool = True, rows_per_request: int = 1):
        B = self.B = batch_size
        self._rows_per_request = rows_per_request
        N = self.rows = B * rows_per_request
        super().__init__(model, max_seq_len, device, 3 * N, B)
        self.V = model.vocab_size
        self.log_capacity = log_capacity
        self._meta_dev_head, self._meta_host_head = self.meta_dev[: 3 * N], self.meta_host[: 3 * N]  # the per-step upload
        self.tokens = self.meta_dev[0:N]
        self.offsets = self.meta_dev[N : 2 * N]
        self.context_lens = self.meta_dev[2 * N : 3 * N]
        self.tables = self.meta_dev[3 * N :].view(self.n_layers, B, self.max_pages)
        self.tables_np = self.meta_np[3 * N :].reshape(self.n_layers, B, self.max_pages)
        self.next_tokens = torch.zeros(N, dtype=torch.int32, device=self.device)
        self.out_log = torch.full((log_capacity * B,), -1, dtype=torch.int32, device=self.device)
        self.step_counter = torch.zeros(1, dtype=torch.int32, device=self.device)
        # per slot: the request group (its per-layer cache objects) the table rows reflect
        self._recs: list[_SlotRecord | None] = [None] * B
        self._tables_dirty = True
        self.h2d_bytes = 0  # bytes copied host -> device by step() / decode_on_device() so far
        self._graph_loop = None
        self.graph_replays = 0
        self.kernels_per_step = 0
        attn0 = model.layers_inner[0].self_attn
        self.fused = bool(fused) and not attn0.rope.traditional and attn0.rope.dims == self.D and self.D % 2 == 0
        self._packed = model.packed_layers() if self.fused else None
        # one-launch attention (q/k norm + rope + append + paged GQA) when the head layout allows it
        # The one-launch attention is a latency design (few CTAs, K/V rows staged per lane): it wins while the
        # step is launch-bound.  With many slots or long contexts the K/V stream dominates and the step uses
        # q/k norm + rope + append as one small launch followed by tl_paged_attention, whose long-context path
        # is the TMA + wgmma streaming kernel (attention_prefill_tc.cu).
        self._attention_fused = self.fused and DecodeEngine.fused_attention_applies(model, self.B * self.max_seq_len)
        if self._attention_fused:
            # the model's scaled table when it has one (every site reads it); else the fused kernel's own unscaled table
            self._rope_inv_freq = attn0.rope.inv_freq if attn0.rope.inv_freq is not None else ext.rope_inv_freq_table(self.D, attn0.rope.base, self.device)
            self._attn_ws = torch.empty(ext.decode_attention_fused_workspace(self.B, self.Hq, self.Hkv, rows_per_request=rows_per_request),
                                        dtype=torch.float32, device=self.device)
        # Row variants: the scheduler fills slots from index 0 (batch.py:220-226), so while few requests are live the
        # occupied slots are a prefix of the table.  A step graph over the first 16 / 32 rows is captured beside the
        # full one and step() replays the smallest that covers the highest occupied slot: every kernel of the wide
        # path costs by rows (swap-AB column count, attention CTAs, reduction planes).  All variants stay on the
        # >= 9-row kernels and the split counts do not depend on the row count, so a row's result is bit-identical
        # whichever variant computed it.  (Config 4 runs 64 slots with ~20 live.)  _row_variants=False keeps only the
        # full-width graph: the reference those bits are tested against.
        self._variants = sorted({r for r in (16, 32, 64) if r < self.B} | {self.B}) if (self.fused and self.B > 16 and _row_variants) else [self.B]
        self._graphs: dict = {}
        self.variant_replays = {r: 0 for r in self._variants}
        # decode_on_device(sampling=...): per-slot parameters in their own pinned block (seed i64 | temperature f32 |
        # top_k i32 | top_p f32, B each), uploaded only when they change; the sampled graph is captured on first use
        self._graph_sample = None
        self.kernels_per_sampled_step = 0
        self._samp_host = torch.zeros(20 * B, dtype=torch.uint8, pin_memory=True)
        self._samp_dev = self._samp_host.to(self.device, copy=True)
        self._samp_key = None
        self._samp_seed = self._samp_dev[: 8 * B].view(torch.int64)
        self._samp_temperature = self._samp_dev[8 * B : 12 * B].view(torch.float32)
        self._samp_top_k = self._samp_dev[12 * B : 16 * B].view(torch.int32)
        self._samp_top_p = self._samp_dev[16 * B : 20 * B].view(torch.float32)
        # decode_on_device(logprobs=...): one more graph per (greedy | sampled) step, the same body plus one tl_logprobs
        # launch on the step's tokens, logging into [log_capacity, B(, max_n)] buffers at the step counter; per-slot
        # top-N counts in their own pinned block.  All of it is allocated / captured on first use.
        self._graph_lp: dict = {}
        self._lp_max_n = None
        self._lp_log = None
        self._lp_host = None
        self._lp_dev = None
        self._lp_key = None
        self.kernels_per_logprobs_step = 0
        # decode_on_device(sampling=<penalised>): the penalised sampled graph, the per-slot token state [B, V] it reads and
        # counts into, and the penalty parameters in their own pinned block (repetition | presence | frequency | min_p
        # f32, B each), all on first use
        self._graph_pen = None
        self.kernels_per_penalized_step = 0
        self.token_counts = None
        self._pen_host = None
        self._pen_dev = None
        self._pen_key = None
        # decode_on_device(sampling=<constrained>): one graph per (penalised, logprobs N or None), the step with
        # tl_sample_constrained as its token choice, over a [B, 5] int64 slab of tl_constraint_row descriptors whose
        # states the launches advance; all on first use
        self._graph_con: dict = {}
        self.kernels_per_constrained_step = 0
        # decode_on_device(sampling=<with a JSON-mode slot>): one graph per (penalised, logprobs N or None), the
        # constrained step between tl_json_token_masks and tl_json_advance over a B-row ConstraintRows (descriptors,
        # JSON states and mask buffers; regex and plain slots ride along); all on first use
        self._graph_json: dict = {}
        self.kernels_per_json_step = 0
        self._json_tab = None
        self._json_key = None
        # decode_on_device(sampling=<with a JSON Schema slot>): one graph per (penalised, logprobs N or None, any JSON
        # slot), the constrained step between the schema (and JSON) rows' masks and their advances over a B-row
        # ConstraintRows of its own; all on first use
        self._graph_schema: dict = {}
        self.kernels_per_schema_step = 0
        self._schema_tab = None
        self._schema_key = None
        # decode_on_device(sampling=..., keep_logits=True): the sampled step plus one tl_log_rows launch that keeps the
        # step's logits rows in a [capacity, B, V] log at the step counter (a speculative draft's q rows); on first use
        self._graph_keep = None
        self._logits_log = None
        # VerifyEngine.verify(sampling=...): the verify pass with tl_speculative_sample as its token choice, one graph
        # per draft-logits buffer it reads
        self._graph_spec: dict = {}
        self._con_host = None
        self._con_dev = None
        self._con_key = None
        # beam_step(): the greedy step body, then tl_logprobs' top N = B + E of every row into fixed buffers and
        # tl_beam_select, one graph per EOS tuple (the ids are kernel arguments, and they fix N); the beams' cumulative
        # log-probabilities live in beam_cum, which the select rewrites in place; all on first use
        self._graph_beam: dict = {}
        self._beam_bufs: dict = {}
        self.beam_cum = None
        self.kernels_per_beam_step = 0
        # decode_on_device(groups=...): grouped twins of the sampled step (with and without logprobs), whose attention is
        # q/k norm + RoPE + append then tl_shared_prefix_attention over the (first_slot, count, shared_pages) descriptors
        # of the call; one graph per logprobs N (None: none), all on first use
        self._graph_grp: dict = {}
        self._grp_host = None
        self._grp_dev = None
        self._grp_ws = None
        self.kernels_per_grouped_step = 0
        if self.lora is not None:
            if rows_per_request != 1 or not self.fused:
                raise ValueError("a model with adapters runs one row per slot on the fused decode step")
            self._alloc_adapter_ids(B, (-1,) * B)

    @staticmethod
    def fused_attention_applies(model, slot_tokens: int) -> bool:
        """The one-launch attention's conditions on the model, for ``slots x max_seq_len`` = ``slot_tokens``."""
        attn0 = model.layers_inner[0].self_attn
        rope = attn0.rope
        return (not rope.traditional and rope.dims == attn0.head_dim and attn0.head_dim == 128
                and attn0.num_heads // attn0.num_kv_heads <= 4 and model.embedding.weight.scales.dtype == torch.bfloat16
                and slot_tokens <= FUSED_ATTENTION_MAX_SLOT_TOKENS)

    def reserve_pools(self, pages_per_layer: int | None = None) -> None:
        super().reserve_pools(pages_per_layer if pages_per_layer is not None else self.B * self.max_pages + 1)

    # ------------------------------------------------------------ graph body --
    def _next_tokens(self, logits, R: int, sampled: bool, penalized: bool = False, constrained: bool = False, spec_draft=None) -> None:
        """The step's token per row: ``tl_argmax``, or (the sampled graph) ``tl_sample`` with the per-slot parameters at
        position ``context_lens``, the index of the token being drawn, or (the penalised graph) ``tl_sample_penalized``
        over ``token_counts``, or (a constrained graph) ``tl_sample_constrained`` over the slot descriptors, or (the
        sampled verify graph, ``spec_draft`` the draft's logits rows) ``tl_speculative_sample`` on the proposals.
        ``constrained == "json"`` (the JSON graph) draws over the JSON table's descriptors, between the JSON rows' mask
        launch and their state advance; ``constrained == "schema"`` (the schema graph) likewise over the schema table,
        with the schema rows' launches (and the JSON rows' when the table holds any); the masks launch stages the tables
        in the shared memory the table held at capture."""
        if spec_draft is not None:
            ext.speculative_sample(logits, spec_draft, self.tokens[1:R], *self._spec_params, self.context_lens[:R], out=self.next_tokens[:R])
            return
        if constrained:
            pen = ()
            if penalized:
                p = self._pen_dev.view(torch.float32).view(4, self.B)
                pen = (p[0, :R], p[1, :R], p[2, :R], p[3, :R], self.token_counts[:R])
            tab = self._json_tab if constrained == "json" else self._schema_tab if constrained == "schema" else None
            if tab is not None and tab.has_json:
                ext.json_token_masks(tab.descriptors[:R], tab.json_states[:R], self.V)
            if tab is not None and tab.has_schema:
                ext.schema_token_masks(tab.descriptors[:R], tab.schema_states[:R], self.V, tab.schema_smem_bytes)
            descriptors = self._con_dev.view(self.B, -1)[:R] if tab is None else tab.descriptors[:R]
            tokens = ext.sample_constrained(logits, self._samp_temperature[:R], self._samp_top_k[:R], self._samp_top_p[:R], self._samp_seed[:R],
                                            self.context_lens[:R], descriptors, *pen)
            if tab is not None and tab.has_json:
                ext.json_advance(tab.descriptors[:R], tab.json_states[:R], tokens, self.context_lens[:R])
            if tab is not None and tab.has_schema:
                ext.schema_advance(tab.descriptors[:R], tab.schema_states[:R], tokens, self.context_lens[:R])
        elif penalized:
            pen = self._pen_dev.view(torch.float32).view(4, self.B)
            tokens = ext.sample_penalized(logits, self._samp_temperature[:R], self._samp_top_k[:R], self._samp_top_p[:R], self._samp_seed[:R],
                                          self.context_lens[:R], pen[0, :R], pen[1, :R], pen[2, :R], pen[3, :R], self.token_counts[:R])
        elif sampled:
            tokens = ext.sample(logits, self._samp_temperature[:R], self._samp_top_k[:R], self._samp_top_p[:R], self._samp_seed[:R],
                                self.context_lens[:R])
        else:
            tokens = ext.argmax(logits)
        self.next_tokens[:R].copy_(tokens)

    def _forward_unfused(self, sampled: bool = False, penalized: bool = False, constrained: bool = False) -> None:
        """One decode step over the static buffers, operator by operator (the
        call sequence of qwen3_week3.py:55-121,139-146,196-207,320-338 at L == 1)."""
        m = self.model
        B, Hq, Hkv, D = self.B, self.Hq, self.Hkv, self.D
        emb = m.embedding.weight
        x = ext.quantized_embedding(self.tokens, emb.scales, emb.biases, emb.weight, emb.group_size, emb.bits)  # [B, H]

        for i, block in enumerate(m.layers_inner):
            at = block.self_attn
            pool = m.page_pools[i]
            h = _normed(x, block.input_layernorm)
            q = _proj(h, at.wq).view(B, 1, Hq, D)
            k = _proj(h, at.wk).view(B, 1, Hkv, D)
            v = _proj(h, at.wv).view(B, Hkv, 1, D)
            q = ext.rms_norm(q, at.q_norm._weight_as(x.dtype, x.device), at.q_norm.eps)
            k = ext.rms_norm(k, at.k_norm._weight_as(x.dtype, x.device), at.k_norm.eps)
            q = at.rope(q, self.offsets)
            k = at.rope(k, self.offsets)
            ext.paged_cache_append_decode(pool._key_pages, pool._value_pages, k.view(B, Hkv, 1, D), v, self.tables[i], self.context_lens)
            y = ext.paged_attention(q.view(B * Hq, 1, D), pool._key_pages, pool._value_pages, self.tables[i], self.context_lens,
                                    at.scale, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
            x = ext.add(x, _proj(y.view(B, Hq * D), at.wo))
            h = _normed(x, block.post_attention_layernorm)
            mlp = block.mlp
            if isinstance(mlp, Moe):
                x = _moe_mlp(mlp, x, h)
                continue
            x = ext.add(x, _proj(ext.swiglu(_proj(h, mlp.w_gate), _proj(h, mlp.w_up)), mlp.w_down))
        x = _normed(x, m.norm)
        head = m.w_lm_head if m.w_lm_head is not None else m.embedding.weight
        logits = _proj(x, head)
        self._next_tokens(logits, B, sampled, penalized, constrained)
        if self.logits is None:
            self.logits = torch.empty_like(logits)
        self.logits.copy_(logits)

    def _forward_fused(self, rows: int | None = None, sampled: bool = False, penalized: bool = False, constrained: bool = False,
                       spec_draft=None, grouped: bool = False) -> None:
        """Same step in ~7 launches per layer: norm / SwiGLU / residual folded into
        the streaming projections, q/k norm + RoPE + K/V append in one kernel.
        Every rounding point of the operator-by-operator sequence is kept.
        ``rows``: only the first ``rows`` slots (a row variant, see __init__)."""
        m = self.model
        R = self.rows if rows is None else rows
        emb = m.embedding.weight
        x = ext.quantized_embedding(self.tokens[:R], emb.scales, emb.biases, emb.weight, emb.group_size, emb.bits)
        head = m.w_lm_head if m.w_lm_head is not None else m.embedding.weight
        if self.lora is not None:
            x = _normed(_lora_layers(m, x, self.adapter_ids[:R], self._qkv_attention(R)), m.norm)
            logits = ext.quantized_matmul_fused(head.scales, head.biases, head.weight, x)
        elif self.B > 8:
            h = _swap_ab_layers(m, x, self._swap_ab_attention(R, grouped))
            logits = ext.quantized_matmul_fused(head.scales, head.biases, head.weight, h)
        else:
            x = self._matvec_layers(x, grouped)
            logits = ext.quantized_matmul_fused(head.scales, head.biases, head.weight, x, m.norm._weight_as(x.dtype, x.device),
                                                prologue=ext.PRO_RMSNORM, eps=m.norm.eps)
        self._next_tokens(logits, R, sampled, penalized, constrained, spec_draft)
        if self.logits is None:
            self.logits = torch.zeros((self.rows, logits.shape[-1]), dtype=logits.dtype, device=logits.device)
        self.logits[:R].copy_(logits)

    def _grouped_attention(self, i: int, at, q):
        """``tl_shared_prefix_attention`` of all B slots over the descriptors of the call (layer ``i``)."""
        pool = self.model.page_pools[i]
        return ext.shared_prefix_attention(q.view(self.B * self.Hq, 1, self.D), pool._key_pages, pool._value_pages, self.tables[i],
                                           self.context_lens, self._grp_dev, self._grp_host, at.scale, self.Hkv, self.Hq,
                                           workspace=self._grp_ws)

    def _swap_ab_attention(self, R: int, grouped: bool = False):
        """The attention of ``_swap_ab_layers`` for the first ``R`` slots (``grouped``: all B, shared-prefix attention)."""
        m, Hq, Hkv, D = self.model, self.Hq, self.Hkv, self.D
        offsets, context_lens = self.offsets[:R], self.context_lens[:R]

        def attention(i, block, h):
            at, pk, pool = block.self_attn, self._packed[i], m.page_pools[i]
            if self._attention_fused and not grouped:
                qkv = ext.quantized_matmul_fused(pk.qkv.scales, pk.qkv.biases, pk.qkv.weight, h)
                return ext.decode_attention_fused(qkv, at.q_norm._weight_as(h.dtype, h.device), at.k_norm._weight_as(h.dtype, h.device),
                                                  offsets, self.tables[i][:R], context_lens, self._rope_inv_freq,
                                                  pool._key_pages, pool._value_pages, Hq, Hkv, at.q_norm.eps, at.scale,
                                                  self.max_seq_len, workspace=self._attn_ws)
            # projection + q/k norm + RoPE + append: the split-reduction planes feed the second kernel, q|k|v is never written
            q = ext.qkv_project_rope_append(pk.qkv.scales, pk.qkv.biases, pk.qkv.weight, h, at.q_norm._weight_as(h.dtype, h.device),
                                            at.k_norm._weight_as(h.dtype, h.device), offsets, self.tables[i][:R], context_lens,
                                            pool._key_pages, pool._value_pages, Hq, Hkv, at.rope.base, at.q_norm.eps, inv_freq=at.rope.inv_freq)
            if grouped:
                return self._grouped_attention(i, at, q).view(R, Hq * D)
            y = ext.paged_attention(q.view(R * Hq, 1, D), pool._key_pages, pool._value_pages, self.tables[i][:R], context_lens,
                                    at.scale, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
            return y.view(R, Hq * D)

        return attention

    def _qkv_attention(self, R: int):
        """The attention of ``_lora_layers`` for the first ``R`` slots, from q|k|v rows the adapters were already added to."""
        m, Hq, Hkv, D = self.model, self.Hq, self.Hkv, self.D
        offsets, context_lens = self.offsets[:R], self.context_lens[:R]

        def attention(i, block, qkv):
            at, pool = block.self_attn, m.page_pools[i]
            qw, kw = at.q_norm._weight_as(qkv.dtype, qkv.device), at.k_norm._weight_as(qkv.dtype, qkv.device)
            if self._attention_fused:
                return ext.decode_attention_fused(qkv, qw, kw, offsets, self.tables[i][:R], context_lens, self._rope_inv_freq,
                                                  pool._key_pages, pool._value_pages, Hq, Hkv, at.q_norm.eps, at.scale,
                                                  self.max_seq_len, workspace=self._attn_ws)
            q = ext.decode_qk_norm_rope_append(qkv, qw, kw, offsets, self.tables[i][:R], context_lens, pool._key_pages, pool._value_pages,
                                               Hq, Hkv, at.rope.base, at.q_norm.eps, inv_freq=at.rope.inv_freq)
            y = ext.paged_attention(q.view(R * Hq, 1, D), pool._key_pages, pool._value_pages, self.tables[i][:R], context_lens,
                                    at.scale, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
            return y.view(R, Hq * D)

        return attention

    def _matvec_layers(self, x, grouped: bool = False):
        """The layer stack for at most 8 slots on the streaming matvec kernel, with RMSNorm as its prologue and the
        residual add as its epilogue; returns the residual stream before the final norm.  ``grouped``: the attention is
        q/k norm + RoPE + append and ``tl_shared_prefix_attention``."""
        m = self.model
        B, Hq, Hkv, D = x.shape[0], self.Hq, self.Hkv, self.D
        for i, block in enumerate(m.layers_inner):
            at, pk, pool = block.self_attn, self._packed[i], m.page_pools[i]
            ln1, ln2 = block.input_layernorm, block.post_attention_layernorm
            qkv = ext.quantized_matmul_fused(pk.qkv.scales, pk.qkv.biases, pk.qkv.weight, x, ln1._weight_as(x.dtype, x.device),
                                             prologue=ext.PRO_RMSNORM, eps=ln1.eps)
            if self._attention_fused and not grouped:
                y = ext.decode_attention_fused(qkv, at.q_norm._weight_as(x.dtype, x.device), at.k_norm._weight_as(x.dtype, x.device),
                                               self.offsets, self.tables[i], self.context_lens, self._rope_inv_freq,
                                               pool._key_pages, pool._value_pages, Hq, Hkv, at.q_norm.eps, at.scale,
                                               self.max_seq_len, workspace=self._attn_ws, rows_per_request=self._rows_per_request)
            else:
                q = ext.decode_qk_norm_rope_append(qkv, at.q_norm._weight_as(x.dtype, x.device), at.k_norm._weight_as(x.dtype, x.device),
                                                   self.offsets, self.tables[i], self.context_lens, pool._key_pages, pool._value_pages,
                                                   Hq, Hkv, at.rope.base, at.q_norm.eps, inv_freq=at.rope.inv_freq)
                if grouped:
                    y = self._grouped_attention(i, at, q)
                else:
                    y = ext.paged_attention(q.view(B * Hq, 1, D), pool._key_pages, pool._value_pages, self.tables[i], self.context_lens,
                                            at.scale, is_causal=True, num_kv_heads=Hkv, num_heads=Hq)
            x = ext.quantized_matmul_fused(at.wo.scales, at.wo.biases, at.wo.weight, y.view(B, Hq * D), residual=x, epilogue=ext.EPI_RESIDUAL)
            if isinstance(block.mlp, Moe):
                x = _moe_mlp(block.mlp, x, ln2=ln2)
                continue
            wd = block.mlp.w_down
            act = ext.quantized_matmul_fused(pk.gate_up.scales, pk.gate_up.biases, pk.gate_up.weight, x, ln2._weight_as(x.dtype, x.device),
                                             prologue=ext.PRO_RMSNORM, eps=ln2.eps, epilogue=ext.EPI_SWIGLU_PAIRS)  # [B, inter]
            x = ext.quantized_matmul_fused(wd.scales, wd.biases, wd.weight, act, residual=x, epilogue=ext.EPI_RESIDUAL)
        return x

    def _set_idle(self) -> None:
        self.meta_dev[2 * self.rows : 3 * self.rows].zero_()  # context_lens
        self.meta_dev[3 * self.rows :].fill_(-1)
        self._tables_dirty = True

    def _capture_graphs(self) -> None:
        forward = self._forward_fused if self.fused else self._forward_unfused

        def self_advancing_step():
            forward()
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        self._graph = self._graph_of(forward)
        self._graphs = {self.B: self._graph}
        self._graph_sample = None  # captured again on first use, over the current slabs
        self._graph_pen = None
        self._graph_lp = {}
        self._graph_con = {}
        self._graph_json = {}
        self._graph_schema = {}
        self._graph_keep = None
        self._graph_spec = {}
        self._graph_beam = {}
        self._graph_grp = {}
        if self._rows_per_request > 1:  # a verify pass: no self-advancing loop, no row variants
            self.kernels_per_step = self._launches
            return
        # the same step (already warmed up) with token feedback and position advance, for decode_on_device
        self._graph_loop = self._graph_of(self_advancing_step, pool=self._graph.pool(), warmups=0)
        self.kernels_per_step = self._launches  # kernels of libtiny_llm_b200.so recorded into one self-advancing step
        self._graphs = {self.B: self._graph}
        for rows in self._variants:
            if rows != self.B:  # the warm-ups run with the metadata still all-idle: the narrower kernels set their attributes lazily
                self._graphs[rows] = self._graph_of(lambda: forward(rows), pool=self._graph.pool())

    def _ensure_sample_graph(self) -> None:
        """Capture the sampled self-advancing step (after ``_ensure_graph``, before the metadata upload: the warm-up
        runs over all-idle metadata, as every capture does)."""
        if self._graph_sample is not None:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def sampled_step():
            forward(sampled=True)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self._graph_sample = self._graph_of(sampled_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_sampled_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _ensure_keep_graph(self, steps: int) -> None:
        """Capture the sampled self-advancing step that also logs its logits rows at ``step_counter`` (same conditions as
        ``_ensure_sample_graph``).  The log holds at least 8 steps and grows, with a new capture, for longer calls."""
        if self._logits_log is None or self._logits_log.shape[0] < steps:
            self._logits_log = torch.zeros((max(8, steps), self.B, self.V), dtype=self.logits.dtype, device=self.device)
            self._graph_keep = None
        if self._graph_keep is not None:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def keep_step():
            forward(sampled=True)
            ext.log_rows(self.logits, self._logits_log, self.step_counter)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self.step_counter.zero_()
            self._graph_keep = self._graph_of(keep_step, pool=self._graph.pool(), warmups=1)
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def beam_buffers(self, eos_ids: tuple):
        """The fixed buffers of the beam step for ``eos_ids``: the beams' ``cum`` (float32 ``[B]``, shared by every EOS
        tuple), ``tl_logprobs``' outputs ``[1, B(, N)]`` with their zero ``out_index``, and the packed select result."""
        if self.beam_cum is None:
            self.beam_cum = torch.zeros(self.B, dtype=torch.float32, device=self.device)
        bufs = self._beam_bufs.get(eos_ids)
        if bufs is None:
            B, N, dev = self.B, self.B + len(eos_ids), self.device
            lp = (torch.empty((1, B), dtype=torch.float32, device=dev), torch.empty((1, B), dtype=torch.float32, device=dev),
                  torch.empty((1, B), dtype=torch.int32, device=dev), torch.empty((1, B, N), dtype=torch.int32, device=dev),
                  torch.empty((1, B, N), dtype=torch.float32, device=dev))
            bufs = self._beam_bufs[eos_ids] = (lp, torch.zeros(1, dtype=torch.int32, device=dev),
                                                 torch.zeros(ext.BEAM_RESULT_WORDS, dtype=torch.int32, device=dev))
        return bufs

    def _ensure_beam_graph(self, eos_ids: tuple) -> None:
        """Capture the beam step for ``eos_ids`` (same conditions as ``_ensure_sample_graph``).  Its warm-up runs the
        select once, so ``beam_cum`` is kept aside and put back."""
        if eos_ids in self._graph_beam:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused
        lp, index, result = self.beam_buffers(eos_ids)
        N = self.B + len(eos_ids)

        def beam_step():
            forward()
            ext.logprobs(self.logits, None, None, N, out=lp, out_index=index)
            ext.beam_select(lp[4][0], lp[3][0], self.beam_cum, self.B, eos_ids, result)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            kept = self.beam_cum.clone()
            self._set_idle()
            self._graph_beam[eos_ids] = self._graph_of(beam_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_beam_step = self._launches
            self.beam_cum.copy_(kept)
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _ensure_grouped_graph(self, max_n: int | None) -> None:
        """Capture the grouped twin of the sampled step, with one ``tl_logprobs`` launch when ``max_n`` is given (same
        conditions as ``_ensure_sample_graph``; the descriptors are all-unused during the warm-up)."""
        if self._grp_host is None:
            self._grp_host = torch.zeros((self.B, 3), dtype=torch.int32, pin_memory=True)
            self._grp_dev = self._grp_host.to(self.device, copy=True)
            nbytes = ext.shared_prefix_attention_workspace(self.B, self.Hq, self.Hkv, self.page_size, self.max_pages)
            self._grp_ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        if max_n in self._graph_grp:
            return
        forward = self._forward_fused

        def grouped_step():
            forward(sampled=True, grouped=True)
            if max_n is not None:
                ext.logprobs(self.logits, self.next_tokens, self._lp_dev, max_n, out=self._lp_log, out_index=self.step_counter)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self._grp_host.zero_()
            self._grp_dev.zero_()
            self.step_counter.zero_()
            self._graph_grp[max_n] = self._graph_of(grouped_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_grouped_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _group_descriptors(self, groups, offsets) -> list:
        """``(first_slot, count, shared_pages)`` of each group of ``groups`` (``(first_slot, count)`` pairs), from the
        host block tables after this call's pages are allocated; ``shared_pages`` is 0 where the selection rule
        (``shared_prefix_attention_applies``) keeps the plain attention.  Malformed groups raise ``ValueError``."""
        taken = [False] * self.B
        out = []
        for first, count in groups:
            first, count = int(first), int(count)
            if count < 1 or first < 0 or first + count > self.B:
                raise ValueError(f"group ({first}, {count}) leaves the engine's {self.B} slots")
            if any(taken[first : first + count]):
                raise ValueError(f"group ({first}, {count}) overlaps another group")
            taken[first : first + count] = [True] * count
            if self._recs[first] is None or any(self._recs[b] is None for b in range(first, first + count)):
                raise ValueError(f"group ({first}, {count}) holds an idle slot")
            pages = shared_run(self.tables_np, first, count, min(int(offsets[b]) for b in range(first, first + count)), self.page_size)
            if not shared_prefix_attention_applies(count, pages * self.page_size, self.model):
                pages = 0
            out.append((first, count, pages))
        return out

    def _ensure_penalized_graph(self) -> None:
        """Capture the penalised sampled self-advancing step (same conditions as ``_ensure_sample_graph``; the warm-up
        runs at context 0, so it counts nothing)."""
        if self._graph_pen is not None:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def penalized_step():
            forward(sampled=True, penalized=True)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self._graph_pen = self._graph_of(penalized_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_penalized_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _ensure_logprobs_graph(self, sampled: bool, max_n: int, penalized: bool = False) -> None:
        """Capture the self-advancing step with one ``tl_logprobs`` launch after the token choice (targets: the tokens it
        just wrote), logging at ``step_counter`` (same conditions as ``_ensure_sample_graph``).  One graph per
        (sampled, penalized)."""
        self._alloc_logprobs(max_n)
        if (sampled, penalized) in self._graph_lp:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def logprobs_step():
            forward(sampled=sampled, penalized=penalized)
            ext.logprobs(self.logits, self.next_tokens, self._lp_dev, max_n, out=self._lp_log, out_index=self.step_counter)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self.step_counter.zero_()  # the warm-up logs at the counter: a previous run may have left it at log_capacity
            self._graph_lp[(sampled, penalized)] = self._graph_of(logprobs_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_logprobs_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _alloc_logprobs(self, max_n: int) -> None:
        """The logs and the top-N block for ``max_n`` (the graphs that log into older buffers are dropped)."""
        if self._lp_max_n != max_n:
            B, cap, dev = self.B, self.log_capacity, self.device
            self._graph_lp = {}
            self._graph_con = {k: g for k, g in self._graph_con.items() if k[1] is None}
            self._graph_json = {k: g for k, g in self._graph_json.items() if k[1] is None}
            self._graph_schema = {k: g for k, g in self._graph_schema.items() if k[1] is None}
            self._lp_max_n = max_n
            self._lp_log = (torch.zeros((cap, B), dtype=torch.float32, device=dev), torch.zeros((cap, B), dtype=torch.float32, device=dev),
                            torch.zeros((cap, B), dtype=torch.int32, device=dev), torch.zeros((cap, B, max_n), dtype=torch.int32, device=dev),
                            torch.zeros((cap, B, max_n), dtype=torch.float32, device=dev))
            if self._lp_host is None:
                self._lp_host = torch.zeros(B, dtype=torch.int32, pin_memory=True)
                self._lp_dev = self._lp_host.to(self.device, copy=True)
            self._lp_key = None

    def _ensure_constrained_graph(self, penalized: bool, max_n: int | None) -> None:
        """Capture the constrained self-advancing step, with one ``tl_logprobs`` launch when ``max_n`` is given (same
        conditions as ``_ensure_sample_graph``; the warm-up runs at context 0, so it advances no state).  One graph per
        (penalized, max_n)."""
        if (penalized, max_n) in self._graph_con:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def constrained_step():
            forward(sampled=True, penalized=penalized, constrained=True)
            if max_n is not None:
                ext.logprobs(self.logits, self.next_tokens, self._lp_dev, max_n, out=self._lp_log, out_index=self.step_counter)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self.step_counter.zero_()
            self._graph_con[(penalized, max_n)] = self._graph_of(constrained_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_constrained_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _ensure_json_graph(self, penalized: bool, max_n: int | None) -> None:
        """Capture the JSON-mode step: the constrained step with the JSON rows' masks before the draw and their advance
        after it (the warm-up runs at context 0, so it advances no state).  One graph per (penalized, max_n)."""
        if (penalized, max_n) in self._graph_json:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def json_step():
            forward(sampled=True, penalized=penalized, constrained="json")
            if max_n is not None:
                ext.logprobs(self.logits, self.next_tokens, self._lp_dev, max_n, out=self._lp_log, out_index=self.step_counter)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self.step_counter.zero_()
            self._graph_json[(penalized, max_n)] = self._graph_of(json_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_json_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _ensure_schema_graph(self, penalized: bool, max_n: int | None, json: bool) -> None:
        """Capture the JSON Schema step: the constrained step with the schema rows' masks before the draw and their
        advance after it, and the JSON rows' too when ``json`` (the warm-up runs at context 0, so it advances no
        state).  One graph per (penalized, max_n, json)."""
        if (penalized, max_n, json) in self._graph_schema:
            return
        forward = self._forward_fused if self.fused else self._forward_unfused

        def schema_step():
            forward(sampled=True, penalized=penalized, constrained="schema")
            if max_n is not None:
                ext.logprobs(self.logits, self.next_tokens, self._lp_dev, max_n, out=self._lp_log, out_index=self.step_counter)
            ext.decode_advance(self.tokens, self.next_tokens, self.offsets, self.context_lens, self.out_log, self.step_counter)

        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self.step_counter.zero_()
            self._graph_schema[(penalized, max_n, json)] = self._graph_of(schema_step, pool=self._graph.pool(), warmups=1)
            self.kernels_per_schema_step = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _set_json_constraints(self, per: list, history, schema: bool = False) -> None:
        """The JSON table's rows for the slots' constraints (JSON, regex or none), as ``_set_constraints`` sets the
        descriptors: a slot with a ``history`` entry starts from the host walk of its generated ids (refused when they
        leave the language), a slot with a new constraint from the start state, and every other constrained slot
        keeps its device state."""
        from .json_mode import JsonConstraint

        B = self.B
        cons = [None if p is None else p.constraint for p in per]
        if history is not None:
            history = list(history)
            if len(history) != B:
                raise ValueError(f"history must hold one (prompt_ids, generated_ids) or None per slot ({B})")
        walked = {}
        for b, c in enumerate(cons):
            if c is None or history is None or history[b] is None:
                continue
            rows = isinstance(c, (JsonConstraint, JsonSchemaConstraint))
            state = c.walk(history[b][1]) if rows else c.walk(c.start_state, history[b][1])
            if state is None or (not rows and state < 0):
                raise ValueError(f"slot {b}: its generated ids leave the constraint's language")
            walked[b] = state
        key = tuple(cons)
        tab, old = (self._schema_tab, self._schema_key) if schema else (self._json_tab, self._json_key)
        if old is not None and all(x is y for x, y in zip(key, old)) and not walked:
            return
        torch.cuda.current_stream(self.device).wait_stream(self._stream)  # the previous call's replays read the table
        for b, c in enumerate(cons):
            if b in walked or old is None or old[b] is not c or c is None:
                tab.set_row(b, c, walked.get(b))
        if schema:
            self._schema_key = key
        else:
            self._json_key = key

    def _set_constraints(self, per: list, history) -> None:
        """Upload the slot descriptors when the slots' constraints change or ``history`` is given.  A slot whose
        ``history`` entry is ``(prompt_ids, generated_ids)`` starts from the host walk of its generated ids; a slot with a
        new constraint and no history from the start state; every other constrained slot keeps its device state."""
        from .constrained import descriptor_state, descriptor_values

        B = self.B
        cons = [None if p is None else p.constraint for p in per]
        if history is not None:
            history = list(history)
            if len(history) != B:
                raise ValueError(f"history must hold one (prompt_ids, generated_ids) or None per slot ({B})")
        walked = {b: c.walk(c.start_state, history[b][1]) for b, c in enumerate(cons)
                  if c is not None and history is not None and history[b] is not None}
        key = tuple(cons)  # holds the constraints, whose device tables the descriptors point into
        if self._con_key is not None and all(x is y for x, y in zip(key, self._con_key)) and not walked:
            return
        kept = {b for b, c in enumerate(cons) if c is not None and b not in walked and self._con_key is not None and self._con_key[b] is c}
        current = descriptor_state(self._con_dev.view(B, -1)).tolist() if kept else None  # one read, only when states carry over
        self._host_write_begin()
        host = self._con_host.numpy().reshape(B, -1)
        for b, c in enumerate(cons):
            state = walked.get(b, current[b] if b in kept else 0)
            if c is not None and state < 0:
                raise ValueError(f"slot {b}: its generated ids leave the constraint's language")
            host[b] = descriptor_values(c, state)
        self._upload_meta(self._con_dev, self._con_host)
        self.h2d_bytes += self._con_host.numel() * 8
        self._con_key = key

    def _set_top_n(self, per: list[int]) -> None:
        """Write the per-slot top-N counts into their pinned block and upload it if they changed."""
        key = tuple(per)
        if key == self._lp_key:
            return
        self._host_write_begin()
        self._lp_host.numpy()[:] = per
        self._upload_meta(self._lp_dev, self._lp_host)
        self.h2d_bytes += 4 * self.B
        self._lp_key = key

    def _per_slot_sampling(self, sampling) -> list:
        from .sampler import SamplingParams

        B = self.B
        per = [sampling] * B if isinstance(sampling, SamplingParams) else list(sampling)
        if len(per) != B or not all(p is None or isinstance(p, SamplingParams) for p in per):
            raise ValueError(f"sampling must be one SamplingParams or a list of {B} (one per slot)")
        return per

    def _alloc_penalties(self) -> None:
        """The token counts and the penalty block, on first use (before the penalised graphs are captured over them)."""
        if self.token_counts is None:
            self.token_counts = torch.zeros((self.B, self.V), dtype=torch.int32, device=self.device)
            self._pen_host = torch.zeros(16 * self.B, dtype=torch.uint8, pin_memory=True)
            self._pen_dev = self._pen_host.to(self.device, copy=True)

    def _set_penalties(self, per: list, history) -> None:
        """Rebuild the token-count rows ``history`` gives (per slot ``(prompt_ids, generated_ids)`` or None: keep the
        row) and upload the penalty parameters if they changed."""
        from .sampler import penalty_tensors, token_state_row

        B = self.B
        if history is not None:
            history = list(history)
            if len(history) != B:
                raise ValueError(f"history must hold one (prompt_ids, generated_ids) or None per slot ({B})")
            for b, h in enumerate(history):
                if h is not None:
                    prompt_ids, generated_ids = h
                    token_state_row(prompt_ids, generated_ids, self.V, out=self.token_counts[b])
        key = tuple(per)
        if key == self._pen_key:
            return
        self._host_write_begin()
        host = self._pen_host.numpy()
        for j, t in enumerate(penalty_tensors(per, "cpu")):
            host[4 * B * j : 4 * B * (j + 1)] = t.numpy().view(np.uint8)
        self._upload_meta(self._pen_dev, self._pen_host)
        self.h2d_bytes += 16 * B
        self._pen_key = key

    def _set_sampling(self, sampling) -> None:
        """Write the per-slot parameters into their pinned block (one ``SamplingParams`` for all slots or one per
        slot, None: greedy) and upload it if they changed."""
        from .sampler import sampling_tensors

        B = self.B
        per = self._per_slot_sampling(sampling)
        key = tuple(per)
        if key == self._samp_key:
            return
        self._host_write_begin()
        temperature, top_k, top_p, seed = (t.numpy() for t in sampling_tensors(per, "cpu"))
        host = self._samp_host.numpy()
        host[: 8 * B] = seed.view(np.uint8)
        host[8 * B : 12 * B] = temperature.view(np.uint8)
        host[12 * B : 16 * B] = top_k.view(np.uint8)
        host[16 * B : 20 * B] = top_p.view(np.uint8)
        self._upload_meta(self._samp_dev, self._samp_host)
        self.h2d_bytes += 20 * B
        self._samp_key = key

    # ------------------------------------------------------- host bookkeeping --
    def _slot_caches(self, caches, layer: int):
        """The per-slot request caches of one layer: a BatchingKvCache table, or a
        single request's cache list (B == 1)."""
        entry = caches[layer]
        if isinstance(entry, BatchingKvCache):
            return entry.kv_caches
        return [entry]

    def _drop(self, b: int) -> None:
        rec = self._recs[b]
        if rec is not None:
            rec.group.settle()
            for c in rec.group.caches:
                if c._lazy is rec.group:
                    c._lazy = None
            self.tables_np[:, b, :] = -1
            self._tables_dirty = True
            self._recs[b] = None

    def _register(self, b: int, caches) -> "_SlotRecord":
        """Slow path, once per request admission: take the request's per-layer cache objects as a
        group, check that they really are in lockstep (same page ids / fill / offset in every layer,
        which is what the schedulers of batch.py / generate.py produce: SURVEY section 7) and mirror
        their page ids into the table rows."""
        self._drop(b)
        group_caches = [self._slot_caches(caches, layer)[b] for layer in range(self.n_layers)]
        c0 = group_caches[0]
        for c in group_caches:
            if not isinstance(c, TinyKvPagedCache):
                raise ValueError("the decode engine needs paged request caches")
            if c._lazy is not None:
                c._lazy.settle()
        n = len(c0.page_ids)
        if n > self.max_pages:
            raise ValueError("request exceeds the engine's max_seq_len")
        lockstep = all(type(c) is TinyKvPagedCache and c.page_ids == c0.page_ids and c._page_lens == c0._page_lens and c._offset == c0._offset
                       for c in group_caches)
        if lockstep:
            self.tables_np[:, b, :n] = c0.page_ids
            self.tables_np[:, b, n:] = -1
        else:
            for layer, c in enumerate(group_caches):
                k = len(c.page_ids)
                if k > self.max_pages:
                    raise ValueError("request exceeds the engine's max_seq_len")
                self.tables_np[layer, b, :k] = c.page_ids
                self.tables_np[layer, b, k:] = -1
        self._tables_dirty = True
        group = _LockstepGroup(group_caches)
        if lockstep:
            for c in group_caches:
                c._lazy = group
        rec = _SlotRecord(c0, group, lockstep)
        self._recs[b] = rec
        return rec

    def _advance_host(self, caches, steps: int = 1) -> list[int]:
        """Account for ``steps`` one-token appends of every active request (host integers only) and
        bring the table rows up to date.  Returns the context length each slot will have after the
        FIRST of those steps.

        Cost per step at B = 64: one identity check per slot; the 36 per-layer cache objects of a
        request are touched only when its tail page overflows (once per ``page_size`` tokens) - the
        one-token appends in between are deferred (``TinyKvPagedCache._lazy``) and settled when
        somebody reads ``page_lens`` / ``offset``, instead of walking 36 x B objects every step."""
        first_ctx = [0] * self.B
        slots0 = self._slot_caches(caches, 0)
        page = self.page_size
        for b, c0 in enumerate(slots0):
            rec = self._recs[b]
            if c0 is None:
                if rec is not None:
                    self._drop(b)
                continue
            if (rec is None or rec.c0 is not c0 or rec.epoch != c0.epoch
                    or (rec.lockstep and (c0._lazy is not rec.group or c0._offset + rec.group.pending != rec.offset or len(c0.page_ids) != rec.pages))):
                rec = self._register(b, caches)
            if not rec.lockstep:  # layers disagree: walk them (always correct, never taken by the in-tree schedulers)
                self._advance_slow(b, rec, caches, steps)
                first_ctx[b] = rec.offset - steps + 1
                continue
            tail = rec.offset - (rec.pages - 1) * page if rec.pages else page
            if tail + steps <= page:
                rec.group.pending += steps
                rec.offset += steps
            else:
                self._advance_pages(b, rec, steps)
            first_ctx[b] = rec.offset - steps + 1
        return first_ctx

    def _check_headroom(self, group_caches, steps: int) -> None:
        """All layers must be able to take the new pages BEFORE any of them is touched (a shortage
        used to surface at layer k with layers < k already advanced: ADVICE round 1)."""
        for c in group_caches:
            tail = c._page_lens[-1] if c.page_ids else self.page_size
            need = max(0, -(-(tail + steps - self.page_size) // self.page_size))
            if len(c.page_ids) + need > self.max_pages:
                raise ValueError("request exceeds the engine's max_seq_len")
            if need and need > c.pool.pages_available():
                raise RuntimeError("page pool slab exhausted: reserve() more pages before decoding")

    def _advance_pages(self, b: int, rec: "_SlotRecord", steps: int) -> None:
        rec.group.settle()
        self._check_headroom(rec.group.caches, steps)
        old = rec.pages
        for layer, c in enumerate(rec.group.caches):
            for _ in range(steps):
                c.append_token_slot()
            self.tables_np[layer, b, old:len(c.page_ids)] = c.page_ids[old:]
        c0 = rec.c0
        rec.pages, rec.offset = len(c0.page_ids), c0._offset
        self._tables_dirty = True

    def _advance_slow(self, b: int, rec: "_SlotRecord", caches, steps: int) -> None:
        group_caches = [self._slot_caches(caches, layer)[b] for layer in range(self.n_layers)]
        self._check_headroom(group_caches, steps)
        for layer, c in enumerate(group_caches):
            for _ in range(steps):
                c.append_token_slot()
            k = len(c.page_ids)
            self.tables_np[layer, b, :k] = c.page_ids
            self.tables_np[layer, b, k:] = -1
        rec.group.caches = group_caches
        rec.offset = group_caches[0]._offset
        rec.pages = len(group_caches[0].page_ids)
        self._tables_dirty = True

    def _upload(self) -> None:
        if self._tables_dirty:
            self._upload_meta(self.meta_dev, self.meta_host)
            self.h2d_bytes += self._meta_len * 4
            self._tables_dirty = False
        else:  # tokens | offsets | context_lens only: the block tables on the device are current
            self._upload_meta(self._meta_dev_head, self._meta_host_head)
            self.h2d_bytes += 3 * self.rows * 4

    def upload_bytes_per_step(self) -> int:
        """Host -> device bytes of a steady-state step (block tables travel only when a page was added)."""
        return 3 * self.rows * 4

    # ------------------------------------------------------------------ steps --
    def _adapters_of_call(self, adapter_ids) -> None:
        """Take the slots' adapter ids of a ``step`` / ``decode_on_device`` call (None: every slot on the base model)."""
        if self.lora is None:
            if adapter_ids is not None and any(int(i) >= 0 for i in adapter_ids):
                raise ValueError("adapter_ids given to an engine of a model without adapters")
            return
        ids = [-1] * self.B if adapter_ids is None else [int(i) for i in adapter_ids]
        if len(ids) != self.B or any(i >= len(self.lora.names) for i in ids):
            raise ValueError(f"adapter_ids must hold one loaded adapter id (or -1) per slot ({self.B})")
        self.h2d_bytes += self._set_adapter_ids(tuple(ids))

    def step(self, tokens, offsets, caches, adapter_ids=None):
        """One decode step.  ``tokens``: B ids (list or tensor), ``offsets``: B
        RoPE positions; returns (logits [B, 1, V] static buffer, next_tokens [B]).  ``adapter_ids`` (LoRA engines): one
        ``AdapterSet`` id per slot, -1 or None for the base model; the same graph serves every mix."""
        B = self.B
        self._host_write_begin()
        ctx = self._advance_host(caches, 1)
        self._ensure_graph()
        self._adapters_of_call(adapter_ids)
        if isinstance(tokens, torch.Tensor):
            tok_host = None
        else:
            tok_host = tokens
            self.meta_np[0:B] = tok_host
        self.meta_np[B : 2 * B] = offsets
        self.meta_np[2 * B : 3 * B] = ctx
        # upload and replay on the CALLER's stream (the side stream is only needed for capture): two stream waits and a
        # stream-context switch less per step - host time here is serial with the GPU step when the caller reads every token
        self._upload()
        if tok_host is None:
            self.tokens.copy_(tokens.reshape(-1) if tokens.dtype == torch.int32 else tokens.reshape(-1).to(torch.int32), non_blocking=True)
        rows = B
        if len(self._variants) > 1:
            hi = 0
            for b, rec in enumerate(self._recs):
                if rec is not None:
                    hi = b + 1
            rows = next(r for r in self._variants if r >= hi)
            self.variant_replays[rows] += 1
        self._graphs[rows].replay()
        self.graph_replays += 1
        return self.logits.view(B, 1, self.V), self.next_tokens

    def decode_on_device(self, tokens, offsets, caches, steps: int, sampling=None, logprobs=None, history=None, adapter_ids=None,
                         keep_logits: bool = False, groups=None):
        """``steps`` greedy decode steps with no host round trip: pages for all
        steps are allocated ahead, then the self-advancing graph is replayed
        back to back.  Returns the sampled tokens ``[steps, B]`` (device).
        ``sampling`` (one ``SamplingParams`` or one per slot, None entries greedy) replays the sampled graph instead:
        slot b's token at position p is ``tl_sample``'s draw with its parameters, p = its offset + 1.
        ``logprobs`` (an int N in [0, 20] for every slot, or one per slot) replays the same step with one ``tl_logprobs``
        launch on the tokens it chose and returns ``(tokens, (logprob [steps, B], rank [steps, B], top_ids [steps, B, N],
        top_logprobs [steps, B, N]))``, device views of the engine's logs (overwritten by the next call).
        With a penalised slot in ``sampling`` the step is ``tl_sample_penalized`` over ``token_counts [B, V]``, which
        it updates at every drawn token.  ``history`` (per slot ``(prompt_ids, generated_ids)``, or None) rebuilds those
        slots' rows first; None continues from the rows as the engine holds them.  A call without a penalised slot
        replays the graphs it would without penalties and does not read ``history``.
        With a constrained slot (``SamplingParams.constraint``) the step is ``tl_sample_constrained`` over the engine's
        slot descriptors, captured on first use per (penalised, logprobs); each launch advances the slots' automaton
        states.  ``history`` also sets a constrained slot's state to the walk of its generated ids; without it a slot
        keeps its state while its constraint stays the same and starts at the start state otherwise.  With a JSON-mode
        slot (``JsonConstraint``) the step is a graph of its own: the JSON rows' masks, the constrained draw and their
        state advance, with the same rules for ``history``.  With a JSON Schema slot (``JsonSchemaConstraint``) the
        step is the schema graph kind, which runs the schema rows' (and any JSON rows') masks and advances.
        ``adapter_ids`` (LoRA engines): one ``AdapterSet`` id per slot as in ``step``, for every graph kind above.
        ``keep_logits=True`` (plain ``sampling``: no penalty, constraint or logprobs) replays the sampled step with one
        more launch that keeps each step's logits rows, and returns ``(tokens, logits [steps, B, V])``, a device view of
        the engine's log (overwritten by the next call): the rows a speculative draft's proposals were drawn from.
        ``groups`` (``(first_slot, count)`` pairs of slots forked from one prompt, ``paged_kv_cache.fork``): for the
        plain sampled step, with or without logprobs, on a fused engine without adapters, the leading full pages every
        layer of a group's slots shares are attended once for all its rows (``tl_shared_prefix_attention``) wherever
        ``shared_prefix_attention_applies``; every other call, and a call where no group qualifies, replays the graph
        it would without ``groups``.  Groups that leave the slots, overlap, hold an idle slot or whose layers do not
        share the same pages raise ``ValueError``."""
        if steps > self.log_capacity:
            raise ValueError("steps exceed the engine's token log capacity")
        if keep_logits:
            from .sampler import any_constrained, any_penalized

            per = None if sampling is None else self._per_slot_sampling(sampling)
            if per is None or logprobs is not None or any_penalized(per) or any_constrained(per):
                raise ValueError("keep_logits takes plain sampling: no penalties, min-p, constraint or logprobs")
        B = self.B
        top_n = None
        if logprobs is not None:
            from .logprobs import _check_n

            top_n = [_check_n(logprobs)] * B if isinstance(logprobs, int) else [_check_n(0 if n is None else n) for n in logprobs]
            if len(top_n) != B:
                raise ValueError(f"logprobs must be one int or a list of {B} (one per slot)")
        penalized = constrained = False
        if sampling is not None:
            from .sampler import any_constrained, any_penalized

            per = self._per_slot_sampling(sampling)
            penalized, constrained = any_penalized(per), any_constrained(per)
            for p in per:
                if p is not None and p.constraint is not None and p.constraint.vocab_size != self.V:
                    raise ValueError(f"the constraint's vocabulary has {p.constraint.vocab_size} ids, the model {self.V}")
        self._host_write_begin()
        ctx = self._advance_host(caches, steps)
        self._ensure_graph()
        descriptors = None
        if groups is not None:
            descriptors = self._group_descriptors(groups, offsets)
            plain = (sampling is not None and not penalized and not constrained and not keep_logits and self.fused
                     and self.lora is None and self._rows_per_request == 1)
            if not plain or not any(d[2] for d in descriptors):
                descriptors = None
        self._adapters_of_call(adapter_ids)
        if penalized:
            self._alloc_penalties()
        json = constrained and any(isinstance(p.constraint, JsonConstraint) for p in per if p is not None)
        schema = constrained and any(isinstance(p.constraint, JsonSchemaConstraint) for p in per if p is not None)
        if schema:
            if self._schema_tab is None:
                self._schema_tab = ConstraintRows(B, self.V, self.device, json=json, schema=True)
            if json:
                self._schema_tab.ensure_json()
            if top_n is not None:
                self._alloc_logprobs(max(top_n))
                self._set_top_n(top_n)
            self._set_json_constraints(self._per_slot_sampling(sampling), history, schema=True)
            self._ensure_schema_graph(penalized, None if top_n is None else max(top_n), self._schema_tab.has_json)
        elif json:
            if self._json_tab is None:
                self._json_tab = ConstraintRows(B, self.V, self.device, json=True)
            if top_n is not None:
                self._alloc_logprobs(max(top_n))
                self._set_top_n(top_n)
            self._ensure_json_graph(penalized, None if top_n is None else max(top_n))
        elif constrained:
            if self._con_dev is None:
                self._con_host = torch.zeros(5 * B, dtype=torch.int64, pin_memory=True)
                self._con_dev = self._con_host.to(self.device, copy=True)
            if top_n is not None:
                self._alloc_logprobs(max(top_n))
                self._set_top_n(top_n)
            self._ensure_constrained_graph(penalized, None if top_n is None else max(top_n))
        elif descriptors is not None:
            if top_n is not None:
                self._alloc_logprobs(max(top_n))
                self._set_top_n(top_n)
            self._ensure_grouped_graph(None if top_n is None else max(top_n))
            self._grp_host.zero_()
            for j, d in enumerate(descriptors):
                self._grp_host[j] = torch.tensor(d, dtype=torch.int32)
        elif top_n is not None:
            self._ensure_logprobs_graph(sampling is not None, max(top_n), penalized)
            self._set_top_n(top_n)
        elif penalized:
            self._ensure_penalized_graph()
        elif keep_logits:
            self._ensure_keep_graph(steps)
        elif sampling is not None:
            self._ensure_sample_graph()
        if sampling is not None:
            self._set_sampling(sampling)
        if penalized:
            self._set_penalties(self._per_slot_sampling(sampling), history)
        if schema:
            pass  # the schema table's rows are set above, before its graph is captured, which sizes its masks launch
        elif json:
            self._set_json_constraints(self._per_slot_sampling(sampling), history)
        elif constrained:
            self._set_constraints(self._per_slot_sampling(sampling), history)
        self.meta_np[0:B] = tokens
        self.meta_np[B : 2 * B] = offsets
        self.meta_np[2 * B : 3 * B] = ctx
        if schema:
            graph = self._graph_schema[(penalized, None if top_n is None else max(top_n), self._schema_tab.has_json)]
        elif json:
            graph = self._graph_json[(penalized, None if top_n is None else max(top_n))]
        elif constrained:
            graph = self._graph_con[(penalized, None if top_n is None else max(top_n))]
        elif descriptors is not None:
            graph = self._graph_grp[None if top_n is None else max(top_n)]
        elif top_n is not None:
            graph = self._graph_lp[(sampling is not None, penalized)]
        elif penalized:
            graph = self._graph_pen
        elif keep_logits:
            graph = self._graph_keep
        else:
            graph = self._graph_loop if sampling is None else self._graph_sample
        cur = torch.cuda.current_stream(self.device)
        self._stream.wait_stream(cur)
        with torch.cuda.stream(self._stream):
            self._upload()
            if descriptors is not None:
                self._grp_dev.copy_(self._grp_host, non_blocking=True)
                self._upload_event.record()
            self.step_counter.zero_()
            for i in range(steps):
                graph.replay()
        cur.wait_stream(self._stream)
        self.graph_replays += steps
        out = self.out_log[: steps * B].view(steps, B)
        if keep_logits:
            return out, self._logits_log[:steps]
        if top_n is None:
            return out
        _, lp, rank, ids, top = self._lp_log
        return out, (lp[:steps], rank[:steps], ids[:steps], top[:steps])


    def beam_step(self, tokens, offsets, caches, eos_ids: tuple):
        """One step of beam search over the B slots (``generate.beam_search_ids``): append ``tokens`` at ``offsets`` to
        the slots' caches (``caches`` as for ``step``; an empty slot takes token 0 at offset 0 and its ``beam_cum`` entry
        must be -inf), then choose the next beams from every row's top ``B + len(eos_ids)`` tokens and ``beam_cum``.
        Returns the packed ``tl_beam_select`` result (int32 ``[BEAM_RESULT_WORDS]``, device), overwritten by the next
        call; ``beam_cum`` then holds the new beams' sums."""
        B = self.B
        self._host_write_begin()
        ctx = self._advance_host(caches, 1)
        self._ensure_graph()
        self.beam_buffers(eos_ids)
        self._ensure_beam_graph(eos_ids)
        self.meta_np[0:B] = tokens
        self.meta_np[B : 2 * B] = offsets
        self.meta_np[2 * B : 3 * B] = ctx
        self._upload()
        self._graph_beam[eos_ids].replay()
        self.graph_replays += 1
        return self._beam_bufs[eos_ids][2]


class VerifyEngine(DecodeEngine):
    """The verify pass of speculative decoding as one CUDA graph: ``T`` (2..8) consecutive tokens of ONE request, i.e.
    ``T`` decode steps in a single pass over the weights.  Metadata block: ``tokens [T] | offsets [T] | context_lens [T]
    | block tables [Ly, 1, MP]``, row j at position ``ctx0 + j`` with context ``ctx0 + j + 1``.

    It runs the B = 1 decode step's launches at M = T: embedding, the matvec layer stack with the T-row fused attention
    (``decode_attention_fused(rows_per_request=T)``), the RMSNorm-prologue head and argmax.  The streaming projections
    compute every row as they do alone and the attention row j as the decode step with rows < j appended, so logits,
    argmax and the appended K/V equal, bit for bit, T successive B = 1 decode steps at the same ``max_seq_len``.  The
    host bookkeeping is ``DecodeEngine``'s (one slot, ``_advance_host(caches, T)``)."""

    def __init__(self, model, rows: int, max_seq_len: int, device):
        if not 2 <= rows <= 8:
            raise ValueError("the verify step takes 2 to 8 rows")
        if not VerifyEngine.supported(model, device, max_seq_len):
            raise ValueError("the verify step needs the B = 1 decode step's fused matvec + fused attention path")
        super().__init__(model, 1, max_seq_len, device, rows_per_request=rows)
        self.T = rows
        assert self.fused and self._attention_fused and self._variants == [1]
        # verify(sampling=...): the request's parameters for all T rows (seed i64 | temperature f32 | top_k i32 | top_p
        # f32, T each) in a pinned block, uploaded when they change
        self._spec_host = torch.zeros(20 * rows, dtype=torch.uint8, pin_memory=True)
        self._spec_dev = self._spec_host.to(self.device, copy=True)
        self._spec_key = None
        T = rows
        self._spec_params = (self._spec_dev[8 * T : 12 * T].view(torch.float32), self._spec_dev[12 * T : 16 * T].view(torch.int32),
                             self._spec_dev[16 * T : 20 * T].view(torch.float32), self._spec_dev[: 8 * T].view(torch.int64))
        self.kernels_per_sampled_verify = 0

    @staticmethod
    def supported(model, device, max_seq_len: int) -> bool:
        """Where the B = 1 decode engine itself runs fused matvec + fused attention, on dense models only (the verify pass
        does not take the MoE block) without adapters (speculative decoding does not take them)."""
        return (torch.device(device).type == "cuda" and DecodeEngine.fused_attention_applies(model, max_seq_len)
                and not any(isinstance(b.mlp, Moe) for b in model.layers_inner) and getattr(model, "adapters", None) is None)

    def reserve_pools(self, pages_per_layer: int | None = None) -> None:
        raise RuntimeError("the verify step shares the B = 1 decode engine's pool reservation")

    def step(self, tokens, offsets, caches):
        raise TypeError("a verify engine runs verify(), not decode steps")

    def decode_on_device(self, tokens, offsets, caches, steps: int):
        raise TypeError("a verify engine runs verify(), not decode steps")

    def _ensure_spec_graph(self, draft) -> None:
        """Capture the sampled verify pass over the draft-logits buffer ``draft`` (after ``_ensure_graph``, before the
        metadata upload, as every capture)."""
        key = (draft.data_ptr(), draft.dtype)
        if key in self._graph_spec:
            return
        with torch.cuda.stream(self._stream):
            self._stream.wait_stream(torch.cuda.current_stream(self.device))
            self._set_idle()
            self._graph_spec[key] = self._graph_of(lambda: self._forward_fused(spec_draft=draft), pool=self._graph.pool(), warmups=1)
            self.kernels_per_sampled_verify = self._launches
        torch.cuda.current_stream(self.device).wait_stream(self._stream)

    def _set_spec_params(self, sampling) -> None:
        from .sampler import sampling_tensors

        if sampling == self._spec_key:
            return
        T = self.T
        self._host_write_begin()
        temperature, top_k, top_p, seed = (t.numpy() for t in sampling_tensors([sampling] * T, "cpu"))
        host = self._spec_host.numpy()
        host[: 8 * T] = seed.view(np.uint8)
        host[8 * T : 12 * T] = temperature.view(np.uint8)
        host[12 * T : 16 * T] = top_k.view(np.uint8)
        host[16 * T : 20 * T] = top_p.view(np.uint8)
        self._upload_meta(self._spec_dev, self._spec_host)
        self.h2d_bytes += 20 * T
        self._spec_key = sampling

    def verify(self, token: int, proposals, offset: int, caches, sampling=None, draft_logits=None):
        """Append ``[token, *proposals]`` (T ids at positions ``offset``..; ``proposals`` a list, or an int32 device tensor
        that never visits the host) to the request's caches and return (logits [T, V] static buffer, greedy next token
        per row [T]).
        ``sampling`` (a plain ``SamplingParams``: no penalty, min-p or constraint) with ``draft_logits`` (``[T - 1, V]``,
        device, the rows the proposals were drawn from) replays the sampled verify graph instead: the second result is
        then ``tl_speculative_sample``'s tokens, row j the proposal when accepted, else the residual draw, row T - 1 the
        bonus draw.  The draft rows are read device to device; one graph is kept per draft buffer."""
        T = self.T
        spec = sampling is not None
        if spec:
            if sampling.penalized or sampling.constraint is not None:
                raise ValueError("the sampled verify pass takes plain sampling: no penalties, min-p or constraint")
            if draft_logits is None or tuple(draft_logits.shape) != (T - 1, self.V) or not draft_logits.is_contiguous():
                raise ValueError(f"the sampled verify pass needs the draft's contiguous logits rows [{T - 1}, {self.V}]")
        self._host_write_begin()
        self._advance_host(caches, T)
        self._ensure_graph()
        if spec:
            self._ensure_spec_graph(draft_logits)
            self._set_spec_params(sampling)
        on_device = isinstance(proposals, torch.Tensor)
        self.meta_np[0] = token
        if not on_device:
            self.meta_np[1:T] = proposals
        pos = np.arange(T, dtype=np.int32) + offset
        self.meta_np[T : 2 * T] = pos
        self.meta_np[2 * T : 3 * T] = pos + 1
        self._upload()
        if on_device:
            self.tokens[1:].copy_(proposals.reshape(-1).to(torch.int32), non_blocking=True)
        (self._graph_spec[(draft_logits.data_ptr(), draft_logits.dtype)] if spec else self._graph).replay()
        self.graph_replays += 1
        return self.logits, self.next_tokens


class PrefillEngine(_GraphEngine):
    """CUDA-graph replay of ONE chunked-prefill step (``Request.try_prefill``: B = 1, up to ``chunk`` prompt tokens,
    ``src/tiny_llm_ref/batch.py:48-76``) for the Week-3 paged model.

    The reference (and the operator path of this backend) issues ~20 operator calls per layer per chunk from
    Python: ~700 launches, whose host time exceeds the GPU work of a 128-token chunk.  Here the
    chunk's whole forward pass is captured once over static buffers; what changes between chunks is DATA in one
    pinned block: the token ids, per-token RoPE positions and post-append lengths, the request's block-table
    row per layer and the final context length.  A short (tail) chunk is RIGHT-aligned in the ``chunk`` rows:
    the padding rows in front carry context length 0 (nothing is appended for them) and the bottom-right causal
    rule of paged attention (``key <= row + ctx - L``) then gives every real row exactly its own prefix.

    Per layer: rms_norm -> q|k|v projection (one launch) -> q/k norm + RoPE + K/V append for all rows (one
    launch, ``tl_chunk_qk_norm_rope_append``) -> paged FlashAttention (wgmma) -> o projection + residual ->
    rms_norm -> gate|up (+ SwiGLU) -> down + residual.  Rounding points are those of the operator sequence.
    Chunks of up to 128 tokens run the layer stack the wide decode step uses (``_swap_ab_layers``), with the
    model's one packed weight copy (``Qwen3ModelWeek3.packed_layers``).
    Integer page bookkeeping stays in the request's ``TinyKvPagedCache`` objects (``append_slots``)."""

    def __init__(self, model, chunk: int, max_seq_len: int, device):
        L = self.L = int(chunk)
        # one int32 block: tokens [L] | offsets [L] | context_lens [L] | ctx_after [1] | tables [Ly, MP]
        super().__init__(model, max_seq_len, device, 3 * L + 1, 1)
        self.tokens = self.meta_dev[0:L].view(1, L)
        self.offsets = self.meta_dev[L:2 * L]
        self.ctxs = self.meta_dev[2 * L:3 * L]
        self.ctx_after = self.meta_dev[3 * L:3 * L + 1]
        self.tables = self.meta_dev[3 * L + 1:].view(self.n_layers, self.max_pages)
        self.tables_np = self.meta_np[3 * L + 1:].reshape(self.n_layers, self.max_pages)
        self.next_token = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.replays = 0
        self.kernels_per_chunk = 0
        self._packed = model.packed_layers()
        # A window above 8,192 keys (a long prefix): the chunk's attention splits the prefix's key range over more CTAs and
        # merges the partials into the token-major output; windows up to 8,192 keep the unsplit launch (no workspace).
        ws = ext.paged_attention_token_major_workspace(self.Hq, L, model.page_size, self.max_pages)
        self._attn_ws = torch.empty(ws, dtype=torch.uint8, device=self.device) if ws else None
        if self.lora is not None:  # one id per chunk, broadcast to its rows (padding rows carry it too: they are never stored)
            self._alloc_adapter_ids(L, -1)

    @staticmethod
    def supported(model, device) -> bool:
        attn = model.layers_inner[0].self_attn
        rope = attn.rope
        return (torch.device(device).type == "cuda" and attn.head_dim == 128 and not rope.traditional and rope.dims == attn.head_dim
                and model.embedding.weight.scales.dtype == torch.bfloat16 and model.page_size % 64 == 0
                and 128 % (attn.num_heads // attn.num_kv_heads) == 0)

    def _attention(self, i, block, h):
        """Layer ``i``'s q|k|v projection, q/k norm + RoPE + K/V append and paged FlashAttention for the chunk's rows
        -> ``[L, Hq * D]`` (the wgmma kernel writes the o-projection's layout itself; else attention + one transpose copy)."""
        at, pk, pool = block.self_attn, self._packed[i], self.model.page_pools[i]
        Hq, Hkv = self.Hq, self.Hkv
        if self.L <= 128:  # projection + q/k norm + RoPE + append: the split-reduction planes feed the second kernel
            q = ext.qkv_project_rope_append(pk.qkv.scales, pk.qkv.biases, pk.qkv.weight, h, at.q_norm._weight_as(h.dtype, h.device),
                                            at.k_norm._weight_as(h.dtype, h.device), self.offsets, self.tables[i], self.ctxs,
                                            pool._key_pages, pool._value_pages, Hq, Hkv, at.rope.base, at.q_norm.eps, chunk=True, inv_freq=at.rope.inv_freq)  # [Hq, L, D]
        else:
            q = ext.chunk_qk_norm_rope_append(_proj(h, pk.qkv), at.q_norm._weight_as(h.dtype, h.device), at.k_norm._weight_as(h.dtype, h.device),
                                              self.offsets, self.tables[i], self.ctxs, pool._key_pages, pool._value_pages,
                                              Hq, Hkv, at.rope.base, at.q_norm.eps, inv_freq=at.rope.inv_freq)  # [Hq, L, D]
        return ext.paged_attention_token_major(q, pool._key_pages, pool._value_pages, self.tables[i:i + 1], self.ctx_after, at.scale,
                                               True, Hkv, Hq, workspace=self._attn_ws)

    def _qkv_attention(self, i, block, qkv):
        """``_attention`` from q|k|v rows the adapters were already added to (LoRA engines, any chunk length)."""
        at, pool = block.self_attn, self.model.page_pools[i]
        q = ext.chunk_qk_norm_rope_append(qkv, at.q_norm._weight_as(qkv.dtype, qkv.device), at.k_norm._weight_as(qkv.dtype, qkv.device),
                                          self.offsets, self.tables[i], self.ctxs, pool._key_pages, pool._value_pages,
                                          self.Hq, self.Hkv, at.rope.base, at.q_norm.eps, inv_freq=at.rope.inv_freq)  # [Hq, L, D]
        return ext.paged_attention_token_major(q, pool._key_pages, pool._value_pages, self.tables[i:i + 1], self.ctx_after, at.scale,
                                               True, self.Hkv, self.Hq, workspace=self._attn_ws)

    def _forward(self) -> None:
        m, L = self.model, self.L
        emb = m.embedding.weight
        x = ext.quantized_embedding(self.tokens, emb.scales, emb.biases, emb.weight, emb.group_size, emb.bits).view(L, -1)
        if self.lora is not None:
            x = _lora_layers(m, x, self.adapter_ids, self._qkv_attention)
            self._finish(_normed(x[L - 1:L], m.norm))
            return
        # logits_to_keep = 1: the hidden state is sliced before the final norm (qwen3_week3.py:330-338); RMSNorm is row-wise,
        # so the last row of the already normalised chunk is the same thing
        if L <= 128:  # the fused epilogues live in the <= 128-row tensor-core kernel; longer chunks use the 128 x 128-tile GEMM
            last = _swap_ab_layers(m, x, self._attention)[L - 1:L]
        else:
            for i, block in enumerate(m.layers_inner):
                h = _normed(x, block.input_layernorm)
                x = ext.add(x, _proj(self._attention(i, block, h), block.self_attn.wo))
                h = _normed(x, block.post_attention_layernorm)
                if isinstance(block.mlp, Moe):
                    x = _moe_mlp(block.mlp, x, h)
                    continue
                x = ext.add(x, _proj(ext.swiglu(_proj(h, block.mlp.w_gate), _proj(h, block.mlp.w_up)), block.mlp.w_down))
            last = _normed(x[L - 1:L], m.norm)
        self._finish(last)

    def _finish(self, last) -> None:
        m = self.model
        head = m.w_lm_head if m.w_lm_head is not None else m.embedding.weight
        logits = _proj(last, head)
        self.next_token.copy_(ext.argmax(logits))
        if self.logits is None:
            self.logits = torch.empty_like(logits)
        self.logits.copy_(logits)

    def _set_idle(self) -> None:
        self.meta_dev[2 * self.L:3 * self.L + 1].zero_()  # all rows padding (context 0 -> no append), no visible keys
        self.meta_dev[3 * self.L + 1:].fill_(-1)

    def _capture_graphs(self) -> None:
        self._graph = self._graph_of(self._forward)
        self.kernels_per_chunk = self._launches

    def applies(self, tokens: int, offset: int, cache) -> bool:
        if not (0 < tokens <= self.L) or offset + tokens > self.max_seq_len:
            return False
        for layer_cache, pool in zip(cache, self.model.page_pools):
            if type(layer_cache) is not TinyKvPagedCache or layer_cache.pool is not pool or layer_cache.offset != offset:
                return False
            if pool._key_pages is None or pool._key_pages.dtype != torch.bfloat16:
                return False
            fresh = -(-(offset + tokens) // self.page_size) - len(layer_cache.page_ids)
            if fresh > 0 and fresh > pool.pages_available():
                return False
        return True

    def prefill_chunk(self, token_ids, offset: int, cache, adapter_id: int = -1):
        """Append ``token_ids`` (1..chunk ids at positions offset.., a list or an int32 device tensor) to the request's
        caches and return (logits [1, 1, V] of the last token - a static buffer -, greedy next token [1]).
        ``adapter_id`` (LoRA engines): the request's ``AdapterSet`` id, -1 for the base model."""
        on_device = isinstance(token_ids, torch.Tensor)
        if self.lora is None and adapter_id >= 0:
            raise ValueError("adapter_id given to an engine of a model without adapters")
        r, L = (int(token_ids.numel()) if on_device else len(token_ids)), self.L
        self._host_write_begin()
        for layer, layer_cache in enumerate(cache):
            layer_cache.append_slots(r)
            n = len(layer_cache.page_ids)
            self.tables_np[layer, :n] = layer_cache.page_ids
            self.tables_np[layer, n:] = -1
        self._ensure_graph()
        if self.lora is not None:
            if adapter_id >= len(self.lora.names):
                raise ValueError(f"adapter_id {adapter_id} exceeds the {len(self.lora.names)} loaded adapters")
            self._set_adapter_ids(int(adapter_id))
        pad = L - r
        meta = self.meta_np
        meta[0:L] = 0
        if not on_device:
            meta[pad:L] = token_ids
        pos = np.arange(L, dtype=np.int32) - pad + offset
        meta[L:2 * L] = pos
        meta[2 * L:3 * L] = np.where(np.arange(L) >= pad, pos + 1, 0)
        meta[3 * L] = offset + r
        cur = torch.cuda.current_stream(self.device)
        self._stream.wait_stream(cur)
        with torch.cuda.stream(self._stream):
            self._upload_meta(self.meta_dev, self.meta_host)
            if on_device:  # ids stay on the device: no host round trip for the prompt
                self.meta_dev[pad:L].copy_(token_ids.reshape(-1).to(torch.int32), non_blocking=True)
            self._graph.replay()
        cur.wait_stream(self._stream)
        self.replays += 1
        return self.logits.view(1, 1, -1), self.next_token
