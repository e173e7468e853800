"""Continuous batching with chunked prefill
(``src/tiny_llm_ref/batch.py``).

Scheduling policy, verbatim from the reference loop (batch.py:164-270): at most
one request is being prefilled, ``prefill_step`` tokens per iteration and always
as a ``B=1`` call; when its prompt is consumed it moves into the first idle
decode slot; every iteration that has at least one occupied slot runs ONE decode
step over all ``batch_size`` slots (idle slots carry token 0 / offset 0 and are
masked out by ``context_lens == 0``).  Each live cache is released exactly once,
also on failure (batch.py:271-284).

``ContinuousBatcher`` holds that loop as an object so that a serving front end
can step it; ``batch_generate`` is the reference's function on top of it.
"""

from __future__ import annotations

import time
from datetime import datetime

import torch

from extensions_b200 import tiny_llm_ext_b200

from .kv_cache import BatchingKvCache
from .logprobs import _check_n, token_logprobs
from .lora import adapter_ids_of
from .json_mode import ConstraintRows
from .sampler import any_constrained, any_penalized, sample_tokens, sampling_per_request, token_state_row


def greedy_tokens(logits: torch.Tensor) -> torch.Tensor:
    """argmax over the vocabulary of ``[rows, vocab]`` logits.  The reference
    subtracts logsumexp first (batch.py:10-12), which cannot change the argmax;
    CUDA logits use the extension's reduction kernel, host tensors (fake models
    in scheduler tests) plain torch."""
    if logits.is_cuda:
        return tiny_llm_ext_b200.argmax(logits.contiguous())
    return torch.argmax(logits, dim=-1)


def _step(model, y, offsets, kv_cache, **lora):
    """One model call -> one greedy token per row (batch.py:8-13).  ``lora``: the rows' ``adapter_ids``, when any is named."""
    logits = model(y, offsets, kv_cache, logits_to_keep=1, **lora)
    return greedy_tokens(logits[:, -1, :])


class _TokenLog:
    """Detokenizer stand-in for token-id workloads (no tokenizer): keeps ids."""

    def __init__(self, _=None):
        self.tokens: list[int] = []

    def add_token(self, token: int) -> None:
        self.tokens.append(token)

    @property
    def text(self) -> str:
        return " ".join(map(str, self.tokens))


class Request:
    """One prompt moving through prefill then decode (batch.py:16-96).

    ``prompt`` is a string (encoded with ``tokenizer``) or, for synthetic
    serving runs, a sequence of token ids (``tokenizer`` may then be ``None``;
    pass ``eos_token_id`` explicitly if one is wanted).  ``sampling`` (a
    ``SamplingParams``) draws the request's tokens with the seeded ``tl_sample``
    kernel; None keeps them greedy.  A penalised ``sampling`` draws the first
    token against the prompt-only token state (``token_state_row``).  A constrained ``sampling`` draws the first token
    under the start state of ``constraint_row``, its one-row ``ConstraintRows``, which that launch advances.  ``logprobs``
    (an int N) records one ``TokenLogprobs`` per generated token in
    ``logprob_entries``."""

    def __init__(
        self,
        model,
        tokenizer,
        prompt,
        prefill_max_step: int = 128,
        prompt_idx: int = 0,
        max_seq_len: int | None = None,
        eos_token_id: int | None = None,
        device=None,
        sampling=None,
        logprobs=None,
        prefix_cache=None,
        adapter_id: int = -1,
    ):
        self.prompt = prompt
        self.adapter_id = adapter_id  # the request's id in the model's AdapterSet, -1: the base model
        self.sampling = sampling
        self.logprobs = logprobs
        self.logprob_entries: list = []
        self.constraint_row = None  # one-row ConstraintRows, made with the first token's draw
        self.model = model
        if isinstance(prompt, str):
            ids = tokenizer.encode(prompt, add_special_tokens=False)
        else:
            ids = [int(t) for t in prompt]
        if tokenizer is not None:
            self.detokenizer = tokenizer.detokenizer.__class__(tokenizer._tokenizer)
            self.eos_token_id = tokenizer.eos_token_id
        else:
            self.detokenizer = _TokenLog()
            self.eos_token_id = eos_token_id
        self.prefill_tokens = torch.tensor(ids, dtype=torch.int32, device=device)
        if max_seq_len is not None and self.prefill_tokens.numel() > max_seq_len:
            raise ValueError(f"Prompt has {self.prefill_tokens.numel()} tokens, which exceeds max_seq_len={max_seq_len}")
        self.kv_cache = model.create_kv_cache()
        self.prefill_max_step = prefill_max_step
        self.max_seq_len = max_seq_len
        self.is_done = False
        self.is_prefill_done = False
        self.finish_reason = None
        self.next_token = None
        self.offset = 0
        self.prompt_idx = prompt_idx
        # prefix caching: the request starts on the cached pages of the longest indexed prefix of its prompt and
        # prefills from there; its prompt is indexed once prefilled
        self.prefix_cache = prefix_cache
        self.prompt_ids = ids if prefix_cache is not None else None
        self.reused_tokens = 0
        if prefix_cache is not None:
            match = prefix_cache.lookup(ids) if adapter_id < 0 else prefix_cache.lookup(ids, adapter_id)
            self.reused_tokens = self.offset = prefix_cache.adopt(match, self.kv_cache)

    def _lora(self) -> dict:
        """The adapter keyword of the request's model calls (nothing for the base model)."""
        return {} if self.adapter_id < 0 else {"adapter_ids": [self.adapter_id]}

    def try_prefill(self):
        """Advance the prompt by at most ``prefill_max_step`` tokens (batch.py:48-76)."""
        if self.is_prefill_done:
            raise ValueError("prefill called after done")
        total = self.prefill_tokens.numel()
        chunk = min(self.prefill_max_step, total - self.offset)
        ids = self.prefill_tokens[self.offset : self.offset + chunk][None]
        entry = None
        if self.sampling is None and self.logprobs is None:
            token = _step(self.model, ids, [self.offset], self.kv_cache, **self._lora())
        else:  # only the last chunk's token is used: the prompt's first token is drawn at position `total`
            logits = self.model(ids, [self.offset], self.kv_cache, logits_to_keep=1, **self._lora())[:, -1, :]
            token = None
            if self.offset + chunk == total:
                if self.sampling is None:
                    token = greedy_tokens(logits)
                else:
                    state = None
                    if self.sampling.penalized:
                        state = token_state_row(self.prefill_tokens, [], logits.shape[-1], device=logits.device)[None]
                    if self.sampling.constraint is not None:
                        self.constraint_row = ConstraintRows.build([self.sampling], logits.shape[-1], logits.device)
                    token = sample_tokens(logits, [self.sampling], [total], state, self.constraint_row)
                if self.logprobs is not None:
                    entry = token_logprobs(logits, token, self.logprobs)[0]
        self.offset += chunk
        for layer_cache in self.kv_cache:
            layer_cache.materialize()
        if self.offset == total:
            self.is_prefill_done = True
            if self.prefix_cache is not None:
                if self.adapter_id < 0:
                    self.prefix_cache.insert(self.prompt_ids, self.kv_cache)
                else:
                    self.prefix_cache.insert(self.prompt_ids, self.kv_cache, self.adapter_id)
            if self.max_seq_len is not None and self.offset >= self.max_seq_len:
                self.is_done = True
                self.finish_reason = "max seq len"
            else:
                self.decode_done(int(token.reshape(-1)[0]), False, entry)

    def decode_done(self, token, update_offset=True, entry=None):
        if self.is_done:
            raise ValueError("decode called after done")
        if token == self.eos_token_id:
            self.is_done = True
            self.finish_reason = "EOS"
            return
        if entry is not None:
            self.logprob_entries.append(entry)
        self.detokenizer.add_token(token)
        self.next_token = token
        if update_offset:
            self.offset += 1

    def text(self):
        return self.detokenizer.text

    def reaches_max_seq_len(self, max_seq_len: int) -> bool:
        # next_token is emitted but not yet in the KV cache: it sits at `offset`.
        return self.next_token is not None and self.offset + 1 >= max_seq_len


def _print_progress(slots, pending, queued: int, tick: int, started: datetime):
    """batch.py:99-133."""
    print(f"  --- {datetime.now() - started}")
    frames = ["⠋", "⠙", "⠹", "⠸", "⠼", "⠴", "⠦", "⠧", "⠇", "⠏"]
    frame = frames[tick % len(frames)]
    for i, request in enumerate(slots):
        if request is None:
            print(f"  Decode #{i}: idle", flush=True)
        else:
            tail = request.text()[-80:].replace("\n", " ")
            print(f"{frame} Decode [req {request.prompt_idx}, {request.offset}]: {tail}", flush=True)
    if pending is None:
        print(f"  Prefill: idle, {queued} requests in queue", flush=True)
    elif pending.is_prefill_done:
        print(f"  Prefill [req {pending.prompt_idx}]: done, waiting for slot, {queued} requests in queue", flush=True)
    else:
        total = pending.prefill_tokens.numel()
        print(
            f"{frame} Prefill [req {pending.prompt_idx}]: {pending.offset / total * 100:.2f}% "
            f"({total - pending.offset} remaining tokens)",
            flush=True,
        )


class ContinuousBatcher:
    """The reference scheduling loop as a steppable object.  ``sampling``: None (greedy, the reference's loop), one
    ``SamplingParams`` for every prompt or a list with one per prompt; a request's tokens are then drawn by the seeded
    ``tl_sample`` kernel from its last prefill chunk's and every decode step's logits, and do not depend on its slot or
    on the other requests.  ``logprobs`` (an int N in [0, 20]) fills ``self.logprobs[prompt_idx]`` with one
    ``TokenLogprobs`` per generated token: the first from the prompt's last prefill chunk, the others from the decode
    step that produced them (one ``ext.logprobs`` launch over all slots per step, idle slots with target -1).

    ``prefix_cache=True`` turns on the model's prefix index (``Qwen3ModelWeek3.enable_prefix_cache``): a request
    admitted to prefill starts on the cached KV pages of the longest indexed prefix of its prompt and prefills only the
    rest; its prompt is indexed once prefilled.  ``reused_tokens[prompt_idx]`` and ``self.reused_total`` record the
    reuse; tokens, sampling, penalties and logprobs are those of a full prefill.

    Penalised requests (``SamplingParams.penalized``) keep their token state in one int32 ``[batch_size, vocab]`` slab,
    allocated when the first of them enters a slot.  From then on every admission rebuilds the slot's row from the
    prompt and the first token, and every decode step with a penalised slot is one ``tl_sample_penalized`` launch over
    all slots (idle slots at position 0, so their rows do not change); the kernel counts each drawn token.

    Constrained requests (``SamplingParams.constraint``) keep their automaton state in one ``ConstraintRows`` of
    ``batch_size`` rows (``tl_constraint_row`` descriptors, plus JSON states and mask buffers once a JSON request
    enters), allocated when the first of them enters a slot.  Admission copies the
    request's row (advanced by its prefill draw) into the slot on the device; idle and unconstrained slots hold zero
    rows.  Every decode step with a constrained slot is one ``tl_sample_constrained`` launch over all slots.

    ``adapters`` (None, one name for every prompt, or one name or None per prompt) runs each request under that LoRA
    adapter of the model's ``AdapterSet`` (``Qwen3ModelWeek3.load_adapters``): its prefill chunks carry its id, its slot
    carries it from admission to release (``slot_adapter_ids``, -1 for idle and base-model slots), and its prefix-cache
    lookups see only pages computed under the same adapter.  A request's tokens are those it gets alone."""

    def __init__(self, model, tokenizer, prompts, max_seq_len=512, batch_size=5, prefill_step=128, verbose=True,
                 eos_token_id=None, device=None, max_new_tokens=None, sampling=None, logprobs=None, prefix_cache=False, adapters=None):
        if max_seq_len <= 0:
            raise ValueError("max_seq_len must be positive")
        if batch_size <= 0:
            raise ValueError("batch_size must be positive")
        if prefill_step <= 0:
            raise ValueError("prefill_step must be positive")
        self.model = model
        self.tokenizer = tokenizer
        self.queue = list(prompts)
        self.sampling = sampling_per_request(sampling, len(self.queue))
        self.adapter_ids = adapter_ids_of(model, adapters, len(self.queue))  # per prompt, None: no request names one
        self.slot_adapter_ids = [-1] * batch_size
        self.logprobs_n = None if logprobs is None else _check_n(logprobs)
        self.logprobs: dict[int, list] = {}
        self.max_seq_len = max_seq_len
        self.batch_size = batch_size
        self.prefill_step = prefill_step
        self.verbose = verbose
        self.eos_token_id = eos_token_id
        self.device = device
        self.max_new_tokens = max_new_tokens  # optional per-request budgets (synthetic serving)
        self.slots: list[Request | None] = [None] * batch_size
        self.kv_cache = [BatchingKvCache(max_active_requests=batch_size, max_seq_len=max_seq_len) for _ in range(model.num_hidden_layers)]
        self.pending: Request | None = None
        self.results: list[tuple[int, str]] = []
        self.next_request_idx = 0
        self.tick = 0
        self.started = datetime.now()
        self.decode_steps = 0
        self.decode_tokens = 0
        self.prefill_tokens = 0
        self.generated: dict[int, int] = {}
        # serving metrics in the spirit of benches/bench.py:351-572 (ServingMetrics): wall time of every
        # decode step / prefill chunk (the host reads the sampled tokens each step, so wall == device time
        # + host scheduling), peak concurrently live requests and KV pages (all layers)
        self.record_timing = False
        self.decode_step_ms: list[float] = []   # wall time per decode step (host reads the tokens: includes queued GPU work)
        self.prefill_chunk_ms: list[float] = []  # wall time per prefill chunk (enqueue only unless it is a prompt's last chunk)
        self._gpu_events: list[tuple[str, object, object]] = []  # (kind, start, end) CUDA events on the current stream
        self.peak_active_requests = 0
        self.peak_live_pages = 0
        self.token_state: torch.Tensor | None = None  # [batch_size, vocab] int32, on first penalised admission
        self.constraint_rows: ConstraintRows | None = None  # batch_size rows, on first constrained admission
        self.prefix_cache = model.enable_prefix_cache() if prefix_cache else None
        self.reused_tokens: dict[int, int] = {}
        self.reused_total = 0

    # -- bookkeeping ---------------------------------------------------------
    def idle(self) -> bool:
        return not self.queue and self.pending is None and all(s is None for s in self.slots)

    def _progress(self):
        if self.verbose:
            _print_progress(self.slots, self.pending, len(self.queue), self.tick, self.started)
        self.tick += 1

    def _gpu_span(self, kind: str):
        """CUDA events around one scheduler phase (device time without the host: an intermediate prefill chunk is not
        synchronised by the scheduler, so its GPU work would otherwise be charged to the decode step behind it)."""
        if not (self.record_timing and torch.cuda.is_available() and self.device is not None and torch.device(self.device).type == "cuda"):
            return None
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        self._gpu_events.append((kind, start, end))
        return end

    def gpu_phase_ms(self) -> dict:
        """Per-phase device times (ms) from the recorded CUDA events; call after the run (synchronises)."""
        out: dict = {"prefill": [], "decode": []}
        if self._gpu_events:
            torch.cuda.synchronize()
        for kind, start, end in self._gpu_events:
            out[kind].append(start.elapsed_time(end))
        return out

    def _record_cache_state(self) -> None:
        live = [s for s in self.slots if s is not None]
        if self.pending is not None:
            live.append(self.pending)
        self.peak_active_requests = max(self.peak_active_requests, len(live))
        if self.prefix_cache is None:
            pages = sum(len(getattr(r.kv_cache[0], "page_ids", ())) for r in live) * len(self.kv_cache)  # layers move in lockstep
        else:  # a page shared through the prefix cache counts once
            pages = len({p for r in live for p in r.kv_cache[0].page_ids}) * len(self.kv_cache)
        self.peak_live_pages = max(self.peak_live_pages, pages)

    def _admit_state(self, request: Request, slot: int) -> None:
        """Rebuild the slot's token-state row from the request's prompt and first token (allocating the slab when the
        first penalised request arrives)."""
        if self.token_state is None:
            if request.sampling is None or not request.sampling.penalized:
                return
            vocab = self.model.vocab_size
            self.token_state = torch.zeros((self.batch_size, vocab), dtype=torch.int32, device=request.prefill_tokens.device)
        token_state_row(request.prefill_tokens, [request.next_token], self.token_state.shape[1], out=self.token_state[slot])

    def _admit_constraint(self, request: Request, slot: int) -> None:
        """Copy the request's constraint row into the slot's row (a device copy of its state), or clear the row.  The
        JSON state and mask buffers are allocated with the first JSON request."""
        if self.constraint_rows is None:
            if request.constraint_row is None:
                return
            src = request.constraint_row
            self.constraint_rows = ConstraintRows(self.batch_size, src.vocab, src.device, src.has_json, src.has_schema)
        if request.constraint_row is None:
            self.constraint_rows.clear_row(slot)
        else:
            self.constraint_rows.copy_row(slot, request.constraint_row)

    def _budget_spent(self, request: Request) -> bool:
        if self.max_new_tokens is None:
            return False
        return self.generated.get(request.prompt_idx, 0) >= self.max_new_tokens[request.prompt_idx]

    # -- one scheduler iteration ----------------------------------------------
    def step(self) -> None:
        if self.queue and self.pending is None:
            prompt = self.queue.pop(0)
            self.pending = Request(
                self.model, self.tokenizer, prompt, self.prefill_step, self.next_request_idx,
                max_seq_len=self.max_seq_len, eos_token_id=self.eos_token_id, device=self.device,
                sampling=None if self.sampling is None else self.sampling[self.next_request_idx],
                logprobs=self.logprobs_n, prefix_cache=self.prefix_cache,
                adapter_id=-1 if self.adapter_ids is None else self.adapter_ids[self.next_request_idx],
            )
            if self.prefix_cache is not None:
                self.reused_tokens[self.next_request_idx] = self.pending.reused_tokens
                self.reused_total += self.pending.reused_tokens
            if self.logprobs_n is not None:
                self.logprobs[self.next_request_idx] = self.pending.logprob_entries
            self.next_request_idx += 1

        if self.pending is not None:
            moved = False
            request = self.pending
            if not request.is_prefill_done:
                before = request.offset
                t0 = time.perf_counter() if self.record_timing else 0.0
                span = self._gpu_span("prefill")
                request.try_prefill()
                if span is not None:
                    span.record()
                if self.record_timing:
                    self.prefill_chunk_ms.append((time.perf_counter() - t0) * 1e3)
                self.prefill_tokens += request.offset - before
                if request.is_prefill_done and request.next_token is not None:
                    self.generated[request.prompt_idx] = 1
                moved = True
            if request.is_prefill_done:
                if request.is_done or request.reaches_max_seq_len(self.max_seq_len) or self._budget_spent(request):
                    text = request.text()
                    for layer_cache in request.kv_cache:
                        layer_cache.release()
                    self.results.append((request.prompt_idx, text))
                    self.pending = None
                    moved = True
                else:
                    for i in range(self.batch_size):
                        if self.slots[i] is None:
                            for layer_cache, table in zip(request.kv_cache, self.kv_cache):
                                table.add_request(layer_cache, i)
                            self._admit_state(request, i)
                            self._admit_constraint(request, i)
                            self.slot_adapter_ids[i] = request.adapter_id
                            self.slots[i] = request
                            self.pending = None
                            moved = True
                            break
            if moved:
                self._progress()

        if any(s is not None for s in self.slots):
            tokens = [0 if s is None else s.next_token for s in self.slots]
            offsets = [0 if s is None else s.offset for s in self.slots]
            if self.record_timing:
                self._record_cache_state()
            t0 = time.perf_counter() if self.record_timing else 0.0
            span = self._gpu_span("decode")
            batch = torch.tensor(tokens, dtype=torch.int32, device=self.device).reshape(-1, 1)
            entries = None
            lora = {} if self.adapter_ids is None else {"adapter_ids": list(self.slot_adapter_ids)}
            if self.sampling is None and self.logprobs_n is None:
                sampled = _step(self.model, batch, offsets, self.kv_cache, **lora)
            else:  # slot i draws the token at position offset + 1; idle and greedy slots get argmax's token
                logits = self.model(batch, offsets, self.kv_cache, logits_to_keep=1, **lora)[:, -1, :]
                if self.sampling is None:
                    sampled = greedy_tokens(logits)
                else:  # idle slots draw greedily at position 0: a penalised launch leaves their state rows alone
                    params = [None if s is None else s.sampling for s in self.slots]
                    positions = [0 if s is None else o + 1 for s, o in zip(self.slots, offsets)]
                    sampled = sample_tokens(logits, params, positions, self.token_state if any_penalized(params) else None,
                                            self.constraint_rows if any_constrained(params) else None)
                if self.logprobs_n is not None:
                    live = torch.tensor([s is not None for s in self.slots], device=sampled.device)
                    targets = torch.where(live, sampled.reshape(-1).to(torch.int32), -1)
                    entries = token_logprobs(logits, targets, self.logprobs_n)
            if span is not None:
                span.record()
            # one device->host read per step (with logprobs, the entries carry the tokens: idle slots hold -1 and are skipped)
            host = sampled.reshape(-1).tolist() if entries is None else [e.token for e in entries]
            if self.record_timing:
                self.decode_step_ms.append((time.perf_counter() - t0) * 1e3)
            self.decode_steps += 1
            for i, request in enumerate(self.slots):
                if request is None:
                    continue
                request.decode_done(int(host[i]), entry=None if entries is None else entries[i])
                self.decode_tokens += 1
                self.generated[request.prompt_idx] = self.generated.get(request.prompt_idx, 0) + (0 if request.is_done else 1)
                reason = None
                if request.is_done:
                    reason = request.finish_reason
                elif request.reaches_max_seq_len(self.max_seq_len):
                    reason = "max seq len"
                elif self._budget_spent(request):
                    reason = "max new tokens"
                if reason is not None:
                    if self.verbose:
                        print(f"Removing request {i} due to {reason}", flush=True)
                    text = request.text()
                    for table in self.kv_cache:
                        table.remove_request(i)
                    if self.constraint_rows is not None:
                        self.constraint_rows.clear_row(i)
                    self.results.append((request.prompt_idx, text))
                    self.slot_adapter_ids[i] = -1
                    self.slots[i] = None
            self._progress()

    def release_all(self) -> None:
        """Release every live cache object exactly once (batch.py:271-284)."""
        live = {}
        if self.pending is not None:
            for layer_cache in self.pending.kv_cache:
                live[id(layer_cache)] = layer_cache
        for table in self.kv_cache:
            for layer_cache in table.kv_caches:
                if layer_cache is not None:
                    live[id(layer_cache)] = layer_cache
            table.kv_caches = [None] * table.max_active_requests
        for layer_cache in live.values():
            layer_cache.release()

    def run(self) -> list[tuple[int, str]]:
        try:
            while not self.idle():
                self.step()
        finally:
            self.release_all()
        return self.results


def batch_generate(model, tokenizer, prompts, max_seq_len=512, batch_size=5, prefill_step=128, verbose=True, **kwargs):
    """batch.py:136-285 - returns ``[(prompt_idx, text), ...]`` in completion order.  With ``logprobs=N`` it returns
    ``(results, logprobs)`` instead, ``logprobs[prompt_idx]`` the request's ``TokenLogprobs`` (``ContinuousBatcher``)."""
    batcher = ContinuousBatcher(
        model, tokenizer, prompts, max_seq_len=max_seq_len, batch_size=batch_size, prefill_step=prefill_step,
        verbose=verbose, **kwargs
    )
    results = batcher.run()
    return results if kwargs.get("logprobs") is None else (results, batcher.logprobs)
