"""Single-request greedy generation with a KV cache
(``src/tiny_llm_ref/generate.py:49-81``)."""

from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200

from .batch import greedy_tokens
from .json_mode import ConstraintRows
from .kv_cache import BatchingKvCache
from .logprobs import _check_n, _host_rows, entries_from_host, token_logprobs
from .logit_controls import ControlRows
from .lora import adapter_ids_of
from .sampler import mirostat_start, sample_tokens, token_state_row


def _release_kv_cache(kv_cache) -> None:
    if kv_cache is not None:
        for layer_cache in kv_cache:
            layer_cache.release()


def greedy_generate_ids(model, prompt_ids, max_new_tokens: int, eos_token_id: int | None = None, device=None, on_token=None, sampler=None,
                        sampling=None, logprobs: int | None = None, prefix_cache: bool = False, adapter: str | None = None):
    """The loop of ``simple_generate_with_kv_cache`` on token ids: the whole
    prompt is prefilled at offset 0 (its last-row logits give the first token),
    then one token per step at a growing offset.  Returns the generated ids.
    ``sampler`` (``make_sampler``; CUDA extension - the reference's cached loop is greedy only) draws
    from ``logits - logsumexp`` instead of taking the arg-max.  ``sampling`` (a ``SamplingParams``) draws each token
    with the seeded ``tl_sample`` kernel instead, at its position in the sequence: the ids equal a prefill plus
    ``DecodeEngine.decode_on_device(sampling=...)``.  A penalised ``sampling`` keeps the request's ``[1, vocab]`` token
    state, built from the prompt; each launch counts the token it draws.  A constrained ``sampling`` keeps the
    request's one-row constraint descriptor: the prompt's first token is drawn under the start state and every launch
    advances it on the device.  A ``sampling`` with logits controls keeps the request's one-row ``ControlRows``, built
    from the prompt: the first token is drawn from the prompt's last row with 0 tokens generated, and every launch
    appends the step's input token to the row's history tail.  ``min_tokens`` holds back ``eos_token_id``, and is
    refused without one.
    ``logprobs`` (an int N in [0, 20]) returns ``(ids, entries)`` instead: one ``TokenLogprobs`` per generated id, from
    the logits row it was chosen from (raw log-probability, rank and the N most likely alternatives).
    ``prefix_cache=True`` starts the request on the model's prefix index (``Qwen3ModelWeek3.enable_prefix_cache``):
    only the prompt past its longest cached prefix is prefilled, and the prompt is indexed afterwards.
    ``adapter`` names a LoRA adapter of the model's ``AdapterSet`` (``Qwen3ModelWeek3.load_adapters``): every model call
    of the request runs under it, and its prefix-cache pages are kept apart from other adapters'."""
    if sampler is not None and sampling is not None:
        raise ValueError("give sampler or sampling, not both")
    if logprobs is not None:
        _check_n(logprobs)
    if sampling is not None and sampling.min_tokens > 0 and eos_token_id is None:
        raise ValueError("min_tokens needs the loop's EOS token id: this loop knows none")
    lora = adapter_ids_of(model, adapter, 1)
    lora_kw = {} if lora is None else {"adapter_ids": lora}
    root = () if lora is None else (lora[0],)  # the prefix index's subtree
    kv_cache = model.create_kv_cache()
    produced: list[int] = []
    entries: list = []
    state = constraints = controls = mu = None
    try:
        ids = [int(t) for t in prompt_ids]
        prompt = torch.as_tensor(ids, dtype=torch.int32, device=device)
        index = model.enable_prefix_cache() if prefix_cache else None
        offset = 0 if index is None else index.adopt(index.lookup(ids, *root), kv_cache)
        tokens = prompt[offset:]
        while len(produced) < max_new_tokens:
            logits = model(tokens[None], offset, kv_cache, logits_to_keep=1, **lora_kw)
            if index is not None and offset + tokens.numel() == len(ids):
                index.insert(ids, kv_cache, *root)
            if sampling is not None:
                if sampling.penalized and state is None:
                    state = token_state_row(prompt, [], logits.shape[-1], device=logits.device)[None]
                if sampling.constraint is not None and constraints is None:
                    constraints = ConstraintRows.build([sampling], logits.shape[-1], logits.device)
                if sampling.controls and controls is None:
                    controls = ControlRows(1, logits.shape[-1], logits.device, history_capacity=len(ids) + max_new_tokens)
                    controls.set_row(0, sampling, ids, (), () if eos_token_id is None else (eos_token_id,))
                if sampling.mirostat and mu is None:  # Mirostat's mu, from 2 tau at the first token on
                    mu = torch.full((1,), mirostat_start(sampling), dtype=torch.float32, device=logits.device)
                token = sample_tokens(logits[:, -1, :], [sampling], [offset + tokens.numel()], state, constraints, controls, tokens[-1:],
                                      **({} if mu is None else {"mirostat_mu": mu}))
            elif sampler is None:
                token = greedy_tokens(logits[:, -1, :])
            else:
                row = logits[:, -1, :].to(torch.float32)
                token = sampler(row - torch.logsumexp(row, dim=-1, keepdim=True))
            value = int(token.reshape(-1)[0])  # device->host read, one per step (mx.eval + .item())
            if eos_token_id is not None and value == eos_token_id:
                break
            produced.append(value)
            if logprobs is not None:
                entries.extend(token_logprobs(logits[:, -1, :], [value], logprobs))
            if on_token is not None:
                on_token(value)
            offset += tokens.numel()
            tokens = token.reshape(1).to(torch.int32)
    finally:
        _release_kv_cache(kv_cache)
    return produced if logprobs is None else (produced, entries)


def simple_generate_with_kv_cache(model, tokenizer, prompt: str, max_new_tokens: int = 1 << 30) -> str:
    """generate.py:49-81 - streams the text to stdout and returns it."""
    detokenizer = tokenizer.detokenizer
    detokenizer.reset()

    def emit(token: int) -> None:
        detokenizer.add_token(token)
        print(detokenizer.last_segment, end="", flush=True)

    device = getattr(model, "device", None)
    greedy_generate_ids(
        model,
        tokenizer.encode(prompt, add_special_tokens=False),
        max_new_tokens,
        eos_token_id=tokenizer.eos_token_id,
        device=device,
        on_token=emit,
    )
    return detokenizer.text


# ------------------------------------------------------------------ speculative decoding --
# A draft model proposes k tokens; the target checks all of them in one pass over k + 1 rows and keeps the longest
# prefix it agrees with, plus its own next token.  The target's greedy output comes out unchanged, in fewer target passes
# (``src/tiny_llm_ref/generate.py:84-322``).  ``_speculate`` is the protocol; a ``_Runner`` executes its three model
# actions (prefill, draft k tokens, verify T rows).


class _GenericRunner:
    """Every model action as a ``model(...)`` call, exactly as the reference issues them (any model, any device).
    With ``sampling`` (a plain ``SamplingParams``, temperature > 0) every token is ``tl_sample``'s draw at its position,
    the draft keeps the logits row each proposal was drawn from, and ``verify`` returns ``tl_speculative_sample``'s
    tokens on the target's T rows in place of the argmax predictions (DESIGN.md section 8d)."""

    def __init__(self, model, draft_model, device, sampling=None, proposer=None):
        self.model, self.draft_model, self.device = model, draft_model, device
        self.sampling = sampling
        self.proposer = proposer  # prompt lookup (draft_model None): an ``NgramProposer`` or a stand-in
        self._draft_rows: list = []

    def round_fits(self, offset: int, k: int) -> bool:
        """Whether a round of ``k`` proposals at ``offset`` can run on this runner (``model(...)`` takes any length)."""
        return True

    def _step(self, model, ids, offset, cache, n_tokens=1):
        y = torch.as_tensor(ids, dtype=torch.int32, device=self.device)
        logits = model(y[None], offset, cache, logits_to_keep=n_tokens)
        rows = logits[0, -n_tokens:, :]
        if self.sampling is None:
            return [int(v) for v in greedy_tokens(rows).reshape(-1).tolist()]
        self._last_rows = rows
        first = offset + len(ids) - n_tokens + 1  # the position of the token row 0 predicts
        return [int(v) for v in sample_tokens(rows, [self.sampling] * n_tokens, range(first, first + n_tokens)).tolist()]

    def prefill(self, model, ids, cache) -> int:
        return self._step(model, ids, 0, cache)[0]

    def target_step(self, token, offset, cache) -> int:
        return self._step(self.model, [token], offset, cache)[0]

    def draft(self, token, offset, cache, k, eos) -> list[int]:
        """Up to ``k`` draft tokens after ``token``; stops after a draft EOS (reference ``_draft_generate``)."""
        out = []
        self._draft_rows = []
        for _ in range(k):
            token = self._step(self.draft_model, [token], offset, cache)[0]
            if self.sampling is not None:
                self._draft_rows.append(self._last_rows)
            out.append(token)
            offset += 1
            if token in eos:
                break
        return out

    def propose(self, committed, token):
        """Prompt lookup: the proposer's k proposals after ``token`` as host ids, or None when the history has no match.
        Sampled, the draft rows are the proposer's one-hot rows: q is the point mass at each proposal."""
        match, ids, _, onehot = self.proposer(committed, token)
        if not match:
            return None
        if self.sampling is not None:
            self._draft_rows = list(onehot.split(1))
        return ids

    def verify(self, token, proposals, offset, cache) -> tuple[list[int], list[int]]:
        """(target predictions for rows [token, *proposals], the proposals as host ids)."""
        ids = [token, *proposals]
        if self.sampling is None:
            return self._step(self.model, ids, offset, cache, len(ids)), list(proposals)
        from extensions_b200 import tiny_llm_ext_b200 as ext

        from .sampler import sampling_tensors

        T = len(ids)
        y = torch.as_tensor(ids, dtype=torch.int32, device=self.device)
        target = self.model(y[None], offset, cache, logits_to_keep=T)[0, -T:, :].contiguous()
        draft = torch.cat(self._draft_rows[: T - 1]).to(target.dtype) if T > 1 else target[:0]
        params = sampling_tensors([self.sampling] * T, target.device)
        positions = torch.arange(offset + 1, offset + T + 1, dtype=torch.int32, device=target.device)
        out = ext.speculative_sample(target, draft.contiguous(), y[1:].contiguous(), *params, positions)
        return [int(v) for v in out.tolist()], list(proposals)


class _GraphRunner(_GenericRunner):
    """CUDA Week-3 models: the draft proposes with its B = 1 decode engine's ``decode_on_device(k)`` (always k tokens:
    the device cannot stop at a draft EOS), the target's verify graph reads those proposals device to device, and the
    round's one device->host read brings back the T predictions together with the k proposals.  Proposals after a
    draft EOS are verified and discarded by the protocol: rows j of the verify pass see only tokens <= j, so the
    outcome is the reference's early stop."""

    def round_fits(self, offset: int, k: int) -> bool:
        """The graph engines hold ``decode_graph_max_seq_len`` tokens; ``model(...)`` leaves its decode graph at the same
        limit.  A round appends up to ``offset + k + 1`` tokens to either cache (k proposals, the verify rows, the draft's
        catch-up), so past that point the protocol continues target-only through ``model(...)``, as greedy does."""
        limit = min(m.decode_graph_max_seq_len for m in (self.model, self.draft_model) if m is not None)
        return offset + k + 1 <= limit

    def propose(self, committed, token):
        """Prompt lookup: the proposals as the proposer's device tensor, which the verify graph reads device to device
        (the host ids came back with the match length in the proposer's one read)."""
        match, _, proposals, onehot = self.proposer(committed, token)
        if not match:
            return None
        if self.sampling is not None:
            self._draft_rows = onehot  # a buffer of fixed address: one sampled verify graph per k
        return proposals

    def draft(self, token, offset, cache, k, eos):
        engine = self.draft_model.decode_engine(1, self.draft_model.decode_graph_max_seq_len)
        if self.sampling is None:
            return engine.decode_on_device([token], [offset], cache, k).reshape(-1)
        out, rows = engine.decode_on_device([token], [offset], cache, k, sampling=self.sampling, keep_logits=True)
        self._draft_rows = rows.view(k, -1)  # the log's first k rows: a buffer whose address the verify graph keys on
        return out.reshape(-1)

    def verify(self, token, proposals, offset, cache):
        k = int(proposals.numel())
        kw = {} if self.sampling is None else {"sampling": self.sampling, "draft_logits": self._draft_rows}
        _, nxt = self.model.verify_engine(k + 1).verify(token, proposals, offset, cache, **kw)
        both = torch.cat([nxt, proposals.to(torch.int32)]).tolist()  # one device->host read per round
        return [int(v) for v in both[: k + 1]], [int(v) for v in both[k + 1 :]]


def _graph_runner_applies(model, draft_model, device, k) -> bool:
    from .qwen3_week3 import Qwen3ModelWeek3

    if not (1 <= k <= 7) or not (device is None or torch.device(device).type == "cuda"):
        return False
    return all(isinstance(m, Qwen3ModelWeek3) and m.verify_applies() for m in (model, draft_model) if m is not None)


def _rewind(cache, n: int) -> None:
    if n and cache is not None:
        for layer in cache:
            layer.rewind(n)


def _check_offset(cache, expected: int, what: str) -> None:
    """Every layer of ``cache`` holds ``expected`` tokens (the reference's ``_assert_cache_offset``)."""
    for layer in cache:
        logical = getattr(layer, "logical_offset", None)
        got = logical() if callable(logical) else getattr(layer, "offset", expected)
        if got != expected:
            raise RuntimeError(f"speculative decoding: {what} cache holds {got} tokens, expected {expected}")


def _speculate(runner, model, draft_model, prompt_ids, max_new_tokens, proposal_length, eos, emit):
    """The reference protocol on token ids.  ``emit(ids)`` receives each accepted run; returns the per-round
    (proposed, accepted) counts.  Every page of both caches goes back to its pool on return or on an exception.
    With ``draft_model`` None the proposals come from ``runner.propose`` (prompt lookup): there is no draft cache, and
    a round whose history has no match is one target step, recorded as (0, 0)."""
    stats: list[tuple[int, int]] = []
    produced = [0]
    committed = list(prompt_ids) if draft_model is None else None  # the proposer's view: prompt + emitted ids

    def out(ids) -> bool:  # emit up to the budget; True once it is spent
        ids = list(ids)[: max_new_tokens - produced[0]]
        if ids:
            produced[0] += len(ids)
            if committed is not None:
                committed.extend(ids)
            emit(ids)
        return produced[0] >= max_new_tokens

    def target_only(token, offset):
        while token not in eos and not out([token]):
            token = runner.target_step(token, offset, cache)
            offset += 1
            _check_offset(cache, offset, "target")

    cache = model.create_kv_cache()
    draft_cache = None
    try:
        if max_new_tokens <= 0:
            return stats
        token = runner.prefill(model, prompt_ids, cache)
        offset = len(prompt_ids)
        _check_offset(cache, offset, "target")
        if token in eos:
            return stats
        if proposal_length == 0 or not runner.round_fits(offset, proposal_length):
            target_only(token, offset)
            return stats
        if draft_model is not None:
            draft_cache = draft_model.create_kv_cache()
            draft_token = runner.prefill(draft_model, prompt_ids, draft_cache)
            _check_offset(draft_cache, offset, "draft")
            if draft_token in eos:
                target_only(token, offset)
                return stats
        while True:
            if not runner.round_fits(offset, proposal_length):  # past the graph engines' length: target-only, as greedy
                target_only(token, offset)
                return stats
            if draft_cache is None:
                proposals = runner.propose(committed, token)
                if proposals is None:  # no match: one target step
                    stats.append((0, 0))
                    if out([token]):
                        return stats
                    token = runner.target_step(token, offset, cache)
                    offset += 1
                    _check_offset(cache, offset, "target")
                    if token in eos:
                        return stats
                    continue
            else:
                proposals = runner.draft(token, offset, draft_cache, proposal_length, eos)
            predictions, drafted = runner.verify(token, proposals, offset, cache)
            n = len(drafted)  # tokens appended to the draft cache; the target appended n + 1
            _check_offset(cache, offset + n + 1, "target")
            if draft_cache is not None:
                _check_offset(draft_cache, offset + n, "draft")
            aligned = [token, *predictions[:-1]]
            checked = [token, *drafted]
            stop = None  # (index, terminal)
            for i, (t, d) in enumerate(zip(aligned, checked)):
                if t != d:
                    stop = (i, False)
                    break
                if t in eos:
                    stop = (i, True)
                    break
            if stop is not None:
                i, terminal = stop
                stats.append((n, i if terminal else i - 1))
                _rewind(cache, n + 1 - i)
                _rewind(draft_cache, n - i)
                _check_offset(cache, offset + i, "target")
                if draft_cache is not None:
                    _check_offset(draft_cache, offset + i, "draft")
                if out(aligned[:i]) or terminal:
                    return stats
                token = aligned[i]
                offset += i
                if token in eos:
                    return stats
                continue
            stats.append((n, n))
            if out(aligned):
                return stats
            offset += n + 1
            token = predictions[-1]
            if token in eos:
                return stats
            if draft_cache is not None:
                runner.draft(checked[-1], offset - 1, draft_cache, 1, ())  # the draft catches up on its last proposal
                _check_offset(draft_cache, offset, "draft")
    finally:
        _release_kv_cache(draft_cache)
        _release_kv_cache(cache)


def _check_proposal_length(proposal_length) -> None:
    if not isinstance(proposal_length, int) or isinstance(proposal_length, bool) or proposal_length < 0:
        raise ValueError("proposal_length must be a non-negative integer")


def _spec_sampling(sampling, constraint):
    """The ``SamplingParams`` speculative decoding samples with (None: greedy), refusing what it does not take."""
    from .grammar import GrammarConstraint

    if isinstance(constraint, GrammarConstraint):
        raise ValueError("speculative decoding is greedy and unconstrained: it takes no grammar")
    if constraint is not None:
        raise ValueError("speculative decoding is greedy and unconstrained: it takes no constraint")
    if sampling is None:
        return None
    from .sampler import SamplingParams

    if not isinstance(sampling, SamplingParams):
        raise ValueError(f"sampling must be None or a SamplingParams, got {type(sampling).__name__}")
    if sampling.grammar:
        raise ValueError("speculative decoding and prompt lookup are unconstrained: sampling must carry no grammar")
    if sampling.constraint is not None:
        raise ValueError("speculative decoding is unconstrained: sampling must carry no constraint")
    if sampling.xtc:
        raise ValueError("speculative decoding and prompt lookup take no XTC: xtc_probability must be 0")
    _refuse_truncation(sampling, "speculative decoding and prompt lookup take")
    if sampling.dry:
        raise ValueError("speculative decoding and prompt lookup take no DRY: dry_multiplier must be 0")
    if sampling.penalized:
        raise ValueError("speculative sampling takes temperature, top-k and top-p only: no penalties or min-p")
    if sampling.controls:
        raise ValueError("speculative decoding takes no logit_bias, allowed_token_ids, bad_words_ids or min_tokens")
    return None if sampling.temperature == 0 else sampling


def _refuse_truncation(sampling, what: str) -> None:
    """The ValueError for a truncation sampler (DESIGN.md section 25) where ``what`` (a phrase ending in a verb) has
    none: the message names the field."""
    if sampling.typical_p < 1:
        raise ValueError(f"{what} no typical sampling: typical_p must be 1")
    if sampling.top_n_sigma > 0:
        raise ValueError(f"{what} no top-n-sigma: top_n_sigma must be 0")
    if sampling.mirostat:
        raise ValueError(f"{what} no Mirostat: mirostat must be 0")


def speculative_generate_ids(draft_model, model, prompt_ids, max_new_tokens: int, proposal_length: int = 4, eos_token_ids=(),
                             device=None, on_token=None, constraint=None, sampling=None):
    """Greedy generation of ``model`` with ``draft_model`` proposing ``proposal_length`` tokens per round.  Returns
    ``(ids, stats)``: the generated ids (those of ``greedy_generate_ids(model, ...)``, token for token) and the per-round
    ``(proposed, accepted)`` counts.  CUDA Week-3 models with ``1 <= proposal_length <= 7`` verify in one captured graph
    per round (``Qwen3ModelWeek3.verify_engine``); everything else runs the same protocol through ``model(...)``.
    Speculative decoding is unconstrained: a ``constraint`` is refused with ``ValueError``.
    ``sampling`` (a ``SamplingParams`` with temperature, top-k, top-p and seed; temperature 0 is the greedy path) samples
    instead (DESIGN.md section 8d): the draft draws each proposal with ``tl_sample`` and every verify round keeps or
    replaces it by the rejection rule of ``tl_speculative_sample``, so each emitted token is distributed as the target's
    own ``tl_sample`` draw at its position.  With the target's weights as draft the ids equal
    ``greedy_generate_ids(model, sampling=...)``.  Penalties, min-p and constraints are refused with ``ValueError``."""
    _check_proposal_length(proposal_length)
    sampling = _spec_sampling(sampling, constraint)
    prompt_ids = [int(t) for t in prompt_ids]
    if not prompt_ids:
        raise ValueError("prompt must encode to at least one token")
    eos = {int(t) for t in eos_token_ids}
    fast = _graph_runner_applies(model, draft_model, device, proposal_length)
    runner = (_GraphRunner if fast else _GenericRunner)(model, draft_model, device, sampling)
    produced: list[int] = []

    def emit(ids):
        for t in ids:
            produced.append(int(t))
            if on_token is not None:
                on_token(int(t))

    stats = _speculate(runner, model, draft_model, prompt_ids, max_new_tokens, proposal_length, eos, emit)
    return produced, stats


# ------------------------------------------------------------------ prompt lookup --
# The proposals are the tokens that followed the latest, longest earlier occurrence of the history's last n tokens
# (``tl_ngram_propose``, DESIGN.md section 14): no second model, no second cache and no draft pass.  The rounds are
# ``_speculate``'s with ``draft_model`` None.


class NgramProposer:
    """Prompt lookup's proposer for one request.  The history (prompt, emitted ids, pending token) lives in a device
    buffer: the prompt is uploaded once, and each call appends the ids emitted since the previous call as kernel
    arguments, runs one ``ngram_propose`` launch and reads back the match length and the k proposals (one small
    device->host read).  With ``onehot_dtype`` the proposer also keeps the ``[k, vocab]`` one-hot rows of its current
    proposals (the draft distribution of the sampled verify pass) at a fixed address, in the model's logits dtype."""

    def __init__(self, model, prompt_ids, k: int, ngram, device=None, sampled: bool = False, capacity: int = 0):
        from extensions_b200 import tiny_llm_ext_b200 as ext

        self._ext = ext
        scales = model.embedding.weight.scales  # the activation dtype: that of the verify pass's logits
        device = scales.device if device is None else device
        self.k, (self.n_min, self.n_max) = k, ngram
        prompt = torch.as_tensor([int(t) for t in prompt_ids], dtype=torch.int32)
        self.length = prompt.numel()
        self.history = torch.empty(max(capacity, self.length + ext.NGRAM_MAX_APPEND), dtype=torch.int32, device=device)
        self.history[: self.length].copy_(prompt)
        self.out = torch.empty(2 + k, dtype=torch.int32, device=device)
        self.state = torch.zeros(ext.NGRAM_STATE_WORDS, dtype=torch.int32, device=device)
        self.onehot = None
        if sampled:
            self.onehot = torch.full((k, model.vocab_size), float("-inf"), dtype=scales.dtype, device=device)

    def __call__(self, committed, token):
        """-> (match length, host proposals, device proposals [k], one-hot rows or None) for the history
        ``committed + [token]``, of which the first ``self.length`` ids are already on the device."""
        new = [*committed[self.length :], int(token)]
        if self.length + len(new) > self.history.numel():  # grow by doubling, device to device
            grown = torch.empty(2 * (self.length + len(new)), dtype=torch.int32, device=self.history.device)
            grown[: self.length].copy_(self.history[: self.length])
            self.history = grown
        self._ext.ngram_propose(self.history, self.length, new, self.k, self.n_min, self.n_max, self.out, self.state, self.onehot)
        self.length += len(new)
        host = self.out.tolist()  # the round's one added device->host read
        return host[0], host[2:] if host[0] else [], self.out[2:], self.onehot


def _check_prompt_lookup(proposal_length, ngram) -> tuple[int, int]:
    if not isinstance(proposal_length, int) or isinstance(proposal_length, bool) or not 1 <= proposal_length <= 7:
        raise ValueError("proposal_length must be an integer in [1, 7] for prompt lookup")
    try:
        n_min, n_max = (int(n) for n in ngram)
    except (TypeError, ValueError):
        raise ValueError("ngram must be a pair (n_min, n_max)") from None
    if not 1 <= n_min <= n_max <= 8 or any(isinstance(n, bool) or int(n) != n for n in ngram):
        raise ValueError("ngram must satisfy 1 <= n_min <= n_max <= 8")
    return n_min, n_max


def prompt_lookup_generate_ids(model, prompt_ids, max_new_tokens: int, proposal_length: int = 4, ngram=(2, 3), eos_token_ids=(),
                               device=None, on_token=None, sampling=None):
    """Speculative generation of ``model`` whose proposals come from the request's own tokens (prompt lookup): each round
    proposes the ``proposal_length`` tokens that followed the latest occurrence of the longest suffix of the history
    of ``ngram = (n_min, n_max)`` tokens, on the device (``NgramProposer``), and verifies them with ``_speculate``'s
    protocol.  A round with no match is one target step.  Returns ``(ids, stats)`` with per-round ``(proposed,
    accepted)`` counts, ``(0, 0)`` for a round without a match.  CUDA Week-3 models verify in one captured graph per
    round, reading the proposals device to device; MoE models and other devices verify through ``model(...)``.
    Greedy (``sampling`` None or temperature 0), the ids equal ``greedy_generate_ids(model, ...)`` token for token.
    Sampled, the draft distribution is the point mass at each proposal, so ``tl_speculative_sample`` accepts proposal
    d with probability p_d and otherwise draws from p restricted to i != d: each emitted token is distributed as the
    target's ``tl_sample`` draw at its position, but the ids need not equal ``greedy_generate_ids(model,
    sampling=...)``'s (the acceptance and residual draws use their own Philox streams).  Constraints, penalties and
    min-p are refused with ``ValueError``, as are ``proposal_length`` outside [1, 7] and ``ngram`` outside
    ``1 <= n_min <= n_max <= 8``."""
    ngram = _check_prompt_lookup(proposal_length, ngram)
    sampling = _spec_sampling(sampling, None)
    prompt_ids = [int(t) for t in prompt_ids]
    if not prompt_ids:
        raise ValueError("prompt must encode to at least one token")
    eos = {int(t) for t in eos_token_ids}
    fast = _graph_runner_applies(model, None, device, proposal_length)
    capacity = len(prompt_ids) + min(max(max_new_tokens, 0), 1 << 16) + 8
    proposer = NgramProposer(model, prompt_ids, proposal_length, ngram, device, sampling is not None, capacity)
    runner = (_GraphRunner if fast else _GenericRunner)(model, None, device, sampling, proposer=proposer)
    produced: list[int] = []

    def emit(ids):
        for t in ids:
            produced.append(int(t))
            if on_token is not None:
                on_token(int(t))

    stats = _speculate(runner, model, None, prompt_ids, max_new_tokens, proposal_length, eos, emit)
    return produced, stats


def speculative_generate(draft_model, model, draft_tokenizer, tokenizer, prompt: str, proposal_length: int = 4) -> str:
    """generate.py:84-322 - prints each accepted run as ``+n <text tail>`` and the final text, and returns the text."""
    _check_proposal_length(proposal_length)

    def _encode(tok):
        return [int(t) for t in tok.encode(prompt, add_special_tokens=False)]

    def _eos_ids(tok):
        ids = getattr(tok, "eos_token_ids", None)
        if ids is None:
            ids = {tok.eos_token_id}
        return {int(t) for t in ids}

    target_prompt = _encode(tokenizer)
    draft_prompt = _encode(draft_tokenizer)
    if not target_prompt:
        raise ValueError("prompt must encode to at least one token")
    if target_prompt != draft_prompt:
        raise ValueError("draft and target tokenizers encode the prompt differently")
    if _eos_ids(tokenizer) != _eos_ids(draft_tokenizer):
        raise ValueError("draft and target tokenizers use different EOS token ids")
    target_vocab, draft_vocab = getattr(tokenizer, "get_vocab", None), getattr(draft_tokenizer, "get_vocab", None)
    if not callable(target_vocab) or not callable(draft_vocab):
        raise ValueError("draft and target tokenizers must expose comparable vocabularies")
    if target_vocab() != draft_vocab():
        raise ValueError("draft and target tokenizers use different token ids")
    detokenizer = tokenizer.detokenizer
    detokenizer.reset()

    def emit(ids):
        for t in ids:
            detokenizer.add_token(t)
        print(f"+{len(ids)} {detokenizer.text.replace(chr(10), ' ')[-80:]}")

    device = getattr(model, "device", None)
    eos = _eos_ids(tokenizer)
    fast = _graph_runner_applies(model, draft_model, device, proposal_length)
    runner = (_GraphRunner if fast else _GenericRunner)(model, draft_model, device)
    _speculate(runner, model, draft_model, target_prompt, 1 << 62, proposal_length, eos, emit)
    finalize = getattr(detokenizer, "finalize", None)
    if callable(finalize):
        finalize()
    text = detokenizer.text
    print(text)
    return text


# ------------------------------------------------------------------ beam search --
# Each step scores every live beam's top W + E tokens, ``tl_logprobs``' top-N lists, and ``tl_beam_select`` walks the
# candidates of all beams in one order (DESIGN.md section 15).  Beam j decodes in slot j of a W-row step; a parent's
# first child takes over the parent's caches and the others fork them (``paged_kv_cache.fork``: shared full pages, a
# copied tail page).


@dataclass
class BeamHypothesis:
    """One result of ``beam_search_ids``: the generated ids (an ending EOS is not included), the sum of their
    log-probabilities (with the EOS's), ``sum_logprob / L**length_penalty`` with L the length including the EOS, and
    whether the hypothesis ended in an EOS (False: cut by ``max_new_tokens``)."""

    ids: list
    sum_logprob: float
    score: float
    finished: bool


def unpack_beam_result(words):
    """The packed ``tl_beam_select`` result (``BEAM_RESULT_WORDS`` int32 words) as ``(live, finished)``: live beams
    ``(parent, token, cum)`` and finished records ``(parent, eos id, sum, walk position)``, in walk order."""
    w = np.asarray(words, dtype=np.int32)
    f = w.view(np.float32)
    M = tiny_llm_ext_b200.BEAM_MAX_WIDTH
    a, b = 2, 2 + 3 * M
    live = [(int(w[a + j]), int(w[a + M + j]), float(f[a + 2 * M + j])) for j in range(int(w[0]))]
    finished = [(int(w[b + j]), int(w[b + M + j]), float(f[b + 2 * M + j]), int(w[b + 3 * M + j])) for j in range(int(w[1]))]
    return live, finished


def _beam_score(total: float, length: int, length_penalty: float) -> float:
    return float(total) / (float(length) ** length_penalty)


class _BeamRunner:
    """Beam search's model actions through ``model(...)`` (any paged model, any device): a step is one call over the W
    slots (``BatchingKvCache`` per layer) and eager ``logprobs`` + ``beam_select`` launches on its W rows."""

    def __init__(self, model, width: int, eos: tuple, device):
        self.model, self.W, self.eos, self.device = model, width, eos, device
        self.N = width + len(eos)
        self.cum = self.result = None

    def _buffers(self, device):
        if self.cum is None:
            self.cum = torch.zeros(self.W, dtype=torch.float32, device=device)
            self.result = torch.zeros(tiny_llm_ext_b200.BEAM_RESULT_WORDS, dtype=torch.int32, device=device)

    def _select(self, rows):
        _, _, _, ids, top = tiny_llm_ext_b200.logprobs(rows.contiguous(), None, None, self.N)
        tiny_llm_ext_b200.beam_select(top, ids, self.cum, self.W, self.eos, self.result)
        return self.result.tolist()  # the step's one device->host read

    def first(self, row):
        """Select from the prompt's last logits row ``[1, V]`` with ``cum = [0]``."""
        self._buffers(row.device)
        self.cum.zero_()
        return self._select(row)

    def step(self, tokens, offsets, caches):
        y = torch.as_tensor(tokens, dtype=torch.int32, device=self.device).view(self.W, 1)
        logits = self.model(y, list(offsets), caches, logits_to_keep=1)
        return self._select(logits[:, -1, :])


class _BeamGraphRunner(_BeamRunner):
    """CUDA Week-3 models: every step after the first is one replay of the W-slot decode engine's beam step graph
    (``DecodeEngine.beam_step``), whose ``beam_cum`` the first, eager select writes."""

    def __init__(self, model, width: int, eos: tuple, device):
        super().__init__(model, width, eos, device)
        self.engine = model.decode_engine(width, model.decode_graph_max_seq_len)
        _, _, self.result = self.engine.beam_buffers(eos)
        self.cum = self.engine.beam_cum

    def step(self, tokens, offsets, caches):
        return self.engine.beam_step(tokens, offsets, caches, self.eos).tolist()


def _beam_graph_applies(model, device, tokens: int) -> bool:
    from .qwen3_week3 import Qwen3ModelWeek3

    return (isinstance(model, Qwen3ModelWeek3) and model._paged and model.use_decode_graph is not False
            and getattr(model, "adapters", None) is None and torch.device(device).type == "cuda"
            and tokens <= model.decode_graph_max_seq_len)


def _check_beam_args(num_beams, length_penalty, num_return_sequences, max_new_tokens, eos) -> None:
    width, max_eos = tiny_llm_ext_b200.BEAM_MAX_WIDTH, tiny_llm_ext_b200.BEAM_MAX_EOS
    if not isinstance(num_beams, int) or isinstance(num_beams, bool) or not 1 <= num_beams <= width:
        raise ValueError(f"num_beams must be an integer in [1, {width}]")
    if len(eos) > max_eos:
        raise ValueError(f"beam search takes at most {max_eos} EOS ids")
    if (not isinstance(num_return_sequences, int) or isinstance(num_return_sequences, bool)
            or not 1 <= num_return_sequences <= num_beams):
        raise ValueError("num_return_sequences must be an integer in [1, num_beams]")
    if not math.isfinite(float(length_penalty)):
        raise ValueError("length_penalty must be finite")
    if not isinstance(max_new_tokens, int) or max_new_tokens < 0:
        raise ValueError("max_new_tokens must be a non-negative integer")


def beam_search_ids(model, prompt_ids, max_new_tokens: int, num_beams: int = 4, length_penalty: float = 1.0,
                    early_stopping: bool = False, num_return_sequences: int = 1, eos_token_ids=(), device=None):
    """Deterministic beam search of ``num_beams`` (1..8) beams (DESIGN.md section 15; ``tests/beam_ref.py`` states the
    rule in plain loops).  Each step walks every live beam's top ``num_beams + len(eos_token_ids)`` tokens in the order
    (score descending, beam, rank): an EOS among the first ``num_beams`` finishes a hypothesis, other tokens become the
    next beams.  A hypothesis of L tokens (its EOS included) scores ``sum_logprob / L**length_penalty``; at most
    ``num_beams`` finished ones are kept.  The search ends when no beam is left, when ``num_beams`` are kept and
    ``early_stopping`` is set or no live beam's score beats the worst kept one, or after ``max_new_tokens`` steps, when
    the live beams join the pool unfinished.  Returns the best ``num_return_sequences`` ``BeamHypothesis``, best first.
    With ``num_beams=1`` and ``early_stopping=True`` the ids are ``greedy_generate_ids``'.
    CUDA Week-3 models whose decode graph window holds prompt + ``max_new_tokens`` run each step as one replay of the
    W-slot beam step graph; other paged models run the same protocol through ``model(...)``.  Refused with
    ``ValueError`` before any work: ``num_beams`` outside 1..8, more than 4 EOS ids, ``num_return_sequences`` outside
    1..num_beams, a non-finite ``length_penalty``, a negative ``max_new_tokens``, an empty prompt and non-paged caches."""
    eos = tuple(dict.fromkeys(int(t) for t in eos_token_ids))
    _check_beam_args(num_beams, length_penalty, num_return_sequences, max_new_tokens, eos)
    prompt = [int(t) for t in prompt_ids]
    if not prompt:
        raise ValueError("prompt must encode to at least one token")
    from .paged_kv_cache import TinyKvPagedCache, fork

    cache = model.create_kv_cache()
    if not all(isinstance(c, TinyKvPagedCache) for c in cache):
        _release_kv_cache(cache)
        raise ValueError("beam search needs paged KV caches (the Week-3 model)")
    if max_new_tokens == 0:
        _release_kv_cache(cache)
        return []
    W, alpha = num_beams, float(length_penalty)
    if device is None:
        scales = getattr(getattr(getattr(model, "embedding", None), "weight", None), "scales", None)
        device = None if scales is None else scales.device
    graph = device is not None and _beam_graph_applies(model, device, len(prompt) + max_new_tokens)
    runner = (_BeamGraphRunner if graph else _BeamRunner)(model, W, eos, device)
    kept: list = []  # (hypothesis, (step, walk position)), best first, at most W

    def keep(hyp, order):
        kept.append((hyp, order))
        kept.sort(key=lambda h: (-h[0].score, h[1]))
        del kept[W:]

    beams: list = []  # (per-layer caches, ids) of the live beams, beam j in slot j
    try:
        logits = model(torch.as_tensor(prompt, dtype=torch.int32, device=device)[None], 0, cache, logits_to_keep=1)
        words = runner.first(logits[:, -1, :])
        beams, cache = [(cache, [])], None
        slots = [BatchingKvCache(W) for _ in range(len(beams[0][0]))]
        step = 0
        while True:
            live, finished = unpack_beam_result(words)
            for parent, _, total, pos in finished:
                ids = beams[parent][1]
                keep(BeamHypothesis(list(ids), total, _beam_score(total, len(ids) + 1, alpha), True), (step, pos))
            step += 1
            if not live:
                break
            if len(kept) == W and (early_stopping or max(_beam_score(c, len(beams[p][1]) + 1, alpha) for p, _, c in live) <= kept[-1][0].score):
                break
            if step == max_new_tokens:
                for j, (p, tok, c) in enumerate(live):
                    ids = [*beams[p][1], tok]
                    keep(BeamHypothesis(ids, c, _beam_score(c, len(ids), alpha), False), (max_new_tokens, j))
                break
            children: dict = {}
            for p, _, _ in live:
                children[p] = children.get(p, 0) + 1
            for i, (caches, ids) in enumerate(beams):  # before the forks: the pages held stay within W beams' worth
                if i not in children:
                    _release_kv_cache(caches)
                    beams[i] = (None, ids)
            extra = [p for p in children if children[p] > 1]
            forks = dict(zip(extra, fork([(beams[p][0], children[p] - 1) for p in extra])))
            taken: set = set()
            new = []
            for p, tok, _ in live:
                if p in taken:
                    caches = forks[p].pop()
                else:
                    taken.add(p)
                    caches = beams[p][0]
                new.append((caches, [*beams[p][1], tok]))
            beams = new
            tokens, offsets = [0] * W, [0] * W
            for j, (caches, ids) in enumerate(beams):
                tokens[j], offsets[j] = ids[-1], len(prompt) + len(ids) - 1
            for layer, slot in enumerate(slots):
                slot.kv_caches = [beams[j][0][layer] if j < len(beams) else None for j in range(W)]
            words = runner.step(tokens, offsets, slots)
    finally:
        _release_kv_cache(cache)
        for caches, _ in beams:
            _release_kv_cache(caches)
    return [h for h, _ in kept[:num_return_sequences]]


# ------------------------------------------------------------------ parallel sampling --
# n seeded samples of each prompt from one prefill: the prompt's cache is forked n - 1 ways (``paged_kv_cache.fork``),
# prompt i's samples decode in slots i*n .. i*n+n-1 of one P*n-slot step, and each such range is a group of
# ``DecodeEngine.decode_on_device(groups=...)``, whose shared prompt pages are attended once per step (DESIGN.md
# section 16).

PARALLEL_MAX_SAMPLES = 16  # n x G <= 128 for every Qwen3 head ratio up to G = 8
PARALLEL_MAX_SLOTS = 64
PARALLEL_ROUND = 16  # decode steps between two reads of the tokens


@dataclass
class ParallelSample:
    """One sample of ``parallel_sample_ids``: the generated ids (an ending EOS is not included), ``"stop"`` (an EOS)
    or ``"length"`` (``max_new_tokens``), and one ``TokenLogprobs`` per id when logprobs were asked for (else None)."""

    ids: list
    finish_reason: str
    logprobs: list | None = None


def sample_seed(seed: int, j: int) -> int:
    """The seed of sample ``j`` of a request seeded ``seed``: ``(seed + j) mod 2**64`` (the CLI's "request i uses
    seed + i"), as the signed 64-bit value ``SamplingParams`` holds."""
    v = (int(seed) + int(j)) % (1 << 64)
    return v - (1 << 64) if v >= (1 << 63) else v


def _check_parallel_args(model, prompts, num_samples, sampling, max_new_tokens, logprobs, adapter) -> list:
    from .sampler import SamplingParams

    if adapter is not None:
        raise ValueError("parallel sampling takes no adapter")
    if not isinstance(num_samples, int) or isinstance(num_samples, bool) or not 1 <= num_samples <= PARALLEL_MAX_SAMPLES:
        raise ValueError(f"num_samples must be an integer in [1, {PARALLEL_MAX_SAMPLES}]")
    if not prompts or len(prompts) * num_samples > PARALLEL_MAX_SLOTS:
        raise ValueError(f"prompts x num_samples must be in [1, {PARALLEL_MAX_SLOTS}]")
    if any(len(p) == 0 for p in prompts):
        raise ValueError("prompt must encode to at least one token")
    if not isinstance(max_new_tokens, int) or isinstance(max_new_tokens, bool) or max_new_tokens < 0:
        raise ValueError("max_new_tokens must be a non-negative integer")
    if logprobs is not None:
        _check_n(logprobs)
    per = [sampling] * len(prompts) if isinstance(sampling, SamplingParams) else list(sampling)
    if len(per) != len(prompts) or not all(isinstance(p, SamplingParams) for p in per):
        raise ValueError("sampling must be one SamplingParams or one per prompt")
    if any(p.dry for p in per):
        raise ValueError("parallel sampling takes no DRY: dry_multiplier must be 0")
    if any(p.controls for p in per):
        raise ValueError("parallel sampling takes no logit_bias, allowed_token_ids, bad_words_ids or min_tokens")
    if num_samples > 1 and any(p.temperature == 0 for p in per):
        raise ValueError("temperature 0 is greedy: every sample would be the same; give num_samples=1")
    return per


def parallel_sample_ids(model, prompts, num_samples: int, sampling, max_new_tokens: int, eos_token_ids=(), logprobs=None, device=None,
                        adapter=None):
    """``num_samples`` independent seeded samples of each prompt of ``prompts`` (lists of ids) from one prefill each.
    Sample j of a prompt draws with ``replace(sampling, seed=(seed + j) mod 2**64)`` (``sampling``: one
    ``SamplingParams`` or one per prompt), so it is the ``greedy_generate_ids(sampling=...)`` run of that seed.  Each
    sample ends at its first EOS (not returned) or after ``max_new_tokens``.  Returns one list per prompt of
    ``num_samples`` ``ParallelSample``.
    The prompt's cache is forked ``num_samples - 1`` ways; all samples decode together, in rounds of
    ``decode_on_device`` on a CUDA Week-3 model whose graph window holds the prompt and budget (with grouped attention
    over each prompt's shared pages where ``shared_prefix_attention_applies``), else through ``model(...)``.  Every
    page goes back to its pool on return and on an exception.  Refused with ``ValueError`` before any work:
    ``num_samples`` outside 1..16, more than 64 samples in all, an empty prompt, a negative budget, non-paged caches,
    temperature 0 with ``num_samples > 1`` and an ``adapter``."""
    from dataclasses import replace

    from .paged_kv_cache import TinyKvPagedCache, fork
    from .sampler import token_state_row

    prompts = [[int(t) for t in p] for p in prompts]
    per = _check_parallel_args(model, prompts, num_samples, sampling, max_new_tokens, logprobs, adapter)
    probe = model.create_kv_cache()
    paged = all(isinstance(c, TinyKvPagedCache) for c in probe)
    _release_kv_cache(probe)
    if not paged:
        raise ValueError("parallel sampling needs paged KV caches (the Week-3 model)")
    n, P = num_samples, len(prompts)
    eos = {int(t) for t in eos_token_ids}
    params = [replace(per[i], seed=sample_seed(per[i].seed, j)) for i in range(P) for j in range(n)]
    out = [[ParallelSample([], "length", [] if logprobs is not None else None) for _ in range(n)] for _ in range(P)]
    if max_new_tokens == 0:
        return out
    if device is None:
        scales = getattr(getattr(getattr(model, "embedding", None), "weight", None), "scales", None)
        device = None if scales is None else scales.device
    longest = max(len(p) for p in prompts) + max_new_tokens
    graph = device is not None and _beam_graph_applies(model, device, longest)
    slots: list = [None] * (P * n)  # per-layer caches of each sample
    done = [False] * (P * n)
    penalized = any(p.penalized for p in params)
    constrained = any(p.constraint is not None for p in params)
    mirostat = any(p.mirostat for p in params)
    state = constraints = mu = None
    mu_first = None  # the samples' mu after their first tokens, handed to the first decode_on_device round

    def take(b, token, entry) -> None:
        if done[b]:
            return
        s = out[b // n][b % n]
        if token in eos:
            done[b], s.finish_reason = True, "stop"
            return
        s.ids.append(int(token))
        if entry is not None:
            s.logprobs.append(entry)
        if len(s.ids) >= max_new_tokens:
            done[b] = True

    try:
        firsts = []
        for i, prompt in enumerate(prompts):
            cache = model.create_kv_cache()
            slots[i * n] = cache
            logits = model(torch.as_tensor(prompt, dtype=torch.int32, device=device)[None], 0, cache, logits_to_keep=1)
            rows = logits[:, -1, :].expand(n, -1).contiguous()
            st = con = None
            if penalized:
                st = torch.stack([token_state_row(torch.as_tensor(prompt), [], rows.shape[-1], device=rows.device)] * n)
            if constrained:
                con = ConstraintRows.build(params[i * n : i * n + n], rows.shape[-1], rows.device)
            m = None
            if mirostat:
                m = torch.tensor([mirostat_start(p) if p.mirostat else 0.0 for p in params[i * n : i * n + n]], dtype=torch.float32,
                                 device=rows.device)
            tok = sample_tokens(rows, params[i * n : i * n + n], [len(prompt)] * n, st, con, **({} if m is None else {"mirostat_mu": m}))
            ent = token_logprobs(rows, tok, logprobs) if logprobs is not None else [None] * n
            firsts.append((tok.tolist(), ent, st, con, m))
            if n > 1:
                slots[i * n + 1 : i * n + n] = fork([(cache, n - 1)])[0]
        tokens = [0] * (P * n)
        for i, (tok, ent, st, con, _) in enumerate(firsts):
            for j in range(n):
                tokens[i * n + j] = tok[j]
                take(i * n + j, tok[j], ent[j])
        if not graph:
            state = torch.cat([f[2] for f in firsts]) if penalized else None
            constraints = ConstraintRows.concat([f[3] for f in firsts]) if constrained else None
            mu = torch.cat([f[4] for f in firsts]) if mirostat else None
        elif mirostat:
            mu_first = [float(v) if p.mirostat else None for v, p in zip(torch.cat([f[4] for f in firsts]).tolist(), params)]
        offsets = [len(prompts[b // n]) for b in range(P * n)]
        batch = [BatchingKvCache(P * n) for _ in range(len(slots[0]))]
        for layer, slot in enumerate(batch):
            slot.kv_caches = [slots[b][layer] for b in range(P * n)]
        groups = [(i * n, n) for i in range(P)] if n > 1 else None
        engine = model.decode_engine(P * n, model.decode_graph_max_seq_len) if graph else None
        while not all(done):
            steps = min(PARALLEL_ROUND, max_new_tokens - min(len(out[b // n][b % n].ids) for b in range(P * n) if not done[b]))
            if graph:
                history = None
                if penalized or constrained:
                    history = [(prompts[b // n], out[b // n][b % n].ids) for b in range(P * n)]
                got = engine.decode_on_device(tokens, offsets, batch, steps, sampling=params, logprobs=logprobs, history=history, groups=groups,
                                              **({} if mu_first is None else {"mirostat_mu": mu_first}))
                mu_first = None  # later rounds go on from the device's mu
                ids, lp = (got, None) if logprobs is None else got
                host = ids.tolist()  # the round's device->host read
                lp_host = None if lp is None else [_host_rows(ids[s], *[t[s] for t in lp]) for s in range(steps)]
                for s in range(steps):
                    ent = entries_from_host(*lp_host[s]) if lp_host is not None else [None] * (P * n)
                    for b in range(P * n):
                        take(b, host[s][b], ent[b])
                tokens = host[-1]
                offsets = [o + steps for o in offsets]
            else:
                for _ in range(steps):
                    y = torch.as_tensor(tokens, dtype=torch.int32, device=device).view(P * n, 1)
                    rows = model(y, list(offsets), batch, logits_to_keep=1)[:, -1, :]
                    tok = sample_tokens(rows, params, [o + 1 for o in offsets], state, constraints, **({} if mu is None else {"mirostat_mu": mu}))
                    ent = token_logprobs(rows, tok, logprobs) if logprobs is not None else [None] * (P * n)
                    tokens = tok.tolist()
                    for b in range(P * n):
                        take(b, tokens[b], ent[b])
                    offsets = [o + 1 for o in offsets]
    finally:
        for caches in slots:
            _release_kv_cache(caches)
    return out
