"""Single-request greedy generation with a KV cache
(``src/tiny_llm_ref/generate.py:49-81``)."""

from __future__ import annotations

import torch

from .batch import greedy_tokens
from .logprobs import _check_n, token_logprobs
from .sampler import sample_tokens, token_state_row


def _release_kv_cache(kv_cache) -> None:
    if kv_cache is not None:
        for layer_cache in kv_cache:
            layer_cache.release()


def greedy_generate_ids(model, prompt_ids, max_new_tokens: int, eos_token_id: int | None = None, device=None, on_token=None, sampler=None,
                        sampling=None, logprobs: int | None = None):
    """The loop of ``simple_generate_with_kv_cache`` on token ids: the whole
    prompt is prefilled at offset 0 (its last-row logits give the first token),
    then one token per step at a growing offset.  Returns the generated ids.
    ``sampler`` (``make_sampler``; CUDA extension - the reference's cached loop is greedy only) draws
    from ``logits - logsumexp`` instead of taking the arg-max.  ``sampling`` (a ``SamplingParams``) draws each token
    with the seeded ``tl_sample`` kernel instead, at its position in the sequence: the ids equal a prefill plus
    ``DecodeEngine.decode_on_device(sampling=...)``.  A penalised ``sampling`` keeps the request's ``[1, vocab]`` token
    state, built from the prompt; each launch counts the token it draws.
    ``logprobs`` (an int N in [0, 20]) returns ``(ids, entries)`` instead: one ``TokenLogprobs`` per generated id, from
    the logits row it was chosen from (raw log-probability, rank and the N most likely alternatives)."""
    if sampler is not None and sampling is not None:
        raise ValueError("give sampler or sampling, not both")
    if logprobs is not None:
        _check_n(logprobs)
    kv_cache = model.create_kv_cache()
    produced: list[int] = []
    entries: list = []
    state = None
    try:
        tokens = torch.as_tensor(list(prompt_ids), dtype=torch.int32, device=device)
        offset = 0
        while len(produced) < max_new_tokens:
            logits = model(tokens[None], offset, kv_cache, logits_to_keep=1)
            if sampling is not None:
                if sampling.penalized and state is None:
                    state = token_state_row(tokens, [], logits.shape[-1], device=logits.device)[None]
                token = sample_tokens(logits[:, -1, :], [sampling], [offset + tokens.numel()], state)
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
    """Every model action as a ``model(...)`` call, exactly as the reference issues them (any model, any device)."""

    def __init__(self, model, draft_model, device):
        self.model, self.draft_model, self.device = model, draft_model, device

    def round_fits(self, offset: int, k: int) -> bool:
        """Whether a round of ``k`` proposals at ``offset`` can run on this runner (``model(...)`` takes any length)."""
        return True

    def _step(self, model, ids, offset, cache, n_tokens=1):
        y = torch.as_tensor(ids, dtype=torch.int32, device=self.device)
        logits = model(y[None], offset, cache, logits_to_keep=n_tokens)
        return [int(v) for v in greedy_tokens(logits[0, -n_tokens:, :]).reshape(-1).tolist()]

    def prefill(self, model, ids, cache) -> int:
        return self._step(model, ids, 0, cache)[0]

    def target_step(self, token, offset, cache) -> int:
        return self._step(self.model, [token], offset, cache)[0]

    def draft(self, token, offset, cache, k, eos) -> list[int]:
        """Up to ``k`` draft tokens after ``token``; stops after a draft EOS (reference ``_draft_generate``)."""
        out = []
        for _ in range(k):
            token = self._step(self.draft_model, [token], offset, cache)[0]
            out.append(token)
            offset += 1
            if token in eos:
                break
        return out

    def verify(self, token, proposals, offset, cache) -> tuple[list[int], list[int]]:
        """(target predictions for rows [token, *proposals], the proposals as host ids)."""
        ids = [token, *proposals]
        return self._step(self.model, ids, offset, cache, len(ids)), list(proposals)


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
        limit = min(self.model.decode_graph_max_seq_len, self.draft_model.decode_graph_max_seq_len)
        return offset + k + 1 <= limit

    def draft(self, token, offset, cache, k, eos):
        engine = self.draft_model.decode_engine(1, self.draft_model.decode_graph_max_seq_len)
        return engine.decode_on_device([token], [offset], cache, k).reshape(-1)

    def verify(self, token, proposals, offset, cache):
        k = int(proposals.numel())
        _, nxt = self.model.verify_engine(k + 1).verify(token, proposals, offset, cache)
        both = torch.cat([nxt, proposals.to(torch.int32)]).tolist()  # one device->host read per round
        return [int(v) for v in both[: k + 1]], [int(v) for v in both[k + 1 :]]


def _graph_runner_applies(model, draft_model, device, k) -> bool:
    from .qwen3_week3 import Qwen3ModelWeek3

    if not (1 <= k <= 7) or not (device is None or torch.device(device).type == "cuda"):
        return False
    return all(isinstance(m, Qwen3ModelWeek3) and m.verify_applies() for m in (model, draft_model))


def _rewind(cache, n: int) -> None:
    if n:
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
    (proposed, accepted) counts.  Every page of both caches goes back to its pool on return or on an exception."""
    stats: list[tuple[int, int]] = []
    produced = [0]

    def out(ids) -> bool:  # emit up to the budget; True once it is spent
        ids = list(ids)[: max_new_tokens - produced[0]]
        if ids:
            produced[0] += len(ids)
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
            proposals = runner.draft(token, offset, draft_cache, proposal_length, eos)
            predictions, drafted = runner.verify(token, proposals, offset, cache)
            n = len(drafted)  # tokens appended to the draft cache; the target appended n + 1
            _check_offset(cache, offset + n + 1, "target")
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
            runner.draft(checked[-1], offset - 1, draft_cache, 1, ())  # the draft catches up on its last proposal
            _check_offset(draft_cache, offset, "draft")
    finally:
        _release_kv_cache(draft_cache)
        _release_kv_cache(cache)


def _check_proposal_length(proposal_length) -> None:
    if not isinstance(proposal_length, int) or isinstance(proposal_length, bool) or proposal_length < 0:
        raise ValueError("proposal_length must be a non-negative integer")


def speculative_generate_ids(draft_model, model, prompt_ids, max_new_tokens: int, proposal_length: int = 4, eos_token_ids=(),
                             device=None, on_token=None):
    """Greedy generation of ``model`` with ``draft_model`` proposing ``proposal_length`` tokens per round.  Returns
    ``(ids, stats)``: the generated ids (those of ``greedy_generate_ids(model, ...)``, token for token) and the per-round
    ``(proposed, accepted)`` counts.  CUDA Week-3 models with ``1 <= proposal_length <= 7`` verify in one captured graph
    per round (``Qwen3ModelWeek3.verify_engine``); everything else runs the same protocol through ``model(...)``."""
    _check_proposal_length(proposal_length)
    prompt_ids = [int(t) for t in prompt_ids]
    if not prompt_ids:
        raise ValueError("prompt must encode to at least one token")
    eos = {int(t) for t in eos_token_ids}
    fast = _graph_runner_applies(model, draft_model, device, proposal_length)
    runner = (_GraphRunner if fast else _GenericRunner)(model, draft_model, device)
    produced: list[int] = []

    def emit(ids):
        for t in ids:
            produced.append(int(t))
            if on_token is not None:
                on_token(int(t))

    stats = _speculate(runner, model, draft_model, prompt_ids, max_new_tokens, proposal_length, eos, emit)
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
