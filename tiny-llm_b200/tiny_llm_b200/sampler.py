"""``make_sampler(temp, top_p, top_k)`` (``src/tiny_llm_ref/sampler.py:5-25``) on
torch tensors: greedy at ``temp == 0``; otherwise mask everything outside the ``top_k`` most likely
tokens, then everything outside the smallest prefix of the sorted distribution whose mass reaches
``top_p`` (a token is kept while the mass BEFORE it is < top_p, ``:19``), divide by ``temp`` and draw
from the categorical distribution.  Runs wherever the log-probabilities live (CUDA in the serving
path: one sort + cumsum over the 151,936-wide row, no host round trip); ``generator`` makes the draw
reproducible."""

from __future__ import annotations

import math
import numbers
from dataclasses import dataclass

import torch


def make_sampler(temp: float, top_p: float | None = None, top_k: int | None = None, generator: torch.Generator | None = None):
    def sample(logprobs: torch.Tensor) -> torch.Tensor:
        if temp == 0:
            return torch.argmax(logprobs, dim=-1)
        lp = logprobs.to(torch.float32).clone()
        if top_k is not None and 0 < top_k < lp.shape[-1]:
            kth = torch.topk(lp, top_k, dim=-1).values[..., -1:]
            lp = torch.where(lp < kth, torch.full_like(lp, float("-inf")), lp)
        if top_p is not None and top_p > 0:
            sorted_lp, sorted_idx = torch.sort(lp, dim=-1, descending=True)
            probs = torch.exp(sorted_lp)
            keep = torch.cumsum(probs, dim=-1) - probs < top_p
            sorted_lp = torch.where(keep, sorted_lp, torch.full_like(sorted_lp, float("-inf")))
            lp = torch.full_like(lp, float("-inf")).scatter(-1, sorted_idx, sorted_lp)
        probs = torch.softmax(lp / temp, dim=-1)
        return torch.multinomial(probs, 1, generator=generator).squeeze(-1)

    return sample


@dataclass(frozen=True)
class SamplingParams:
    """One request's seeded sampling on the CUDA path (``tl_sample``, DESIGN.md section 8).  ``temperature == 0`` is
    greedy, the ``argmax`` token.  Otherwise the token is drawn from ``softmax(logits / temperature)`` restricted to the
    keep set of ``top_k`` (on for ``0 < top_k < vocab``; ties at the k-th value are kept) and ``top_p`` (on for
    ``0 < top_p < 1``; a token is kept while the probability mass strictly above it is ``< top_p``).  The draw is a pure
    function of (logits row, parameters, ``seed``, position of the drawn token): the same request gives the same tokens
    in any batch, slot or engine.

    Token-history penalties and min-p (``tl_sample_penalized``, DESIGN.md section 8b), each off at its default:
    ``repetition_penalty`` (> 0, off at 1) divides a positive logit (multiplies a negative one) of every token seen in
    the prompt or drawn so far; ``frequency_penalty`` subtracts ``frequency_penalty * count`` and ``presence_penalty``
    subtracts itself from every token drawn so far (both may be negative); ``min_p`` (in [0, 1], on above 0) keeps a
    token only when its probability after temperature is at least ``min_p`` times the top one.  The draw, greedy
    included, then runs on the penalised logits.

    ``constraint`` (a ``TokenConstraint``, ``tl_sample_constrained``, DESIGN.md section 8c) restricts every draw to the
    tokens that keep the text a prefix of the pattern's language (EOS once it is a match); greedy under a constraint is
    ``SamplingParams(0.0, constraint=c)``.  With a mask that allows every token the draw is the unconstrained one.
    A ``JsonConstraint`` (JSON mode, DESIGN.md section 20) restricts the text to one JSON object the same way, and a
    ``JsonSchemaConstraint`` (DESIGN.md section 21) to one JSON object that validates against a schema, and a
    ``GrammarConstraint`` (DESIGN.md section 23) to the language of a GBNF grammar.

    Logits controls (``tl_logit_controls``, DESIGN.md section 22), each off at its default and refused together with a
    ``constraint``: ``logit_bias`` (a mapping token id -> finite bias in [-100, 100], at most 1024 entries) adds its
    bias to the token's logit in one fp32 add; ``allowed_token_ids`` (a non-empty collection of ids) sends every other
    token to -inf; ``bad_words_ids`` (at most 64 sequences of 1-16 ids) sends a sequence's last id to -inf whenever its
    other ids are the request's most recent tokens (prompt, then generated ids); ``min_tokens`` sends the EOS ids to
    -inf until that many tokens have been generated.  The draw, greedy included, runs on the controlled row.  They are
    stored normalised: ``logit_bias`` as ``((id, bias), ...)`` sorted by id, ``allowed_token_ids`` as a sorted tuple of
    distinct ids and ``bad_words_ids`` as a tuple of tuples, so a ``SamplingParams`` stays hashable.

    DRY (``tl_dry_penalty``, DESIGN.md section 24), a logits control run after the others: with ``dry_multiplier``
    m > 0, a token that would extend a repeat of an earlier span of the history (prompt, then generated ids) of
    length l >= ``dry_allowed_length`` a loses ``m * dry_base ** (l - a)`` (b > 1), l capped at 64 and taken over
    the last ``dry_penalty_last_n`` tokens (0: all of them); a repeat never runs through a
    ``dry_sequence_breakers`` id (at most 64, stored as a sorted tuple).  XTC (the penalised form, DESIGN.md section
    24): with probability ``xtc_probability`` per draw, every kept token whose probability is at least
    ``xtc_threshold`` but the least likely of them is excluded, when there are two or more.

    Truncation samplers (the penalised form, DESIGN.md section 25), each off at its default: ``top_n_sigma`` n > 0 keeps
    only tokens whose logit is at least ``max - n * sigma`` (sigma the standard deviation of the row's finite logits);
    ``typical_p`` p < 1 (locally typical sampling) keeps, of the tokens left, those closest to the row's entropy in
    surprise until their probability reaches p; ``mirostat=2`` (Mirostat 2.0) keeps the tokens whose surprise
    ``-log2 p`` is at most the request's mu, which starts at ``2 * mirostat_tau`` and after every draw moves by
    ``-mirostat_eta * (surprise - mirostat_tau)``.  Mirostat replaces top-k, top-p, min-p, typical, top-n-sigma and
    XTC, and is refused beside any of them."""

    temperature: float
    top_k: int | None = None
    top_p: float | None = None
    seed: int = 0
    repetition_penalty: float = 1.0
    presence_penalty: float = 0.0
    frequency_penalty: float = 0.0
    min_p: float = 0.0
    constraint: object = None
    logit_bias: object = None
    allowed_token_ids: object = None
    bad_words_ids: object = None
    min_tokens: int = 0
    dry_multiplier: float = 0.0
    dry_base: float = 1.75
    dry_allowed_length: int = 2
    dry_penalty_last_n: int = 0
    dry_sequence_breakers: object = ()
    xtc_threshold: float = 0.1
    xtc_probability: float = 0.0
    typical_p: float = 1.0
    top_n_sigma: float = 0.0
    mirostat: int = 0
    mirostat_tau: float = 5.0
    mirostat_eta: float = 0.1

    def __post_init__(self):
        t = self.temperature
        if isinstance(t, bool) or not isinstance(t, numbers.Real) or not math.isfinite(t) or t < 0:
            raise ValueError(f"temperature must be a finite number >= 0, got {t!r}")
        k = self.top_k
        if k is not None and (isinstance(k, bool) or not isinstance(k, numbers.Integral) or k < 0):
            raise ValueError(f"top_k must be None or an int >= 0, got {k!r}")
        p = self.top_p
        if p is not None and (isinstance(p, bool) or not isinstance(p, numbers.Real) or not math.isfinite(p)):
            raise ValueError(f"top_p must be None or a finite number, got {p!r}")
        s = self.seed
        if isinstance(s, bool) or not isinstance(s, numbers.Integral) or not 0 <= s < 1 << 64:
            raise ValueError(f"seed must be an int in [0, 2**64), got {s!r}")

        def real(v):
            return not isinstance(v, bool) and isinstance(v, numbers.Real) and math.isfinite(v)

        r = self.repetition_penalty
        if not real(r) or not r > 0:
            raise ValueError(f"repetition_penalty must be a finite number > 0, got {r!r}")
        for name in ("presence_penalty", "frequency_penalty"):
            v = getattr(self, name)
            if not real(v):
                raise ValueError(f"{name} must be a finite number, got {v!r}")
        m = self.min_p
        if not real(m) or not 0 <= m <= 1:
            raise ValueError(f"min_p must be a number in [0, 1], got {m!r}")
        q = self.xtc_probability
        if not real(q) or not 0 <= q <= 1:
            raise ValueError(f"xtc_probability must be a number in [0, 1], got {q!r}")
        th = self.xtc_threshold
        if not real(th) or not 0 < th <= 1:
            raise ValueError(f"xtc_threshold must be a number in (0, 1], got {th!r}")
        object.__setattr__(self, "xtc_probability", float(q))
        object.__setattr__(self, "xtc_threshold", float(th))
        tp = self.typical_p
        if not real(tp) or not 0 < tp <= 1:
            raise ValueError(f"typical_p must be a number in (0, 1], got {tp!r}")
        ns = self.top_n_sigma
        if not real(ns) or not ns >= 0:
            raise ValueError(f"top_n_sigma must be a finite number >= 0, got {ns!r}")
        mo = self.mirostat
        if isinstance(mo, bool) or not isinstance(mo, numbers.Integral) or mo not in (0, 1, 2):
            raise ValueError(f"mirostat must be 0 (off) or 2, got {mo!r}")
        if mo == 1:
            raise ValueError("Mirostat 1.0 is not supported; use mirostat=2")
        for name in ("mirostat_tau", "mirostat_eta"):
            v = getattr(self, name)
            if not real(v) or not v > 0:
                raise ValueError(f"{name} must be a finite number > 0, got {v!r}")
            object.__setattr__(self, name, float(v))
        object.__setattr__(self, "typical_p", float(tp))
        object.__setattr__(self, "top_n_sigma", float(ns))
        object.__setattr__(self, "mirostat", int(mo))
        if self.mirostat:
            for name, on in (("top_k", (self.top_k or 0) > 0), ("top_p", self.top_p is not None and 0 < self.top_p < 1),
                             ("min_p", self.min_p > 0), ("typical_p", self.typical_p < 1), ("top_n_sigma", self.top_n_sigma > 0),
                             ("xtc_probability", self.xtc)):
                if on:
                    raise ValueError(f"mirostat=2 replaces the other truncation samplers: {name} must be off beside it")
        from .dry import normalized_dry

        for name, value in normalized_dry(self).items():
            object.__setattr__(self, name, value)
        if self.dry and self.constraint is not None:
            raise ValueError("dry_multiplier takes no constraint")
        if self.constraint is not None:
            from .constrained import TokenConstraint
            from .json_mode import JsonConstraint
            from .json_schema import JsonSchemaConstraint
            from .grammar import GrammarConstraint

            if not isinstance(self.constraint, (TokenConstraint, JsonConstraint, JsonSchemaConstraint, GrammarConstraint)):
                raise ValueError(f"constraint must be None or a TokenConstraint, got {type(self.constraint).__name__}")
        from .logit_controls import normalized_controls

        for name, value in normalized_controls(self).items():
            object.__setattr__(self, name, value)
        if self.controls and self.grammar:
            raise ValueError("logit_bias, allowed_token_ids, bad_words_ids and min_tokens take no grammar constraint")
        if self.controls and self.constraint is not None:
            raise ValueError("logit_bias, allowed_token_ids, bad_words_ids and min_tokens take no constraint")

    @property
    def controls(self) -> bool:
        """Whether the request needs ``tl_logit_controls``: a logit bias, an allow-list, banned sequences or min_tokens."""
        return (self.logit_bias is not None or self.allowed_token_ids is not None or self.bad_words_ids is not None or self.min_tokens > 0
                or self.dry)

    @property
    def dry(self) -> bool:
        """Whether the request needs ``tl_dry_penalty`` (DRY is on: ``dry_multiplier > 0``)."""
        return self.dry_multiplier > 0

    @property
    def xtc(self) -> bool:
        """Whether the draw runs XTC (``xtc_probability > 0``)."""
        return self.xtc_probability > 0

    @property
    def truncation(self) -> bool:
        """Whether the draw runs a truncation sampler: typical (``typical_p < 1``), top-n-sigma or Mirostat."""
        return self.typical_p < 1 or self.top_n_sigma > 0 or self.mirostat == 2

    @property
    def grammar(self) -> bool:
        """Whether the request carries a ``GrammarConstraint``."""
        from .grammar import GrammarConstraint

        return isinstance(self.constraint, GrammarConstraint)

    @property
    def penalized(self) -> bool:
        """Whether the request needs ``tl_sample_penalized``: a penalty, min-p, XTC or a truncation sampler is on."""
        return (self.repetition_penalty != 1 or self.presence_penalty != 0 or self.frequency_penalty != 0 or self.min_p > 0
                or self.xtc or self.truncation)


GREEDY = SamplingParams(0.0)


def sampling_per_request(sampling, n: int) -> list | None:
    """``sampling`` as given to the batcher (None, one ``SamplingParams`` or one per request) -> None or a list of
    ``n`` entries."""
    if sampling is None:
        return None
    if isinstance(sampling, SamplingParams):
        return [sampling] * n
    per = list(sampling)
    if len(per) != n or not all(isinstance(p, SamplingParams) for p in per):
        raise ValueError(f"sampling must be one SamplingParams or a list of {n} (one per prompt)")
    return per


def sampling_tensors(params, device) -> tuple[torch.Tensor, ...]:
    """The per-row device arrays of ``ext.sample`` (temperature, top_k, top_p, seed) for a list of ``SamplingParams``
    (None: greedy)."""
    params = [GREEDY if p is None else p for p in params]
    return (torch.tensor([float(p.temperature) for p in params], dtype=torch.float32, device=device),
            torch.tensor([min(p.top_k or 0, (1 << 31) - 1) for p in params], dtype=torch.int32, device=device),
            torch.tensor([0.0 if p.top_p is None else float(p.top_p) for p in params], dtype=torch.float32, device=device),
            torch.tensor([p.seed - (1 << 64) if p.seed >= 1 << 63 else p.seed for p in params], dtype=torch.int64, device=device))


def any_penalized(params) -> bool:
    return any(p is not None and p.penalized for p in params)


def any_controlled(params) -> bool:
    return any(p is not None and p.controls for p in params)


def any_dry(params) -> bool:
    return any(p is not None and p.dry for p in params)


def any_xtc(params) -> bool:
    return any(p is not None and p.xtc for p in params)


def any_truncation(params) -> bool:
    return any(p is not None and p.truncation for p in params)


def any_mirostat(params) -> bool:
    return any(p is not None and p.mirostat == 2 for p in params)


def any_constrained(params) -> bool:
    return any(p is not None and p.constraint is not None for p in params)


def penalty_tensors(params, device) -> tuple[torch.Tensor, ...]:
    """The per-row device arrays ``ext.sample_penalized`` adds to ``sampling_tensors``' (repetition, presence,
    frequency, min_p) for a list of ``SamplingParams`` (None: greedy, every penalty off)."""
    params = [GREEDY if p is None else p for p in params]
    return tuple(torch.tensor([float(getattr(p, name)) for p in params], dtype=torch.float32, device=device)
                 for name in ("repetition_penalty", "presence_penalty", "frequency_penalty", "min_p"))


def xtc_tensors(params, device) -> tuple[torch.Tensor, ...]:
    """The per-row XTC arrays (threshold, probability) ``ext.sample_penalized`` and ``ext.sample_constrained`` take
    beside ``penalty_tensors``' (None: greedy, XTC off)."""
    params = [GREEDY if p is None else p for p in params]
    return tuple(torch.tensor([float(getattr(p, name)) for p in params], dtype=torch.float32, device=device)
                 for name in ("xtc_threshold", "xtc_probability"))


def truncation_tensors(params, device) -> tuple[torch.Tensor, ...]:
    """The per-row truncation arrays (typical_p, top_n_sigma, mirostat_tau, mirostat_eta) ``ext.sample_penalized`` and
    ``ext.sample_constrained`` take beside ``penalty_tensors``' (None: greedy, all off).  ``mirostat_tau`` is 0 on the
    rows without Mirostat, which turns it off there."""
    params = [GREEDY if p is None else p for p in params]
    return (torch.tensor([p.typical_p for p in params], dtype=torch.float32, device=device),
            torch.tensor([p.top_n_sigma for p in params], dtype=torch.float32, device=device),
            torch.tensor([p.mirostat_tau if p.mirostat == 2 else 0.0 for p in params], dtype=torch.float32, device=device),
            torch.tensor([p.mirostat_eta if p.mirostat == 2 else 0.0 for p in params], dtype=torch.float32, device=device))


def mirostat_start(params) -> float:
    """The mu a Mirostat request starts from: ``2 * mirostat_tau``, in fp32."""
    return float(torch.tensor(2.0 * params.mirostat_tau, dtype=torch.float32))


STATE_PROMPT = 1 << 30  # token state: bit 30 marks a prompt token, bits 0-29 count the draws


def token_state_row(prompt_ids, generated_ids, vocab: int, out: torch.Tensor | None = None, device=None) -> torch.Tensor:
    """One request's int32 token state ``[vocab]`` (``tl_sample_penalized``): bit 30 set for the tokens of
    ``prompt_ids``, bits 0-29 the number of times each token occurs in ``generated_ids``.  Written into ``out`` (a row
    of a state slab) when given."""
    if out is None:
        out = torch.zeros(vocab, dtype=torch.int32, device=device)
    else:
        out.zero_()
    dev = out.device
    prompt = torch.as_tensor(list(prompt_ids) if not isinstance(prompt_ids, torch.Tensor) else prompt_ids, dtype=torch.int64).reshape(-1).to(dev)
    gen = torch.as_tensor(list(generated_ids) if not isinstance(generated_ids, torch.Tensor) else generated_ids, dtype=torch.int64).reshape(-1).to(dev)
    for ids in (prompt, gen):
        if ids.numel() and (int(ids.min()) < 0 or int(ids.max()) >= vocab):
            raise ValueError(f"token ids must be in [0, {vocab})")
    if prompt.numel():
        out.index_fill_(0, prompt, STATE_PROMPT)
    if gen.numel():
        out.index_add_(0, gen, torch.ones_like(gen, dtype=torch.int32))
    return out


def sample_tokens(logits: torch.Tensor, params, positions, state: torch.Tensor | None = None,
                  constraints: torch.Tensor | None = None, controls=None, tokens=None, mirostat_mu: torch.Tensor | None = None) -> torch.Tensor:
    """One seeded token per row of ``logits [rows, vocab]`` with the ``tl_sample`` kernel; ``params`` one
    ``SamplingParams`` (or None: greedy) per row, ``positions`` the index of each drawn token -> int32 ``[rows]``.
    When a row is penalised the launch is ``tl_sample_penalized`` over ``state`` (int32 ``[rows, vocab]``, required
    then), which it updates at the drawn tokens of the rows with position > 0.  When a row carries a constraint the
    launch is ``tl_sample_constrained`` over ``constraints`` (int64 ``[rows, 5]`` descriptor rows, required then: the
    constrained rows' ``TokenConstraint.descriptor``, zero rows elsewhere), whose states it advances likewise.
    ``constraints`` may also be a ``ConstraintRows`` (required for JSON, schema and grammar rows): those rows' masks are
    written before the draw and their states advanced after it.
    When a row carries logits controls, ``tl_logit_controls`` first turns every row into its fp32 controlled row
    (uncontrolled rows are copied exactly) over ``controls`` (a ``ControlRows`` of at least ``rows`` rows, required
    then), appending ``tokens`` (the step's input token per row) to its history tails, and the draw runs on those rows.
    When a row has DRY on, ``tl_dry_penalty`` then penalises those rows in place over ``controls.dry`` and appends
    ``tokens`` to its histories.  XTC rows pass the ``xtc_tensors`` to the penalised or constrained draw, and rows with
    a truncation sampler the ``truncation_tensors``; a Mirostat row needs ``mirostat_mu`` (float32 ``[rows]`` on the
    device, each Mirostat row's mu, updated in place for rows with position > 0).
    Rows of other requests may carry a constraint in the same launch: the constrained draw then runs on their exact
    fp32 copies, which draws the tokens it draws on the raw rows (a request never carries both)."""
    from extensions_b200 import tiny_llm_ext_b200 as ext

    temperature, top_k, top_p, seed = sampling_tensors(params, logits.device)
    pos = torch.as_tensor(positions, dtype=torch.int32).to(logits.device)
    if any_controlled(params):
        if controls is None or tokens is None:
            raise ValueError("a SamplingParams with logits controls needs the request's ControlRows and input tokens")
        n = len(params)
        tok = torch.as_tensor(tokens, dtype=torch.int32).reshape(-1).to(logits.device)
        logits = ext.logit_controls(logits.contiguous(), controls.descriptors[:n], pos, tok, controls.tails[:n])
        if any_dry(params):
            if controls.dry is None:
                raise ValueError("a SamplingParams with DRY needs its history in the ControlRows")
            ext.dry_penalty(logits, controls.dry.table[:n], pos, tok, controls.dry.history[:n], controls.dry.scratch[:n])
    xtc = {}
    if any_xtc(params):
        xtc = dict(zip(("xtc_threshold", "xtc_probability"), xtc_tensors(params, logits.device)))
    if any_truncation(params):
        names = ("typical_p", "top_n_sigma", "mirostat_tau", "mirostat_eta")
        xtc.update(zip(names, truncation_tensors(params, logits.device)))
        if any_mirostat(params):
            if mirostat_mu is None:
                raise ValueError("a Mirostat SamplingParams needs the request's mu (mirostat_mu)")
            xtc["mirostat_mu"] = mirostat_mu[: len(params)]
        else:
            del xtc["mirostat_tau"], xtc["mirostat_eta"]
    if any_constrained(params):
        if constraints is None:
            raise ValueError("a constrained SamplingParams needs the request's constraint descriptor")
        for p in params:
            if p is not None and p.constraint is not None and p.constraint.vocab_size != logits.shape[-1]:
                raise ValueError(f"the constraint's vocabulary has {p.constraint.vocab_size} ids, the logits {logits.shape[-1]}")
        pen = ()
        if any_penalized(params):
            if state is None:
                raise ValueError("a penalised SamplingParams needs the request's token state")
            pen = (*penalty_tensors(params, logits.device), state)
        from .json_mode import ConstraintRows, JsonConstraint
        from .json_schema import JsonSchemaConstraint

        if not isinstance(constraints, ConstraintRows):
            if any(p is not None and isinstance(p.constraint, JsonConstraint) for p in params):
                raise ValueError("a JSON-mode SamplingParams needs the request's ConstraintRows")
            if any(p is not None and isinstance(p.constraint, JsonSchemaConstraint) for p in params):
                raise ValueError("a JSON-schema SamplingParams needs the request's ConstraintRows")
            if any(p is not None and p.grammar for p in params):
                raise ValueError("a grammar SamplingParams needs the request's ConstraintRows")
            return ext.sample_constrained(logits.contiguous(), temperature, top_k, top_p, seed, pos, constraints, *pen, **xtc)
        constraints.before_draw(len(params))
        tokens = ext.sample_constrained(logits.contiguous(), temperature, top_k, top_p, seed, pos, constraints.descriptors[:len(params)], *pen,
                                        **xtc)
        constraints.after_draw(tokens, pos)
        return tokens
    if not any_penalized(params):
        return ext.sample(logits.contiguous(), temperature, top_k, top_p, seed, pos)
    if state is None:
        raise ValueError("a penalised SamplingParams needs the request's token state")
    return ext.sample_penalized(logits.contiguous(), temperature, top_k, top_p, seed, pos, *penalty_tensors(params, logits.device), state, **xtc)
