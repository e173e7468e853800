"""Logits controls (DESIGN.md section 22): ``SamplingParams.logit_bias``, ``allowed_token_ids``, ``bad_words_ids`` and
``min_tokens``, validated here and packed for ``tl_logit_controls``.

A controlled row is one ``tl_control_row`` descriptor (int64 ``[CONTROL_ROW_WORDS]``) pointing at the request's packed
int32 words: the biased ids and their fp32 bias bits, one ``1 + 16``-word record per banned sequence (its length, then
its ids), the EOS ids ``min_tokens`` holds back and, with an allow-list, the ``ceil(vocab / 32)``-word allow mask.
Beside it the request keeps a history tail: its 15 most recent tokens before the step's input token, oldest first,
-1 where the history is shorter.  Each launch appends the step's input token on the device, so decode never needs the
host to keep the tail."""

from __future__ import annotations

import math
import numbers

import numpy as np
import torch

MAX_BIAS = 1024  # TL_CONTROL_MAX_BIAS
BIAS_LIMIT = 100.0
MAX_BAD_WORDS = 64  # TL_CONTROL_MAX_BAD_WORDS
MAX_BAD_WORD_LEN = 16  # TL_CONTROL_MAX_BAD_WORD_LEN
BAD_WORD_WORDS = 1 + MAX_BAD_WORD_LEN
MAX_EOS = 8  # TL_CONTROL_MAX_EOS
TAIL = MAX_BAD_WORD_LEN - 1  # TL_CONTROL_TAIL
ROW_WORDS = 6  # int64 words of one tl_control_row
FLAG_ON = 1
FLAG_ALLOW = 2


def _token_id(name: str, v) -> int:
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or not 0 <= v < 1 << 31:
        raise ValueError(f"{name} token ids must be ints in [0, 2**31), got {v!r}")
    return int(v)


def normalized_controls(p) -> dict:
    """The control fields of ``SamplingParams`` ``p`` validated and normalised (``ValueError`` naming the field)."""
    out = {}
    bias = p.logit_bias
    if bias is not None:
        if isinstance(bias, dict):
            items = list(bias.items())
        else:
            try:
                items = [tuple(e) for e in bias]
            except TypeError:
                raise ValueError(f"logit_bias must be a mapping token id -> bias, got {type(bias).__name__}") from None
            if any(len(e) != 2 for e in items):
                raise ValueError("logit_bias must be a mapping token id -> bias")
            if len({e[0] for e in items}) != len(items):
                raise ValueError("logit_bias lists a token id twice")
        if len(items) > MAX_BIAS:
            raise ValueError(f"logit_bias holds at most {MAX_BIAS} entries, got {len(items)}")
        norm = []
        for t, b in items:
            t = _token_id("logit_bias", t)
            if isinstance(b, bool) or not isinstance(b, numbers.Real) or not math.isfinite(b) or not -BIAS_LIMIT <= b <= BIAS_LIMIT:
                raise ValueError(f"logit_bias values must be finite numbers in [-100, 100], got {b!r} for token {t}")
            norm.append((t, float(b)))
        out["logit_bias"] = tuple(sorted(norm))
    allowed = p.allowed_token_ids
    if allowed is not None:
        if isinstance(allowed, (str, bytes)) or not hasattr(allowed, "__iter__"):
            raise ValueError(f"allowed_token_ids must be a collection of token ids, got {type(allowed).__name__}")
        ids = tuple(sorted({_token_id("allowed_token_ids", t) for t in allowed}))
        if not ids:
            raise ValueError("allowed_token_ids must hold at least one token id")
        out["allowed_token_ids"] = ids
    bad = p.bad_words_ids
    if bad is not None:
        if isinstance(bad, (str, bytes)) or not hasattr(bad, "__iter__"):
            raise ValueError(f"bad_words_ids must be a list of token id sequences, got {type(bad).__name__}")
        seqs = []
        for seq in bad:
            if isinstance(seq, (str, bytes)) or not hasattr(seq, "__iter__"):
                raise ValueError(f"bad_words_ids must be a list of token id sequences, got an entry {seq!r}")
            seq = tuple(_token_id("bad_words_ids", t) for t in seq)
            if not 1 <= len(seq) <= MAX_BAD_WORD_LEN:
                raise ValueError(f"bad_words_ids sequences must hold 1 to {MAX_BAD_WORD_LEN} ids, got {len(seq)}")
            seqs.append(seq)
        if len(seqs) > MAX_BAD_WORDS:
            raise ValueError(f"bad_words_ids holds at most {MAX_BAD_WORDS} sequences, got {len(seqs)}")
        out["bad_words_ids"] = tuple(seqs)
    m = p.min_tokens
    if isinstance(m, bool) or not isinstance(m, numbers.Integral) or not 0 <= m < 1 << 31:
        raise ValueError(f"min_tokens must be an int >= 0, got {m!r}")
    out["min_tokens"] = int(m)
    return out


def check_vocab(p, vocab: int) -> None:
    """Every id of ``p``'s controls lies in [0, vocab) (``ValueError`` naming the field)."""
    for name, ids in (("logit_bias", [t for t, _ in p.logit_bias or ()]), ("allowed_token_ids", p.allowed_token_ids or ()),
                      ("bad_words_ids", [t for s in p.bad_words_ids or () for t in s])):
        bad = [t for t in ids if t >= vocab]
        if bad:
            raise ValueError(f"{name} token id {bad[0]} is outside the vocabulary [0, {vocab})")


def pack_row(p, vocab: int, eos_ids=(), prompt_len: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """``(header, data)`` of one request: the descriptor's ten int32 fields after the data pointer (flags, prompt_len,
    min_tokens, num_bias, bias_off, num_bad, bad_off, num_eos, eos_off, allow_off) and the packed int32 words.  An
    uncontrolled ``p`` (or None) packs to a zero header and no words."""
    header = np.zeros(10, dtype=np.int32)
    if p is None or not p.controls:
        return header, np.zeros(0, dtype=np.int32)
    check_vocab(p, vocab)
    eos = [int(t) for t in eos_ids] if p.min_tokens > 0 else []
    if p.min_tokens > 0 and not eos:
        raise ValueError("min_tokens needs the loop's EOS token id: this loop knows none")
    if len(eos) > MAX_EOS:
        raise ValueError(f"min_tokens holds back at most {MAX_EOS} EOS ids")
    bias = p.logit_bias or ()
    bias_words = np.concatenate([np.array([t for t, _ in bias], dtype=np.int32),
                                 np.array([b for _, b in bias], dtype=np.float32).view(np.int32)])
    bad = np.zeros((len(p.bad_words_ids or ()), BAD_WORD_WORDS), dtype=np.int32)
    for s, seq in enumerate(p.bad_words_ids or ()):
        bad[s, 0] = len(seq)
        bad[s, 1 : 1 + len(seq)] = seq
    allow = np.zeros(0, dtype=np.int32)
    flags = FLAG_ON
    if p.allowed_token_ids is not None:
        words = np.zeros((vocab + 31) // 32, dtype=np.uint32)
        ids = np.array(p.allowed_token_ids, dtype=np.int64)
        np.bitwise_or.at(words, ids >> 5, (np.uint32(1) << (ids & 31).astype(np.uint32)))
        allow = words.view(np.int32)
        flags |= FLAG_ALLOW
    parts = [bias_words, bad.reshape(-1), np.array(eos, dtype=np.int32), allow]
    offs = np.cumsum([0] + [len(a) for a in parts])
    header[:] = (flags, prompt_len, p.min_tokens, len(bias), offs[0], len(bad), offs[1], len(eos), offs[2], offs[3])
    return header, np.concatenate(parts).astype(np.int32)


def history_tail(prompt_ids, generated_ids) -> tuple[np.ndarray, int]:
    """``(tail, input_token)`` of a request about to draw its next token: the input token is the last of
    ``prompt_ids + generated_ids`` (the step appends it on the device), the tail the 15 before it, -1 padded in front."""
    hist = [int(t) for t in prompt_ids] + [int(t) for t in generated_ids]
    if not hist:
        raise ValueError("a controlled request needs at least one prompt token")
    tail = np.full(TAIL, -1, dtype=np.int32)
    before = hist[:-1][-TAIL:]
    if before:
        tail[TAIL - len(before) :] = before
    return tail, hist[-1]


def unpack_row(header, data, vocab: int) -> dict:
    """The controls a packed row carries (the inverse of ``pack_row``, for checks)."""
    flags, prompt_len, min_tokens, nb, bo, nbad, bado, ne, eo, ao = (int(v) for v in header)
    data = np.asarray(data, dtype=np.int32)
    bias = tuple(zip(data[bo : bo + nb].tolist(), data[bo + nb : bo + 2 * nb].view(np.float32).tolist()))
    bad = tuple(tuple(data[bado + BAD_WORD_WORDS * s + 1 : bado + BAD_WORD_WORDS * s + 1 + data[bado + BAD_WORD_WORDS * s]].tolist())
                for s in range(nbad))
    allowed = None
    if flags & FLAG_ALLOW:
        words = data[ao : ao + (vocab + 31) // 32].view(np.uint32)
        allowed = tuple(t for t in range(vocab) if (words[t >> 5] >> (t & 31)) & 1)
    return dict(flags=flags, prompt_len=prompt_len, min_tokens=min_tokens, logit_bias=bias or None, bad_words_ids=bad or None,
                eos_ids=tuple(data[eo : eo + ne].tolist()), allowed_token_ids=allowed)


class ControlRows:
    """The ``tl_logit_controls`` table of ``rows`` rows on ``device``: ``descriptors`` (int64 ``[rows, ROW_WORDS]``,
    zero rows uncontrolled) and ``tails`` (int32 ``[rows, TAIL]``), plus each controlled row's packed words, which the
    table keeps alive while its descriptor points at them.  ``dry`` is the ``tl_dry_penalty`` table beside it
    (``dry.DryRows`` of ``history_capacity`` ids per row), allocated when the first DRY row is written."""

    def __init__(self, rows: int, vocab: int, device, history_capacity: int | None = None):
        self.rows, self.vocab, self.device = rows, vocab, torch.device(device)
        self.descriptors = torch.zeros((rows, ROW_WORDS), dtype=torch.int64, device=self.device)
        self.tails = torch.full((rows, TAIL), -1, dtype=torch.int32, device=self.device)
        self._data: list = [None] * rows
        self.history_capacity = history_capacity
        self.dry = None

    def _set_dry(self, r: int, p, history_ids) -> None:
        from .dry import DryRows

        if p is not None and p.dry and self.dry is None:
            if not self.history_capacity:
                raise ValueError("a DRY request needs a history capacity: this loop allocated none")
            self.dry = DryRows(self.rows, self.history_capacity, self.device)
        if self.dry is not None:
            self.dry.set_row(r, p, history_ids)

    def set_row(self, r: int, p, prompt_ids, generated_ids=(), eos_ids=()) -> int:
        """Write request ``p``'s row ``r`` from its history; returns the step's input token (the last history id).  An
        uncontrolled ``p`` clears the row."""
        tail, last = history_tail(prompt_ids, generated_ids)
        header, words = pack_row(p, self.vocab, eos_ids, len(prompt_ids))
        self._set_dry(r, p, [*prompt_ids, *generated_ids])
        if not header[0]:
            self.clear_row(r)
            return last
        data = torch.from_numpy(words).to(self.device) if words.size else torch.zeros(1, dtype=torch.int32, device=self.device)
        desc = np.zeros(2 * ROW_WORDS, dtype=np.int32)
        desc[2:] = header
        desc = desc.view(np.int64)
        desc[0] = data.data_ptr() if self.device.type == "cuda" else 0
        self.descriptors[r].copy_(torch.from_numpy(desc))
        self.tails[r].copy_(torch.from_numpy(tail))
        self._data[r] = data
        return last

    def clear_row(self, r: int) -> None:
        self.descriptors[r].zero_()
        self.tails[r].fill_(-1)
        self._data[r] = None
        if self.dry is not None:
            self.dry.clear_row(r)

    def row_data(self, r: int):
        return self._data[r]


def control_rows(params, vocab: int, device, eos_ids=(), histories=None, history_capacity=None) -> tuple[ControlRows, list[int]]:
    """One ``ControlRows`` row per entry of ``params`` (``SamplingParams`` or None), each from its history
    ``(prompt_ids, generated_ids)`` in ``histories`` -> ``(rows, input tokens)``: the launch's ``tokens`` argument for
    the row's next draw (the last history id of each row; 0 for rows without a history).  DRY rows need
    ``history_capacity``."""
    table = ControlRows(len(params), vocab, device, history_capacity)
    if histories is None:
        histories = [None] * len(params)
    if len(histories) != len(params):
        raise ValueError(f"histories must hold one (prompt_ids, generated_ids) or None per row ({len(params)})")
    inputs = []
    for r, (p, h) in enumerate(zip(params, histories)):
        if p is not None and p.controls and h is None:
            raise ValueError("a controlled row needs its (prompt_ids, generated_ids) history")
        inputs.append(0 if h is None else table.set_row(r, p, h[0], h[1], eos_ids))
    return table, inputs
