"""Reranking: Qwen3-Reranker relevance scores from packed prefill passes (DESIGN.md section 19).

Qwen3-Reranker is the plain Qwen3 causal LM.  For one query and N documents it runs N prompts that share a leading
part (system prompt, instruction, query) and differ in the rest (document and closing template); a document's score
is ``softmax([logit(false_id), logit(true_id)])[1]`` at its prompt's last position.

A pass of ``max_tokens`` rows holds, per query it serves, the query's shared prefix once as a segment of its own and
then as many of that query's documents as fit.  A prefix row attends its prefix causally; a document row attends the
prefix of its query in that pass and its own document causally (``paged_attention_prefixed_segments``), with RoPE
positions continuing after the prefix, so each document sees exactly the prompt it would see alone.  The LM head is
replaced by ``select_logits``: the final RMSNorm and the two logits of each document's last row.  The layer stack is
``embed.run_packed_pass``; as for embeddings, every segment starts on a ``SEGMENT_ALIGN``-row boundary and every pass
has the same row count, so a document's score does not depend on its siblings, its place in the pass, or the pass."""

from __future__ import annotations

import numpy as np
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext

from .embed import PASS_ALIGN, SEGMENT_ALIGN, _aligned, _check_model, run_packed_pass

# Qwen3-Reranker's prompt template (its model card): the system turn, then per pair the instruction, query and
# document in the user turn, and an empty thinking block before the yes / no answer.
RERANK_SYSTEM = ("<|im_start|>system\nJudge whether the Document meets the requirements based on the Query and the Instruct "
                 "provided. Note that the answer can only be \"yes\" or \"no\".<|im_end|>\n<|im_start|>user\n")
RERANK_SUFFIX = "<|im_end|>\n<|im_start|>assistant\n<think>\n\n</think>\n\n"
RERANK_DEFAULT_INSTRUCTION = "Given a web search query, retrieve relevant passages that answer the query"


def rerank_prompt(query: str, document: str, instruction: str | None = None) -> str:
    """The full Qwen3-Reranker prompt text of one (query, document) pair."""
    instruction = RERANK_DEFAULT_INSTRUCTION if instruction is None else instruction
    return f"{RERANK_SYSTEM}<Instruct>: {instruction}\n<Query>: {query}\n<Document>: {document}{RERANK_SUFFIX}"


def split_shared_prefix(sequences):
    """``(prefix, rests)`` of N >= 1 token-id prompts: ``prefix`` is their longest common leading run, shortened so
    that every rest keeps at least one token, and ``rests[i]`` is prompt i after it.  Working on ids (not text), each
    ``prefix + rests[i]`` is exactly prompt i as tokenised whole."""
    seqs = [[int(t) for t in s] for s in sequences]
    if not seqs:
        raise ValueError("split_shared_prefix needs at least one prompt")
    if any(not s for s in seqs):
        raise ValueError("split_shared_prefix: a prompt is empty")
    n = min(len(s) for s in seqs) - 1
    for k in range(n):
        t = seqs[0][k]
        if any(s[k] != t for s in seqs):
            n = k
            break
    return seqs[0][:n], [s[n:] for s in seqs]


def pack_groups(prefix_lengths, doc_lengths, max_tokens: int) -> list[list[tuple[int, int]]]:
    """Passes of (query, document) entries in row order; document -1 is the query's prefix.

    Queries and their documents are taken in input order.  A document goes to the first pass that holds its query's
    prefix and has room for its ``SEGMENT_ALIGN``-rounded length.  Otherwise the prefix is laid out again with it: the
    pair goes to the first pass with room for both (a new pass when none has).  An empty prefix takes no rows."""
    if max_tokens <= 0 or max_tokens % PASS_ALIGN != 0:
        raise ValueError(f"max_tokens must be a positive multiple of {PASS_ALIGN}, got {max_tokens}")
    if len(prefix_lengths) != len(doc_lengths):
        raise ValueError("one list of document lengths per query")
    passes, used = [], []
    for q, (P, docs) in enumerate(zip(prefix_lengths, doc_lengths)):
        mine = []  # passes holding this query's prefix
        for d, n in enumerate(docs):
            if n < 1:
                raise ValueError(f"query {q} document {d} is empty")
            need = _aligned(n)
            if _aligned(P) + need > max_tokens:
                raise ValueError(f"query {q} document {d}: a prefix of {P} tokens and a document of {n} tokens, each aligned to "
                                 f"{SEGMENT_ALIGN} rows, do not fit max_tokens={max_tokens}")
            for p in mine:
                if used[p] + need <= max_tokens:
                    passes[p].append((q, d))
                    used[p] += need
                    break
            else:
                entries = ([(q, -1)] if P > 0 else []) + [(q, d)]
                need += _aligned(P)
                for p, u in enumerate(used):
                    if u + need <= max_tokens:
                        break
                else:
                    p = len(passes)
                    passes.append([])
                    used.append(0)
                passes[p] += entries
                used[p] += need
                mine.append(p)
    return passes


def group_layout(entries, prefix_lengths, doc_lengths, max_tokens: int):
    """Per-row int32 arrays of one pass holding ``entries`` (``pack_groups``' form) in order: ``(offsets, ctxs,
    segment_start, prefix_start, prefix_end, score_rows, starts)``.

    A prefix row j has RoPE position j, an empty prefix range and its prefix as segment.  A document row j of a query
    with a P-token prefix has position P + j, the rows of its query's prefix in this pass as prefix range, and its
    document as segment.  Every such row has context row + 1 (row r appends its K/V at slot r).  Padding rows have
    context 0, position 0, an empty prefix and segment start ``max_tokens`` (no visible key).  ``score_rows``: the last
    row of each document entry, in entry order; ``starts``: each entry's first row."""
    offsets = np.zeros(max_tokens, dtype=np.int32)
    ctxs = np.zeros(max_tokens, dtype=np.int32)
    seg = np.full(max_tokens, max_tokens, dtype=np.int32)
    pst = np.zeros(max_tokens, dtype=np.int32)
    pen = np.zeros(max_tokens, dtype=np.int32)
    prefix_row, score_rows, starts, r = {}, [], [], 0
    for q, d in entries:
        P = prefix_lengths[q]
        n = P if d < 0 else doc_lengths[q][d]
        if r + n > max_tokens:
            raise ValueError(f"the entries need more than {max_tokens} rows")
        starts.append(r)
        ctxs[r:r + n] = np.arange(r + 1, r + n + 1, dtype=np.int32)
        seg[r:r + n] = r
        if d < 0:
            offsets[r:r + n] = np.arange(n, dtype=np.int32)
            prefix_row[q] = r
        else:
            offsets[r:r + n] = np.arange(P, P + n, dtype=np.int32)
            if P > 0:
                if q not in prefix_row:
                    raise ValueError(f"query {q}'s document {d} precedes its prefix in the pass")
                pst[r:r + n] = prefix_row[q]
                pen[r:r + n] = prefix_row[q] + P
            score_rows.append(r + n - 1)
        r += _aligned(n)
    return offsets, ctxs, seg, pst, pen, np.asarray(score_rows, dtype=np.int32), starts


def _lm_head(model):
    """The packed weight of the LM head: ``w_lm_head``, or the embedding when the head is tied."""
    return model.embedding.weight if model.w_lm_head is None else model.w_lm_head


def _run_pass(model, groups, entries, max_tokens, token_ids, device) -> torch.Tensor:
    """One packed pass: fp32 [documents of ``entries``, 2] log-probabilities over ``token_ids``, in entry order."""
    prefix_lengths = [len(p) for p, _ in groups]
    doc_lengths = [[len(d) for d in docs] for _, docs in groups]
    offsets, ctxs, seg, pst, pen, score_rows, starts = group_layout(entries, prefix_lengths, doc_lengths, max_tokens)
    tokens = np.zeros(max_tokens, dtype=np.int32)
    for (q, d), s in zip(entries, starts):
        ids = groups[q][0] if d < 0 else groups[q][1][d]
        tokens[s:s + len(ids)] = ids
    head_w = _lm_head(model)

    def attend(q, at, pool, table, views):
        return ext.paged_attention_prefixed_segments(q, pool._key_pages, pool._value_pages, table, views[0], views[1], views[2], at.scale,
                                                     at.num_kv_heads, at.num_heads)

    def head(x, views):
        _, logprobs = ext.select_logits(x, model.norm._weight_as(x.dtype, x.device), model.norm.eps, views[3], head_w.weight,
                                        head_w.scales, head_w.biases, views[4])
        return logprobs

    ids = np.asarray(token_ids, dtype=np.int32)
    return run_packed_pass(model, max_tokens, tokens, offsets, ctxs, [seg, pst, pen, score_rows, ids], attend, head, device)


def rerank_ids(model, queries, true_id: int, false_id: int, max_tokens: int = 8192, device=None) -> list[torch.Tensor]:
    """Relevance scores of token-id documents, per query and in input order.

    ``queries``: a list of ``(prefix_ids, [document_ids, ...])``, where ``prefix_ids + document_ids`` is the whole
    prompt of one pair (``split_shared_prefix`` makes this split from whole prompts).  Returns one fp32 tensor per
    query holding, per document, ``P(true_id)`` over ``{false_id, true_id}`` at the prompt's last position.  Documents
    are packed into passes of ``max_tokens`` rows (a multiple of 128), each borrowing ``ceil(max_tokens / page_size)``
    pages per layer from the model's pools and returning them, also on an error.  Qwen3-MoE models, models with
    adapters, empty documents, ids outside the vocabulary, ``true_id == false_id`` and a prefix plus document that
    do not fit one pass raise ``ValueError`` before any work."""
    device = torch.device(device) if device is not None else model.embedding.weight.scales.device
    _check_model(model, device, "rerank")
    V = model.vocab_size
    true_id, false_id = int(true_id), int(false_id)
    for name, t in (("true_id", true_id), ("false_id", false_id)):
        if not 0 <= t < V:
            raise ValueError(f"{name} {t} is outside [0, {V})")
    if true_id == false_id:
        raise ValueError("true_id and false_id must differ")
    groups = []
    for q, (prefix, docs) in enumerate(queries):
        prefix = [int(t) for t in prefix]
        docs = [[int(t) for t in d] for d in docs]
        if any(t < 0 or t >= V for t in prefix):
            raise ValueError(f"query {q}'s prefix holds a token id outside [0, {V})")
        for d, doc in enumerate(docs):
            if any(t < 0 or t >= V for t in doc):
                raise ValueError(f"query {q} document {d} holds a token id outside [0, {V})")
        groups.append((prefix, docs))
    passes = pack_groups([len(p) for p, _ in groups], [[len(d) for d in docs] for _, docs in groups], max_tokens)
    out = [torch.empty(len(docs), dtype=torch.float32, device=device) for _, docs in groups]
    for entries in passes:
        logprobs = _run_pass(model, groups, entries, max_tokens, (false_id, true_id), device)
        scores = logprobs[:, 1].exp()
        docs = [(q, d) for q, d in entries if d >= 0]
        for q in sorted({q for q, _ in docs}):
            sel = [i for i, (qq, _) in enumerate(docs) if qq == q]
            out[q][torch.tensor([docs[i][1] for i in sel], device=device)] = scores[torch.tensor(sel, device=device)]
    return out
