"""Command-line front doors: the equivalents of the reference's ``main.py`` (one prompt,
``main.py:1-190``) and ``batch-main.py`` (continuous batching,
``batch-main.py:1-102``) over a checkpoint DIRECTORY (MLX 4-bit safetensors layout,
see checkpoint.py; there is no hub download here).

    python -m tiny_llm_b200.cli generate --model /path/to/Qwen3-4B-MLX-4bit --prompt "..." [--loader week3]
    python -m tiny_llm_b200.cli batch    --model /path/to/ckpt --prompts-file prompts.txt --batch-size 5
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --max-new-tokens 8   (no files needed)
    python -m tiny_llm_b200.cli generate --model /path/to/Qwen3-30B-A3B-MLX-4bit --prompt "..."   (Qwen3-MoE; --synthetic tiny-moe-d128 without files)
    python -m tiny_llm_b200.cli batch    --synthetic tiny-d128 --prompt-ids "5,17,3;9,2,4" --sampler-temp 0.7 --sampler-top-p 0.9 --seed 3
        (seeded sampling with the tl_sample kernel: the same seed gives the same tokens)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --sampler-temp 0.7 --presence-penalty 1.5 --min-p 0.05
        (token-history penalties and min-p; with --sampler-temp 0 the greedy token of the penalised logits)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --logit-bias 42:5 --bad-words "7,8;9"
        (logits controls: a per-token bias, banned sequences; also --allowed-token-ids and --min-tokens)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --sampler-temp 0.8 --dry-multiplier 0.8 --xtc-probability 0.5
        (DRY penalises tokens that extend a verbatim repeat; XTC drops the most likely choices with a seeded probability)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --sampler-temp 0.8 --typical-p 0.9 --top-n-sigma 1.5
        (locally typical sampling and top-n-sigma; --mirostat 2 --mirostat-tau 5 --mirostat-eta 0.1 for Mirostat 2.0)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --draft-synthetic tiny-d128 --proposal-length 4 --prompt-ids 5,17,3
        (speculative decoding: same ids as greedy; acceptance stats on stderr)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --draft-synthetic tiny-d128 --proposal-length 4 --prompt-ids 5,17,3 --sampler-temp 0.7 --sampler-top-p 0.9 --seed 3
        (speculative sampling: the same ids as the seeded sampled run without the draft)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-lookup 4 --prompt-lookup-ngram 2:3 --prompt-ids 5,17,3,9,5,17
        (prompt-lookup speculative decoding: proposals from the request's own tokens, same ids as greedy)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --num-beams 4 --num-return-sequences 2
        (beam search: the returned hypotheses with their scores, best first)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --logprobs 5
        (each generated token's log-probability, rank and 5 most likely alternatives, after the text)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --num-samples 4 --sampler-temp 0.8 --seed 3
        (parallel sampling: 4 seeded samples from one prefill, sample j uses seed + j)
    python -m tiny_llm_b200.cli score    --model /path/to/ckpt --prompt "The capital of France is Paris." [--logprobs 3]
        (teacher-forced log-probability of every prompt token and the prompt's perplexity)
    python -m tiny_llm_b200.cli batch    --synthetic tiny-d128 --prompt-ids "5,17,3,8;5,17,3,9" --prefix-cache
        (requests share the KV pages of a common prompt prefix; reused tokens per request and cache stats after the text)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --regex "[0-9]{4}-[0-9]{2}-[0-9]{2}"
        (every generated token keeps the text inside the pattern's language; EOS ends it once it is a match)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --json
        (the generated text is one JSON object: every prefix can still complete, EOS only once it has closed)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 \
        --json-schema '{"type": "object", "properties": {"name": {"type": "string"}}, "required": ["name"]}'
        (one JSON object that validates against the schema, keys in the schema's order; FILE_OR_INLINE_JSON)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --grammar 'root ::= [0-9]+ ("+" [0-9]+)*'
        (the generated text stays in the language of a GBNF grammar; FILE_OR_INLINE grammar text)
    python -m tiny_llm_b200.cli batch --synthetic tiny-d128 --synthetic-lora a=16 --synthetic-lora b=8:1 \
        --prompt-ids "5,17,3;5,17,3;5,17,3" --adapters "a;;b"
        (one resident base model, each request under the LoRA adapter it names: --lora NAME=DIR loads a PEFT directory)
    python -m tiny_llm_b200.cli embed --synthetic tiny-d128 --prompt-ids "5,17,3;9,2,4,8" --dimensions 64 [--pooling mean] [--out e.npy]
        (one pooled, L2-normalised embedding per prompt from packed prefill passes; --append-eos for Qwen3-Embedding)
    python -m tiny_llm_b200.cli rerank --synthetic tiny-d128 --prefix-ids "5,17,3" --document-ids "9,2;4,8,1" --true-id 10 --false-id 11
        (one Qwen3-Reranker relevance score per document; with --model: --query, --document / --documents-file, --instruction)
"""

from __future__ import annotations

import argparse
import json
import sys
from pathlib import Path

import torch


TOKENIZER_FILES = ("tokenizer.json", "tokenizer_config.json", "vocab.json", "tokenizer.model")


def _load(args, device):
    from .checkpoint import load_checkpoint, load_tokenizer
    from .synthetic import synthetic_qwen3

    if args.synthetic:
        extra = {} if args.rope_scaling is None else {"rope_scaling": args.rope_scaling}
        return (synthetic_qwen3(args.synthetic, seed=0, device=device, realistic=args.synthetic.startswith("tiny"), bits=args.synthetic_bits,
                                **extra), None,
                "Qwen/Qwen3-synthetic")
    ns = load_checkpoint(args.model, device=device)
    tokenizer = None
    if not any((Path(args.model) / f).exists() for f in TOKENIZER_FILES):
        # transformers would build an empty-vocabulary tokenizer from config.json alone and print every token as ""
        print(f"(no tokenizer files in {args.model}: token ids are printed)", file=sys.stderr)
        return ns, None, "Qwen/Qwen3-" + str(args.model)
    try:
        tokenizer = load_tokenizer(args.model)
    except Exception as exc:  # token-id mode still works without tokenizer files
        print(f"(no tokenizer loaded from {args.model}: {exc})", file=sys.stderr)
    return ns, tokenizer, "Qwen/Qwen3-" + str(args.model)


def _model(args, ns, name):
    from .models import dispatch_model

    if args.loader == "week2":
        if args.max_context is not None:
            raise SystemExit("--max-context needs the paged week3 model")
        return dispatch_model(name, ns, week=2)
    return dispatch_model(name, ns, week=3, enable_paged_attention=not args.disable_paged_attention, max_context=args.max_context)


def _rope_scaling_arg(spec: str) -> dict:
    from .rope_scaling import parse_cli

    try:
        return parse_cli(spec)
    except ValueError as exc:
        raise argparse.ArgumentTypeError(str(exc)) from None


def _positive_int(text: str) -> int:
    try:
        value = int(text)
    except ValueError:
        value = 0
    if value <= 0:
        raise argparse.ArgumentTypeError(f"expected a positive integer (got {text!r})")
    return value


def parse_lora_specs(lora, synthetic_lora):
    """``--lora NAME=DIR`` and ``--synthetic-lora NAME=RANK[:SEED]`` as ``[(name, directory)]`` and ``[(name, rank, seed)]``."""
    loaded, made = [], []
    for spec in lora or []:
        name, sep, path = spec.partition("=")
        if not sep or not name or not path:
            raise SystemExit(f"--lora expects NAME=DIR, got {spec!r}")
        loaded.append((name, path))
    for spec in synthetic_lora or []:
        name, sep, rest = spec.partition("=")
        rank, _, seed = rest.partition(":")
        if not sep or not name or not rank.isdigit() or (seed and not seed.isdigit()):
            raise SystemExit(f"--synthetic-lora expects NAME=RANK[:SEED], got {spec!r}")
        made.append((name, int(rank), int(seed) if seed else 0))
    return loaded, made


def _load_adapters(args, model, ns) -> None:
    """Give ``model`` the adapters the flags name (nothing without them)."""
    from .lora import LoraAdapter

    loaded, made = parse_lora_specs(args.lora, args.synthetic_lora)
    if not loaded and not made:
        return
    if not hasattr(model, "load_adapters"):
        raise SystemExit("--lora / --synthetic-lora need the week3 model")
    try:
        adapters = [LoraAdapter.load(path, name) for name, path in loaded]
        adapters += [LoraAdapter.synthetic(ns.args, rank, seed=seed, name=name) for name, rank, seed in made]
        loaded_set = model.load_adapters(adapters)
    except (ValueError, OSError) as exc:
        raise SystemExit(f"adapters: {exc}")
    if getattr(args, "adapter", None) is not None and args.adapter not in loaded_set.names:
        raise SystemExit(f"--adapter {args.adapter!r} is not among the loaded adapters {loaded_set.names}")


def _prompt_ids(args, tokenizer, prompt: str | None):
    if args.prompt_ids:
        return [int(t) for t in args.prompt_ids.split(",")]
    if tokenizer is None:
        raise SystemExit("a text prompt needs the checkpoint's tokenizer files; use --prompt-ids")
    messages = [{"role": "system", "content": "You are a helpful assistant."}, {"role": "user", "content": prompt}]
    text = tokenizer.apply_chat_template(messages, tokenize=False, add_generation_prompt=True, enable_thinking=args.enable_thinking)
    return tokenizer.encode(text, add_special_tokens=False)


def _token_text(tokenizer, token: int) -> str:
    if tokenizer is None:
        return str(token)
    return repr(tokenizer.decode([token]))


def _print_logprobs(entries, tokenizer, file=None) -> None:
    """One line per entry: the token, its log-probability and rank, then its alternatives."""
    for e in entries:
        alts = ", ".join(f"{_token_text(tokenizer, i)} {v:.4f}" for i, v in e.top)
        print(f"  {_token_text(tokenizer, e.token)}\tlogprob {e.logprob:.4f}\trank {e.rank}" + (f"\t| {alts}" if alts else ""), file=file)


def _penalties(args) -> dict:
    """The ``SamplingParams`` penalty and truncation fields the flags turn on (an empty dict when every one is off)."""
    given = dict(repetition_penalty=args.repetition_penalty, presence_penalty=args.presence_penalty,
                 frequency_penalty=args.frequency_penalty, min_p=args.min_p)
    off = dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_p=0.0)
    return {**{k: v for k, v in given.items() if v != off[k]}, **_truncation(args)}


def _truncation(args) -> dict:
    """The ``SamplingParams`` truncation fields of ``--typical-p``, ``--top-n-sigma`` and ``--mirostat*`` (an empty
    dict when every sampler is off; tau and eta only with ``--mirostat 2``)."""
    out = {}
    if args.typical_p != 1.0:
        out["typical_p"] = args.typical_p
    if args.top_n_sigma != 0.0:
        out["top_n_sigma"] = args.top_n_sigma
    if args.mirostat:
        out.update(mirostat=args.mirostat, mirostat_tau=args.mirostat_tau, mirostat_eta=args.mirostat_eta)
    return out


def _truncation_flags(args) -> list:
    """The truncation flags given, by name."""
    return [f for f, on in (("--typical-p", args.typical_p != 1.0), ("--top-n-sigma", args.top_n_sigma != 0.0),
                            ("--mirostat", args.mirostat != 0)) if on]


def parse_controls(logit_bias=None, allowed_token_ids=None, bad_words=None, min_tokens=0) -> dict:
    """The ``SamplingParams`` logits-control fields of the flags' strings (an empty dict when every one is off):
    ``--logit-bias "ID:B,ID:B"``, ``--allowed-token-ids "ID,ID"``, ``--bad-words "ID,ID;ID"`` (sequences split by
    ``;``) and ``--min-tokens N``.  Malformed strings raise ``ValueError``."""
    out = {}
    try:
        if logit_bias:
            pairs = [e.split(":") for e in logit_bias.split(",") if e.strip()]
            if any(len(e) != 2 for e in pairs):
                raise ValueError
            bias = {}
            for t, b in pairs:
                if int(t) in bias:
                    raise ValueError(f"--logit-bias lists token {int(t)} twice")
                bias[int(t)] = float(b)
            out["logit_bias"] = bias
        if allowed_token_ids:
            out["allowed_token_ids"] = [int(t) for t in allowed_token_ids.split(",") if t.strip()]
        if bad_words:
            out["bad_words_ids"] = [[int(t) for t in seq.split(",") if t.strip()] for seq in bad_words.split(";") if seq.strip()]
    except ValueError as exc:
        raise ValueError(str(exc) or "expected --logit-bias ID:B,ID:B, --allowed-token-ids ID,ID and --bad-words ID,ID;ID") from None
    if min_tokens:
        out["min_tokens"] = min_tokens
    return out


def parse_dry_xtc(dry_multiplier=0.0, dry_base=1.75, dry_allowed_length=2, dry_penalty_last_n=0, dry_sequence_breakers=None,
                  xtc_threshold=0.1, xtc_probability=0.0, tokenizer=None) -> dict:
    """The ``SamplingParams`` DRY and XTC fields of the flags (an empty dict when both samplers are off).
    ``--dry-sequence-breakers`` is either ids (``"13,198"``) or a JSON list of strings (``'["\\n", ":"]'``); a string
    becomes the last id of the tokenizer's encoding of ``"a" + s`` (text-generation-webui's rule), so it needs a
    tokenizer.  Malformed values raise ``ValueError``."""
    out = {}
    if dry_multiplier:
        out.update(dry_multiplier=dry_multiplier, dry_base=dry_base, dry_allowed_length=dry_allowed_length,
                   dry_penalty_last_n=dry_penalty_last_n)
        if dry_sequence_breakers:
            text = dry_sequence_breakers.strip()
            if text.startswith("["):
                try:
                    strings = json.loads(text)
                except json.JSONDecodeError:
                    raise ValueError("--dry-sequence-breakers must be ids ID,ID or a JSON list of strings") from None
                if not isinstance(strings, list) or not all(isinstance(s, str) and s for s in strings):
                    raise ValueError("--dry-sequence-breakers must be ids ID,ID or a JSON list of strings")
                if strings and tokenizer is None:
                    raise ValueError("--dry-sequence-breakers strings need a tokenizer: give ids with --synthetic")
                ids = []
                for s in strings:
                    enc = tokenizer.encode("a" + s, add_special_tokens=False)
                    if enc:
                        ids.append(int(enc[-1]))
                out["dry_sequence_breakers"] = ids
            else:
                try:
                    out["dry_sequence_breakers"] = [int(t) for t in text.split(",") if t.strip()]
                except ValueError:
                    raise ValueError("--dry-sequence-breakers must be ids ID,ID or a JSON list of strings") from None
    if xtc_probability:
        out.update(xtc_probability=xtc_probability, xtc_threshold=xtc_threshold)
    return out


def _dry_xtc(args, tokenizer) -> dict:
    """The DRY and XTC fields of ``--dry-*`` and ``--xtc-*``."""
    try:
        return parse_dry_xtc(args.dry_multiplier, args.dry_base, args.dry_allowed_length, args.dry_penalty_last_n,
                             args.dry_sequence_breakers, args.xtc_threshold, args.xtc_probability, tokenizer)
    except ValueError as exc:
        raise SystemExit(str(exc)) from None


def _controls(args) -> dict:
    """The logits-control fields of ``--logit-bias``, ``--allowed-token-ids``, ``--bad-words`` and ``--min-tokens``."""
    try:
        return parse_controls(args.logit_bias, args.allowed_token_ids, args.bad_words, args.min_tokens)
    except ValueError as exc:
        raise SystemExit(str(exc)) from None


def _constraint(args, model, tokenizer, device):
    """The ``TokenConstraint`` of ``--regex``, the ``JsonConstraint`` of ``--json``, the ``JsonSchemaConstraint`` of
    ``--json-schema`` or the ``GrammarConstraint`` of ``--grammar`` over the checkpoint tokenizer's vocabulary (the
    synthetic vocabulary with ``--synthetic``), or None."""
    grammar_text = getattr(args, "grammar", None)
    if grammar_text is not None and (args.regex is not None or args.json or args.json_schema is not None):
        raise SystemExit("--grammar takes no --regex, --json or --json-schema: give one constraint")
    if grammar_text is not None:
        return _grammar_constraint(args, grammar_text, model, tokenizer, device)
    schema_text = args.json_schema
    given = [f for f, on in (("--regex", args.regex is not None), ("--json", args.json), ("--json-schema", schema_text is not None)) if on]
    if args.regex is not None and args.json:
        raise SystemExit("give --regex or --json, not both")
    if len(given) > 1:
        raise SystemExit(f"give one of {', '.join(given)}, not several")
    if not given:
        return None
    from .constrained import TokenConstraint, TokenVocabulary
    from .json_mode import JsonConstraint
    from .json_schema import JsonSchemaConstraint, load_schema_arg

    flag = given[0]
    schema = None
    if schema_text is not None:
        try:
            schema = load_schema_arg(schema_text)
        except (OSError, ValueError) as exc:
            raise SystemExit(f"--json-schema: not a JSON schema file or inline JSON object: {exc}")
    if device.type != "cuda":
        raise SystemExit(f"{flag} runs on the CUDA sampling kernel: use a cuda --device")
    if args.synthetic:
        vocabulary = TokenVocabulary.synthetic(model.vocab_size)
    elif tokenizer is None:
        raise SystemExit(f"{flag} needs the checkpoint's tokenizer files (or --synthetic)")
    else:
        vocabulary = TokenVocabulary.from_tokenizer(tokenizer, model.vocab_size)
    try:
        if args.json:
            return JsonConstraint(vocabulary, device=device)
        if schema is not None:
            return JsonSchemaConstraint(schema, vocabulary, device=device)
        return TokenConstraint.compile(args.regex, vocabulary, device=device)
    except ValueError as exc:
        raise SystemExit(f"{flag}: {exc}")


def _grammar_constraint(args, text: str, model, tokenizer, device):
    from .constrained import TokenVocabulary
    from .grammar import GrammarConstraint, load_grammar_arg

    try:
        grammar = load_grammar_arg(text)
    except (OSError, UnicodeDecodeError) as exc:
        raise SystemExit(f"--grammar: not a grammar file or inline GBNF grammar: {exc}")
    if device.type != "cuda":
        raise SystemExit("--grammar runs on the CUDA sampling kernel: use a cuda --device")
    if args.synthetic:
        vocabulary = TokenVocabulary.synthetic(model.vocab_size)
    elif tokenizer is None:
        raise SystemExit("--grammar needs the checkpoint's tokenizer files (or --synthetic)")
    else:
        vocabulary = TokenVocabulary.from_tokenizer(tokenizer, model.vocab_size)
    try:
        return GrammarConstraint(grammar, vocabulary, device=device)
    except ValueError as exc:
        raise SystemExit(f"--grammar: {exc}")


def _adapter_kw(args, key: str) -> dict:
    """``{key: name}`` for ``--adapter NAME`` (nothing without it, so models that take no adapters run as before)."""
    return {} if args.adapter is None else {key: args.adapter}


def cmd_generate(args) -> int:
    from .generate import greedy_generate_ids
    from .sampler import SamplingParams, make_sampler

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    _load_adapters(args, model, ns)
    ids = _prompt_ids(args, tokenizer, args.prompt)
    sampler = sampling = None
    penalties = _penalties(args)
    controls = _controls(args)
    dry_xtc = _dry_xtc(args, tokenizer)
    if dry_xtc and (args.num_beams is not None or args.num_samples is not None):
        raise SystemExit("beam search and parallel sampling take no --dry-multiplier or --xtc-probability")
    if controls and (args.num_beams is not None or args.num_samples is not None):
        raise SystemExit("beam search and parallel sampling take no --logit-bias, --allowed-token-ids, --bad-words or --min-tokens")
    if args.num_beams is not None:
        if args.num_samples is not None:
            raise SystemExit("give --num-beams or --num-samples, not both")
        return _beam_search(args, model, tokenizer, ids, penalties, device)
    if args.num_samples is not None:
        return _parallel_sample(args, model, tokenizer, ids, penalties, device)
    drafted = bool(args.draft_model or args.draft_synthetic)
    speculative = drafted or args.prompt_lookup is not None
    if drafted and args.prompt_lookup is not None:
        raise SystemExit("give one proposer: a draft (--draft-model / --draft-synthetic) or --prompt-lookup, not both")
    if speculative and args.regex is not None:
        raise SystemExit("speculative decoding is greedy and unconstrained: drop --regex")
    if speculative and args.json:
        raise SystemExit("speculative decoding is greedy and unconstrained: drop --json")
    if speculative and args.json_schema is not None:
        raise SystemExit("speculative decoding is greedy and unconstrained: drop --json-schema")
    if speculative and args.grammar is not None:
        raise SystemExit("speculative decoding and prompt lookup are greedy and unconstrained: drop --grammar")
    if speculative and dry_xtc:
        raise SystemExit("speculative decoding and prompt lookup take no --dry-multiplier or --xtc-probability")
    if speculative and _truncation_flags(args):
        raise SystemExit(f"speculative decoding and prompt lookup take no {_truncation_flags(args)[0]}: drop it or the proposer")
    if speculative and controls:
        raise SystemExit("speculative decoding takes no --logit-bias, --allowed-token-ids, --bad-words or --min-tokens")
    if controls and args.grammar is not None:
        raise SystemExit("--logit-bias, --allowed-token-ids, --bad-words and --min-tokens take no --grammar")
    constraint = _constraint(args, model, tokenizer, device)
    if constraint is not None:
        if controls:
            raise SystemExit("--logit-bias, --allowed-token-ids, --bad-words and --min-tokens take no --regex, --json or --json-schema")
        penalties["constraint"] = constraint
    penalties.update(controls)
    penalties.update(dry_xtc)
    if args.sampler_temp != 0 or penalties:
        if device.type == "cuda" or penalties or speculative:  # the seeded kernel
            try:
                sampling = SamplingParams(args.sampler_temp, top_k=args.sampler_top_k, top_p=args.sampler_top_p, seed=args.seed, **penalties)
            except ValueError as exc:
                raise SystemExit(str(exc)) from None
        else:
            sampler = make_sampler(args.sampler_temp, top_p=args.sampler_top_p, top_k=args.sampler_top_k)
    if tokenizer is not None:
        tokenizer.detokenizer.reset()

    def emit(token: int) -> None:
        if tokenizer is None:
            print(token, end=" ", flush=True)
        else:
            tokenizer.detokenizer.add_token(token)
            print(tokenizer.detokenizer.last_segment, end="", flush=True)

    eos = getattr(tokenizer, "eos_token_id", None)
    if constraint is not None and args.synthetic:
        eos = constraint.vocabulary.eos_ids[0]
    if controls.get("min_tokens") and eos is None:
        raise SystemExit("--min-tokens holds back the tokenizer's EOS id: this run has none (--synthetic without a tokenizer)")
    if speculative:
        from .generate import _check_prompt_lookup, prompt_lookup_generate_ids, speculative_generate_ids

        if args.adapter is not None or getattr(model, "adapters", None) is not None:
            raise SystemExit("speculative decoding does not take adapters: drop --lora / --synthetic-lora / --adapter")
        if penalties:
            raise SystemExit("speculative sampling takes --sampler-temp, --sampler-top-k, --sampler-top-p and --seed only: "
                             "drop the penalties and --min-p")
        if args.logprobs is not None:
            raise SystemExit("speculative decoding does not report log-probabilities: drop --logprobs")
        if args.draft_model and args.draft_synthetic:
            raise SystemExit("give one draft: --draft-model or --draft-synthetic, not both")
        eos_ids = () if eos is None else (eos,)
        if args.prompt_lookup is not None:
            try:
                ngram = _check_prompt_lookup(args.prompt_lookup, [int(n) for n in args.prompt_lookup_ngram.split(":")])
            except ValueError as exc:
                raise SystemExit(f"--prompt-lookup K --prompt-lookup-ngram MIN:MAX: {exc}") from None
            produced, stats = prompt_lookup_generate_ids(model, ids, args.max_new_tokens, proposal_length=args.prompt_lookup,
                                                         ngram=ngram, eos_token_ids=eos_ids, device=device, on_token=emit,
                                                         sampling=sampling)
            proposed, accepted = sum(p for p, _ in stats), sum(a for _, a in stats)
            matched = sum(1 for p, _ in stats if p)
            print(f"\nspeculative: {len(stats)} rounds, {accepted}/{proposed} proposals accepted"
                  + (f" ({accepted / proposed:.2f})" if proposed else "") + f", {matched} rounds matched", file=sys.stderr)
            print()
            return 0
        draft_args = argparse.Namespace(**{**vars(args), "model": args.draft_model, "synthetic": args.draft_synthetic})
        draft_ns, draft_tokenizer, draft_name = _load(draft_args, device)
        if tokenizer is not None and draft_tokenizer is not None and tokenizer.get_vocab() != draft_tokenizer.get_vocab():
            raise SystemExit("draft and target tokenizers use different token ids")
        draft = _model(args, draft_ns, draft_name)
        produced, stats = speculative_generate_ids(draft, model, ids, args.max_new_tokens, proposal_length=args.proposal_length,
                                                   eos_token_ids=eos_ids, device=device, on_token=emit,
                                                   sampling=sampling)
        proposed, accepted = sum(p for p, _ in stats), sum(a for _, a in stats)
        print(f"\nspeculative: {len(stats)} rounds, {accepted}/{proposed} proposals accepted"
              + (f" ({accepted / proposed:.2f})" if proposed else ""), file=sys.stderr)
        print()
        return 0
    produced = greedy_generate_ids(model, ids, args.max_new_tokens, eos_token_id=eos, device=device,
                                   on_token=emit, sampler=sampler, sampling=sampling, logprobs=args.logprobs, **_adapter_kw(args, "adapter"))
    print()
    if args.logprobs is not None:
        produced, entries = produced
        print("logprobs (raw model distribution):")
        _print_logprobs(entries, tokenizer)
    return 0 if produced is not None else 1


def _parallel_sample(args, model, tokenizer, ids, penalties, device) -> int:
    """``generate --num-samples N``: N seeded samples of the prompt from one prefill (sample j draws with seed
    ``--seed + j``); per sample one line with its seed, finish reason and length, then its text (its ids for
    ``--prompt-ids`` runs), then its log-probabilities with ``--logprobs``."""
    from .generate import parallel_sample_ids, sample_seed
    from .sampler import SamplingParams

    refused = [("adapters", args.adapter is not None or getattr(model, "adapters", None) is not None),
               ("a draft", bool(args.draft_model or args.draft_synthetic)), ("--prompt-lookup", args.prompt_lookup is not None)]
    for what, given in refused:
        if given:
            raise SystemExit(f"parallel sampling takes no {what}: drop it or --num-samples")
    if device.type != "cuda":  # without --num-samples a CPU run draws through make_sampler, which has no per-sample seeds
        raise SystemExit("parallel sampling draws with the seeded CUDA sampling kernel: it needs a CUDA --device")
    constraint = _constraint(args, model, tokenizer, device)
    if constraint is not None:
        penalties["constraint"] = constraint
    sampling = SamplingParams(args.sampler_temp, top_k=args.sampler_top_k, top_p=args.sampler_top_p, seed=args.seed, **penalties)
    eos = getattr(tokenizer, "eos_token_id", None)
    if constraint is not None and args.synthetic:
        eos = constraint.vocabulary.eos_ids[0]
    try:
        samples = parallel_sample_ids(model, [ids], args.num_samples, sampling, args.max_new_tokens,
                                      eos_token_ids=() if eos is None else (eos,), logprobs=args.logprobs, device=device)[0]
    except ValueError as exc:
        raise SystemExit(f"--num-samples: {exc}") from None
    for j, s in enumerate(samples):
        print(f"sample {j}: seed {sample_seed(args.seed, j)}, {s.finish_reason}, {len(s.ids)} tokens")
        print(" ".join(str(t) for t in s.ids) if tokenizer is None else tokenizer.decode(s.ids))
        if s.logprobs is not None:
            print("logprobs (raw model distribution):")
            _print_logprobs(s.logprobs, tokenizer)
    return 0


def _beam_search(args, model, tokenizer, ids, penalties, device) -> int:
    """``generate --num-beams W``: one line per returned hypothesis (rank, score, sum of log-probabilities, length,
    finished or not), then its text (its ids for ``--prompt-ids`` runs)."""
    from .generate import beam_search_ids

    refused = [("a non-zero --sampler-temp", args.sampler_temp != 0), ("--typical-p", args.typical_p != 1.0),
               ("--top-n-sigma", args.top_n_sigma != 0.0), ("--mirostat", args.mirostat != 0), ("penalties or --min-p", bool(penalties)),
               ("--regex", args.regex is not None), ("--json", args.json),
               ("--json-schema", args.json_schema is not None), ("--grammar", args.grammar is not None),
               ("--logprobs", args.logprobs is not None),
               ("adapters", args.adapter is not None or getattr(model, "adapters", None) is not None),
               ("a draft", bool(args.draft_model or args.draft_synthetic)), ("--prompt-lookup", args.prompt_lookup is not None)]
    for what, given in refused:
        if given:
            raise SystemExit(f"beam search is deterministic and takes no {what}: drop it or --num-beams")
    eos = getattr(tokenizer, "eos_token_id", None)
    try:
        hyps = beam_search_ids(model, ids, args.max_new_tokens, num_beams=args.num_beams, length_penalty=args.length_penalty,
                               early_stopping=args.early_stopping, num_return_sequences=args.num_return_sequences,
                               eos_token_ids=() if eos is None else (eos,), device=device)
    except ValueError as exc:
        raise SystemExit(f"--num-beams: {exc}") from None
    for rank, h in enumerate(hyps):
        state = "finished" if h.finished else "unfinished"
        print(f"beam {rank}: score {h.score:.6f}  sum_logprob {h.sum_logprob:.6f}  length {len(h.ids) + int(h.finished)}  {state}")
    for rank, h in enumerate(hyps):
        text = " ".join(str(t) for t in h.ids) if tokenizer is None or args.prompt_ids else tokenizer.decode(h.ids)
        print(f"[{rank}] {text}")
    return 0


def cmd_batch(args) -> int:
    from .batch import ContinuousBatcher
    from .sampler import SamplingParams

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    _load_adapters(args, model, ns)
    if args.prompts_file:
        prompts = [line.strip() for line in open(args.prompts_file) if line.strip()]
    else:
        prompts = [args.prompt or "Give me a short introduction to large language models."]
    if args.prompt_ids or tokenizer is None:
        queue = [[int(t) for t in p.split(",")] for p in (args.prompt_ids.split(";") if args.prompt_ids else prompts)]
    else:
        queue = [tokenizer.apply_chat_template([{"role": "user", "content": p}], tokenize=False, add_generation_prompt=True,
                                               enable_thinking=args.enable_thinking) for p in prompts]
    sampling = None
    penalties = _penalties(args)
    controls = _controls(args)
    if controls and args.grammar is not None:
        raise SystemExit("--logit-bias, --allowed-token-ids, --bad-words and --min-tokens take no --grammar")
    constraint = _constraint(args, model, tokenizer, device)
    if constraint is not None:
        if controls:
            raise SystemExit("--logit-bias, --allowed-token-ids, --bad-words and --min-tokens take no --regex, --json or --json-schema")
        penalties["constraint"] = constraint
    penalties.update(controls)
    penalties.update(_dry_xtc(args, tokenizer))
    if args.sampler_temp != 0 or penalties:  # request i draws with seed `--seed + i`
        try:
            sampling = [SamplingParams(args.sampler_temp, top_k=args.sampler_top_k, top_p=args.sampler_top_p, seed=args.seed + i, **penalties)
                        for i in range(len(queue))]
        except ValueError as exc:
            raise SystemExit(str(exc)) from None
    if args.prefix_cache and not hasattr(model, "enable_prefix_cache"):
        raise SystemExit("--prefix-cache needs the paged week3 model")
    eos = constraint.vocabulary.eos_ids[0] if constraint is not None and args.synthetic else None
    if controls.get("min_tokens") and eos is None and getattr(tokenizer, "eos_token_id", None) is None:
        raise SystemExit("--min-tokens holds back the tokenizer's EOS id: this run has none (--synthetic without a tokenizer)")
    extra = {}
    if args.adapters is not None:  # one name per prompt, empty: the base model
        names = [n.strip() or None for n in args.adapters.split(";")]
        if len(names) != len(queue):
            raise SystemExit(f"--adapters names {len(names)} requests, there are {len(queue)} prompts")
        extra["adapters"] = names
    try:
        batcher = ContinuousBatcher(model, tokenizer, queue, max_seq_len=args.max_seq_len, batch_size=args.batch_size, prefill_step=args.prefill_step,
                                    verbose=not args.quiet, device=device, eos_token_id=eos,
                                    max_new_tokens=[args.max_new_tokens] * len(queue) if args.max_new_tokens else None, sampling=sampling,
                                    logprobs=args.logprobs, prefix_cache=args.prefix_cache, **extra)
    except (KeyError, ValueError) as exc:  # an adapter name that is not loaded
        raise SystemExit(f"batch: {exc}")
    results = batcher.run()
    for idx, text in sorted(results):
        print(f"--- request {idx}\n{text}")
        if args.prefix_cache:
            print(f"reused tokens: {batcher.reused_tokens.get(idx, 0)}")
        if args.logprobs is not None:
            _print_logprobs(batcher.logprobs.get(idx, []), tokenizer)
    if args.prefix_cache:
        print("prefix cache: " + ", ".join(f"{k} {v}" for k, v in batcher.prefix_cache.stats().items()))
    return 0


def cmd_score(args) -> int:
    from .logprobs import score_ids

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    _load_adapters(args, model, ns)
    if args.prompt_ids:
        ids = [int(t) for t in args.prompt_ids.split(",")]
    elif tokenizer is None:
        raise SystemExit("a text prompt needs the checkpoint's tokenizer files; use --prompt-ids")
    else:
        ids = tokenizer.encode(args.prompt, add_special_tokens=False)
    if len(ids) < 2:
        raise SystemExit("scoring needs a prompt of at least two tokens")
    result = score_ids(model, ids, chunk=args.chunk, top_n=args.logprobs or 0, device=device, **_adapter_kw(args, "adapter"))
    print(f"prompt: {len(ids)} tokens; first token {_token_text(tokenizer, ids[0])} is not scored")
    _print_logprobs(result.entries, tokenizer)
    print(f"total nll {result.nll:.4f} nats over {len(result.entries)} tokens, perplexity {result.perplexity:.4f}")
    if result.next_top:
        print("next token: " + ", ".join(f"{_token_text(tokenizer, i)} {v:.4f}" for i, v in result.next_top))
    return 0


def embed_inputs(args, tokenizer) -> list[list[int]]:
    """The token ids ``embed`` runs: ``--prompt-ids`` ("1,2;3,4"), else the ``--prompt`` texts and the lines of
    ``--prompts-file`` encoded by the tokenizer; ``--append-eos`` ends each with the tokenizer's EOS id (what
    Qwen3-Embedding's last-token pooling expects)."""
    if args.prompt_ids:
        prompts = [[int(t) for t in part.split(",") if t.strip()] for part in args.prompt_ids.split(";")]
    else:
        texts = list(args.prompt or [])
        if args.prompts_file:
            with open(args.prompts_file, encoding="utf-8") as f:
                texts += [line.rstrip("\n") for line in f if line.strip()]
        if not texts:
            raise SystemExit("embed needs --prompt-ids, --prompt or --prompts-file")
        if tokenizer is None:
            raise SystemExit("text prompts need the checkpoint's tokenizer files; use --prompt-ids")
        prompts = [list(tokenizer.encode(t, add_special_tokens=False)) for t in texts]
    if args.append_eos:
        eos = None if tokenizer is None else tokenizer.eos_token_id
        if eos is None:
            raise SystemExit("--append-eos needs a tokenizer with an EOS id")
        prompts = [p + [int(eos)] for p in prompts]
    for i, p in enumerate(prompts):
        if not p:
            raise SystemExit(f"prompt {i} is empty")
    return prompts


def cmd_embed(args) -> int:
    from .embed import embed_ids

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    prompts = embed_inputs(args, tokenizer)
    try:
        out = embed_ids(model, prompts, pooling=args.pooling, normalize=not args.no_normalize, dimensions=args.dimensions,
                        max_tokens=args.max_tokens, device=device).cpu()
    except ValueError as exc:
        raise SystemExit(f"embed: {exc}") from None
    for i, row in enumerate(out):
        print(f"[{i}] {len(prompts[i])} tokens, {row.numel()} dims, norm {row.norm().item():.6f}: " + " ".join(f"{v:.6f}" for v in row.tolist()))
    if args.out:
        import numpy as np

        np.save(args.out, out.numpy())
    return 0


def rerank_inputs(args, tokenizer):
    """``(prefix, documents, true_id, false_id)`` for ``rerank``.  With ``--document-ids`` ("a,b;c,d"): the documents'
    ids after ``--prefix-ids``.  Otherwise each ``--document`` and line of ``--documents-file`` is put into the
    Qwen3-Reranker template with ``--query`` and ``--instruction``, each pair is tokenised whole, and the longest
    shared leading run of ids becomes the prefix.  ``--true-id`` / ``--false-id`` default to the tokenizer's "yes" and
    "no"."""
    from .rerank import rerank_prompt, split_shared_prefix

    def ids(text):
        return [int(t) for t in text.split(",") if t.strip()]

    if args.document_ids:
        prefix = ids(args.prefix_ids or "")
        docs = [ids(part) for part in args.document_ids.split(";")]
    else:
        texts = list(args.document or [])
        if args.documents_file:
            with open(args.documents_file, encoding="utf-8") as f:
                texts += [line.rstrip("\n") for line in f if line.strip()]
        if not texts or args.query is None:
            raise SystemExit("rerank needs --document-ids, or --query with --document or --documents-file")
        if tokenizer is None:
            raise SystemExit("text queries and documents need the checkpoint's tokenizer files; use --prefix-ids / --document-ids")
        prompts = [list(tokenizer.encode(rerank_prompt(args.query, t, args.instruction), add_special_tokens=False)) for t in texts]
        prefix, docs = split_shared_prefix(prompts)
    for i, d in enumerate(docs):
        if not d:
            raise SystemExit(f"document {i} is empty")
    true_id, false_id = args.true_id, args.false_id
    if true_id is None or false_id is None:
        if tokenizer is None:
            raise SystemExit("--true-id and --false-id are needed without the checkpoint's tokenizer")
        true_id = tokenizer.convert_tokens_to_ids("yes") if true_id is None else true_id
        false_id = tokenizer.convert_tokens_to_ids("no") if false_id is None else false_id
    return prefix, docs, int(true_id), int(false_id)


def cmd_rerank(args) -> int:
    from .rerank import rerank_ids

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    prefix, docs, true_id, false_id = rerank_inputs(args, tokenizer)
    try:
        scores = rerank_ids(model, [(prefix, docs)], true_id, false_id, max_tokens=args.max_tokens, device=device)[0].cpu()
    except ValueError as exc:
        raise SystemExit(f"rerank: {exc}") from None
    print(f"shared prefix: {len(prefix)} tokens")
    for i, (doc, score) in enumerate(zip(docs, scores.tolist())):
        print(f"[{i}] {len(doc)} tokens: {score:.6f}")
    return 0


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="tiny_llm_b200.cli")
    sub = ap.add_subparsers(dest="command", required=True)
    for name, fn in (("generate", cmd_generate), ("batch", cmd_batch), ("score", cmd_score)):
        p = sub.add_parser(name)
        p.set_defaults(fn=fn)
        p.add_argument("--model", default=None, help="checkpoint directory (config.json + *.safetensors [+ tokenizer files])")
        p.add_argument("--synthetic", default=None, help="random weights of a named shape (tiny, tiny-d128, qwen3-0.6b, qwen3-4b; Qwen3-MoE: "
                       "tiny-moe-d128, qwen3-30b-a3b) instead of --model")
        p.add_argument("--synthetic-bits", type=int, choices=(4, 8), default=4,
                       help="code width of the --synthetic weights, and of a --draft-synthetic draft's (MLX affine, group 128)")
        p.add_argument("--prompt", default="Give me a short introduction to large language models.")
        p.add_argument("--prompt-ids", default=None, help="comma-separated token ids (';' between requests for `batch`)")
        p.add_argument("--loader", choices=["week2", "week3"], default="week3")
        p.add_argument("--rope-scaling", type=_rope_scaling_arg, default=None, metavar="yarn:FACTOR[:ORIGINAL]",
                       help="static YaRN RoPE scaling of the --synthetic model (a checkpoint states its own in config.json)")
        p.add_argument("--max-context", type=_positive_int, default=None, metavar="N",
                       help="context window of the decode / prefill graphs (default 8192); refused if its KV pages do not fit the GPU")
        p.add_argument("--device", default="cuda:0")
        p.add_argument("--disable-paged-attention", action="store_true")
        p.add_argument("--enable-thinking", action="store_true")
        p.add_argument("--max-new-tokens", type=int, default=128)
    for name in ("generate", "batch"):
        sub.choices[name].add_argument("--sampler-temp", type=float, default=0.0)
        sub.choices[name].add_argument("--sampler-top-p", type=float, default=None)
        sub.choices[name].add_argument("--sampler-top-k", type=int, default=None)
        sub.choices[name].add_argument("--seed", type=int, default=0, help="seed of the sampled draw on CUDA (`batch`: request i uses seed + i)")
        sub.choices[name].add_argument("--repetition-penalty", type=float, default=1.0,
                                       help="divide positive (multiply negative) logits of prompt and generated tokens (> 0; 1: off)")
        sub.choices[name].add_argument("--presence-penalty", type=float, default=0.0, help="subtract from the logits of generated tokens")
        sub.choices[name].add_argument("--frequency-penalty", type=float, default=0.0,
                                       help="subtract this times the count of each generated token")
        sub.choices[name].add_argument("--min-p", type=float, default=0.0,
                                       help="keep tokens at least this fraction as likely as the top one (0: off)")
        sub.choices[name].add_argument("--logit-bias", default=None, metavar="ID:B,ID:B",
                                       help="add bias B (in [-100, 100]) to token ID's logit before the draw")
        sub.choices[name].add_argument("--allowed-token-ids", default=None, metavar="ID,ID",
                                       help="draw only from these token ids")
        sub.choices[name].add_argument("--bad-words", default=None, metavar="ID,ID;ID",
                                       help="never complete these token sequences (split by ';'); a single id is banned outright")
        sub.choices[name].add_argument("--min-tokens", type=int, default=0, metavar="N",
                                       help="hold back EOS until N tokens have been generated")
        sub.choices[name].add_argument("--dry-multiplier", type=float, default=0.0,
                                       help="DRY: penalise tokens that extend a verbatim repeat of the history (0: off)")
        sub.choices[name].add_argument("--dry-base", type=float, default=1.75, help="DRY: the penalty's growth per repeated token (> 1)")
        sub.choices[name].add_argument("--dry-allowed-length", type=int, default=2, help="DRY: the longest repeat left alone (>= 1)")
        sub.choices[name].add_argument("--dry-penalty-last-n", type=int, default=0, help="DRY: the window of recent tokens (0: all)")
        sub.choices[name].add_argument("--dry-sequence-breakers", default=None, metavar="ID,ID or JSON",
                                       help='DRY: ids, or a JSON list of strings such as \'["\\n", ":"]\', that no repeat runs through')
        sub.choices[name].add_argument("--xtc-threshold", type=float, default=0.1,
                                       help="XTC: tokens at least this likely are the top choices (in (0, 1])")
        sub.choices[name].add_argument("--xtc-probability", type=float, default=0.0,
                                       help="XTC: the chance per draw of excluding all top choices but the least likely (0: off)")
        sub.choices[name].add_argument("--typical-p", type=float, default=1.0,
                                       help="locally typical sampling: keep the tokens closest to the entropy up to this mass (1: off)")
        sub.choices[name].add_argument("--top-n-sigma", type=float, default=0.0,
                                       help="keep tokens within this many standard deviations of the top logit (0: off)")
        sub.choices[name].add_argument("--mirostat", type=int, default=0, choices=(0, 2),
                                       help="Mirostat 2.0: keep the surprise of each draw near --mirostat-tau (0: off)")
        sub.choices[name].add_argument("--mirostat-tau", type=float, default=5.0, help="Mirostat: the target surprise in bits (> 0)")
        sub.choices[name].add_argument("--mirostat-eta", type=float, default=0.1, help="Mirostat: the learning rate of mu (> 0)")
        sub.choices[name].add_argument("--regex", default=None, metavar="PATTERN",
                                       help="constrain the generated text to fullmatch PATTERN (re.ASCII semantics over UTF-8 bytes)")
        sub.choices[name].add_argument("--json", action="store_true",
                                       help="constrain the generated text to one JSON object (RFC 8259; depth <= 64, whitespace runs <= 32)")
        sub.choices[name].add_argument("--json-schema", default=None, metavar="FILE_OR_INLINE_JSON",
                                       help="constrain the generated text to one JSON object that validates against this JSON Schema "
                                            "(keys in the schema's order; DESIGN.md section 21 lists the keywords)")
        sub.choices[name].add_argument("--grammar", default=None, metavar="FILE_OR_INLINE",
                                       help="constrain the generated text to the language of this GBNF grammar (a file, or the "
                                            "grammar text itself when it holds '::='; start rule root; DESIGN.md section 23)")
    for name in ("generate", "batch", "score"):
        sub.choices[name].add_argument("--logprobs", type=int, default=None, metavar="N",
                                       help="print each token's log-probability, rank and N most likely alternatives (N <= 20)")
        sub.choices[name].add_argument("--lora", action="append", default=None, metavar="NAME=DIR",
                                       help="load a PEFT LoRA adapter directory under NAME (repeatable, up to 32)")
        sub.choices[name].add_argument("--synthetic-lora", action="append", default=None, metavar="NAME=RANK[:SEED]",
                                       help="a seeded random adapter of RANK (8, 16, 32 or 64) on every projection (repeatable)")
    for name in ("generate", "score"):
        sub.choices[name].add_argument("--adapter", default=None, metavar="NAME", help="run the request under this loaded adapter")
    sub.choices["batch"].add_argument("--adapters", default=None, metavar="A;;B",
                                      help="one loaded adapter name per prompt, ';' between them (empty: the base model)")
    sub.choices["score"].add_argument("--chunk", type=int, default=512, help="prompt tokens per forward pass (bounds the live logits)")
    sub.choices["generate"].add_argument("--draft-model", default=None, help="checkpoint directory of a draft model: speculative decoding")
    sub.choices["generate"].add_argument("--draft-synthetic", default=None, help="random-weight draft of a named shape (seed 0, as --synthetic)")
    sub.choices["generate"].add_argument("--proposal-length", type=int, default=4, help="draft tokens proposed per round")
    sub.choices["generate"].add_argument("--num-beams", type=int, default=None, metavar="W",
                                         help="deterministic beam search with W (1..8) beams; prints every returned hypothesis")
    sub.choices["generate"].add_argument("--length-penalty", type=float, default=1.0,
                                         help="beam search: a hypothesis of L tokens scores sum_logprob / L**A")
    sub.choices["generate"].add_argument("--early-stopping", action="store_true",
                                         help="beam search: stop as soon as num_beams hypotheses have finished")
    sub.choices["generate"].add_argument("--num-return-sequences", type=int, default=1, metavar="N",
                                         help="beam search: hypotheses to return (1..W)")
    sub.choices["generate"].add_argument("--num-samples", type=int, default=None, metavar="N",
                                         help="N (1..16) seeded samples of the prompt from one prefill on a CUDA device; sample j uses seed + j")
    sub.choices["generate"].add_argument("--prompt-lookup", type=int, default=None, metavar="K",
                                         help="prompt-lookup speculative decoding: K (1..7) proposals per round from the request's own tokens")
    sub.choices["generate"].add_argument("--prompt-lookup-ngram", default="2:3", metavar="MIN:MAX",
                                         help="suffix lengths prompt lookup matches (1 <= MIN <= MAX <= 8)")
    p = sub.add_parser("embed")
    p.set_defaults(fn=cmd_embed, loader="week3", rope_scaling=None, max_context=None, disable_paged_attention=False, logprobs=None)
    p.add_argument("--model", default=None, help="checkpoint directory (Qwen3 or Qwen3-Embedding, MLX 4- or 8-bit)")
    p.add_argument("--synthetic", default=None, help="random weights of a named shape (tiny-d128, qwen3-0.6b, qwen3-4b) instead of --model")
    p.add_argument("--synthetic-bits", type=int, choices=(4, 8), default=4, help="code width of the --synthetic weights (MLX affine, group 128)")
    p.add_argument("--prompt", action="append", default=None, help="a text to embed (repeatable; needs the tokenizer)")
    p.add_argument("--prompts-file", default=None, help="one text per line")
    p.add_argument("--prompt-ids", default=None, help="comma-separated token ids, ';' between prompts")
    p.add_argument("--append-eos", action="store_true", help="end every prompt with the tokenizer's EOS id")
    p.add_argument("--pooling", choices=["last", "mean"], default="last")
    p.add_argument("--dimensions", type=_positive_int, default=None, metavar="N", help="keep the first N features (default: all)")
    p.add_argument("--no-normalize", action="store_true", help="skip the L2 normalisation")
    p.add_argument("--max-tokens", type=_positive_int, default=8192, metavar="N", help="rows per packed pass (a multiple of 128)")
    p.add_argument("--out", default=None, metavar="FILE.npy", help="also save the [n, d] float32 embeddings")
    p.add_argument("--device", default="cuda:0")
    p = sub.add_parser("rerank")
    p.set_defaults(fn=cmd_rerank, loader="week3", rope_scaling=None, max_context=None, disable_paged_attention=False, logprobs=None)
    p.add_argument("--model", default=None, help="checkpoint directory (Qwen3 or Qwen3-Reranker, MLX 4- or 8-bit)")
    p.add_argument("--synthetic", default=None, help="random weights of a named shape (tiny-d128, qwen3-0.6b, qwen3-4b) instead of --model")
    p.add_argument("--synthetic-bits", type=int, choices=(4, 8), default=4, help="code width of the --synthetic weights (MLX affine, group 128)")
    p.add_argument("--query", default=None, help="the query text (needs the tokenizer)")
    p.add_argument("--document", action="append", default=None, help="a document text (repeatable)")
    p.add_argument("--documents-file", default=None, help="one document text per line")
    p.add_argument("--instruction", default=None, help="the task instruction (default: Qwen3-Reranker's web-search one)")
    p.add_argument("--prefix-ids", default=None, help="comma-separated token ids shared by every prompt")
    p.add_argument("--document-ids", default=None, help="comma-separated token ids of each prompt's rest, ';' between documents")
    p.add_argument("--true-id", type=int, default=None, help="the id whose probability is the score (default: the tokenizer's \"yes\")")
    p.add_argument("--false-id", type=int, default=None, help="the competing id (default: the tokenizer's \"no\")")
    p.add_argument("--max-tokens", type=_positive_int, default=8192, metavar="N", help="rows per packed pass (a multiple of 128)")
    p.add_argument("--device", default="cuda:0")
    sub.choices["batch"].add_argument("--prompts-file", default=None)
    sub.choices["batch"].add_argument("--batch-size", type=int, default=5)
    sub.choices["batch"].add_argument("--prefill-step", type=int, default=128)
    sub.choices["batch"].add_argument("--max-seq-len", type=int, default=512)
    sub.choices["batch"].add_argument("--quiet", action="store_true")
    sub.choices["batch"].add_argument("--prefix-cache", action="store_true",
                                      help="share the KV pages of prompt prefixes computed before (paged week3 model)")
    args = ap.parse_args(argv)
    if not args.model and not args.synthetic:
        ap.error("--model or --synthetic is required")
    if args.rope_scaling is not None and not args.synthetic:
        ap.error("--rope-scaling applies to --synthetic; a checkpoint's config.json states its own rope_scaling")
    if args.synthetic_bits != 4 and not args.synthetic:
        ap.error("--synthetic-bits applies to --synthetic; a checkpoint's config.json states its own quantization")
    if args.command == "batch" and args.max_context is not None and args.max_seq_len > args.max_context:
        ap.error(f"--max-seq-len {args.max_seq_len} exceeds --max-context {args.max_context}")
    if args.logprobs is not None and not 0 <= args.logprobs <= 20:
        ap.error("--logprobs must be in [0, 20]")
    return args.fn(args)


if __name__ == "__main__":
    raise SystemExit(main())
