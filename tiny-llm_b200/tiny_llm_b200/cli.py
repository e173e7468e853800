"""Command-line front doors: the equivalents of the reference's ``main.py`` (one prompt,
``main.py:1-190``) and ``batch-main.py`` (continuous batching,
``batch-main.py:1-102``) over a checkpoint DIRECTORY (MLX 4-bit safetensors layout,
see checkpoint.py; there is no hub download here).

    python -m tiny_llm_b200.cli generate --model /path/to/Qwen3-4B-MLX-4bit --prompt "..." [--loader week3]
    python -m tiny_llm_b200.cli batch    --model /path/to/ckpt --prompts-file prompts.txt --batch-size 5
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --max-new-tokens 8   (no files needed)
    python -m tiny_llm_b200.cli batch    --synthetic tiny-d128 --prompt-ids "5,17,3;9,2,4" --sampler-temp 0.7 --sampler-top-p 0.9 --seed 3
        (seeded sampling with the tl_sample kernel: the same seed gives the same tokens)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --sampler-temp 0.7 --presence-penalty 1.5 --min-p 0.05
        (token-history penalties and min-p; with --sampler-temp 0 the greedy token of the penalised logits)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --draft-synthetic tiny-d128 --proposal-length 4 --prompt-ids 5,17,3
        (speculative decoding: same ids as greedy; acceptance stats on stderr)
    python -m tiny_llm_b200.cli generate --synthetic tiny-d128 --prompt-ids 5,17,3 --logprobs 5
        (each generated token's log-probability, rank and 5 most likely alternatives, after the text)
    python -m tiny_llm_b200.cli score    --model /path/to/ckpt --prompt "The capital of France is Paris." [--logprobs 3]
        (teacher-forced log-probability of every prompt token and the prompt's perplexity)
"""

from __future__ import annotations

import argparse
import sys

import torch


def _load(args, device):
    from .checkpoint import load_checkpoint, load_tokenizer
    from .synthetic import synthetic_qwen3

    if args.synthetic:
        return synthetic_qwen3(args.synthetic, seed=0, device=device, realistic=args.synthetic.startswith("tiny")), None, "Qwen/Qwen3-synthetic"
    ns = load_checkpoint(args.model, device=device)
    tokenizer = None
    try:
        tokenizer = load_tokenizer(args.model)
    except Exception as exc:  # token-id mode still works without tokenizer files
        print(f"(no tokenizer loaded from {args.model}: {exc})", file=sys.stderr)
    return ns, tokenizer, "Qwen/Qwen3-" + str(args.model)


def _model(args, ns, name):
    from .models import dispatch_model

    if args.loader == "week2":
        return dispatch_model(name, ns, week=2)
    return dispatch_model(name, ns, week=3, enable_paged_attention=not args.disable_paged_attention)


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
    """The ``SamplingParams`` penalty fields the flags turn on (an empty dict when every one is off)."""
    given = dict(repetition_penalty=args.repetition_penalty, presence_penalty=args.presence_penalty,
                 frequency_penalty=args.frequency_penalty, min_p=args.min_p)
    off = dict(repetition_penalty=1.0, presence_penalty=0.0, frequency_penalty=0.0, min_p=0.0)
    return {k: v for k, v in given.items() if v != off[k]}


def cmd_generate(args) -> int:
    from .generate import greedy_generate_ids
    from .sampler import SamplingParams, make_sampler

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    ids = _prompt_ids(args, tokenizer, args.prompt)
    sampler = sampling = None
    penalties = _penalties(args)
    if args.sampler_temp != 0 or penalties:
        if device.type == "cuda" or penalties:  # the seeded kernel
            sampling = SamplingParams(args.sampler_temp, top_k=args.sampler_top_k, top_p=args.sampler_top_p, seed=args.seed, **penalties)
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
    if args.draft_model or args.draft_synthetic:
        from .generate import speculative_generate_ids

        if sampler is not None or sampling is not None:
            raise SystemExit("speculative decoding is greedy: drop --sampler-temp")
        if args.logprobs is not None:
            raise SystemExit("speculative decoding does not report log-probabilities: drop --logprobs")
        if args.draft_model and args.draft_synthetic:
            raise SystemExit("give one draft: --draft-model or --draft-synthetic, not both")
        draft_args = argparse.Namespace(**{**vars(args), "model": args.draft_model, "synthetic": args.draft_synthetic})
        draft_ns, draft_tokenizer, draft_name = _load(draft_args, device)
        if tokenizer is not None and draft_tokenizer is not None and tokenizer.get_vocab() != draft_tokenizer.get_vocab():
            raise SystemExit("draft and target tokenizers use different token ids")
        draft = _model(args, draft_ns, draft_name)
        produced, stats = speculative_generate_ids(draft, model, ids, args.max_new_tokens, proposal_length=args.proposal_length,
                                                   eos_token_ids=() if eos is None else (eos,), device=device, on_token=emit)
        proposed, accepted = sum(p for p, _ in stats), sum(a for _, a in stats)
        print(f"\nspeculative: {len(stats)} rounds, {accepted}/{proposed} proposals accepted"
              + (f" ({accepted / proposed:.2f})" if proposed else ""), file=sys.stderr)
        print()
        return 0
    produced = greedy_generate_ids(model, ids, args.max_new_tokens, eos_token_id=eos, device=device,
                                   on_token=emit, sampler=sampler, sampling=sampling, logprobs=args.logprobs)
    print()
    if args.logprobs is not None:
        produced, entries = produced
        print("logprobs (raw model distribution):")
        _print_logprobs(entries, tokenizer)
    return 0 if produced is not None else 1


def cmd_batch(args) -> int:
    from .batch import ContinuousBatcher
    from .sampler import SamplingParams

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
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
    if args.sampler_temp != 0 or penalties:  # request i draws with seed `--seed + i`
        sampling = [SamplingParams(args.sampler_temp, top_k=args.sampler_top_k, top_p=args.sampler_top_p, seed=args.seed + i, **penalties)
                    for i in range(len(queue))]
    batcher = ContinuousBatcher(model, tokenizer, queue, max_seq_len=args.max_seq_len, batch_size=args.batch_size, prefill_step=args.prefill_step,
                                verbose=not args.quiet, device=device,
                                max_new_tokens=[args.max_new_tokens] * len(queue) if args.max_new_tokens else None, sampling=sampling,
                                logprobs=args.logprobs)
    results = batcher.run()
    for idx, text in sorted(results):
        print(f"--- request {idx}\n{text}")
        if args.logprobs is not None:
            _print_logprobs(batcher.logprobs.get(idx, []), tokenizer)
    return 0


def cmd_score(args) -> int:
    from .logprobs import score_ids

    device = torch.device(args.device)
    ns, tokenizer, name = _load(args, device)
    model = _model(args, ns, name)
    if args.prompt_ids:
        ids = [int(t) for t in args.prompt_ids.split(",")]
    elif tokenizer is None:
        raise SystemExit("a text prompt needs the checkpoint's tokenizer files; use --prompt-ids")
    else:
        ids = tokenizer.encode(args.prompt, add_special_tokens=False)
    if len(ids) < 2:
        raise SystemExit("scoring needs a prompt of at least two tokens")
    result = score_ids(model, ids, chunk=args.chunk, top_n=args.logprobs or 0, device=device)
    print(f"prompt: {len(ids)} tokens; first token {_token_text(tokenizer, ids[0])} is not scored")
    _print_logprobs(result.entries, tokenizer)
    print(f"total nll {result.nll:.4f} nats over {len(result.entries)} tokens, perplexity {result.perplexity:.4f}")
    if result.next_top:
        print("next token: " + ", ".join(f"{_token_text(tokenizer, i)} {v:.4f}" for i, v in result.next_top))
    return 0


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(prog="tiny_llm_b200.cli")
    sub = ap.add_subparsers(dest="command", required=True)
    for name, fn in (("generate", cmd_generate), ("batch", cmd_batch), ("score", cmd_score)):
        p = sub.add_parser(name)
        p.set_defaults(fn=fn)
        p.add_argument("--model", default=None, help="checkpoint directory (config.json + *.safetensors [+ tokenizer files])")
        p.add_argument("--synthetic", default=None, help="random weights of a named shape (tiny, tiny-d128, qwen3-0.6b, qwen3-4b) instead of --model")
        p.add_argument("--prompt", default="Give me a short introduction to large language models.")
        p.add_argument("--prompt-ids", default=None, help="comma-separated token ids (';' between requests for `batch`)")
        p.add_argument("--loader", choices=["week2", "week3"], default="week3")
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
    for name in ("generate", "batch", "score"):
        sub.choices[name].add_argument("--logprobs", type=int, default=None, metavar="N",
                                       help="print each token's log-probability, rank and N most likely alternatives (N <= 20)")
    sub.choices["score"].add_argument("--chunk", type=int, default=512, help="prompt tokens per forward pass (bounds the live logits)")
    sub.choices["generate"].add_argument("--draft-model", default=None, help="checkpoint directory of a draft model: speculative decoding")
    sub.choices["generate"].add_argument("--draft-synthetic", default=None, help="random-weight draft of a named shape (seed 0, as --synthetic)")
    sub.choices["generate"].add_argument("--proposal-length", type=int, default=4, help="draft tokens proposed per round")
    sub.choices["batch"].add_argument("--prompts-file", default=None)
    sub.choices["batch"].add_argument("--batch-size", type=int, default=5)
    sub.choices["batch"].add_argument("--prefill-step", type=int, default=128)
    sub.choices["batch"].add_argument("--max-seq-len", type=int, default=512)
    sub.choices["batch"].add_argument("--quiet", action="store_true")
    args = ap.parse_args(argv)
    if not args.model and not args.synthetic:
        ap.error("--model or --synthetic is required")
    if args.logprobs is not None and not 0 <= args.logprobs <= 20:
        ap.error("--logprobs must be in [0, 20]")
    return args.fn(args)


if __name__ == "__main__":
    raise SystemExit(main())
