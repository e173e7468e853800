"""Regex-constrained generation on one GPU (V = 151,936, the seeded synthetic vocabulary):

* compile time of a few patterns: the host DFA (parse, NFA, subset construction, trim) and the ``tl_constraint_token_masks``
  launch (CUDA events, median of 20);
* ``tl_sample_constrained`` (every row masked, bf16 logits, temperature 0.7, top-p 0.9, top-k 50) against ``tl_sample``
  on the same rows, at 1, 8 and 64 rows (CUDA events over 200 launches);
* JSON mode's ``tl_json_token_masks`` per call at 1, 8 and 64 rows, every row inside a string value (nearly every
  token walks its whole length) and every row at a value position (most tokens fail on their first byte);
* JSON Schema's ``tl_schema_token_masks`` per call at 1, 8 and 64 rows under ``SCHEMA`` (11 properties, a nested
  array of objects, an enum, a pattern and a recursive ``$ref``), beside ``tl_json_token_masks`` on the same text in
  the same process, inside a string value and at a value position;
* the grammar kernel's ``tl_grammar_token_masks`` per call at 1, 8 and 64 rows: the expression grammar (inside a
  number, at a term), ``JSON_GBNF`` (JSON as a GBNF grammar) beside ``tl_schema_token_masks`` under ``SCHEMA`` and
  ``tl_json_token_masks`` on the same text, and ``EIGHT`` with eight parses live;
* ``decode_on_device`` tok/s, sampled against sampled under ``[a-z ]+``, under JSON mode, under ``SCHEMA`` and under the
  expression grammar, at B = 1 and B = 8 on Qwen3-4B-shaped synthetic weights, context 128 + steps, alternated in one
  process.

  python tools/constrained_bench.py [--out tools_out/constrained_bench.json]
"""
from __future__ import annotations

import argparse
import json
import statistics
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path[:0] = [str(ROOT), str(ROOT / "tiny-llm_b200"), str(ROOT / "tools")]

from extensions_b200 import tiny_llm_ext_b200 as ext  # noqa: E402
from sample_bench import card, timed  # noqa: E402
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3, SamplingParams  # noqa: E402
from tiny_llm_b200.constrained import TokenConstraint, TokenVocabulary, compile_dfa  # noqa: E402
from tiny_llm_b200.engine import DecodeEngine  # noqa: E402
from tiny_llm_b200.grammar import GRAMMAR_SMEM_BYTES, GrammarConstraint  # noqa: E402
from tiny_llm_b200.json_mode import ConstraintRows, JsonConstraint, JsonWalker  # noqa: E402
from tiny_llm_b200.json_schema import SCHEMA_SMEM_BYTES, JsonSchemaConstraint  # noqa: E402
from tiny_llm_b200.sampler import sampling_tensors  # noqa: E402
from tiny_llm_b200.synthetic import synthetic_qwen3  # noqa: E402

DEV = torch.device("cuda:0")
V = 151936
PATTERNS = {"date": r"[0-9]{4}-[0-9]{2}-[0-9]{2}", "label": r"(?:positive|negative|neutral)",
            "json": r'\{"name": "[a-zA-Z ]{1,20}", "age": [0-9]{1,3}, "tags": \[("[a-z]{1,10}"(, )?){0,4}\]\}',
            "words": r"[a-z ]+"}


def compile_table(vocab) -> dict:
    out = {}
    offsets, data = vocab.csr(DEV)
    eos = torch.tensor(vocab.eos_ids, dtype=torch.int32, device=DEV)
    for name, pattern in PATTERNS.items():
        host = []
        for _ in range(5):
            t0 = time.perf_counter()
            dfa = compile_dfa(pattern)
            host.append((time.perf_counter() - t0) * 1e3)
        table = torch.from_numpy(dfa.table).to(DEV)
        accept = torch.from_numpy(dfa.accept.astype("uint8")).to(DEV)
        kern = []
        for _ in range(20):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            ext.constraint_token_masks(table, accept, offsets, data, eos)
            b.record()
            b.synchronize()
            kern.append(a.elapsed_time(b))
        t0 = time.perf_counter()
        TokenConstraint.compile(pattern, vocab, device=DEV)
        total = (time.perf_counter() - t0) * 1e3
        out[name] = {"states": dfa.num_states, "host_dfa_ms": statistics.median(host), "kernel_ms": statistics.median(kern),
                     "compile_total_ms": total}
        print(f"{name}: {dfa.num_states} states, host DFA {out[name]['host_dfa_ms']:.2f} ms, masks kernel {out[name]['kernel_ms']:.3f} ms, "
              f"TokenConstraint.compile {total:.1f} ms", flush=True)
    return out


def kernel_table(c) -> dict:
    out = {}
    g = torch.Generator(device=DEV).manual_seed(0)
    for rows in (1, 8, 64):
        logits = (torch.randn(rows, V, generator=g, device=DEV) * 3).to(torch.bfloat16)
        zero = torch.zeros(rows, dtype=torch.int32, device=DEV)  # position 0: the states stay as they are
        t, k, p, s = sampling_tensors([SamplingParams(0.7, top_k=50, top_p=0.9, seed=i) for i in range(rows)], DEV)
        desc = torch.stack([c.descriptor()] * rows)
        res = {"sample": timed(lambda: ext.sample(logits, t, k, p, s, zero)),
               "sample_constrained": timed(lambda: ext.sample_constrained(logits, t, k, p, s, zero, desc))}
        out[rows] = res
        print(f"rows {rows}: " + ", ".join(f"{k} {v:.1f} us" for k, v in res.items()), flush=True)
    return out


def json_mask_table(jc) -> dict:
    out = {}
    for rows in (1, 8, 64):
        res = {}
        for where, text in (("in_string", b'{"name": "abc'), ("at_value", b'{"name": ')):
            w = JsonWalker()
            w.walk(text)
            tab = ConstraintRows(rows, V, DEV, json=True)
            for r in range(rows):
                tab.set_row(r, jc, w)
            res[where] = timed(lambda: ext.json_token_masks(tab.descriptors, tab.json_states, V))
        out[rows] = res
        print(f"json masks, rows {rows}: " + ", ".join(f"{k} {v:.1f} us" for k, v in res.items()), flush=True)
    return out


SCHEMA = {
    "type": "object",
    "properties": {
        "name": {"type": "string"},
        "age": {"type": "integer"},
        "email": {"type": "string", "pattern": "^[a-z]{1,16}@[a-z]{1,12}\\.com$"},
        "status": {"enum": ["active", "inactive", "pending", None]},
        "score": {"type": "number"},
        "nickname": {"type": ["string", "null"]},
        "tags": {"type": "array", "items": {"type": "string"}, "maxItems": 8},
        "address": {"type": "object", "properties": {"street": {"type": "string"}, "city": {"type": "string"}, "zip": {"type": "string"}},
                    "required": ["street", "city"]},
        "orders": {"type": "array", "items": {"type": "object", "properties": {"id": {"type": "integer"}, "qty": {"type": "integer"},
                                                                                "note": {"type": "string"}}, "required": ["id", "qty"]}},
        "comments": {"type": "array", "items": {"$ref": "#/$defs/comment"}},
        "active": {"type": "boolean"},
    },
    "required": ["name", "age", "status"],
    "$defs": {"comment": {"type": "object", "properties": {"text": {"type": "string"}, "replies": {"type": "array", "items": {"$ref": "#/$defs/comment"}}},
                          "required": ["text"]}},
}


def schema_mask_table(sc, jc) -> dict:
    """``tl_schema_token_masks`` under SCHEMA beside ``tl_json_token_masks`` on the same text, alternated per size."""
    out = {"blob_bytes": int(sc.compiled.blob.size), "staged": bool(sc.compiled.blob.size <= SCHEMA_SMEM_BYTES),
           "states": sc.compiled.num_states, "classes": sc.compiled.num_classes}
    print(f"schema tables: {out['states']} states, {out['classes']} byte classes, {out['blob_bytes']} bytes "
          f"({'staged in' if out['staged'] else 'read around'} shared memory)", flush=True)
    for rows in (1, 8, 64):
        res = {}
        for where, text in (("in_string", b'{"name": "abc'), ("at_value", b'{"name": ')):
            w = sc.start()
            assert w.walk(text)
            jw = JsonWalker()
            jw.walk(text)
            tab = ConstraintRows(rows, V, DEV, json=False, schema=True)
            jtab = ConstraintRows(rows, V, DEV, json=True)
            for r in range(rows):
                tab.set_row(r, sc, w)
                jtab.set_row(r, jc, jw)
            res[f"schema_{where}"] = timed(lambda: ext.schema_token_masks(tab.descriptors, tab.schema_states, V))
            res[f"json_{where}"] = timed(lambda: ext.json_token_masks(jtab.descriptors, jtab.json_states, V))
        out[rows] = res
        print(f"schema vs json masks, rows {rows}: " + ", ".join(f"{k} {v:.1f} us" for k, v in res.items()), flush=True)
    return out


EXPR = '''root ::= expr
expr ::= term | term "+" expr
term ::= num | "(" expr ")"
num  ::= [0-9]+'''
JSON_GBNF = r'''root   ::= object
value  ::= object | array | string | number | "true" | "false" | "null"
object ::= "{" ws ( string ":" ws value ( "," ws string ":" ws value )* )? "}" ws
array  ::= "[" ws ( value ( "," ws value )* )? "]" ws
string ::= "\"" ( [^"\\\x00-\x1F] | "\\" ( ["\\/bfnrt] | "u" [0-9a-fA-F]{4} ) )* "\"" ws
number ::= "-"? ( "0" | [1-9] [0-9]* ) ( "." [0-9]+ )? ( [eE] [-+]? [0-9]+ )? ws
ws     ::= [ \t\n]{0,8}'''
EIGHT = ('root ::= "ab" tail\ntail ::= ' + " | ".join(f"r{k}" for k in range(1, 9)) + "\n"
         + "\n".join(f'r{k} ::= "x" r{k} "{k}" | "z"' for k in range(1, 9)))


def grammar_mask_table(vocab, sc, jc) -> dict:
    """``tl_grammar_token_masks`` for three grammars, and the schema and JSON-mode kernels on JSON_GBNF's texts."""
    gs = {"expr": GrammarConstraint(EXPR, vocab, device=DEV), "json_gbnf": GrammarConstraint(JSON_GBNF, vocab, device=DEV),
          "eight": GrammarConstraint(EIGHT, vocab, device=DEV)}
    out = {"tables": {k: {"states": g.compiled.num_states, "classes": g.compiled.num_classes, "blob_bytes": int(g.compiled.blob.size),
                          "staged": bool(g.compiled.blob.size <= GRAMMAR_SMEM_BYTES)} for k, g in gs.items()}}
    print(f"grammar tables: {out['tables']}", flush=True)
    cases = [("expr_in_number", "expr", b"(12+(3"), ("expr_at_term", "expr", b"(12+"),
             ("json_gbnf_in_string", "json_gbnf", b'{"name": "abc'), ("json_gbnf_at_value", "json_gbnf", b'{"name": '),
             ("eight_parses", "eight", b"abxx")]
    for rows in (1, 8, 64):
        res = {}
        for name, key, text in cases:
            g = gs[key]
            w = g.start()
            assert w.walk(text), text
            tab = ConstraintRows(rows, V, DEV, json=False, grammar=True)
            for r in range(rows):
                tab.set_row(r, g, w)
            res[f"grammar_{name}"] = timed(lambda: ext.grammar_token_masks(tab.descriptors, tab.grammar_states, V, tab.grammar_smem_bytes))
            res[f"parses_{name}"] = len(w.parses)
        for where, text in (("in_string", b'{"name": "abc'), ("at_value", b'{"name": ')):
            w = sc.start()
            assert w.walk(text)
            jw = JsonWalker()
            jw.walk(text)
            tab = ConstraintRows(rows, V, DEV, json=False, schema=True)
            jtab = ConstraintRows(rows, V, DEV, json=True)
            for r in range(rows):
                tab.set_row(r, sc, w)
                jtab.set_row(r, jc, jw)
            res[f"schema_{where}"] = timed(lambda: ext.schema_token_masks(tab.descriptors, tab.schema_states, V, tab.schema_smem_bytes))
            res[f"json_{where}"] = timed(lambda: ext.json_token_masks(jtab.descriptors, jtab.json_states, V))
        out[rows] = res
        print(f"grammar masks, rows {rows}: " + ", ".join(f"{k} {v:.1f} us" if isinstance(v, float) else f"{k} {v}" for k, v in res.items()),
              flush=True)
    return out


def decode_rates(model, c, jc, sc, gc, B, ctx=128, steps=64, rounds=3) -> dict:
    modes = {"sampled": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1),
             "constrained": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1, constraint=c),
             "json": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1, constraint=jc),
             "schema": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1, constraint=sc),
             "grammar": SamplingParams(0.7, top_k=50, top_p=0.9, seed=1, constraint=gc)}
    msl = ctx + len(modes) * (rounds + 1) * steps + 64
    engine = DecodeEngine(model, B, msl, DEV)
    engine.reserve_pools()
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    for b in range(B):
        cache = model.create_kv_cache()
        for cc, t in zip(cache, tables):
            cc.append_slots(ctx)
            t.add_request(cc, b)
    offsets, tokens = [ctx] * B, [1] * B
    times = {m: [] for m in modes}
    for r in range(rounds + 1):
        for mode, sampling in modes.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            log = engine.decode_on_device(tokens, offsets, tables, steps, sampling=sampling)
            b.record()
            b.synchronize()
            tokens = log[-1].tolist()
            offsets = [o + steps for o in offsets]
            if r:  # round 0 captures the graphs
                times[mode].append(a.elapsed_time(b))
    res = {m: B * steps * len(v) / (sum(v) / 1e3) for m, v in times.items()}
    res["kernels_per_step"] = {"sampled": engine.kernels_per_sampled_step, "constrained": engine.kernels_per_constrained_step,
                               "json": engine.kernels_per_json_step, "schema": engine.kernels_per_schema_step,
                               "grammar": engine.kernels_per_grammar_step}
    for t in tables:  # the next engine reserves its pages from the same pools
        for cc in t.kv_caches:
            if cc is not None:
                cc.release()
    print(f"B {B}: sampled {res['sampled']:.1f} tok/s, constrained {res['constrained']:.1f} tok/s "
          f"({(res['constrained'] / res['sampled'] - 1) * 100:+.2f} %), json {res['json']:.1f} tok/s "
          f"({(res['json'] / res['sampled'] - 1) * 100:+.2f} % against sampled, {(res['json'] / res['constrained'] - 1) * 100:+.2f} % "
          f"against [a-z ]+), schema {res['schema']:.1f} tok/s ({(res['schema'] / res['json'] - 1) * 100:+.2f} % against json), "
          f"grammar {res['grammar']:.1f} tok/s ({(res['grammar'] / res['sampled'] - 1) * 100:+.2f} % against sampled)", flush=True)
    return res


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("constrained_bench needs a CUDA device")
    result = {"card": card()}
    print(f"card: {result['card']}", flush=True)
    vocab = TokenVocabulary.synthetic(V)
    result["compile"] = compile_table(vocab)
    c = TokenConstraint.compile(PATTERNS["words"], vocab, device=DEV)
    result["kernels_us"] = kernel_table(c)
    jc = JsonConstraint(vocab, device=DEV)
    result["json_masks_us"] = json_mask_table(jc)
    sc = JsonSchemaConstraint(SCHEMA, vocab, device=DEV)
    result["schema_masks_us"] = schema_mask_table(sc, jc)
    result["grammar_masks_us"] = grammar_mask_table(vocab, sc, jc)
    gc = GrammarConstraint(EXPR, vocab, device=DEV)
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=DEV)
    model = Qwen3ModelWeek3(ns, page_size=64)
    result["decode"] = {B: decode_rates(model, c, jc, sc, gc, B) for B in (1, 8)}
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(json.dumps(result, indent=1))


if __name__ == "__main__":
    main()
