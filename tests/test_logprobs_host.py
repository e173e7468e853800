"""Host tests of token log-probabilities (DESIGN.md section 8a): the float64 reference against torch, the shim's
argument checks, the C ABI declaration, and the plumbing of generate / the batcher / prompt scoring / the CLI through
the CPU stand-in of ``ext.logprobs``."""

import importlib.util
import math
import re
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from oracle import sampling as sampling_ref
from tiny_llm_b200 import Qwen3ModelWeek3, SamplingParams, TokenLogprobs, score_ids, token_logprobs
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.cli import main as cli_main
from tiny_llm_b200.generate import greedy_generate_ids
from tiny_llm_b200.synthetic import synthetic_qwen3

ROOT = Path(__file__).resolve().parent.parent


def _load_logprobs_ref():
    """The helper next to this file, by path: `tests` is no package of this project."""
    name = "tiny_llm_b200_logprobs_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("logprobs_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


ref = _load_logprobs_ref()


# ------------------------------------------------------------------ reference --
def test_reference_matches_torch_log_softmax_in_float64():
    g = np.random.default_rng(0)
    x = g.standard_normal((6, 1000)) * np.array([[0.1], [1], [3], [10], [30], [1e4]])
    want = torch.log_softmax(torch.from_numpy(x), dim=-1).numpy()
    for r in range(x.shape[0]):
        t = int(g.integers(0, 1000))
        lse, lp, rank, ids, lps = ref.row(x[r], t, 20)
        assert lp == pytest.approx(want[r, t], rel=1e-12, abs=1e-9)
        assert lse == pytest.approx(float(torch.logsumexp(torch.from_numpy(x[r]), 0)), rel=1e-12)
        assert rank == 1 + int((x[r] > x[r, t]).sum())
        top = torch.topk(torch.from_numpy(want[r]), 20)
        assert ids.tolist() == top.indices.tolist()
        np.testing.assert_allclose(lps, top.values.numpy(), rtol=1e-12, atol=1e-9)


def test_reference_ties_go_to_the_lower_id():
    x = np.zeros(50)
    lse, lp, rank, ids, lps = ref.row(x, 7, 5)
    assert ids.tolist() == [0, 1, 2, 3, 4] and rank == 1
    assert lp == pytest.approx(-math.log(50)) and np.allclose(lps, -math.log(50))
    x = np.array([1.0, 3.0, 2.0, 3.0, 2.0, 2.0, 0.0])
    assert ref.row(x, 5, 4)[3].tolist() == [1, 3, 2, 4]  # the tie at the 3rd place straddles the list's end
    assert ref.row(x, 5, 4)[2] == 3


def test_reference_nan_and_minus_inf_rules():
    x = np.array([np.nan, 1.0, -np.inf, 1.0, np.nan, 0.0])
    lse, lp, rank, ids, lps = ref.row(x, 2, 6)
    assert lse == pytest.approx(math.log(2 * math.e + 1))
    assert lp == -np.inf and rank == 4  # -inf is an ordinary entry; NaN never counts
    assert ids.tolist() == [1, 3, 5, 2, -1, -1] and lps[3] == -np.inf and lps[4] == -np.inf
    lse, lp, rank, _, _ = ref.row(x, 0, 0)
    assert math.isnan(lp) and rank == 0
    lse, lp, rank, _, _ = ref.row(x, -1, 0)
    assert math.isnan(lp) and rank == 0


def test_reference_rows_without_a_finite_maximum():
    for x, lse_want in (([1.0, np.inf, 2.0], np.inf), ([-np.inf, -np.inf], -np.inf), ([np.nan, np.nan], np.nan)):
        lse, lp, rank, ids, lps = ref.row(np.array(x), 0, 2)
        assert (math.isnan(lse) and math.isnan(lse_want)) or lse == lse_want
        assert math.isnan(lp) or rank == 0
    _, _, rank, ids, lps = ref.row(np.array([1.0, np.inf, 2.0]), 0, 2)
    assert rank == 3 and ids.tolist() == [1, 2] and np.isnan(lps).all()
    _, _, rank, ids, lps = ref.row(np.array([np.nan, np.nan]), 0, 2)
    assert rank == 0 and ids.tolist() == [-1, -1] and (lps == -np.inf).all()


def test_bound_is_tight_on_exact_rows():
    # 2^j equal maxima, the rest -inf: lp = -j ln 2 and the bound is a few ulp of it
    x = np.full(64, -np.inf)
    x[:8] = 3.0
    lp_b, lse_b = ref.bound(x)
    assert lp_b[0] < 1e-6 and lse_b < 1e-6


# ------------------------------------------------------------------ shim and ABI --
def test_shim_checks_arguments():
    x = torch.zeros(2, 8)
    with pytest.raises(RuntimeError, match="expected 2D float logits"):
        ext.logprobs(torch.zeros(8))
    with pytest.raises(RuntimeError, match="expected 2D float logits"):
        ext.logprobs(torch.zeros(2, 8, dtype=torch.int32))
    with pytest.raises(RuntimeError, match=r"max_n must be an integer in \[0, 20\]"):
        ext.logprobs(x, max_n=21)
    with pytest.raises(RuntimeError, match=r"max_n must be an integer in \[0, 20\]"):
        ext.logprobs(x, max_n=-1)
    with pytest.raises(RuntimeError, match=r"targets must be int32 \[2\]"):
        ext.logprobs(x, targets=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(RuntimeError, match=r"top_n must be int32 \[2\]"):
        ext.logprobs(x, top_n=torch.zeros(3, dtype=torch.int32), max_n=2)
    with pytest.raises(RuntimeError, match="out_index needs out"):
        ext.logprobs(x, out_index=torch.zeros(1, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="logprobs: the course extension is GPU-only"):
        ext.logprobs(x, targets=torch.zeros(2, dtype=torch.int32), max_n=3)


def test_abi_declares_and_exports_tl_logprobs():
    header = (ROOT / "include" / "tiny_llm_b200.h").read_text()
    decl = re.search(r"int tl_logprobs\(([^)]*)\);", header)
    assert decl is not None and "#define TL_LOGPROBS_MAX_N 20" in header
    params = [p.strip() for p in decl.group(1).split(",")]
    restype, argtypes = ext._SIGNATURES["tl_logprobs"]
    assert len(params) == len(argtypes) == 15
    assert ext.LOGPROBS_MAX_N == 20 and "logprobs" in ext.__all__ and "tl_logprobs" in ext.EXPORTED_SYMBOLS
    assert hasattr(ext._lib, "tl_logprobs")


# ------------------------------------------------------------------ plumbing --
@pytest.fixture
def cpu_lp(cpu_ext, monkeypatch):
    """``cpu_ext`` with the float64 references of ``tl_logprobs`` and ``tl_sample``."""
    monkeypatch.setattr(cpu_ext, "logprobs", ref.logprobs_like_ext)
    monkeypatch.setattr(cpu_ext, "sample", sampling_ref.sample_like_ext)
    return cpu_ext


@pytest.fixture(scope="module")
def ns():
    return synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)


PROMPTS = [[5, 17, 3, 250], [9, 2, 4, 6, 8, 11], [300, 1, 77], [42] * 9]


def _teacher_forced(ns, ids):
    """The per-token entries of ``ids[1:]`` from one scoring pass (no top list)."""
    return score_ids(Qwen3ModelWeek3(ns, page_size=16), ids, chunk=5, device="cpu").entries


# The bf16 model rounds a token's activations differently in another chunking, so the same row's log-probabilities
# agree to TOL, not bit for bit; a row off by one position is several nats away.
TOL = 0.1


def _check_against_scoring(ns, prompt, generated, entries):
    assert [e.token for e in entries] == list(generated)
    scored = _teacher_forced(ns, list(prompt) + list(generated))[len(prompt) - 1 :]
    assert len(scored) == len(entries)
    for e, s in zip(entries, scored):
        assert e.token == s.token
        assert e.logprob == pytest.approx(s.logprob, abs=TOL)


def test_token_logprobs_entry(cpu_lp):
    logits = torch.tensor([[0.0, 2.0, 1.0, 2.0], [5.0, 0.0, 0.0, 0.0]])
    a, b = token_logprobs(logits, [2, -1], 2)
    assert isinstance(a, TokenLogprobs) and a.token == 2 and a.rank == 3 and [i for i, _ in a.top] == [1, 3]
    assert a.logprob == pytest.approx(1 - math.log(1 + 2 * math.e**2 + math.e), rel=1e-6)
    assert b.rank == 0 and math.isnan(b.logprob) and b.top[0][0] == 0


def test_generate_without_logprobs_is_unchanged(cpu_lp, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    ids = greedy_generate_ids(model, PROMPTS[0], 5, device="cpu")
    assert isinstance(ids, list)
    out, entries = greedy_generate_ids(model, PROMPTS[0], 5, device="cpu", logprobs=3)
    assert out == ids and len(entries) == 5
    for e in entries:  # greedy: the chosen token is the most likely one and heads its own list
        assert e.rank == 1 and e.top[0] == (e.token, e.logprob) and len(e.top) == 3
    _check_against_scoring(ns, PROMPTS[0], out, entries)


def test_generate_logprobs_follow_sampled_tokens(cpu_lp, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    params = SamplingParams(1.5, seed=4)
    ids = greedy_generate_ids(model, PROMPTS[1], 6, device="cpu", sampling=params)
    out, entries = greedy_generate_ids(model, PROMPTS[1], 6, device="cpu", sampling=params, logprobs=0)
    assert out == ids and all(e.top == () for e in entries)
    _check_against_scoring(ns, PROMPTS[1], out, entries)


def test_generate_refuses_bad_counts(cpu_lp, ns):
    model = Qwen3ModelWeek3(ns, page_size=16)
    for bad in (21, -1, 2.0, True):
        with pytest.raises(ValueError, match="logprobs must be an int"):
            greedy_generate_ids(model, PROMPTS[0], 2, device="cpu", logprobs=bad)


def _batch(ns, prompts, **kw):
    model = Qwen3ModelWeek3(ns, page_size=16)
    b = ContinuousBatcher(model, None, prompts, max_seq_len=64, batch_size=2, prefill_step=3, verbose=False,
                          max_new_tokens=[5] * len(prompts), device="cpu", **kw)
    out = dict(b.run())
    return out, b


@pytest.mark.parametrize("sampling", [None, SamplingParams(1.2, top_k=30, seed=7)])
def test_batcher_entries_line_up_with_tokens(cpu_lp, ns, sampling):
    plain, _ = _batch(ns, PROMPTS, sampling=sampling)
    out, b = _batch(ns, PROMPTS, sampling=sampling, logprobs=2)
    assert out == plain and sorted(b.logprobs) == list(range(len(PROMPTS)))
    for idx, prompt in enumerate(PROMPTS):
        generated = [int(t) for t in out[idx].split()]
        _check_against_scoring(ns, prompt, generated, b.logprobs[idx])  # the first entry: the last prefill chunk's row


def test_score_ids_chunks_agree_and_add_up(cpu_lp, ns):
    ids = [5, 17, 3, 250, 9, 2, 4, 6, 8, 11, 300]
    model = Qwen3ModelWeek3(ns, page_size=16)
    whole = score_ids(model, ids, chunk=64, top_n=3, device="cpu")
    pieces = score_ids(model, ids, chunk=4, top_n=3, device="cpu")
    assert [e.token for e in whole.entries] == ids[1:] and len(whole.next_top) == 3
    for a, b in zip(whole.entries, pieces.entries):
        assert a.token == b.token and a.logprob == pytest.approx(b.logprob, abs=TOL)
    assert whole.nll == pytest.approx(-sum(e.logprob for e in whole.entries))
    assert whole.perplexity == pytest.approx(math.exp(whole.nll / (len(ids) - 1)))
    # the last row is the first generated token's distribution
    first = greedy_generate_ids(model, ids, 1, device="cpu", logprobs=3)[1][0]
    assert first.top[0][0] == whole.next_top[0][0] and first.logprob == pytest.approx(whole.next_top[0][1], abs=TOL)


def test_cli_prints_logprobs_and_perplexity(cpu_lp, capsys):
    common = ["--synthetic", "tiny-d128", "--device", "cpu", "--logprobs", "2"]
    assert cli_main(["generate", "--prompt-ids", "5,17,3", "--max-new-tokens", "3", *common]) == 0
    out = capsys.readouterr().out
    assert out.count("logprob ") == 3 and "rank 1" in out
    assert cli_main(["batch", "--prompt-ids", "5,17,3;9,2,4", "--max-new-tokens", "3", "--quiet", "--max-seq-len", "64", *common]) == 0
    out = capsys.readouterr().out
    assert out.count("logprob ") == 6 and "--- request 1" in out
    assert cli_main(["score", "--prompt-ids", "5,17,3,250,9", "--chunk", "2", *common]) == 0
    out = capsys.readouterr().out
    assert out.count("logprob ") == 4 and "perplexity" in out and "next token:" in out
    with pytest.raises(SystemExit):
        cli_main(["score", "--prompt-ids", "5,17", "--synthetic", "tiny-d128", "--device", "cpu", "--logprobs", "21"])


# ------------------------------------------------------------------ the absorption rows --
def _plan(V):
    """``sample_plan``: CTAs per row and entries per CTA."""
    c = min(-(-V // 4096), 8)
    return c, -(-(-(-V // c)) // 8) * 8


def _kernel_order_lse(x, fixed_point: bool) -> float:
    """``lse`` of the kernel's layout (C CTAs of 512 threads, thread t of a CTA summing entries t, t + 512, ... of its
    slice, a warp butterfly, the 16 warps in order, then the CTAs in order) with the masses summed either as the
    kernel sums them (2^-40 fixed point, exact) or in fp32 in that order."""
    V = len(x)
    C, s = _plan(V)
    x32 = x.astype(np.float32)
    m = np.float32(x32.max())
    e = np.exp((x32 - m).astype(np.float32)).astype(np.float32)
    if fixed_point:
        total = np.float32(float(np.rint(e.astype(np.float64) * 2.0**40).sum()) * 2.0**-40)
    else:
        total = np.float32(0)
        for r in range(C):
            part = e[r * s : min(V, (r + 1) * s)]
            threads = np.zeros(512, np.float32)
            for t in range(512):
                acc = np.float32(0)
                for v in part[t::512]:
                    acc = np.float32(acc + v)
                threads[t] = acc
            w = threads.reshape(16, 32)
            for o in (16, 8, 4, 2, 1):
                w = (w + w[:, np.arange(32) ^ o]).astype(np.float32)
            cta = np.float32(0)
            for k in range(16):
                cta = np.float32(cta + w[k, 0])
            total = np.float32(total + cta)
    return float(np.float32(m + np.float32(np.log(total))))


@pytest.mark.parametrize("V,level", [(4097, -17.0), (151936, -17.0), (151936, -17.5)])
def test_absorption_rows_separate_a_thread_order_fp32_sum(V, level):
    # the GPU test's absorption rows: an fp32 sum in the kernel's thread order leaves the bound, the fixed-point sum not
    x = np.full(V, level)
    x[0] = 0.0
    lse = ref.row(x, -1, 0)[0]
    _, bound = ref.bound(x)
    assert abs(_kernel_order_lse(x, fixed_point=True) - lse) <= bound
    assert abs(_kernel_order_lse(x, fixed_point=False) - lse) > 2 * bound


def test_shim_passes_the_log_capacity(monkeypatch):
    """The log capacity reaches the kernel, which writes nothing for an index outside it."""
    seen = {}

    class FakeLib:
        def tl_logprobs(self, *args):
            seen["args"] = args
            return 0

    monkeypatch.setattr(ext, "_lib", FakeLib())
    monkeypatch.setattr(ext, "_gpu", lambda *a: None)
    monkeypatch.setattr(ext, "_stream_ptr", lambda *a: 0)
    x = torch.zeros(3, 8)
    out = (torch.zeros(5, 3), torch.zeros(5, 3), torch.zeros(5, 3, dtype=torch.int32), torch.zeros(5, 3, 2, dtype=torch.int32),
           torch.zeros(5, 3, 2))
    ext.logprobs(x, None, None, 2, out=out, out_index=torch.zeros(1, dtype=torch.int32))
    assert seen["args"][9:13] == (3, 8, 2, 5)  # rows, vocab, max_n, out_capacity
    ext.logprobs(x, None, None, 2)
    assert seen["args"][3] is None and seen["args"][12] == 1


def test_batch_generate_returns_the_entries_with_logprobs(cpu_lp, ns):
    from tiny_llm_b200 import batch_generate

    kw = dict(max_seq_len=64, batch_size=2, prefill_step=3, verbose=False, max_new_tokens=[4] * len(PROMPTS), device="cpu")
    plain = batch_generate(Qwen3ModelWeek3(ns, page_size=16), None, PROMPTS, **kw)
    results, logprobs = batch_generate(Qwen3ModelWeek3(ns, page_size=16), None, PROMPTS, logprobs=1, **kw)
    assert results == plain
    for idx, text in results:
        assert [e.token for e in logprobs[idx]] == [int(t) for t in text.split()] and all(len(e.top) == 1 for e in logprobs[idx])
