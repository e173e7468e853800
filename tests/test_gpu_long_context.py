"""YaRN RoPE scaling and long context windows on the GPU.

1. Every RoPE site given a YaRN table against float64 RoPE (``yarn_ref.py``) at positions up to 131,071, at every dtype it
   takes, within a bound derived from the fp32 angle (half an ulp of the angle), the fp32 trig and one output rounding.
2. Every site given the unscaled table (``ext.rope_default_inv_freq``) returns exactly the bits of its ``base`` path.
3. A ``tiny-d128`` model with YaRN: decode and chunk graphs equal the independent launch plan (``engine_plan.py``, given the
   table) bit for bit; graphs, operator path and the CPU oracle with the float64 table agree; speculative decoding with a
   YaRN target and draft gives greedy's ids.
4. Windows: a reservation that cannot fit is refused before anything is allocated.
Each test stays well under 16 GB of device memory."""

import importlib.util
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3
from tiny_llm_b200.engine import DecodeEngine, PrefillEngine
from tiny_llm_b200.generate import greedy_generate_ids, speculative_generate_ids
from tiny_llm_b200.rope_scaling import parse_rope_scaling, rope_inv_freq
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


ref = _load("tiny_llm_b200_yarn_ref", "yarn_ref.py")
plan = _load("tiny_llm_b200_engine_plan", "engine_plan.py")

POSITIONS = [0, 1, 32767, 32768, 40960, 65535, 131071]
QWEN3_YARN = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 32768}
BF, F16, F32 = torch.bfloat16, torch.float16, torch.float32


@pytest.fixture(scope="module")
def dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return torch.device("cuda:0")


def _table(dev, D=128, theta=1e6):
    t = rope_inv_freq(D, theta, parse_rope_scaling(QWEN3_YARN, 40960), dev)
    np.testing.assert_allclose(t.cpu().numpy(), ref.yarn_table(theta, D, 4.0, 32768)[0], rtol=1e-14, atol=0)
    return t


def _assert_rope(got, x, positions, table, dtype, what):
    """``got`` [rows, H, D] against float64 RoPE of ``x`` [rows, H, D] at one position per row."""
    inv = table.cpu().numpy()
    pos = torch.tensor(positions, dtype=torch.float64, device=x.device)
    want = ref.rope_f64(x, pos, inv)
    bound = ref.rope_bound(x, pos, inv, dtype)
    err = (got.double() - want).abs()
    bad = err > bound
    assert not bad.any(), f"{what}: {int(bad.sum())} elements beyond the bound; worst excess {float((err - bound).max()):.3g}"


def _qk_setup(dev, dtype, rows, Hq=4, Hkv=2, D=128, page=16, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    qkv = torch.randn(rows, (Hq + 2 * Hkv) * D, generator=g, device=dev).to(dtype)
    qw = (1 + 0.1 * torch.randn(D, generator=g, device=dev)).to(dtype)
    kw = (1 + 0.1 * torch.randn(D, generator=g, device=dev)).to(dtype)
    pages = -(-rows // page) + 1
    kp = torch.zeros(pages * rows, Hkv, page, D, dtype=dtype, device=dev)
    vp = torch.zeros_like(kp)
    return qkv, qw, kw, kp, vp


def _normed(qkv, w, heads, start, D, eps):
    """The q or k heads of ``qkv`` through ``rms_norm`` (the rounding point every fused site keeps)."""
    x = qkv.view(qkv.shape[0], -1, D)[:, start : start + heads].contiguous()
    return ext.rms_norm(x, w, eps)


# ---------------------------------------------------------------- 1 + 2: sites --
@pytest.mark.parametrize("dtype", [F32, F16, BF])
@pytest.mark.parametrize("L", [1, 16])  # 7 x 1 rows: the per-element kernel; 7 x 16: the per-(token, pair) kernel
def test_rope_table_against_float64_and_default_bits(dev, dtype, L):
    table = _table(dev)
    B, H, D = len(POSITIONS), 4, 128
    g = torch.Generator(device=dev).manual_seed(L)
    x = torch.randn(B, L, H, D, generator=g, device=dev).to(dtype)
    off = torch.tensor(POSITIONS, dtype=torch.int32, device=dev)
    assert ext.rope_route(B, L, H, D, D, dtype) == (ext.ROPE_ELEMENT if L == 1 else ext.ROPE_HEADS)
    got = ext.rope_table(x, off, D, table)
    pos = [p + l for p in POSITIONS for l in range(L)]
    _assert_rope(got.reshape(B * L, H, D), x.reshape(B * L, H, D), pos, table, dtype, f"rope_table {dtype} L {L}")
    plain = ext.rope_default_inv_freq(D, 1e6, dev)
    assert torch.equal(ext.rope_table(x, off, D, plain), ext.rope(x, off, D, 1e6))


@pytest.mark.parametrize("dtype", [F32, BF])  # bf16 D 128: the row kernel; f32: the per-head kernel
@pytest.mark.parametrize("form", ["decode", "chunk"])
def test_qk_norm_rope_append_against_float64_and_default_bits(dev, dtype, form):
    table = _table(dev)
    Hq, Hkv, D, page, eps = 4, 2, 128, 16, 1e-6
    rows = len(POSITIONS)
    qkv, qw, kw, kp, vp = _qk_setup(dev, dtype, rows)
    off = torch.tensor(POSITIONS, dtype=torch.int32, device=dev)
    if form == "decode":  # one request per row, each at its own page
        bt = torch.arange(rows, dtype=torch.int32, device=dev).view(rows, 1).contiguous()
        ctx = torch.ones(rows, dtype=torch.int32, device=dev)
        slot = [(r, 0) for r in range(rows)]
        call = ext.decode_qk_norm_rope_append
    else:  # consecutive tokens of one request
        bt = torch.arange(kp.shape[0], dtype=torch.int32, device=dev)
        ctx = torch.arange(1, rows + 1, dtype=torch.int32, device=dev)
        slot = [(r // page, r % page) for r in range(rows)]
        call = ext.chunk_qk_norm_rope_append
    q = call(qkv, qw, kw, off, bt, ctx, kp, vp, Hq, Hkv, 1e6, eps, inv_freq=table)
    q = q if form == "decode" else q.transpose(0, 1)
    _assert_rope(q, _normed(qkv, qw, Hq, 0, D, eps), POSITIONS, table, dtype, f"{form} q {dtype}")
    k = torch.stack([kp[p, :, s] for p, s in slot])
    _assert_rope(k, _normed(qkv, kw, Hkv, Hq, D, eps), POSITIONS, table, dtype, f"{form} k {dtype}")
    v = torch.stack([vp[p, :, s] for p, s in slot])
    assert torch.equal(v, qkv.view(rows, -1, D)[:, Hq + Hkv :])
    # the unscaled table gives the base path's bits (q and the appended pages)
    plain = ext.rope_default_inv_freq(D, 1e6, dev)
    kp2, vp2 = torch.zeros_like(kp), torch.zeros_like(vp)
    kp3, vp3 = torch.zeros_like(kp), torch.zeros_like(vp)
    a = call(qkv, qw, kw, off, bt, ctx, kp2, vp2, Hq, Hkv, 1e6, eps, inv_freq=plain)
    b = call(qkv, qw, kw, off, bt, ctx, kp3, vp3, Hq, Hkv, 1e6, eps)
    assert torch.equal(a, b) and torch.equal(kp2, kp3) and torch.equal(vp2, vp3)


@pytest.mark.parametrize("rows", [7, 16])  # 7: q|k|v materialised; 16: split-reduction planes feed the norm / RoPE kernel
@pytest.mark.parametrize("chunk", [False, True])
def test_qkv_project_rope_append_against_float64_and_default_bits(dev, rows, chunk):
    table = _table(dev)
    Hq, Hkv, D, N, page, eps = 4, 2, 128, 256, 16, 1e-6
    K = (Hq + 2 * Hkv) * D
    g = torch.Generator().manual_seed(rows)
    words = torch.randint(-(2**31), 2**31, (K, N // 8), dtype=torch.int64, generator=g).to(torch.int32).to(dev)
    scales = (torch.randn(K, N // 128, generator=g) * 0.02).to(BF).to(dev)
    biases = (-7.5 * scales.float().cpu() + torch.randn(K, N // 128, generator=g) * 0.02).to(BF).to(dev)
    p0 = torch.randn(rows, N, generator=g).to(BF).to(dev)
    qw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF).to(dev)
    kw = (1 + 0.1 * torch.randn(D, generator=g)).to(BF).to(dev)
    positions = [POSITIONS[r % len(POSITIONS)] for r in range(rows)]
    off = torch.tensor(positions, dtype=torch.int32, device=dev)
    if chunk:
        kp = torch.zeros(-(-rows // page) + 1, Hkv, page, D, dtype=BF, device=dev)
        bt = torch.arange(kp.shape[0], dtype=torch.int32, device=dev)
        ctx = torch.arange(1, rows + 1, dtype=torch.int32, device=dev)
        slot = [(r // page, r % page) for r in range(rows)]
    else:
        kp = torch.zeros(rows, Hkv, page, D, dtype=BF, device=dev)
        bt = torch.arange(rows, dtype=torch.int32, device=dev).view(rows, 1).contiguous()
        ctx = torch.ones(rows, dtype=torch.int32, device=dev)
        slot = [(r, 0) for r in range(rows)]
    vp = torch.zeros_like(kp)
    q = ext.qkv_project_rope_append(scales, biases, words, p0, qw, kw, off, bt, ctx, kp, vp, Hq, Hkv, 1e6, eps, chunk=chunk, inv_freq=table)
    q = q.transpose(0, 1) if chunk else q
    qkv = ext.quantized_matmul_fused(scales, biases, words, p0)  # the projection's own result
    _assert_rope(q, _normed(qkv, qw, Hq, 0, D, eps), positions, table, BF, f"qkv_project q rows {rows} chunk {chunk}")
    k = torch.stack([kp[p, :, s] for p, s in slot])
    _assert_rope(k, _normed(qkv, kw, Hkv, Hq, D, eps), positions, table, BF, f"qkv_project k rows {rows} chunk {chunk}")
    plain = ext.rope_default_inv_freq(D, 1e6, dev)
    outs = []
    for extra in ({"inv_freq": plain}, {}):
        kp2, vp2 = torch.zeros_like(kp), torch.zeros_like(vp)
        outs.append((ext.qkv_project_rope_append(scales, biases, words, p0, qw, kw, off, bt, ctx, kp2, vp2, Hq, Hkv, 1e6, eps, chunk=chunk, **extra),
                     kp2, vp2))
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_decode_attention_fused_appends_yarn_keys(dev):
    """The fused decode attention reads the same table: the key it appends at each probe position."""
    table = _table(dev)
    Hq, Hkv, D, page, eps = 4, 2, 128, 16, 1e-6
    rows = len(POSITIONS)
    qkv, qw, kw, kp, vp = _qk_setup(dev, BF, rows)
    off = torch.tensor(POSITIONS, dtype=torch.int32, device=dev)
    bt = torch.arange(rows, dtype=torch.int32, device=dev).view(rows, 1).contiguous()
    ctx = torch.ones(rows, dtype=torch.int32, device=dev)
    ext.decode_attention_fused(qkv, qw, kw, off, bt, ctx, table, kp, vp, Hq, Hkv, eps, 128**-0.5, page)
    k = kp[:rows, :, 0]
    _assert_rope(k, _normed(qkv, kw, Hkv, Hq, D, eps), POSITIONS, table, BF, "decode_attention_fused k")


# ------------------------------------------------------------------ 3: model --
SMALL_YARN = {"rope_type": "yarn", "factor": 4.0, "original_max_position_embeddings": 64}  # interpolation acts at test lengths


def _ns(dev, seed=0, **kw):
    return synthetic_qwen3("tiny-d128", seed=seed, device=dev, realistic=True, max_position_embeddings=512, rope_scaling=SMALL_YARN, **kw)


class _TableExt:
    """``ext`` as the plan calls it, with the model's table passed to every RoPE site (the plan names ``base``)."""

    def __init__(self, table):
        self._t = table

    def __getattr__(self, name):
        return getattr(ext, name)

    def decode_qk_norm_rope_append(self, *a, **k):
        return ext.decode_qk_norm_rope_append(*a, **k, inv_freq=self._t)

    def chunk_qk_norm_rope_append(self, *a, **k):
        return ext.chunk_qk_norm_rope_append(*a, **k, inv_freq=self._t)

    def qkv_project_rope_append(self, *a, **k):
        return ext.qkv_project_rope_append(*a, **k, inv_freq=self._t)

    def paged_attention_token_major(self, q, kp, vp, table, *a, **k):  # the chunk engine's split above 8,192 keys
        ws = ext.paged_attention_token_major_workspace(q.shape[0], q.shape[1], kp.shape[2], table.shape[1])
        w = torch.empty(ws, dtype=torch.uint8, device=q.device) if ws else None
        return ext.paged_attention_token_major(q, kp, vp, table, *a, **k, workspace=w)


def _plan(model, monkeypatch):
    monkeypatch.setattr(plan, "ext", _TableExt(model.rope_inv_freq))
    P = plan.Plan(model)
    P.inv_freq = model.rope_inv_freq
    assert P.scale == model.layers_inner[0].self_attn.scale
    return P


@pytest.mark.parametrize("msl", [256, 32768])  # fused attention; past 16K slot-tokens, norm/RoPE/append + paged attention
def test_yarn_decode_and_chunk_graphs_equal_the_plan(dev, monkeypatch, msl):
    model = Qwen3ModelWeek3(_ns(dev), page_size=64)  # 64-slot pages: the chunk's wgmma attention, split at msl 32768
    P = _plan(model, monkeypatch)
    pre = PrefillEngine(model, 32, msl, dev)
    assert (pre._attn_ws is not None) == (msl > 8192)
    pre.reserve_pools(2 * pre.max_pages + 2)
    cache = model.create_kv_cache()
    g = torch.Generator().manual_seed(3)
    for r in (32, 32, 13):
        ids = torch.randint(1, model.vocab_size, (r,), generator=g).tolist()
        off = cache[0].offset
        before = [(p._key_pages.clone(), p._value_pages.clone()) for p in model.page_pools]
        pre.prefill_chunk(ids, off, cache)
        meta = plan.prefill_metadata(cache, ids, off, 32, pre.max_pages)
        logits, nxt = P.prefill(meta, before)
        assert torch.equal(pre.logits, logits), f"chunk at {off}: logits differ from the plan"
        for p, (k, v) in zip(model.page_pools, before):
            assert torch.equal(p._key_pages, k) and torch.equal(p._value_pages, v)
    dec = DecodeEngine(model, 1, msl, dev)
    dec.reserve_pools(2 * dec.max_pages + 2)
    assert dec._attention_fused == (msl <= 16384)
    assert not dec._attention_fused or dec._rope_inv_freq is model.rope_inv_freq
    tok = int(nxt)
    for _ in range(3):
        before = [(p._key_pages.clone(), p._value_pages.clone()) for p in model.page_pools]
        dec.step([tok], [cache[0].offset], cache)
        meta = plan.decode_metadata(cache, [tok], dec.max_pages)
        logits, nxt = P.decode(meta, before, dec._attention_fused, rows=1)
        assert torch.equal(dec.logits[:1], logits), "decode step differs from the plan"
        for p, (k, v) in zip(model.page_pools, before):
            assert torch.equal(p._key_pages, k) and torch.equal(p._value_pages, v)
        tok = int(nxt[0])


def test_yarn_model_paths_and_oracle_agree(dev):
    ns_cpu = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, rope_scaling=SMALL_YARN)
    oracle = ref.yarn_reference_model(ns_cpu, 4.0, 64)
    from oracle.model import greedy_decode

    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11] * 12  # 108 tokens: past L0 = 64, where interpolation acts
    ref_tokens, ref_lp = greedy_decode(oracle, prompt, 6, return_logprobs=True)
    for graphs in (True, False):
        model = Qwen3ModelWeek3(_ns(dev), page_size=16)
        model.set_max_context(512)
        if not graphs:
            model.use_decode_graph = False
        else:
            model.prefill_graph_len = 32
            model.decode_engine(1)  # reserve, so prefill chunks take the chunk graph
        cache = model.create_kv_cache()
        feed, offset = prompt, 0
        steps = []
        for tok, lp_ref in zip(ref_tokens, ref_lp):
            while feed:  # 32-token pieces: the chunk graph when graphs are on
                piece, feed = feed[:32], feed[32:]
                logits = model(torch.tensor([piece], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1)[0, -1].float().cpu()
                offset += len(piece)
            lp = logits - torch.logsumexp(logits, dim=-1)
            top = torch.topk(lp_ref, 4).indices
            torch.testing.assert_close(lp[top], lp_ref[top], rtol=0, atol=0.25)
            steps.append(int(lp.argmax()))
            feed = [tok]
        assert steps == ref_tokens, f"graphs={graphs}: greedy ids {steps} differ from the float64-table oracle's {ref_tokens}"
        for c in cache:
            c.release()


def test_speculative_decoding_with_yarn_target_and_draft_matches_greedy(dev):
    target = Qwen3ModelWeek3(_ns(dev), page_size=16)
    target.set_max_context(512)
    draft = Qwen3ModelWeek3(_ns(dev, seed=1), page_size=16)
    draft.set_max_context(512)
    prompt = list(range(3, 83))
    want = greedy_generate_ids(target, prompt, 24, device=dev)
    got, stats = speculative_generate_ids(draft, target, prompt, 24, proposal_length=4, device=dev)
    assert list(got) == list(want)
    assert target._verify_engines, "the verify graph did not run"


# ------------------------------------------------------- 5: split chunk attention --
def _attention_f64(q, kp, vp, pages, ctx, L, G, scale):
    """float64 causal attention of the chunk's rows (query row l sees keys [0, ctx - L + l]) -> [L, Hq, D], and the bound
    sum_j p_j |v_j| per element (the scale of the bf16 rounding of P and of the output)."""
    Hq, _, D = q.shape
    Hkv = kp.shape[1]
    out = torch.empty(L, Hq, D, dtype=torch.float64, device=q.device)
    mag = torch.empty_like(out)
    last = torch.arange(ctx - L, ctx, device=q.device)
    keys = torch.arange(ctx, device=q.device)
    mask = keys[None, :] > last[:, None]
    for h in range(Hkv):
        k = kp[pages, h].reshape(-1, D)[:ctx].double()
        v = vp[pages, h].reshape(-1, D)[:ctx].double()
        for g in range(G):
            hq = h * G + g
            s = (q[hq].double() @ k.T) * scale
            s.masked_fill_(mask, float("-inf"))
            p = torch.softmax(s, dim=-1)
            out[:, hq] = p @ v
            mag[:, hq] = p @ v.abs()
    return out, mag


@pytest.mark.parametrize("prefix", [1000, 16384, 65536, 131072 - 128])
def test_split_chunk_attention_against_float64(dev, prefix):
    """A 128-row chunk after ``prefix`` keys, Qwen3-4B heads, a block table of 131,072 + 128 keys: split (two launches,
    token-major merge) and unsplit both within the bound of float64.  At prefix 1,000 every split holds one 64-key tile,
    so the last split lies wholly past the last visible key of the early rows of a query block (an empty partial)."""
    Hq, Hkv, D, page, L = 32, 8, 128, 128, 128
    G, scale = Hq // Hkv, D**-0.5
    max_pages = 131072 // page + 1
    ctx = prefix + L
    n = -(-ctx // page)
    g = torch.Generator(device=dev).manual_seed(prefix)
    kp = torch.randn(n, Hkv, page, D, generator=g, device=dev).to(BF)
    vp = torch.randn(n, Hkv, page, D, generator=g, device=dev).to(BF)
    q = (3 * torch.randn(Hq, L, D, generator=g, device=dev)).to(BF)  # peaked scores: outputs well above the rounding
    table = torch.full((1, max_pages), -1, dtype=torch.int32, device=dev)
    table[0, :n] = torch.randperm(n, device=dev, generator=g).to(torch.int32)
    cl = torch.tensor([ctx], dtype=torch.int32, device=dev)
    ws_bytes = ext.paged_attention_token_major_workspace(Hq, L, page, max_pages)
    assert ws_bytes == Hq * L * 32 * (D + 2) * 4
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    n0 = ext.launch_count()
    split = ext.paged_attention_token_major(q, kp, vp, table, cl, scale, True, Hkv, Hq, workspace=ws)
    assert ext.launch_count() - n0 == 2, "the split form is the attention launch plus the merge"
    n0 = ext.launch_count()
    plain = ext.paged_attention_token_major(q, kp, vp, table, cl, scale, True, Hkv, Hq)
    assert ext.launch_count() - n0 == 1
    want, mag = _attention_f64(q, kp, vp, table[0, :n].long(), ctx, L, G, scale)
    bound = 2.0**-7 * mag + 2.0**-8 * want.abs() + 1e-6
    for name, got in (("split", split), ("unsplit", plain)):
        err = (got.view(L, Hq, D).double() - want).abs()
        assert not (err > bound).any(), f"{name} at prefix {prefix}: worst excess {float((err - bound).max()):.3g}"


def test_windows_up_to_8192_never_split(dev):
    for max_pages, page in ((64, 128), (128, 64), (8192 // 16, 16)):
        assert ext.paged_attention_token_major_workspace(32, 128, page, max_pages) == 0
    assert ext.paged_attention_token_major_workspace(32, 128, 128, 65) > 0
    model = Qwen3ModelWeek3(_ns(dev), page_size=64)
    assert PrefillEngine(model, 32, 8192, dev)._attn_ws is None
    assert PrefillEngine(model, 32, 8256, dev)._attn_ws is not None


# ---------------------------------------------------------------- 4: windows --
def test_long_window_prompt_in_one_call_and_decode_at_131071(dev, monkeypatch):
    """One-layer Qwen3-4B-shaped model with YaRN and a 131,072-token window: a 131,071-token prompt in one call (run as
    8,192-token pieces) against the same prompt fed in 16 calls, then the B = 1 decode graph at position 131,071 against
    its launch plan."""
    W = 131072
    ns = synthetic_qwen3("qwen3-4b", seed=0, device=dev, num_hidden_layers=1, rope_scaling=QWEN3_YARN)
    model = Qwen3ModelWeek3(ns, page_size=128, max_context=W)
    ids = torch.randint(1, 151936, (1, W - 1), generator=torch.Generator().manual_seed(5), dtype=torch.int64).to(torch.int32).to(dev)
    assert model._needs_pieces(1, W - 1, 1) and not model._needs_pieces(1, 4096, 1)
    one = model.create_kv_cache()
    a = model(ids, 0, one, logits_to_keep=1)[0, -1].float()
    pieces = model.create_kv_cache()
    step = -(-(W - 1) // 16)
    for s0 in range(0, W - 1, step):
        b = model(ids[:, s0:s0 + step], s0, pieces, logits_to_keep=1)[0, -1].float()
    torch.testing.assert_close(a, b, rtol=0, atol=0.05)
    for c in pieces:
        c.release()
    P = _plan(model, monkeypatch)
    dec = model.decode_engine(1)
    assert dec.max_seq_len == W and not dec._attention_fused
    tok = int(a.argmax())
    before = [(p._key_pages.clone(), p._value_pages.clone()) for p in model.page_pools]
    dec.step([tok], [W - 1], one)
    meta = plan.decode_metadata(one, [tok], dec.max_pages)
    assert meta.offsets == [W - 1]
    logits, _ = P.decode(meta, before, dec._attention_fused, rows=1)
    assert torch.equal(dec.logits[:1], logits), "decode at position 131,071 differs from the plan"
    for p, (k, v) in zip(model.page_pools, before):
        assert torch.equal(p._key_pages, k) and torch.equal(p._value_pages, v)
    assert one[0].offset == W


# ---------------------------------------------------------------- 4: refusal --
def test_window_that_cannot_fit_is_refused_before_allocation(dev):
    model = Qwen3ModelWeek3(synthetic_qwen3("qwen3-4b", seed=0, device=dev, num_hidden_layers=1, vocab_size=1024), page_size=128)
    # free as the model counts it: the device's free memory plus blocks torch's allocator holds cached for reuse
    free = torch.cuda.mem_get_info(dev)[0] + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    window = 131072
    per_slot = model.kv_reservation_bytes(window, 2) - model.kv_reservation_bytes(window, 1)
    batch = 2 + free // per_slot  # more slots than the free memory holds
    before = torch.cuda.memory_allocated(dev)
    with pytest.raises(MemoryError, match=rf"context window {window} for {batch} slot\(s\) needs \d+ bytes"):
        model.set_max_context(window, batch_size=batch)
    with pytest.raises(MemoryError, match="needs"):
        model.decode_engine(batch, window)
    assert torch.cuda.memory_allocated(dev) == before and all(p.capacity == 0 for p in model.page_pools)
    assert not model._decode_engines and model.max_context == 8192
    model.set_max_context(window)  # B = 1 at one layer: 2049 pages of 512 KiB
    assert model.max_context == window
