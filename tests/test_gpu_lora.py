"""``tl_lora_apply`` on the GPU against the float64 reference of ``tests/lora_ref.py``, exact probes, row independence,
and adapters through the model, the graph engines and the batcher."""

import importlib.util
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.engine import DecodeEngine, PrefillEngine
from tiny_llm_b200.generate import greedy_generate_ids
from tiny_llm_b200.lora import LoraAdapter
from tiny_llm_b200.synthetic import synthetic_qwen3

pytestmark = pytest.mark.gpu


def _load_ref():
    name = "tiny_llm_b200_lora_ref"
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name("lora_ref.py"))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


lora_reference, random_site, site_to = (getattr(_load_ref(), n) for n in ("lora_reference", "random_site", "site_to"))

# (N, segment widths): the four sites of tiny-d128, Qwen3-0.6B and Qwen3-4B
SITES = {
    "d128-qkv": (256, [512, 256, 256]), "d128-o": (512, [256]), "d128-gate_up": (256, [384, 384]), "d128-down": (384, [256]),
    "0.6b-qkv": (1024, [2048, 1024, 1024]), "0.6b-o": (2048, [1024]), "0.6b-gate_up": (1024, [3072, 3072]), "0.6b-down": (3072, [1024]),
    "4b-qkv": (2560, [4096, 1024, 1024]), "4b-o": (4096, [2560]), "4b-gate_up": (2560, [9728, 9728]), "4b-down": (9728, [2560]),
}


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


def run_case(dev, gen, site_cpu, M, with_residual, ids=None):
    N, Ks = site_cpu.N, site_cpu.K
    x = torch.randn(M, N, generator=gen).to(torch.bfloat16)
    base = [torch.randn(M, K, generator=gen).to(torch.bfloat16) for K in Ks]
    res = [torch.randn(M, K, generator=gen).to(torch.bfloat16) for K in Ks] if with_residual else None
    if ids is None:
        ids = torch.randint(-1, site_cpu.n_adapters, (M,), generator=gen).tolist()
    site = site_to(site_cpu, dev)
    y = torch.cat(base, dim=1).to(dev)
    got = ext.lora_apply(x.to(dev), y, torch.tensor(ids, dtype=torch.int32, device=dev), site,
                         residual=None if res is None else torch.cat(res, dim=1).to(dev))
    return x, base, res, ids, list(torch.split(got.cpu(), Ks, dim=1))


@pytest.mark.parametrize("with_residual", [False, True])
@pytest.mark.parametrize("M", [1, 3, 8, 9, 64, 65, 128, 1000])
@pytest.mark.parametrize("name", list(SITES))
def test_kernel_against_float64(dev, name, M, with_residual):
    N, Ks = SITES[name]
    if with_residual and len(Ks) > 1:
        pytest.skip("only the single-segment sites (o, down) carry the residual")
    if M == 1000 and not name.startswith("d128") and name != "4b-qkv":
        pytest.skip("the float64 reference of 1,000 wide rows is run on one large site")
    gen = torch.Generator().manual_seed(list(SITES).index(name) * 10000 + M * 2 + int(with_residual))
    site_cpu = random_site(gen, N, Ks, [8, 16, 32, 64])
    assert ext.lora_apply_route(M, site_cpu) == (ext.LORA_TILES if M > 64 else ext.LORA_ROWS)
    check_rows = range(M) if M <= 128 else list(range(0, M, 37)) + [M - 1]
    x, base, res, ids, got = run_case(dev, gen, site_cpu, M, with_residual)
    rows = torch.tensor(list(check_rows))
    want, bound = lora_reference(x[rows], [b[rows] for b in base], [ids[i] for i in check_rows], site_cpu,
                                 None if res is None else [r[rows] for r in res])
    for s in range(len(Ks)):
        err = (got[s][rows].to(torch.float64) - want[s]).abs()
        assert bool((err <= bound[s] * 1.0001).all()), f"segment {s}: worst excess {float((err - bound[s]).max())}"
        idle = torch.tensor([ids[i] < 0 for i in check_rows])
        if idle.any() and res is None:
            assert torch.equal(got[s][rows][idle], base[s][rows][idle]), "rows without an adapter keep the base's bits"


def test_exact_probes_power_of_two(dev):
    """Power-of-two A, B, scale and a needle activation: every product and sum is exact, so the result is known bit for bit."""
    N, Ks, r = 256, [128, 64], 8
    A = torch.zeros(1, 2 * r, N, dtype=torch.bfloat16)
    A[0, 3, 17] = 0.5    # segment 0: t_3 = 0.5 * x_17
    A[0, r + 1, 200] = 2.0  # segment 1: t_1 = 2 * x_200
    B0 = torch.zeros(1, 128, r, dtype=torch.bfloat16)
    B0[0, 5, 3] = 4.0
    B1 = torch.zeros(1, 64, r, dtype=torch.bfloat16)
    B1[0, 63, 1] = -0.25
    site = ext.LoraSite(A.to(dev), [B0.to(dev), B1.to(dev)], torch.tensor([2.0], device=dev), torch.tensor([r], dtype=torch.int32, device=dev),
                        torch.tensor([3], dtype=torch.int32, device=dev))
    x = torch.zeros(3, N, dtype=torch.bfloat16)
    x[:, 17], x[:, 200] = 1.0, 8.0
    base = torch.ones(5, 192, dtype=torch.bfloat16)  # two more rows than the launch covers
    y = base.to(dev)
    ext.lora_apply(x.to(dev), y[:3], torch.tensor([0, -1, 0], dtype=torch.int32, device=dev), site)
    want = base.clone()
    for m in (0, 2):
        want[m, 5] = 1.0 + 2.0 * 4.0 * 0.5
        want[m, 128 + 63] = 1.0 + 2.0 * -0.25 * 16.0
    assert torch.equal(y.cpu(), want), "id -1 rows, untouched outputs and rows outside the launch keep their bits"
    # an untargeted segment keeps the base's bits
    site1 = ext.LoraSite(site.a, site.b, site.scales, site.ranks, torch.tensor([1], dtype=torch.int32, device=dev))
    y = base.to(dev)
    ext.lora_apply(x.to(dev), y[:3], torch.tensor([0, 0, 0], dtype=torch.int32, device=dev), site1)
    assert torch.equal(y.cpu()[:, 128:], base[:, 128:]) and float(y[0, 5]) == 5.0


def test_rank_padding_changes_no_bit(dev):
    gen = torch.Generator().manual_seed(3)
    N, Ks = 2560, [4096, 1024, 1024]
    small = random_site(gen, N, Ks, [8])
    A = torch.zeros(1, 3 * 64, N, dtype=torch.bfloat16)
    Bs = [torch.zeros(1, K, 64, dtype=torch.bfloat16) for K in Ks]
    for s in range(3):
        A[0, s * 64 : s * 64 + 8] = small.a[0, s * 8 : s * 8 + 8]
        Bs[s][0, :, :8] = small.b[s][0]
    padded = ext.LoraSite(A, Bs, small.scales, small.ranks, small.seg_mask)
    for M in (5, 70):
        state = gen.get_state()
        a = run_case(dev, gen, small, M, False, ids=[0] * M)[-1]
        gen.set_state(state)
        b = run_case(dev, gen, padded, M, False, ids=[0] * M)[-1]
        assert all(torch.equal(p, q) for p, q in zip(a, b))


def test_row_independence_routes_and_graph_replay(dev):
    """A row's output is the same bits alone, at every index of a 64-row launch among other adapters, inside uniform and
    mixed 8-row tiles of the M > 64 route, on a second launch and under graph capture and replay."""
    gen = torch.Generator().manual_seed(11)
    N, Ks = 1024, [2048, 1024, 1024]
    site = site_to(random_site(gen, N, Ks, [16, 64, 8]), dev)
    row = torch.randn(1, N, generator=gen).to(torch.bfloat16).to(dev)
    base_row = torch.randn(1, sum(Ks), generator=gen).to(torch.bfloat16).to(dev)
    one = torch.tensor([1], dtype=torch.int32, device=dev)
    alone = ext.lora_apply(row, base_row.clone(), one, site)
    assert torch.equal(alone, ext.lora_apply(row, base_row.clone(), one, site))
    for M in (64, 200):
        x = torch.randn(M, N, generator=gen).to(torch.bfloat16).to(dev)
        base = torch.randn(M, sum(Ks), generator=gen).to(torch.bfloat16).to(dev)
        ids = torch.randint(-1, 3, (M,), generator=gen).to(torch.int32).to(dev)
        spots = range(M) if M == 64 else (0, 7, 8, 15, 64, 199)
        for i in spots:
            xi, bi, idi = x.clone(), base.clone(), ids.clone()
            xi[i], bi[i], idi[i] = row[0], base_row[0], 1
            if M == 200 and i in (8, 15):
                idi[8:16] = 1  # a uniform tile
            assert torch.equal(ext.lora_apply(xi, bi, idi, site)[i], alone[0]), f"M = {M}, row {i}"
    x = torch.randn(8, N, generator=gen).to(torch.bfloat16).to(dev)
    x[3] = row[0]
    ids = torch.tensor([0, 2, -1, 1, 1, 0, 2, -1], dtype=torch.int32, device=dev)
    static_y = torch.empty(8, sum(Ks), dtype=torch.bfloat16, device=dev)
    base = torch.randn(8, sum(Ks), generator=gen).to(torch.bfloat16).to(dev)
    base[3] = base_row[0]
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        static_y.copy_(base)
        ext.lora_apply(x, static_y, ids, site)
        stream.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=stream):
            static_y.copy_(base)
            ext.lora_apply(x, static_y, ids, site)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(static_y[3], alone[0])


# ------------------------------------------------------------------ model, engines, batcher --
@pytest.fixture(scope="module")
def tiny_gpu(dev):
    return synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512, device=dev)


def adapters_for(ns):
    return [LoraAdapter.synthetic(ns.args, 16, seed=0, name="a"), LoraAdapter.synthetic(ns.args, 8, seed=1, name="b"),
            LoraAdapter.synthetic(ns.args, 64, targets=("q", "v", "down"), seed=2, name="c")]


def lora_model(ns, page_size=8, graphs=True):
    model = Qwen3ModelWeek3(ns, page_size=page_size)
    model.load_adapters(adapters_for(ns))
    if not graphs:
        model.use_decode_graph = False
    return model


def test_zero_b_adapter_gives_the_base_logits_bit_for_bit(dev, tiny_gpu):
    args = tiny_gpu.args
    zero = LoraAdapter.synthetic(args, 16, seed=5, name="zero")
    zero.tensors = {k: (A, torch.zeros_like(B)) for k, (A, B) in zero.tensors.items()}
    model = Qwen3ModelWeek3(tiny_gpu, page_size=64)
    model.load_adapters([zero])
    model.use_decode_graph = False
    plain = Qwen3ModelWeek3(tiny_gpu, page_size=64)
    plain.use_decode_graph = False
    ids = torch.tensor([[5, 17, 3, 250, 99, 42, 7]], dtype=torch.int32, device=dev)
    base = plain(ids, 0, plain.create_kv_cache())
    assert torch.equal(model(ids, 0, model.create_kv_cache(), adapter_ids=[0]), base)
    moved = lora_model(tiny_gpu, page_size=64, graphs=False)
    assert not torch.equal(moved(ids, 0, moved.create_kv_cache(), adapter_ids=[0]), base), "a non-zero adapter must move the logits"


class _MergedWeight:
    """``W + sc B A`` in float32 in place of a dense bf16 weight of the CPU oracle model: ``x @ merged.T`` multiplies in
    float32 and rounds the product to the activation dtype, as the oracle's own ``linear`` rounds its output."""

    def __init__(self, dense, A, B, scale):
        self.w = dense.float() + scale * (B.float() @ A.float())

    @property
    def T(self):
        return self

    def __rmatmul__(self, x):
        return (x.float() @ self.w.T).to(x.dtype)


@pytest.mark.parametrize("targets", [("q", "k", "v", "o", "gate", "up", "down"), ("q", "v", "down"), ("k", "o", "gate"), ("up",)])
def test_operator_path_against_the_cpu_oracle_with_the_adapter_merged_in_float(dev, tiny_gpu, targets):
    """Whole-model check of the wiring (which input each site reads, which segment is which, the scale convention), against
    an implementation that shares none of it: the CPU oracle model with ``W_deq + (alpha / r) B A`` as its dense weights.
    Teacher-forced over a prefill and five decode steps, within DESIGN section 2's 0.25 nat on the oracle's top candidates."""
    from oracle.model import ReferenceCpuModel, greedy_decode

    ns_cpu = synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)
    adapter = LoraAdapter.synthetic(ns_cpu.args, 16, targets=targets, seed=9, name="m", alpha=48.0)
    ref = ReferenceCpuModel(ns_cpu)
    prompt = [5, 17, 3, 250, 99, 42, 7, 300, 11]
    base_tokens, base_lp = greedy_decode(ref, prompt, 6, return_logprobs=True)
    where = {"q": ("attn", "wq"), "k": ("attn", "wk"), "v": ("attn", "wv"), "o": ("attn", "wo"),
             "gate": (None, "w_gate"), "up": (None, "w_up"), "down": (None, "w_down")}
    for (layer, proj), (A, B) in adapter.tensors.items():
        part, attr = where[proj]
        holder = ref.blocks[layer] if part is None else getattr(ref.blocks[layer], part)
        setattr(holder, attr, _MergedWeight(getattr(holder, attr), A, B, adapter.scale))
    ref_tokens, ref_lp = greedy_decode(ref, prompt, 6, return_logprobs=True)
    assert float((ref_lp[0] - base_lp[0]).abs().max()) > 0.5, "the adapter must move the oracle's distribution well beyond the tolerance"

    model = Qwen3ModelWeek3(tiny_gpu, page_size=64)
    model.load_adapters([LoraAdapter.synthetic(tiny_gpu.args, 8, seed=1, name="other"), adapter])
    model.use_decode_graph = False
    cache = model.create_kv_cache()
    feed, offset = prompt, 0
    for tok, lp_ref in zip(ref_tokens, ref_lp):
        logits = model(torch.tensor([feed], dtype=torch.int32, device=dev), offset, cache, logits_to_keep=1, adapter_ids=[1])[0, -1].float().cpu()
        lp = logits - torch.logsumexp(logits, dim=-1)
        top = torch.topk(lp_ref, 4).indices
        torch.testing.assert_close(lp[top], lp_ref[top], rtol=0, atol=0.25)
        offset += len(feed)
        feed = [tok]
    for c in cache:
        c.release()


def prefill(model, dev, prompt, adapter_id):
    cache = model.create_kv_cache()
    was, model.use_decode_graph = model.use_decode_graph, False
    logits = model(torch.tensor([prompt], dtype=torch.int32, device=dev), 0, cache, logits_to_keep=1, adapter_ids=[adapter_id])
    model.use_decode_graph = was
    return cache, int(torch.argmax(logits[0, -1].float()))


def slots_setup(dev, ns, B, graphs):
    """A model with the three adapters, ``B`` slots of which a prefix is live on ids -1, 0, 1, 2, -1, ..., each prefilled
    on the operator path: (model, per-layer slot tables, tokens, offsets, slot ids, live slots)."""
    from tiny_llm_b200.kv_cache import BatchingKvCache

    model = lora_model(ns, graphs=graphs)
    live = list(range(B)) if B <= 8 else list(range(12))  # B = 16 / 32: the occupied prefix picks a row variant
    slot_ids = [(b % 4) - 1 if b in live else -1 for b in range(B)]
    g = torch.Generator().manual_seed(B)
    table = [BatchingKvCache(max_active_requests=B, max_seq_len=128) for _ in range(model.num_hidden_layers)]
    toks, offs = [0] * B, [0] * B
    for b in live:
        prompt = torch.randint(1, 500, (5 + b % 3,), generator=g).tolist()
        cache, toks[b] = prefill(model, dev, prompt, slot_ids[b])
        for layer_cache, t in zip(cache, table):
            t.add_request(layer_cache, b)
        offs[b] = len(prompt)
    return model, table, toks, offs, slot_ids, live


@pytest.mark.parametrize("B", [1, 8, 16, 32])
def test_decode_engine_matches_the_operator_path(dev, tiny_gpu, B):
    """``step`` over 24 steps against the operator path with the same ids, slots on different adapters and on none; half
    way the slots change adapters, which is data and not a new graph."""
    ref_model, ref_table, toks, offs, slot_ids, live = slots_setup(dev, tiny_gpu, B, graphs=False)
    model, table, toks2, _, _, _ = slots_setup(dev, tiny_gpu, B, graphs=True)
    assert toks == toks2
    engine = model.decode_engine(B, 128)
    rows = torch.tensor(live, device=dev)
    worst, captures = 0.0, None
    for step in range(24):
        batch = torch.tensor(toks, dtype=torch.int32, device=dev).reshape(-1, 1)
        want = ref_model(batch, offs, ref_table, logits_to_keep=1, adapter_ids=slot_ids)
        got, nxt = engine.step(toks, offs, table, adapter_ids=slot_ids)
        worst = max(worst, float((got.view_as(want)[rows].float() - want[rows].float()).abs().max()))
        torch.testing.assert_close(got.view_as(want)[rows].float(), want[rows].float(), rtol=0, atol=0.06)
        for b in live:
            toks[b] = int(torch.argmax(want[b, -1].float()))
            offs[b] += 1
        if step == 11:
            captures = engine.captures
            slot_ids = [((i + 2) % 4) - 1 if b in live else -1 for b, i in enumerate(slot_ids)]
    assert engine.captures == captures
    assert engine.kernels_per_step == 13 * model.num_hidden_layers + 6, engine.kernels_per_step
    print(f"B = {B}: kernels_per_step {engine.kernels_per_step}, worst |logit difference| against the operator path {worst}")


@pytest.mark.parametrize("B", [1, 8, 32])
def test_decode_on_device_gives_the_tokens_of_step(dev, tiny_gpu, B):
    from tiny_llm_b200.sampler import SamplingParams

    steps = 24
    model, table, toks, offs, slot_ids, live = slots_setup(dev, tiny_gpu, B, graphs=True)
    engine = model.decode_engine(B, 128)
    rows = torch.tensor(live, device=dev)
    want = []
    for _ in range(steps):
        _, nxt = engine.step(toks, offs, table, adapter_ids=slot_ids)
        want.append(nxt[rows].clone())
        toks = [int(t) if b in live else 0 for b, t in enumerate(nxt.tolist())]
        offs = [o + 1 if b in live else 0 for b, o in enumerate(offs)]
    model2, table2, toks2, offs2, _, _ = slots_setup(dev, tiny_gpu, B, graphs=True)
    out = model2.decode_engine(B, 128).decode_on_device(toks2, offs2, table2, steps, adapter_ids=slot_ids)
    assert torch.equal(out[:, rows], torch.stack(want))
    # sampled with logprobs: the graph's tokens and log-probabilities are those of step() plus the eager tl_sample and
    # tl_logprobs launches on its logits, so the sampled and logprobs graphs read the same adapter ids as the greedy one
    from tiny_llm_b200.sampler import sampling_tensors

    params = SamplingParams(0.8, top_k=20, top_p=0.9, seed=7)
    m1, t1, tk, of, _, _ = slots_setup(dev, tiny_gpu, B, graphs=True)
    e1 = m1.decode_engine(B, 128)
    e1.step(tk, of, t1, adapter_ids=slot_ids)
    logits = e1.logits[rows].clone()
    temperature, top_k, top_p, seed = (t.to(dev) for t in sampling_tensors([params] * len(live), "cpu"))
    positions = torch.tensor([of[b] + 1 for b in live], dtype=torch.int32, device=dev)
    eager = ext.sample(logits, temperature, top_k, top_p, seed, positions)
    _, eager_lp, eager_rank, eager_ids, eager_top = ext.logprobs(logits, eager, None, 5)
    m2, t2, tk2, of2, _, _ = slots_setup(dev, tiny_gpu, B, graphs=True)
    tokens, (lp, rank, ids, top) = m2.decode_engine(B, 128).decode_on_device(tk2, of2, t2, 1, sampling=params, logprobs=5, adapter_ids=slot_ids)
    assert torch.equal(tokens[0, rows], eager)
    assert torch.equal(lp[0, rows], eager_lp) and torch.equal(rank[0, rows], eager_rank)
    assert torch.equal(ids[0, rows], eager_ids) and torch.equal(top[0, rows], eager_top)
    # the same slots on the base model draw from other logits
    m3, t3, tk3, of3, _, _ = slots_setup(dev, tiny_gpu, B, graphs=True)
    _, (lp_base, _, _, _) = m3.decode_engine(B, 128).decode_on_device(tk3, of3, t3, 1, sampling=params, logprobs=5)
    on_adapter = torch.tensor([i for i, b in enumerate(live) if slot_ids[b] >= 0], device=dev)
    if on_adapter.numel():
        assert not torch.equal(lp_base[0, rows][on_adapter], eager_lp[on_adapter])


def test_no_adapter_model_keeps_its_launch_count_and_matches_the_operator_path(dev, tiny_gpu):
    """A model without adapters builds the base engine (5 launches per layer + 5) and its step matches the plain operator
    path as the existing engine tests hold it; so does a LoRA engine with its slot at -1, at 13 launches per layer + 6."""
    plain = Qwen3ModelWeek3(tiny_gpu, page_size=8)
    plain.use_decode_graph = False
    model = Qwen3ModelWeek3(tiny_gpu, page_size=8)
    with_set = lora_model(tiny_gpu)
    e0, e1 = DecodeEngine(model, 1, 128, dev), DecodeEngine(with_set, 1, 128, dev)
    for e in (e0, e1):
        e.reserve_pools()
    layers = model.num_hidden_layers
    cp, tok = prefill(plain, dev, [5, 17, 3], -1)
    c0, _ = prefill(model, dev, [5, 17, 3], -1)
    c1, _ = prefill(with_set, dev, [5, 17, 3], -1)
    for step in range(6):
        want = plain(torch.tensor([[tok]], dtype=torch.int32, device=dev), 3 + step, cp, logits_to_keep=1)
        a, _ = e0.step([tok], [3 + step], c0)
        b, _ = e1.step([tok], [3 + step], c1)
        torch.testing.assert_close(a.float().view_as(want), want.float(), rtol=0, atol=0.06)
        torch.testing.assert_close(b.float().view_as(want), want.float(), rtol=0, atol=0.06)
        tok = int(torch.argmax(want[0, -1].float()))
    assert e0.lora is None and e0.kernels_per_step == 5 * layers + 5, e0.kernels_per_step
    assert e1.kernels_per_step == 13 * layers + 6, e1.kernels_per_step


@pytest.mark.parametrize("chunk,length", [(32, 32), (32, 7), (128, 128), (128, 50), (256, 256), (256, 130)])
def test_prefill_engine_matches_the_operator_path(dev, tiny_gpu, chunk, length):
    ref_model = lora_model(tiny_gpu, page_size=64, graphs=False)
    model = lora_model(tiny_gpu, page_size=64)
    engine = PrefillEngine(model, chunk, 512, dev)
    engine.reserve_pools(16)
    # up to 128 rows the projections take the fused entry (never the tile GEMM there); longer chunks the plain entry, whose
    # route for these shapes is the 128-token wgmma tile GEMM, not the streaming matvec
    from tiny_llm_b200.engine import lora_projection_is_fused

    assert lora_projection_is_fused(chunk) == (chunk <= 128)
    w = model.layers_inner[0].mlp.w_down
    x = torch.zeros((chunk, w.weight.shape[1] * 8), dtype=torch.bfloat16, device=dev)
    route = ext.quantized_matmul_route(chunk, x.shape[1], w.weight.shape[0], x.shape[1], ext.PRO_NONE, chunk <= 128, True, x.dtype, x, w.weight,
                                       w.scales, w.biases)[0]
    assert route == (ext.W4_TILES if chunk > 128 else ext.W4_SKINNY)
    g = torch.Generator().manual_seed(chunk + length)
    for adapter_id in (1, -1, 2):  # one graph, the id is data
        prompt = torch.randint(1, 500, (length,), generator=g).tolist()
        want = ref_model(torch.tensor([prompt], dtype=torch.int32, device=dev), 0, ref_model.create_kv_cache(), logits_to_keep=1, adapter_ids=[adapter_id])
        cache = model.create_kv_cache()
        got, _ = engine.prefill_chunk(prompt, 0, cache, adapter_id=adapter_id)
        torch.testing.assert_close(got.float().reshape(-1), want.float().reshape(-1), rtol=0, atol=0.08)
        for c in cache:
            c.release()
    assert engine.captures == 1


@pytest.mark.parametrize("order", [[0, 1, 2, 3], [3, 1, 0, 2]])
def test_batcher_gives_each_request_its_own_adapters_tokens(dev, tiny_gpu, order):
    prompts = [[5, 17, 3, 9], [5, 17, 3, 9], [5, 17, 3, 9], [8, 1, 300]]
    names = ["a", None, "b", "a"]
    model = lora_model(tiny_gpu, page_size=64)
    # the graph and operator paths agree to a tolerance, not bit for bit: build the engines first, so that every request,
    # alone or batched, prefills and decodes on the graph path
    greedy_generate_ids(model, prompts[0], 2, device=dev)
    alone = [greedy_generate_ids(model, p, 10, device=dev, adapter=n) for p, n in zip(prompts, names)]
    assert alone[0] != alone[1] and alone[1] != alone[2] and alone[0] != alone[2]
    batcher = ContinuousBatcher(model, None, [prompts[i] for i in order], max_seq_len=64, batch_size=3, prefill_step=128, verbose=False,
                                device=dev, max_new_tokens=[10] * 4, adapters=[names[i] for i in order])
    seen = []
    while not batcher.idle():
        batcher.step()
        seen.append(list(batcher.slot_adapter_ids))
    batcher.release_all()
    got = {idx: [int(t) for t in text.split()] for idx, text in batcher.results}
    for pos, i in enumerate(order):
        assert got[pos] == alone[i], f"request {i} ({names[i]})"
    assert seen[-1] == [-1, -1, -1] and any(s != [-1, -1, -1] for s in seen)


def test_prefix_cache_is_kept_apart_per_adapter(dev, tiny_gpu):
    model = lora_model(tiny_gpu, page_size=8)
    prompt = list(range(3, 3 + 20))
    names = ["a", "b", "a", None, None]
    alone = {n: greedy_generate_ids(model, prompt, 6, device=dev, adapter=n) for n in set(names)}
    batcher = ContinuousBatcher(model, None, [prompt] * 5, max_seq_len=64, batch_size=2, prefill_step=128, verbose=False, device=dev,
                                max_new_tokens=[6] * 5, adapters=names, prefix_cache=True)
    results = dict(batcher.run())
    assert [batcher.reused_tokens[i] for i in range(5)] == [0, 0, 19, 0, 19]
    for i, n in enumerate(names):
        assert [int(t) for t in results[i].split()] == alone[n]
