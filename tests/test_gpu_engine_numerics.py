"""The graph engines against an independent eager statement of their launches, and each launch in place against float64.

``tests/engine_plan.py`` restates one decode step of ``DecodeEngine`` and one chunk of ``PrefillEngine`` from the C ABI,
the model's unpacked weights and the request caches.  The kernels are deterministic, so for every case below:

(a) after each engine step (or chunk) the logits, the next tokens and every layer's WHOLE K and V slab are bit-identical
    (``torch.equal``) to the plan run on clones of the slabs taken just before the step; comparing whole slabs proves that
    nothing outside the target slots was written.  The engine's launch count per step equals the plan's.
(b) every launch the plan recorded is checked, teacher-forced on the inputs it actually received, against the float64
    references and bounds of the kernel suites (w4a16_ref, elementwise_ref, attention_ref), with norm weights, positions
    and projections taken from the model's per-layer unpacked weights: a wrong layer, norm, packing or position fails at
    the stage where it happens, and the bounds do not compound.

Each case asserts the engine branch it reaches; ``test_the_cases_reach_every_engine_branch`` requires all of them."""

import importlib.util
import math
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import BatchingKvCache, Qwen3ModelWeek3
from tiny_llm_b200.engine import DecodeEngine, PrefillEngine
from tiny_llm_b200.synthetic import synthetic_qwen3


def _load(name, file):
    """A helper next to this file, by path: `tests` is no package of this project, and another installed `tests`
    package may already own that name."""
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


wr = _load("tiny_llm_b200_w4a16_ref", "w4a16_ref.py")
er = _load("tiny_llm_b200_elementwise_ref", "elementwise_ref.py")
ar = _load("tiny_llm_b200_attention_ref", "attention_ref.py")
plan = _load("tiny_llm_b200_engine_plan", "engine_plan.py")

pytestmark = pytest.mark.gpu
F64, BF16 = torch.float64, torch.bfloat16
PATHS = {ext.W4_VANILLA: "vanilla", ext.W4_STREAM: "stream", ext.W4_SKINNY: "skinny", ext.W4_TILES: "tiles"}
MATMULS = {"qkv", "o", "gate_up", "down", "head", "o_norm", "down_norm", "gate", "up"}
MODELS = {
    "d128": ("tiny-d128", dict(seed=5, realistic=True, max_position_embeddings=8192)),
    "4b": ("qwen3-4b", dict(seed=1, num_hidden_layers=2, vocab_size=4096)),
    "0.6b": ("qwen3-0.6b", dict(seed=2, num_hidden_layers=2, vocab_size=4096)),
}
REACHED: dict = {}
RATIOS: dict = {}  # stage -> largest error / bound seen


def reach(branch, case):
    REACHED.setdefault(branch, case)


@pytest.fixture(scope="module")
def dev(cuda_device):
    return cuda_device


_NS: dict = {}


def make_model(key, page, dev):
    if key not in _NS:
        name, kw = MODELS[key]
        _NS[key] = synthetic_qwen3(name, device=dev, **kw)
    return Qwen3ModelWeek3(_NS[key], page_size=page)


def randomize_slabs(model, seed):
    """Every slab element random: an append to any slot but its target shows in the whole-slab comparison."""
    g = torch.Generator(device=model.page_pools[0]._key_pages.device).manual_seed(seed)
    for pool in model.page_pools:
        pool._key_pages.normal_(generator=g)
        pool._value_pages.normal_(generator=g)


def slabs(model):
    return [(p._key_pages.clone(), p._value_pages.clone()) for p in model.page_pools]


def assert_slabs_equal(model, pages, what):
    for i, (pool, (kp, vp)) in enumerate(zip(model.page_pools, pages)):
        for name, got, want in (("K", pool._key_pages, kp), ("V", pool._value_pages, vp)):
            if not torch.equal(got, want):
                bad = (got.view(torch.int16) != want.view(torch.int16)).nonzero()
                raise AssertionError(f"{what}: layer {i} {name} slab differs from the plan in {len(bad)} elements; first [page, head, slot, d] "
                                     f"{bad[:4].tolist()}")


# ------------------------------------------------------------- stage checks --
class Checker:
    """float64 references of the plan's recorded stages, from the model's unpacked weights."""

    def __init__(self, model, P):
        self.model, self.P = model, P
        self._w: dict = {}
        at = model.layers_inner[0].self_attn
        self.Hq, self.Hkv, self.D, self.scale, self.base = at.num_heads, at.num_kv_heads, at.head_dim, at.scale, at.rope.base

    def W(self, key, rounded):
        k = (key, rounded)
        if k not in self._w:
            kind, i = key
            build = lambda q: wr.Weights.build(q.weight.view(torch.int32) if q.weight.dtype == torch.uint32 else q.weight, q.scales, q.biases,  # noqa: E731
                                               rounded=rounded)
            if kind == "qkv":
                at = self.model.layers_inner[i].self_attn
                parts = [build(w) for w in (at.wq, at.wk, at.wv)]
                self._w[k] = wr.Weights(*(torch.cat([getattr(p, f) for p in parts]) for f in ("w", "absw", "abs_s", "abs_b")), BF16, rounded)
            elif kind == "gate_up":
                mlp = self.model.layers_inner[i].mlp
                g, u = build(mlp.w_gate), build(mlp.w_up)
                gi, ui = wr.pairs_index(g.w.shape[0], g.w.device)

                def inter(a, b):
                    out = torch.empty((2 * a.shape[0], a.shape[1]), dtype=a.dtype, device=a.device)
                    out[gi], out[ui] = a, b
                    return out

                self._w[k] = wr.Weights(inter(g.w, u.w), inter(g.absw, u.absw), inter(g.abs_s, u.abs_s), inter(g.abs_b, u.abs_b), BF16, rounded)
            else:
                b = self.model.layers_inner[i] if i is not None else None
                q = {"o": lambda: b.self_attn.wo, "down": lambda: b.mlp.w_down, "gate": lambda: b.mlp.w_gate, "up": lambda: b.mlp.w_up,
                     "head": lambda: self.model.w_lm_head or self.model.embedding.weight}[kind]()
                self._w[k] = build(q)
        return self._w[k]

    def norm(self, key):
        """The model's own norm object for a key (not the plan's lookup)."""
        kind, i = key
        if kind == "final":
            return self.model.norm
        b = self.model.layers_inner[i]
        return {"ln1": b.input_layernorm, "ln2": b.post_attention_layernorm, "q": b.self_attn.q_norm, "k": b.self_attn.k_norm}[kind]

    def note(self, stage, ratio):
        RATIOS[stage] = max(RATIOS.get(stage, 0.0), ratio)

    def check(self, before, after, what):
        """``before``: the slabs the plan started from; ``after``: the plan's slabs after the step."""
        for st in self.P.stages:
            label = f"{what}: {st.name} (layer {st.layer})"
            fn = getattr(self, "_" + st.name) if st.name not in MATMULS else self._matmul
            fn(st, before, after, label)

    def _embedding(self, st, before, after, label):
        emb = self.model.embedding.weight
        wr.assert_exact(st.out, er.embedding_ref(st.args["ids"], emb.scales, emb.biases, emb.weight.view(torch.int32), BF16), label)

    def _rms_norm(self, st, before, after, label):
        n = self.norm(st.args["norm"])
        b = er.rms_norm_ref(st.args["x"], n.weight, n.eps, BF16)
        self.note("rms_norm", er.assert_within(st.out, b.pre, b.tol, label))

    def _matmul(self, st, before, after, label):
        a = st.args
        path, splits, gbps = PATHS[st.route[0]], st.route[1], st.route[2]
        W = self.W(a["w"], path in ("skinny", "tiles"))
        pro = wr.PRO_RMSNORM if a["norm"] is not None else wr.PRO_NONE
        n = self.norm(a["norm"]) if a["norm"] is not None else None
        nxt = self.norm(a["next_norm"]) if a.get("next_norm") is not None else None
        r = wr.reference(W, a["a"], p1=None if n is None else n.weight, prologue=pro, epilogue=a["epilogue"], residual=a["residual"],
                         eps=0.0 if n is None else n.eps, norm_weight=None if nxt is None else nxt.weight, norm_eps=0.0 if nxt is None else nxt.eps)
        b = wr.error_bound(r, W, path, splits=splits, gb_per_split=gbps)
        out = st.out[0] if isinstance(st.out, tuple) else st.out
        self.note(f"{st.name} {path}", wr.assert_within(out, b.pre, b.tol, label))
        if nxt is not None:
            self.note(f"{st.name} {path} normed", wr.assert_within(st.out[1], b.normed_pre, b.normed_tol, label + " normed"))

    def _qk(self, st, qkv, q_out, before, after, label, chunk, inv_freq=None):
        """q against qk_norm_rope_ref; the appended K rows within its bound, V rows bit for bit, nothing else touched."""
        i, a = st.layer, st.args
        qn, kn = self.norm(("q", i)), self.norm(("k", i))
        ref = er.qk_norm_rope_ref(qkv, qn.weight, kn.weight, a["offsets"], self.Hq, self.Hkv, self.base, qn.eps, inv_freq=inv_freq)
        if q_out is not None:
            got = q_out.permute(1, 0, 2) if chunk else q_out.view(-1, self.Hq, self.D)
            self.note("q", er.assert_within(got, ref.q.pre, ref.q.tol, label + " q"))
        (k0, v0), (k1, v1) = before[i], after[i]
        slots = er.append_slots(a["ctx"], a["table"], k0.shape[2], k0.shape[0], chunk=chunk)
        self.note("appended k", er.check_pages(k0, k1, slots, None, tol=ref.k.tol, pre=ref.k.pre, what=label + " K pages"))
        er.check_pages(v0, v1, slots, ref.v, label + " V pages")
        return ref

    def _qk_norm_rope_append(self, st, before, after, label):
        self._qk(st, st.args["qkv"], st.out, before, after, label, chunk=False)

    def _chunk_qk_norm_rope_append(self, st, before, after, label):
        self._qk(st, st.args["qkv"], st.out, before, after, label, chunk=True)

    def _qkv_rope_append(self, st, before, after, label):
        """The projection is not written by the launch: the same rows through quantized_matmul_fused give the q|k|v it
        rounds (the header: same results as the two calls), checked against the reference, then the q/k half on it."""
        a = st.args
        w = self.P.qkv[st.layer]
        qkv = ext.quantized_matmul_fused(w.scales, w.biases, w.weight, a["a"])
        path, splits, gbps = PATHS[st.route[0][0]], st.route[0][1], st.route[0][2]
        W = self.W(a["w"], path in ("skinny", "tiles"))
        b = wr.error_bound(wr.reference(W, a["a"]), W, path, splits=splits, gb_per_split=gbps)
        self.note(f"qkv {path}", wr.assert_within(qkv, b.pre, b.tol, label + " projection"))
        self._qk(st, qkv, st.out, before, after, label, chunk=a["chunk"])

    def _attention(self, st, before, after, label):
        a = st.args
        kp, vp = after[st.layer]
        q = a["q"]
        if a["token_major"]:  # q [Hq, L, D], out [L, Hq * D]
            got = st.out.view(a["L"], self.Hq, self.D).permute(1, 0, 2)
        else:
            got = st.out.view(q.shape)
        ref, A, smax, nvis = ar.paged_reference(q, kp, vp, a["table"], a["ctx"], self.scale, True, self.Hkv, self.Hq)
        tol = ar.error_bound(ref, A, smax, nvis, self.D, BF16, p_rounded=st.route in (ext.PAGED_FLASH, ext.PAGED_WGMMA))
        ar.assert_within(got, ref, tol, label)

    def _attention_fused(self, st, before, after, label):
        """The kernel does not expose the q it rotates: form it with qk_norm_rope_ref and widen the bound by what q's
        rounding ambiguity can do.  The kernel's q is within dq = tol + |T(pre) - pre| of the reference's T(pre), which
        moves a score by at most scale * sum_d dq_d max_j |k_jd| (max over the keys the row sees), and a score moved by at
        most delta moves the output by at most (e^(2 delta) - 1) A; this adds to the fp32 score error of the bound."""
        a = st.args
        ref_q = self._qk(st, a["qkv"], None, before, after, label, chunk=False, inv_freq=self.P.inv_freq)
        kp, vp = after[st.layer]
        R, Hq, Hkv, D = a["qkv"].shape[0], self.Hq, self.Hkv, self.D
        G = Hq // Hkv
        q = ref_q.q.out  # [R, Hq, D]
        dq = ref_q.q.tol + (ref_q.q.out - ref_q.q.pre).abs()
        ref, A, smax, nvis = ar.paged_reference(q.reshape(R * Hq, 1, D), kp, vp, a["table"], a["ctx"], self.scale, True, Hkv, Hq)
        dscore = torch.zeros(R, Hq, dtype=F64, device=q.device)
        page = kp.shape[2]
        for b, n in enumerate(a["ctx"].tolist()):
            if n <= 0:
                continue
            npg = -(-n // page)
            ids = a["table"][b, :npg].long()
            K = kp[ids].to(F64).permute(1, 0, 2, 3).reshape(Hkv, npg * page, D)[:, :n]
            kmax = K.abs().amax(1).repeat_interleave(G, 0)  # [Hq, D]
            dscore[b] = self.scale * (dq[b] * kmax).sum(-1)
        delta = (2 * D + 16) * 2.0**-24 * smax + 2.0**-20 + dscore.reshape(R * Hq, 1)
        tol = (2.0**-8 + 2.0**-23) * ref.abs() + (torch.expm1(2 * delta) + (nvis.to(F64) / 4 + 64) * 2.0**-23)[..., None] * A
        ar.assert_within(st.out.view(R * Hq, 1, D), ref, tol, label)

    def _add(self, st, before, after, label):
        wr.assert_exact(st.out, er.add_ref(st.args["a"], st.args["b"], BF16), label)

    def _swiglu(self, st, before, after, label):
        b = er.swiglu_ref(st.args["gate"], st.args["up"], BF16)
        self.note("swiglu", er.assert_within(st.out, b.pre, b.tol, label))

    def _argmax(self, st, before, after, label):
        wr.assert_exact(st.out, er.argmax_ref(st.args["logits"]).to(F64), label)


# ----------------------------------------------------------------- drivers --
def admit(model, B, msl, lens):
    """Requests with the given context lengths in their slots (pages through the caches' own bookkeeping), behind
    per-layer BatchingKvCache tables (or one request's cache list when B == 1)."""
    if B == 1:
        cache = model.create_kv_cache()
        for c in cache:
            c.append_slots(lens[0])
        return cache
    tables = [BatchingKvCache(max_active_requests=B, max_seq_len=msl) for _ in range(model.num_hidden_layers)]
    add(model, tables, lens)
    return tables


def add(model, tables, lens):
    for b, n in lens.items():
        cache = model.create_kv_cache()
        for c, t in zip(cache, tables):
            c.append_slots(n)
            t.add_request(c, b)


def occupied(caches):
    first = caches[0]
    return list(first.kv_caches) if isinstance(first, BatchingKvCache) else [first]


def decode_step(model, engine, P, caches, tokens, what, check):
    """One engine step against the plan; returns the plan's next tokens."""
    slot0 = occupied(caches)
    offsets = [c.offset if c is not None else 0 for c in slot0]
    tokens = [t if c is not None else 0 for t, c in zip(tokens, slot0)]
    before = slabs(model)
    engine.step(tokens, offsets, caches)
    hi = max(b + 1 for b, c in enumerate(slot0) if c is not None)
    rows = next(r for r in engine._variants if r >= hi)
    meta = plan.decode_metadata(caches, tokens, engine.max_pages)
    assert meta.offsets == offsets
    pages = [(k.clone(), v.clone()) for k, v in before]
    P.stages = []
    n0 = ext.launch_count()
    logits, nxt = P.decode(meta, pages, engine._attention_fused, rows=rows)
    launches = ext.launch_count() - n0
    if rows == engine.B:
        assert engine.kernels_per_step == launches + 1, (engine.kernels_per_step, launches)  # + decode_advance
    assert torch.equal(engine.logits[:rows], logits), f"{what}: logits differ from the plan"
    assert torch.equal(engine.next_tokens[:rows], nxt), f"{what}: next tokens differ from the plan"
    assert_slabs_equal(model, pages, what)
    if check:
        Checker(model, P).check(before, pages, what)
    branch = ("matvec" if engine.B <= 8 else "swap-AB") + (" + fused attention" if engine._attention_fused else " + unfused attention")
    reach(branch, what)
    if len(engine._variants) > 1:
        reach(f"row variant {rows if rows < engine.B else 'full'}", what)
    return nxt.tolist() + [0] * (engine.B - rows)


def attention_routes(P):
    return {st.route for st in P.stages if st.name == "attention"}


def run_decode(dev, key, B, msl, page, phases, steps, *, fused, seed, check_every=None):
    """``phases``: a list of {slot: context} admissions; each phase then runs ``steps`` steps."""
    model = make_model(key, page, dev)
    engine = DecodeEngine(model, B, msl, dev)
    engine.reserve_pools()
    assert engine._attention_fused == fused and B * engine.max_seq_len == B * msl
    caches = None
    g = torch.Generator().manual_seed(seed)
    P = plan.Plan(model)
    for ph, lens in enumerate(phases):
        if caches is None:
            caches = admit(model, B, msl, lens)
        else:
            add(model, caches, lens)
        randomize_slabs(model, seed + ph)
        tokens = torch.randint(0, model.vocab_size, (B,), generator=g).tolist()
        for s in range(steps):
            check = s in (0, steps - 1) if check_every is None else s % check_every == 0
            tokens = decode_step(model, engine, P, caches, tokens, f"{key} B {B} msl {msl} phase {ph} step {s}", check)
    return model, engine, caches, P


# ------------------------------------------------------------------ decode --
def test_decode_b1_fused_reaches_the_tables_last_slot(dev):
    """B = 1, 20 steps from context 44 behind a 64-token table of 16-slot pages: crosses pages at 48, and the last append
    lands in the table's last slot (post-append length = max_seq_len)."""
    model, engine, caches, _ = run_decode(dev, "d128", 1, 64, 16, [{0: 44}], 20, fused=True, seed=1)
    assert caches[0].offset == 64 == engine.max_seq_len


@pytest.mark.parametrize("key", ["d128", "4b", "0.6b"])
def test_decode_b3_fused_with_an_idle_slot_and_ragged_contexts(dev, key):
    run_decode(dev, key, 3, 256, 16, [{0: 30, 2: 95}], 20, fused=True, seed=3)


@pytest.mark.parametrize("key", ["d128", "4b"])
def test_decode_b8_unfused_attention_on_the_matvec_stack(dev, key):
    """B x max_seq_len = 32 K > 16 K: decode_qk_norm_rope_append + paged_attention on the matvec stack.  The 4096-token
    table sends paged_attention to its split wgmma route; slot 0 (1100 keys) and slot 7 (2000) fill several splits."""
    _, engine, _, P = run_decode(dev, key, 8, 4096, 64, [{0: 1100, 1: 5, 2: 63, 3: 64, 5: 300, 7: 2000}], 3, fused=False, seed=8)
    assert attention_routes(P) == {ext.PAGED_WGMMA}
    assert not engine._attention_fused and engine.B <= 8


@pytest.mark.parametrize("msl,fused", [(1024, True), (1088, False)])
def test_decode_b16_swap_ab(dev, msl, fused):
    """B x max_seq_len exactly 16 K keeps the fused attention; one page more (1088) does not."""
    lens = {b: 3 + 61 * b for b in range(16) if b % 5 != 2}
    run_decode(dev, "d128", 16, msl, 64, [lens], 3, fused=fused, seed=16)


def test_decode_b16_unfused_at_head_ratio_2_width(dev):
    run_decode(dev, "0.6b", 16, 1088, 64, [{b: 7 + 50 * b for b in range(16) if b % 3}], 2, fused=False, seed=61)


def test_decode_b32_serving_configuration_row_variants(dev):
    """32 slots behind 1024-token tables of 64-slot pages, as the serving configuration runs it: slots 0..12 occupied
    replay the 16-row graph, then slot 31 joins and the full 32-row graph runs."""
    _, engine, _, P = run_decode(dev, "d128", 32, 1024, 64, [{b: 9 + 13 * b for b in range(13) if b % 4 != 2}, {31: 700}], 3, fused=False, seed=32)
    assert engine.variant_replays[16] == 3 and engine.variant_replays[32] == 3
    assert attention_routes(P) == {ext.PAGED_WGMMA}


def test_decode_b64_row_variants(dev):
    _, engine, _, _ = run_decode(dev, "d128", 64, 128, 16, [{b: 4 + b for b in range(10)}, {20: 33}, {63: 100}], 2, fused=True, seed=64)
    assert engine.variant_replays == {16: 2, 32: 2, 64: 2}


@pytest.mark.parametrize("B,msl,fused", [(3, 256, True), (8, 4096, False)])
def test_decode_on_device_equals_the_plan_with_its_own_feedback(dev, B, msl, fused):
    """N = 24 self-advancing replays against 24 plan steps fed by the plan's own argmax: the token log, the step counter,
    the final logits and the slabs."""
    steps, page = 24, 64
    model = make_model("d128", page, dev)
    engine = DecodeEngine(model, B, msl, dev)
    engine.reserve_pools()
    assert engine._attention_fused == fused
    lens = {0: 40, 2: 63} if B == 3 else {0: 1030, 1: 9, 4: 64, 7: 500}
    caches = admit(model, B, msl, lens)
    randomize_slabs(model, B)
    slot0 = occupied(caches)
    tokens = [(17 * b + 3) if c is not None else 0 for b, c in enumerate(slot0)]
    offsets = [c.offset if c is not None else 0 for c in slot0]
    before = slabs(model)
    log = engine.decode_on_device(tokens, offsets, caches, steps)
    meta = plan.decode_metadata(caches, tokens, engine.max_pages, steps=steps)
    assert meta.offsets == offsets
    pages = [(k.clone(), v.clone()) for k, v in before]
    P = plan.Plan(model)
    want = []
    for s in range(steps):
        P.stages = []
        logits, nxt = P.decode(meta, pages, fused)
        want.append([t if c > 0 else -1 for t, c in zip(nxt.tolist(), meta.context_lens)])
        meta.tokens = [t if c > 0 else 0 for t, c in zip(nxt.tolist(), meta.context_lens)]
        meta.offsets = [o + 1 if c > 0 else o for o, c in zip(meta.offsets, meta.context_lens)]
        meta.context_lens = [c + 1 if c > 0 else 0 for c in meta.context_lens]
    assert log.tolist() == want
    assert int(engine.step_counter) == steps
    assert torch.equal(engine.logits, logits)
    assert_slabs_equal(model, pages, f"decode_on_device B {B}")
    reach("decode_on_device", f"B {B}")


def test_recapture_after_slab_growth_equals_the_plan(dev):
    """A second engine reserves more pages, the slabs move and the first engine re-captures: its warm-up passes run with
    all-idle metadata, so the replay equals the plan bit for bit on the new slabs - including the pages that request A
    released and request B was handed."""
    model = make_model("d128", 8, dev)
    small = DecodeEngine(model, 1, 64, dev)
    small.reserve_pools()
    P = plan.Plan(model)
    a = admit(model, 1, 64, {0: 7})
    randomize_slabs(model, 100)
    decode_step(model, small, P, a, [5], "recapture: request A", True)
    released = list(a[0].page_ids)
    for c in a:
        c.release()  # A's pages go back to the free list ...
    b = admit(model, 1, 64, {0: 9})  # ... and are handed to B
    assert set(released) <= set(b[0].page_ids)
    big = DecodeEngine(model, 4, 256, dev)
    big.reserve_pools()  # the slabs move
    randomize_slabs(model, 101)
    decode_step(model, small, P, b, [9], "recapture: request B after slab growth", True)
    assert small.captures == 2
    reach("re-capture", "B 1 after a 4-slot engine reserved")


# ----------------------------------------------------------------- prefill --
def prefill_case(dev, key, chunk, msl, sizes, seed, what):
    """Feed ``sizes`` tokens chunk by chunk through a PrefillEngine, each chunk against the plan, then one decode step on the
    same caches."""
    page = 64
    model = make_model(key, page, dev)
    engine = PrefillEngine(model, chunk, msl, dev)
    engine.reserve_pools(engine.max_pages + 2)
    randomize_slabs(model, seed)
    g = torch.Generator().manual_seed(seed)
    cache = model.create_kv_cache()
    P = plan.Plan(model)
    for r in sizes:
        ids = torch.randint(1, model.vocab_size, (r,), generator=g).tolist()
        off = cache[0].offset
        before = slabs(model)
        engine.prefill_chunk(ids, off, cache)
        meta = plan.prefill_metadata(cache, ids, off, chunk, engine.max_pages)
        pages = [(k.clone(), v.clone()) for k, v in before]
        P.stages = []
        n0 = ext.launch_count()
        logits, nxt = P.prefill(meta, pages)
        assert ext.launch_count() - n0 == engine.kernels_per_chunk
        label = f"{what} chunk at {off} ({r} of {chunk} rows)"
        assert torch.equal(engine.logits, logits), f"{label}: logits differ from the plan"
        assert torch.equal(engine.next_token, nxt), label
        assert_slabs_equal(model, pages, label)
        Checker(model, P).check(before, pages, label)
        reach("prefill L <= 128" if chunk <= 128 else "prefill L > 128", label)
        if r < chunk:
            reach("right-aligned tail chunk", label)
    dec = DecodeEngine(model, 1, msl, dev)
    dec.reserve_pools()  # the slabs keep the prefill's pages
    decode_step(model, dec, P, cache, [int(nxt)], f"{what}: decode after prefill", True)


def test_prefill_chunk32_right_aligned_tail(dev):
    prefill_case(dev, "d128", 32, 256, [32, 32, 13], 77, "d128 chunk 32")


def test_prefill_chunk128_mid_page_at_4b_width(dev):
    prefill_case(dev, "4b", 128, 512, [44, 128, 128], 300, "4b chunk 128")


@pytest.mark.parametrize("key", ["d128", "4b"])
@pytest.mark.parametrize("sizes", [[256, 256, 88], [2]], ids=["600", "2-at-0"])
def test_prefill_chunk256_operator_stack(dev, key, sizes):
    """L > 128: the 128-token-tile GEMM, chunk_qk_norm_rope_append, separate add / rms_norm; the 2-token first chunk has
    254 padding rows at negative positions."""
    prefill_case(dev, key, 256, 1024, sizes, 600 + len(sizes), f"{key} chunk 256")


def test_prefill_chunk1024(dev):
    prefill_case(dev, "d128", 1024, 2048, [1024], 1024, "d128 chunk 1024")


# ---------------------------------------------------------------- coverage --
BRANCHES = {
    "matvec + fused attention", "matvec + unfused attention", "swap-AB + fused attention", "swap-AB + unfused attention",
    "row variant 16", "row variant 32", "row variant full", "decode_on_device", "re-capture", "prefill L <= 128",
    "prefill L > 128", "right-aligned tail chunk",
}


def test_the_cases_reach_every_engine_branch(dev, capsys):
    with capsys.disabled():
        print("\nengine branches:")
        for b in sorted(REACHED):
            print(f"  {b:30s} <- {REACHED[b]}")
        print("largest error / bound per stage:")
        for k in sorted(RATIOS):
            print(f"  {k:28s} {RATIOS[k]:.4f}")
    assert BRANCHES <= set(REACHED), sorted(BRANCHES - set(REACHED))
    assert math.isfinite(max(RATIOS.values(), default=0.0))
