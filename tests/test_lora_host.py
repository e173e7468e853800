"""Host logic of multi-LoRA serving, with ``ext.lora_apply`` replaced by its CPU stand-in (``tests/lora_ref.py``): the
PEFT round trip and refusals, rank padding and the packed layout, the batcher's slot ids, prefix-cache isolation, the
CLI flags, and the stand-in against the float64 reference."""

import importlib.util
import json
import sys
from pathlib import Path

import pytest
import torch

from extensions_b200 import tiny_llm_ext_b200 as ext
from tiny_llm_b200 import Qwen3ModelWeek3
from tiny_llm_b200.batch import ContinuousBatcher
from tiny_llm_b200.cli import main as cli_main, parse_lora_specs
from tiny_llm_b200.generate import greedy_generate_ids
from tiny_llm_b200.lora import AdapterSet, LoraAdapter, adapter_ids_of, projection_shapes
from tiny_llm_b200.synthetic import make_args, synthetic_qwen3


def _load(name, file):
    if name not in sys.modules:
        spec = importlib.util.spec_from_file_location(name, Path(__file__).with_name(file))
        module = importlib.util.module_from_spec(spec)
        sys.modules[name] = module
        spec.loader.exec_module(module)
    return sys.modules[name]


lref = _load("tiny_llm_b200_lora_ref", "lora_ref.py")
pcref = _load("tiny_llm_b200_prefix_cache_ref", "prefix_cache_ref.py")
ARGS = make_args("tiny-d128")


@pytest.fixture
def lora_ext(cpu_ext, monkeypatch):
    lref.install(cpu_ext, monkeypatch)
    pcref.install(cpu_ext, monkeypatch)
    return cpu_ext


def test_peft_round_trip(tmp_path):
    adapter = LoraAdapter.synthetic(ARGS, 16, targets=("q", "v", "down"), seed=3, name="x")
    adapter.save(tmp_path / "x")
    config = json.loads((tmp_path / "x" / "adapter_config.json").read_text())
    assert config["r"] == 16 and config["lora_alpha"] == 32.0 and config["target_modules"] == ["q_proj", "v_proj", "down_proj"]
    back = LoraAdapter.load(tmp_path / "x")
    assert back.name == "x" and back.rank == 16 and back.alpha == 32.0 and back.targets == ("q", "v", "down")
    assert back.tensors.keys() == adapter.tensors.keys()
    for key, (A, B) in adapter.tensors.items():
        assert torch.equal(back.tensors[key][0], A) and torch.equal(back.tensors[key][1], B)
        assert float(B.abs().max()) > 0, "a synthetic adapter must not have B = 0"


def _saved(tmp_path, edit_config=None, edit_tensors=None):
    from safetensors.torch import load_file, save_file

    LoraAdapter.synthetic(ARGS, 8, targets=("q",), name="t").save(tmp_path)
    if edit_config:
        config = json.loads((tmp_path / "adapter_config.json").read_text())
        edit_config(config)
        (tmp_path / "adapter_config.json").write_text(json.dumps(config))
    if edit_tensors:
        tensors = load_file(str(tmp_path / "adapter_model.safetensors"))
        edit_tensors(tensors)
        save_file(tensors, str(tmp_path / "adapter_model.safetensors"))
    return tmp_path


@pytest.mark.parametrize("case,message", [
    ("dora", "use_dora is not supported"), ("rslora", "use_rslora is not supported"), ("bias", "bias = 'all' is not supported"),
    ("no-r", "lacks 'r'"), ("unknown-key", "unknown tensor 'base_model.model.lm_head.lora_A.weight'"), ("half", "has lora_A only"),
    ("targets", "target_modules = ['k']"), ("rank", "LoRA rank must be one of"),
])
def test_load_refusals(tmp_path, case, message):
    q0 = "base_model.model.model.layers.0.self_attn.q_proj"
    edits = {
        "dora": (lambda c: c.update(use_dora=True), None), "rslora": (lambda c: c.update(use_rslora=True), None),
        "bias": (lambda c: c.update(bias="all"), None), "no-r": (lambda c: c.pop("r"), None),
        "unknown-key": (None, lambda t: t.update({"base_model.model.lm_head.lora_A.weight": torch.zeros(8, 8)})),
        "half": (None, lambda t: t.pop(q0 + ".lora_B.weight")), "targets": (lambda c: c.update(target_modules=["k_proj"]), None),
        "rank": (lambda c: c.update(r=12), None),
    }[case]
    with pytest.raises(ValueError, match=message.replace("[", r"\[").replace("]", r"\]")):
        LoraAdapter.load(_saved(tmp_path, *edits))


def test_shapes_that_do_not_match_the_base_and_set_limits():
    other = make_args("tiny")
    with pytest.raises(ValueError, match=r"layer 0 q_proj is A \(8, 128\).*the base projection is \[512, 256\]"):
        AdapterSet(ARGS, [LoraAdapter.synthetic(other, 8, name="o")])
    a = LoraAdapter.synthetic(ARGS, 8, name="a")
    with pytest.raises(ValueError, match="names must be unique"):
        AdapterSet(ARGS, [a, a])
    with pytest.raises(ValueError, match="1 to 32 adapters"):
        AdapterSet(ARGS, [LoraAdapter("n%d" % i, 8, 16, {}) for i in range(33)])
    with pytest.raises(KeyError, match="no adapter named 'zz'"):
        AdapterSet(ARGS, [a]).id_of("zz")


def test_packing_layout_and_rank_padding():
    a = LoraAdapter.synthetic(ARGS, 8, targets=("q", "v", "gate"), seed=1, name="a")
    b = LoraAdapter.synthetic(ARGS, 32, targets=("k", "o"), seed=2, name="b")
    aset = AdapterSet(ARGS, [a, b])
    assert aset.r_max == 32 and aset.id_of("b") == 1 and aset.id_of(None) == -1
    shapes = projection_shapes(ARGS)
    for layer, sites in enumerate(aset.sites):
        qkv = sites.qkv
        assert sites.down is None and qkv.nseg == 3 and qkv.K == [shapes[p][0] for p in "qkv"] and qkv.N == 256
        assert qkv.seg_mask.tolist() == [0b101, 0b010] and qkv.ranks.tolist() == [8, 32] and qkv.scales.tolist() == [2.0, 2.0]
        assert tuple(qkv.a.shape) == (2, 96, 256) and [tuple(t.shape) for t in qkv.b] == [(2, 512, 32), (2, 256, 32), (2, 256, 32)]
        A, B = a.tensors[(layer, "v")]
        assert torch.equal(qkv.a[0, 64:72], A) and not qkv.a[0, 72:96].any() and not qkv.a[0, 32:64].any()
        assert torch.equal(qkv.b[2][0, :, :8], B) and not qkv.b[2][0, :, 8:].any()
        assert torch.equal(qkv.a[1, 32:64], b.tensors[(layer, "k")][0])
        assert sites.gate_up.seg_mask.tolist() == [1, 0] and sites.o.seg_mask.tolist() == [0, 1]


def test_cpu_stand_in_against_the_reference_and_padding():
    gen = torch.Generator().manual_seed(0)
    site = lref.random_site(gen, 256, [128, 64], [8, 16], masks=[3, 2])
    x = torch.randn(5, 256, generator=gen).to(torch.bfloat16)
    base = torch.randn(5, 192, generator=gen).to(torch.bfloat16)
    ids = torch.tensor([0, -1, 1, 1, 0], dtype=torch.int32)
    y = lref.lora_apply_like_ext(x, base.clone(), ids, site)
    assert torch.equal(y[1], base[1]) and torch.equal(y[2, :128], base[2, :128]) and not torch.equal(y[0], base[0])
    want, bound = lref.lora_reference(x, list(torch.split(base, [128, 64], dim=1)), ids.tolist(), site)
    assert torch.equal(y, torch.cat(want, dim=1).to(torch.bfloat16)) and float(bound[0][1].max()) == 0.0 and float(bound[0][0].min()) > 0
    t = site.a[0, :8].double() @ x[0].double()
    d = 2.0 * (site.b[0][0, :, :8].double() @ lref.bf16_round(t))
    assert torch.equal(y[0, :128].double(), lref.bf16_round(base[0, :128].double() + d))
    res = torch.randn(5, 192, generator=gen).to(torch.bfloat16)
    z = lref.lora_apply_like_ext(x, base.clone(), ids, site, residual=res)
    assert torch.equal(z, (res.double() + y.double()).to(torch.bfloat16))
    with pytest.raises(RuntimeError, match="one row per adapter id"):
        ext.lora_apply(x[:4], base.clone(), ids, site)
    with pytest.raises(RuntimeError, match="GPU-only"):
        ext.lora_apply(x, base.clone(), ids, site)


def _model(ns):
    model = Qwen3ModelWeek3(ns, page_size=8)
    model.load_adapters([LoraAdapter.synthetic(ns.args, 16, seed=0, name="a"), LoraAdapter.synthetic(ns.args, 8, seed=1, name="b")])
    return model


@pytest.fixture(scope="module")
def tiny_ns():
    return synthetic_qwen3("tiny-d128", seed=0, realistic=True, max_position_embeddings=512)


def test_model_refusals(lora_ext, tiny_ns):
    model = _model(tiny_ns)
    with pytest.raises(RuntimeError, match="already has its adapter set"):
        model.load_adapters([])
    plain = Qwen3ModelWeek3(tiny_ns, page_size=8)
    ids = torch.tensor([[5, 17, 3]], dtype=torch.int32)
    with pytest.raises(ValueError, match="the model has none loaded"):
        plain(ids, 0, plain.create_kv_cache(), adapter_ids=[0])
    with pytest.raises(ValueError, match="the model has none loaded"):
        adapter_ids_of(plain, "a", 1)
    with pytest.raises(ValueError, match="exceed the 2 loaded adapters"):
        model(ids, 0, model.create_kv_cache(), adapter_ids=[2])
    moe = Qwen3ModelWeek3(synthetic_qwen3("tiny-moe-d128", seed=0), page_size=8)
    with pytest.raises(ValueError, match="Qwen3-MoE models are not supported"):
        moe.load_adapters([LoraAdapter.synthetic(make_args("tiny-moe-d128"), 8, targets=("q",))])
    plain._decode_engines[(1, 8)] = object()
    with pytest.raises(RuntimeError, match="before the first decode or prefill graph engine"):
        plain.load_adapters([LoraAdapter.synthetic(tiny_ns.args, 8)])


@pytest.mark.parametrize("order", [[0, 1, 2, 3], [2, 3, 1, 0]])
def test_batcher_slot_ids_and_tokens_under_two_queue_orders(lora_ext, tiny_ns, order):
    prompts, names = [[5, 17, 3, 9], [5, 17, 3, 9], [5, 17, 3, 9], [8, 1, 300]], ["a", None, "b", "a"]
    model = _model(tiny_ns)
    alone = [greedy_generate_ids(model, p, 5, adapter=n) for p, n in zip(prompts, names)]
    assert alone[0] != alone[1] != alone[2] != alone[0]
    batcher = ContinuousBatcher(model, None, [prompts[i] for i in order], max_seq_len=64, batch_size=2, verbose=False,
                                max_new_tokens=[5] * 4, adapters=[names[i] for i in order])
    while not batcher.idle():
        batcher.step()
        for slot, request in enumerate(batcher.slots):
            assert batcher.slot_adapter_ids[slot] == (-1 if request is None else request.adapter_id)
    batcher.release_all()
    got = {idx: [int(t) for t in text.split()] for idx, text in batcher.results}
    assert [got[pos] for pos in range(4)] == [alone[i] for i in order]
    assert batcher.slot_adapter_ids == [-1, -1]


def test_prefix_cache_roots_are_kept_apart_per_adapter(lora_ext, tiny_ns):
    model = _model(tiny_ns)
    prompt = list(range(3, 23))
    names = ["a", "b", "a", None, None]
    alone = {n: greedy_generate_ids(model, prompt, 4, adapter=n) for n in set(names)}
    batcher = ContinuousBatcher(model, None, [prompt] * 5, max_seq_len=64, batch_size=2, verbose=False, max_new_tokens=[4] * 5,
                                adapters=names, prefix_cache=True)
    results = dict(batcher.run())
    assert [batcher.reused_tokens[i] for i in range(5)] == [0, 0, 19, 0, 19]
    assert [[int(t) for t in results[i].split()] for i in range(5)] == [alone[n] for n in names]
    model.prefix_cache.clear()
    assert model.prefix_cache.lookup(prompt, 0).reused == 0 and model.prefix_cache.stats()["cached_pages"] == 0


def test_cli_flags():
    assert parse_lora_specs(["x=/some/dir"], ["a=16", "b=8:1"]) == ([("x", "/some/dir")], [("a", 16, 0), ("b", 8, 1)])
    for bad in (["nodir"], ["=d"]):
        with pytest.raises(SystemExit, match="--lora expects NAME=DIR"):
            parse_lora_specs(bad, None)
    for bad in (["a"], ["a=x"], ["a=8:y"]):
        with pytest.raises(SystemExit, match="--synthetic-lora expects NAME=RANK"):
            parse_lora_specs(None, bad)


def test_cli_batch_runs_each_request_under_its_adapter(lora_ext, capsys):
    base = ["batch", "--synthetic", "tiny-d128", "--device", "cpu", "--quiet", "--max-new-tokens", "4", "--prompt-ids", "5,17,3;5,17,3;5,17,3"]
    assert cli_main(base + ["--synthetic-lora", "a=16", "--synthetic-lora", "b=8:1", "--adapters", "a;;b"]) == 0
    texts = capsys.readouterr().out.split("--- request ")[1:]
    assert len({t.split("\n")[1] for t in texts}) == 3
    assert cli_main(base) == 0
    plain = capsys.readouterr().out.split("--- request ")[1:]
    assert texts[1] == plain[1]
    with pytest.raises(SystemExit, match="names 2 requests, there are 3 prompts"):
        cli_main(base + ["--synthetic-lora", "a=16", "--adapters", "a;"])
    with pytest.raises(SystemExit, match="no adapter named 'zz'"):
        cli_main(base + ["--synthetic-lora", "a=16", "--adapters", "a;zz;"])
    with pytest.raises(SystemExit, match="rank must be one of"):
        cli_main(base + ["--synthetic-lora", "a=12"])
