"""Un-merged LoRA adapters (params.json `lora` block) on the CPU: the oracle's rounding chain pinned against the reference's own
LoRALinear model (tests/golden/reference/lora_pins.safetensors, written by oracle/make_lora_pins.py), and the host side of
mistral_inference_b200: state-dict keys, both checkpoint layouts, load_lora semantics, pipeline-rank filtering and the
configurations that are refused."""
import json

import pytest
import torch

import synth
from mistral_inference_b200.args import TransformerArgs
from mistral_inference_b200.transformer import Transformer
from mistral_inference_b200.transformer_layers import LoraAdapter
from oracle import lora as OL
from oracle import restatement as R
from oracle.make_lora_pins import (LORA_ADAPTER_SEED, LORA_CASES, LORA_PINS_FILE, LORA_RANKS, LORA_SCALINGS, lora_key,
                                   prompts_for)

from .util import oracle_args, same_machine_as_golden


@pytest.fixture(scope="module")
def pins():
    import safetensors
    import safetensors.torch

    with safetensors.safe_open(str(LORA_PINS_FILE), "pt") as f:
        meta = f.metadata()
    return safetensors.torch.load_file(str(LORA_PINS_FILE)), meta


def _tol(dtype):  # tests/test_oracle_vs_reference.py
    return 1e-4 if dtype == torch.float32 else 6e-2


def _oracle(p, dtype, rank, scaling, max_batch=3, adapter=True):
    w = synth.synth_state_dict(p, 3, dtype)
    ad = synth.synth_lora_state_dict(p, rank, LORA_ADAPTER_SEED, dtype) if adapter else {
        k: torch.zeros_like(v) for k, v in synth.synth_lora_state_dict(p, rank, LORA_ADAPTER_SEED, dtype).items()}
    return OL.OracleLoraTransformer(oracle_args(p, max_batch), OL.lora_weights(w, ad), scaling)


def _compare_generate(gold, meta, key, t_or, lp_or, dtype):
    t_ref = gold[f"{key}/tokens"].tolist()
    lp_ref = torch.split(gold[f"{key}/logprobs"], gold[f"{key}/lengths"].tolist())
    if same_machine_as_golden(meta):
        assert t_ref == t_or
        assert [x.tolist() for x in lp_ref] == lp_or
        return
    for tr, to, lr, lo in zip(t_ref, t_or, lp_ref, lp_or):
        n = next((i for i, (a, b) in enumerate(zip(tr, to)) if a != b), len(tr))
        m = len(lo) - len(to) + n
        torch.testing.assert_close(torch.tensor(lo[:m], dtype=torch.float64), lr[:m], rtol=0, atol=_tol(dtype))


@pytest.mark.parametrize("shape,over", LORA_CASES)
@pytest.mark.parametrize("rank", LORA_RANKS)
@pytest.mark.parametrize("scaling", LORA_SCALINGS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_generate_vs_reference(pins, shape, over, rank, scaling, dtype):
    gold, meta = pins
    p = synth.shape(shape, **over)
    t_or, lp_or = R.generate(prompts_for(p), _oracle(p, dtype, rank, scaling), max_tokens=9, chunk_size=4)
    _compare_generate(gold, meta, f"generate/{lora_key(shape, over, dtype, rank, scaling)}", t_or, lp_or, dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_forward_without_cache_vs_reference(pins, dtype):
    gold, meta = pins
    p = synth.shape("tiny")
    with torch.inference_mode():
        b = _oracle(p, dtype, 8, 2.0, max_batch=2).forward(torch.tensor(synth.synth_prompt(13, p["vocab_size"], 5)), [6, 7])
    a = gold[f"forward_no_cache/{str(dtype).split('.')[-1]}"]
    if same_machine_as_golden(meta):
        assert torch.equal(a, b)
    else:
        torch.testing.assert_close(b, a, rtol=0, atol=_tol(dtype))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_lora_term_is_far_above_tolerance(pins, dtype):
    """Negative control: the oracle without the adapter, or with the scaling applied twice, misses the pinned cache-less logits
    by far more than the tolerance the comparisons above allow."""
    gold, _ = pins
    p = synth.shape("tiny")
    a = gold[f"forward_no_cache/{str(dtype).split('.')[-1]}"]
    toks = torch.tensor(synth.synth_prompt(13, p["vocab_size"], 5))
    with torch.inference_mode():
        dropped = _oracle(p, dtype, 8, 2.0, max_batch=2, adapter=False).forward(toks, [6, 7])
        twice = _oracle(p, dtype, 8, 4.0, max_batch=2).forward(toks, [6, 7])
        plain = R.OracleTransformer(oracle_args(p, 2), synth.synth_state_dict(p, 3, dtype)).forward(toks, [6, 7])
    assert torch.equal(dropped, plain)  # a zero adapter is the plain model
    for wrong in (dropped, twice):
        assert (wrong - a).abs().max().item() > 20 * _tol(dtype)


def test_load_lora_scaling_argument_is_ignored(pins):
    gold, _ = pins
    for d in ("bfloat16", "float32"):
        key = lora_key("tiny", {}, getattr(torch, d), 4, 0.3)
        assert torch.equal(gold[f"load_scaling_7/{d}/tokens"], gold[f"generate/{key}/tokens"])
        assert torch.equal(gold[f"load_scaling_7/{d}/logprobs"], gold[f"generate/{key}/logprobs"])
    p = synth.shape("tiny")
    m = _cpu_model(p, rank=4, scaling=0.3)
    m._load_lora_state_dict(synth.synth_lora_state_dict(p, 4, 1), scaling=7.0)
    assert {a.scaling for a in m.modules() if isinstance(a, LoraAdapter)} == {0.3}


# ----------------------------------------------------------------------------- host model (CPU tensors: loading only)
def _args(p, rank=8, scaling=2.0, max_batch=1):
    a = TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=scaling)))
    a.max_batch_size = max_batch
    return a


def _cpu_model(p, rank=8, scaling=2.0, **kw):
    m = Transformer.empty(_args(p, rank, scaling), device="cpu", dtype=torch.bfloat16, **kw)
    m.load_state_dict(synth.synth_state_dict(p, 3))
    return m


def test_state_dict_keys_match_reference(pins):
    _, meta = pins
    want = json.loads(meta["state_dict_keys"])
    m = _cpu_model(synth.shape("tiny"))
    assert sorted(m.state_dict().keys()) == sorted(want)
    assert sum(".lora_A." in k for k in want) == 7 * 2


def test_views_are_zero_copy_and_packed():
    p = synth.shape("tiny")
    m = _cpu_model(p, rank=8)
    ad = synth.synth_lora_state_dict(p, 8, 1)
    m._load_lora_state_dict(ad)
    sd = m.state_dict()
    att, ff = m.layers["0"].attention, m.layers["0"].feed_forward
    for name in ("attention.wq", "attention.wk", "attention.wv", "attention.wo", "feed_forward.w1", "feed_forward.w2", "feed_forward.w3"):
        for part in ("lora_A", "lora_B"):
            assert torch.equal(sd[f"layers.0.{name}.{part}.weight"], ad[f"layers.0.{name}.{part}.weight"])
    assert sd["layers.0.attention.wk.lora_A.weight"].data_ptr() == att.wqkv_lora.a.data_ptr() + 8 * p["dim"] * 2
    # packing: B_exp holds each segment's lora_B in its own columns, zeros elsewhere; the w13 rows interleave like w13
    q, kv, r = 4 * 128, 2 * 128, 8
    b = att.wqkv_lora.b
    assert att.wqkv_lora.rank_cols == 64 and b.shape == (q + 2 * kv, 64)
    assert torch.equal(b[:q, :r], ad["layers.0.attention.wq.lora_B.weight"]) and not b[:q, r:].any()
    assert torch.equal(b[q + kv:, 2 * r:3 * r], ad["layers.0.attention.wv.lora_B.weight"]) and not b[q + kv:, :2 * r].any()
    b13 = ff.w13_lora.b.view(p["hidden_dim"], 2, 64)
    assert torch.equal(b13[:, 0, :r], ad["layers.0.feed_forward.w1.lora_B.weight"]) and not b13[:, 0, r:].any()
    assert torch.equal(b13[:, 1, r:2 * r], ad["layers.0.feed_forward.w3.lora_B.weight"]) and not b13[:, 1, :r].any()
    assert not att.wqkv_lora.a[3 * r:].any()  # padding rows


def test_both_checkpoint_layouts_load(tmp_path):
    p = synth.shape("tiny")
    plain = synth.synth_state_dict(p, 3)
    ad = synth.synth_lora_state_dict(p, 8, 1)
    full = OL.lora_weights(plain, ad)
    a = _cpu_model(p)
    a.load_state_dict(full)
    sd = a.state_dict()
    assert set(sd) == set(full) and all(torch.equal(sd[k], v) for k, v in full.items())
    # a plain checkpoint on top zeroes every adapter (lora.py:76-89) and keeps the base weights
    a.load_state_dict(plain)
    sd = a.state_dict()
    for k, v in OL.lora_weights(plain, {k: torch.zeros_like(v) for k, v in ad.items()}).items():
        assert torch.equal(sd[k], v), k
    # missing base weights still raise; missing adapters do not
    with pytest.raises(AssertionError, match="missing keys"):
        a.load_state_dict({k: v for k, v in plain.items() if k != "layers.1.attention.wo.weight"})
    a.load_state_dict({k: v for k, v in full.items() if "lora_" not in k})
    # from_folder: a full checkpoint with a lora params.json, and a LoRA-layout checkpoint
    import safetensors.torch

    synth.write_model_folder(tmp_path / "plain", p, seed=3, lora=dict(rank=8, scaling=2.0))
    m = Transformer.from_folder(tmp_path / "plain", device="cpu")
    assert m.args.lora.rank == 8 and not any(v.any() for k, v in m.state_dict().items() if "lora_" in k)
    (tmp_path / "lora").mkdir()
    (tmp_path / "lora" / "params.json").write_text(json.dumps(dict(p, lora=dict(rank=8, scaling=2.0))))
    safetensors.torch.save_file({k: v.contiguous() for k, v in full.items()}, str(tmp_path / "lora" / "consolidated.safetensors"))
    m = Transformer.from_folder(tmp_path / "lora", device="cpu")
    sd = m.state_dict()
    assert all(torch.equal(sd[k], v) for k, v in full.items())


def test_load_lora_replaces_instead_of_accumulating(tmp_path):
    import safetensors.torch

    p = synth.shape("tiny")
    m = _cpu_model(p)
    base = {k: v.clone() for k, v in m.state_dict().items() if k.endswith(".linear.weight")}
    ad_a, ad_b = synth.synth_lora_state_dict(p, 8, 1), synth.synth_lora_state_dict(p, 8, 2)
    safetensors.torch.save_file(ad_a, str(tmp_path / "a.safetensors"))
    safetensors.torch.save_file(ad_b, str(tmp_path / "b.safetensors"))
    m.load_lora(tmp_path / "a.safetensors")
    first = {k: v.clone() for k, v in m.state_dict().items()}
    m.load_lora(tmp_path / "b.safetensors")
    assert all(torch.equal(m.state_dict()[k], v) for k, v in ad_b.items())
    m.load_lora(tmp_path / "a.safetensors")
    sd = m.state_dict()
    assert all(torch.equal(sd[k], v) for k, v in first.items())
    assert all(torch.equal(sd[k], v) for k, v in base.items())  # base weights never change


def test_load_lora_checks():
    p = synth.shape("tiny")
    m = _cpu_model(p, rank=8)
    with pytest.raises(AssertionError, match="shape"):
        m._load_lora_state_dict(synth.synth_lora_state_dict(p, 4, 1))  # rank 4 into rank-8 slots
    with pytest.raises(AssertionError, match="dtype"):
        m._load_lora_state_dict(synth.synth_lora_state_dict(p, 8, 1, dtype=torch.float32))
    with pytest.raises(AssertionError):
        m._load_lora_state_dict({"layers.0.attention.wq.weight": torch.zeros(512, 256, dtype=torch.bfloat16)})


def test_pipeline_ranks_load_their_own_layers():
    p = synth.shape("tiny")
    ad = synth.synth_lora_state_dict(p, 8, 1)
    for rank in (0, 1):
        m = Transformer.empty(_args(p), device="cpu", dtype=torch.bfloat16, pipeline_rank=rank, num_pipeline_ranks=2)
        m.load_state_dict(synth.synth_state_dict(p, 3), strict=False)
        m._load_lora_state_dict(ad)  # the other rank's layer is skipped, not an error
        sd = m.state_dict()
        mine = [k for k in ad if k.startswith(f"layers.{rank}.")]
        assert mine and all(torch.equal(sd[k], ad[k]) for k in mine)
        assert not any(k.startswith(f"layers.{1 - rank}.") for k in sd)


def test_moe_with_lora_is_refused_before_allocation():
    p = synth.shape("tiny-moe")
    with pytest.raises(NotImplementedError, match="mixture-of-experts"):
        Transformer(_args(p))


def test_vision_tower_has_no_adapters():
    p = synth.shape("pixtral-ref-test")
    m = Transformer.empty(_args(p), device="cpu", dtype=torch.bfloat16)
    keys = list(m.state_dict())
    assert any(k.startswith("layers.0.attention.wq.lora_A") for k in keys)
    assert not any("lora" in k or ".linear." in k for k in keys if not k.startswith("layers."))
    assert "output.weight" in keys and all("gate" not in k for k in keys)
    m.load_state_dict(synth.synth_state_dict(p, 3))
