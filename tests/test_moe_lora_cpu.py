"""Un-merged LoRA on FP8 experts without a GPU: the host side of `Transformer(..., expert_weights="fp8")` with a `lora` block --
state-dict keys against the reference's, both checkpoint layouts, load_lora semantics, rank and shard filtering, and the
configurations that stay refused.  The e4m3 quantiser runs on the device; here its CPU restatement (oracle/fp8.py) stands in, so
these tests check where each tensor goes, not the quantiser's bits (tests/test_gpu_moe_lora.py does)."""
import json

import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import moe as M
from mistral_inference_b200.transformer import Transformer
from mistral_inference_b200.transformer_layers import LoraAdapter
from oracle import fp8 as F8
from oracle import moe_lora as OM
from oracle.make_moe_lora_pins import MOE_LORA_PINS_FILE, MOE_LORA_SHAPE


def _args(p, rank=4, scaling=2.0):
    a = mi.TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=scaling)))
    a.max_batch_size = 1
    return a


@pytest.fixture
def cpu_quantiser(monkeypatch):
    def quantize_rows_(name, w, q, s):
        assert tuple(w.shape) == tuple(q.shape), f"{name}: shape {tuple(w.shape)} != expected {tuple(q.shape)}"
        qq, ss = F8.quantize_rows(w.to(torch.bfloat16))
        q.copy_(qq)
        s.copy_(ss)

    monkeypatch.setattr(M, "quantize_rows_", quantize_rows_)


def _model(p, rank=4, scaling=2.0, **kw):
    return Transformer.empty(_args(p, rank, scaling), device="cpu", dtype=torch.bfloat16, expert_weights="fp8", **kw)


def _reference_keys():
    import safetensors

    with safetensors.safe_open(str(MOE_LORA_PINS_FILE), "pt") as f:
        return json.loads(f.metadata()["state_dict_keys"])


def _renamed(keys):
    """The reference's keys with every expert base `.linear.weight` stored as `.linear.weight_e4m3` and `.linear.weight_scale`."""
    out = []
    for k in keys:
        if ".experts." in k and k.endswith(".linear.weight"):
            out += [k[: -len(".weight")] + ".weight_e4m3", k[: -len(".weight")] + ".weight_scale"]
        else:
            out.append(k)
    return out


def test_state_dict_keys_match_reference():
    p = synth.shape(MOE_LORA_SHAPE)
    m = _model(p)
    ref = _reference_keys()
    assert sorted(m.state_dict()) == sorted(_renamed(ref))
    E = p["moe"]["num_experts"]
    assert sum(".experts." in k and k.endswith(".lora_A.weight") for k in ref) == p["n_layers"] * E * 3
    assert m._missing_keys(set(ref)) == set()
    assert m._missing_keys(set(synth.synth_state_dict(p, 1))) == set()  # a plain checkpoint: zero adapters
    ex = m.layers["0"].feed_forward.experts["3"]
    assert isinstance(ex, M.Fp8Expert) and ex.w13_lora.interleaved and ex.w13_lora.rank_cols == 64 and ex.w2_lora.rank_cols == 64
    assert ex.w13_lora.a.dtype == torch.bfloat16 and ex.w13_q.dtype == torch.uint8


def test_both_layouts_load_and_a_plain_checkpoint_zeroes_the_adapters(cpu_quantiser):
    p = synth.shape(MOE_LORA_SHAPE)
    plain = synth.synth_state_dict(p, 3)
    ad = OM.synth_moe_lora_state_dict(p, 4, 7)
    base = Transformer.empty(mi.TransformerArgs.from_dict(dict(p)), device="cpu", dtype=torch.bfloat16, expert_weights="fp8")
    base.load_state_dict(plain)

    m = _model(p)
    m.load_state_dict(OM.moe_lora_weights(plain, ad))  # the reference's LoRA layout
    sd = m.state_dict()
    for k, v in ad.items():
        assert torch.equal(sd[k], v), k
    _assert_same_base(m, base)

    m.load_state_dict(plain)  # a plain checkpoint on top: zero adapters, the same base
    sd = m.state_dict()
    assert all(not sd[k].any() for k in ad)
    for mod in m.modules():
        if isinstance(mod, LoraAdapter):
            assert not mod.a.any() and not mod.b.any()
    _assert_same_base(m, base)


def _assert_same_base(m, base):
    """Every quantised expert matrix and scale, and the attention weights, equal those of the plain FP8 load bit for bit."""
    for lid, blk in m.layers.items():
        for e, ex in blk.feed_forward.experts.items():
            ex0 = base.layers[lid].feed_forward.experts[e]
            for t in ("w13_q", "w2_q", "w13_scale_bits", "w2_scale_bits"):
                assert torch.equal(getattr(ex, t), getattr(ex0, t)), (lid, e, t)
        assert torch.equal(blk.attention.wqkv, base.layers[lid].attention.wqkv)
        assert torch.equal(blk.feed_forward.gate_weight, base.layers[lid].feed_forward.gate_weight)


def test_load_lora_replaces_and_ignores_scaling(cpu_quantiser):
    p = synth.shape(MOE_LORA_SHAPE)
    m = _model(p, scaling=0.5)
    m.load_state_dict(synth.synth_state_dict(p, 3))
    a, b = OM.synth_moe_lora_state_dict(p, 4, 7), OM.synth_moe_lora_state_dict(p, 4, 8)
    ptrs = [t.data_ptr() for t in m.parameters()]
    m._load_lora_state_dict(b, scaling=7.0)
    m._load_lora_state_dict(a, scaling=7.0)
    sd = m.state_dict()
    assert all(torch.equal(sd[k], v) for k, v in a.items())
    assert {x.scaling for x in m.modules() if isinstance(x, LoraAdapter)} == {0.5}
    assert [t.data_ptr() for t in m.parameters()] == ptrs  # copied in place: captured decode graphs keep their pointers
    half = {k: v for k, v in b.items() if ".experts.2." in k}
    m._load_lora_state_dict(half)  # replaces the Linears it names, and only those
    sd = m.state_dict()
    assert all(torch.equal(sd[k], (half if k in half else a)[k]) for k in a)


def test_wrong_rank_or_dtype_is_refused():
    p = synth.shape(MOE_LORA_SHAPE)
    m = _model(p, rank=4)
    with pytest.raises(AssertionError):
        m._load_lora_state_dict({k: v for k, v in OM.synth_moe_lora_state_dict(p, 8, 7).items() if ".experts." in k})
    with pytest.raises(AssertionError):
        m._load_lora_state_dict({k: v.float() for k, v in OM.synth_moe_lora_state_dict(p, 4, 7).items()})


def test_pipeline_ranks_and_expert_shards_load_their_own_part(cpu_quantiser):
    p = synth.shape(MOE_LORA_SHAPE)
    full = OM.moe_lora_weights(synth.synth_state_dict(p, 3), OM.synth_moe_lora_state_dict(p, 4, 7))
    for rank in (0, 1):
        m = _model(p, pipeline_rank=rank, num_pipeline_ranks=2)
        m.load_state_dict(full, strict=False)
        m._load_lora_state_dict(OM.synth_moe_lora_state_dict(p, 4, 7))  # the other rank's layer is skipped, not an error
        sd = m.state_dict()
        mine = [k for k in full if k.startswith(f"layers.{rank}.") and "lora_" in k]
        assert mine and all(torch.equal(sd[k], full[k]) for k in mine)
        assert not any(k.startswith(f"layers.{1 - rank}.") for k in sd)
    for g in (0, 1):
        m = _model(p, expert_parallel=(g, 2))
        assert m._owns_key("layers.0.feed_forward.experts.3.w1.lora_A.weight") == (g == 1)
        m.load_state_dict(full, strict=False)
        m._load_lora_state_dict(OM.synth_moe_lora_state_dict(p, 4, 7))
        sd = m.state_dict()
        ex_keys = [k for k in full if ".experts." in k and "lora_" in k]
        mine = [k for k in ex_keys if int(k.split(".")[4]) % 2 == g]
        assert all(torch.equal(sd[k], full[k]) for k in mine)
        assert not any(k in sd for k in ex_keys if k not in mine)
        assert m._missing_keys({k for k in full if m._owns_key(k)}) == set()


def test_refused_configurations_before_allocation():
    p = synth.shape(MOE_LORA_SHAPE)
    with torch.device("meta"):
        with pytest.raises(NotImplementedError, match="INT4 expert"):
            Transformer(_args(p), expert_weights="int4")
        with pytest.raises(NotImplementedError, match="INT4"):
            Transformer(_args(p), expert_weights="int4", dense_weights="int4")
        with pytest.raises(NotImplementedError, match="mixture-of-experts"):
            Transformer(_args(p))
        with pytest.raises(ValueError):
            Transformer(_args(p), expert_weights="fp8", dense_weights="fp8")
        m = Transformer(_args(p), expert_weights="fp8")  # the combination that is built
    assert m._megakernel_ok(1) is False
    merged = Transformer.empty(mi.TransformerArgs.from_dict(dict(p)), device="cpu", dtype=torch.bfloat16, expert_weights="fp8")
    with pytest.raises(NotImplementedError):  # merging into FP8 experts stays refused
        merged._load_lora_state_dict({k: v for k, v in OM.synth_moe_lora_state_dict(p, 4, 7).items() if ".experts.0." in k})
