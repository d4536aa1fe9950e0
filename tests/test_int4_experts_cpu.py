"""INT4 expert weights without a GPU: the host side of `Transformer(..., expert_weights="int4")` -- the Int4Expert storage and its
zero-copy views into the interleaved w13 rows (checked against the restatement in tests/int4_dense_ref.py), state-dict keys, the
refusals before allocation -- and of `dense_weights="int4"` on mixture-of-experts models, which quantises the attention Linears only."""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200.moe import EXPERT_WEIGHTS, Fp8Expert, Int4Expert, MoeLayer
from mistral_inference_b200.transformer import Transformer
from tests import int4_dense_ref as I4


def moe_args(**overrides):
    p = synth.shape("tiny-moe", **overrides)
    return p, mi.TransformerArgs.from_dict(dict(p))


def rand_bf16(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * torch.logspace(-3, 3, shape[0])[:, None]).to(torch.bfloat16)


# ----------------------------------------------------------------------------- storage and views
def test_expert_weights_keyword_and_storage():
    assert EXPERT_WEIGHTS == ("bf16", "fp8", "int4")
    _, args = moe_args()
    m = Transformer(args, expert_weights="int4")
    assert m.expert_weights == "int4"
    ff = m.layers["1"].feed_forward
    assert isinstance(ff, MoeLayer) and ff.expert_weights == "int4" and not ff.fp8
    ex = ff.experts["5"]
    assert isinstance(ex, Int4Expert)
    dim, hidden = args.dim, args.hidden_dim
    assert ex.w13.dtype == torch.uint8 and tuple(ex.w13.shape) == (2 * hidden, dim // 2)
    assert ex.w2_weight.dtype == torch.uint8 and tuple(ex.w2_weight.shape) == (dim, hidden // 2)
    assert ex.w13_gscale_bits.dtype == torch.int16 and tuple(ex.w13_gscale_bits.shape) == (2 * hidden, dim // 128)
    assert ex.w2_gscale_bits.dtype == torch.int16 and tuple(ex.w2_gscale_bits.shape) == (dim, hidden // 128)
    # the attention stays bf16 unless dense_weights says otherwise
    assert m.layers["0"].attention.wqkv.dtype == torch.float32 and not m.layers["0"].attention.int4


def test_scales_survive_module_to_bf16():
    _, args = moe_args()
    m = Transformer(args, expert_weights="int4")
    ex = m.layers["0"].feed_forward.experts["0"]
    with torch.no_grad():
        ex.w13_gscale.copy_(torch.linspace(1e-30, 3e30, ex.w13_gscale.numel()).view_as(ex.w13_gscale))
        ex.w2_gscale.copy_(torch.linspace(-5.0, 5.0, ex.w2_gscale.numel()).view_as(ex.w2_gscale))
    before = (ex.w13_gscale_bits.clone(), ex.w2_gscale_bits.clone())
    m = m.to(torch.bfloat16)
    ex = m.layers["0"].feed_forward.experts["0"]
    assert torch.equal(ex.w13_gscale_bits, before[0]) and torch.equal(ex.w2_gscale_bits, before[1])
    assert ex.w13.dtype == torch.uint8 and m.dtype == torch.bfloat16


def test_views_land_in_the_interleaved_rows():
    dim, hidden = 256, 384
    ex = Int4Expert(dim, hidden)
    w1, w3, w2 = rand_bf16((hidden, dim), 1), rand_bf16((hidden, dim), 2), rand_bf16((dim, hidden), 3)
    with torch.no_grad():
        for name, w in (("w1", w1), ("w3", w3), ("w2", w2)):
            c, s = I4.quantize(w)
            ex.weight_int4(name).copy_(c)
            ex.weight_gscale(name).copy_(s)
    # what the quantiser's row strides produce: the restatement of the packed gate/up matrix, row 2i = w1[i], row 2i + 1 = w3[i]
    w13 = torch.stack((w1, w3), dim=1).reshape(2 * hidden, dim)
    c13, s13 = I4.quantize(w13)
    assert torch.equal(ex.w13, c13) and torch.equal(ex.w13_gscale.view(torch.int16), s13.view(torch.int16))
    c2, s2 = I4.quantize(w2)
    assert torch.equal(ex.w2_weight, c2) and torch.equal(ex.w2_gscale.view(torch.int16), s2.view(torch.int16))
    assert torch.equal(I4.dequantize(ex.w13, ex.w13_gscale)[1::2], I4.dequantize(*I4.quantize(w3)))
    # zero-copy, with the packing strides
    G = dim // 128
    c1, c3 = ex.weight_int4("w1"), ex.weight_int4("w3")
    assert c1.stride() == (dim, 1) and c1.data_ptr() == ex.w13.data_ptr() and c3.data_ptr() == ex.w13.data_ptr() + dim // 2
    g1, g3 = ex.weight_gscale("w1"), ex.weight_gscale("w3")
    assert g1.dtype == torch.bfloat16 and g1.stride() == (2 * G, 1) and g3.data_ptr() == ex.w13_gscale_bits.data_ptr() + 2 * G
    assert ex.weight_int4("w2").data_ptr() == ex.w2_weight.data_ptr()
    with pytest.raises(ValueError):
        ex.weight_int4("w4")


def test_expert_bytes_are_a_quarter_plus_the_scales():
    _, args = moe_args(n_layers=2)
    m = Transformer.empty(args, device="cpu", expert_weights="int4")
    expert_bytes = sum(t.numel() * t.element_size() for n, t in m.named_parameters() if ".experts." in n)
    mats = 3 * args.dim * args.hidden_dim
    assert expert_bytes == args.n_layers * args.moe.num_experts * (mats // 2 + 2 * mats // 128)


def test_state_dict_keys_are_zero_copy_views():
    p, args = moe_args()
    m = Transformer(args, expert_weights="int4").to(torch.bfloat16)
    sd = m.state_dict()
    ref = set(synth.synth_state_dict(p, 1))
    experts = {k for k in ref if ".experts." in k}
    want = (ref - experts) | {k[: -len(".weight")] + s for k in experts for s in (".weight_int4", ".weight_gscale")}
    assert set(sd) == want
    ex = m.layers["0"].feed_forward.experts["3"]
    d = args.dim
    w1, w3, w2 = (sd[f"layers.0.feed_forward.experts.3.{n}.weight_int4"] for n in ("w1", "w3", "w2"))
    assert w1.dtype == torch.uint8 and w1.data_ptr() == ex.w13.data_ptr() and w3.data_ptr() == ex.w13.data_ptr() + d // 2
    assert w2.data_ptr() == ex.w2_weight.data_ptr()
    s3 = sd["layers.0.feed_forward.experts.3.w3.weight_gscale"]
    assert s3.dtype == torch.bfloat16 and s3.data_ptr() == ex.w13_gscale_bits.data_ptr() + 2 * (d // 128)
    # the reference's bf16 expert keys provide these entries, and a missing one is named
    assert m._missing_keys(ref) == set()
    assert m._missing_keys(ref - {"layers.1.feed_forward.experts.6.w2.weight"}) == {"layers.1.feed_forward.experts.6.w2.weight_int4",
                                                                                   "layers.1.feed_forward.experts.6.w2.weight_gscale"}
    # the views round-trip: a second model filled through the first one's keys holds the same bytes
    m2 = Transformer(args, expert_weights="int4").to(torch.bfloat16)
    with torch.no_grad():
        for k, v in m.state_dict().items():
            if v.dtype == torch.uint8:
                v.copy_(torch.randint(0, 256, v.shape, dtype=torch.uint8))
        for k, v in m2.state_dict().items():
            v.copy_(m.state_dict()[k])
    for (n1, t1), (n2, t2) in zip(m.named_parameters(), m2.named_parameters()):
        assert n1 == n2 and torch.equal(t1.view(torch.uint8), t2.view(torch.uint8)), n1  # bytes: uninitialised bf16 may hold NaNs


def test_expert_parallel_shard_allocates_its_own_experts_only():
    _, args = moe_args()
    m = Transformer(args, expert_parallel=(1, 2), expert_weights="int4")
    ff = m.layers["0"].feed_forward
    assert ff.local_expert_ids == [1, 3, 5, 7] and all(isinstance(e, Int4Expert) for e in ff.experts.values())
    assert m._owns_key("layers.0.feed_forward.experts.3.w1.weight") and not m._owns_key("layers.0.feed_forward.experts.2.w1.weight")


# ----------------------------------------------------------------------------- refusals
def test_refusals_before_allocation():
    with pytest.raises(ValueError, match="mixture-of-experts"):
        Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape("tiny"))), device="meta", expert_weights="int4")
    for bad in (dict(hidden_dim=320), dict(hidden_dim=192), dict(dim=320)):
        _, args = moe_args(**bad)
        with pytest.raises(ValueError, match="multiples of 128"):
            Transformer.empty(args, device="meta", expert_weights="int4")
        Transformer.empty(args, device="meta", expert_weights="fp8")  # FP8 experts have no 128-wide groups
    for name in ("mixtral-8x7b", "mixtral-8x22b"):
        Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape(name, n_layers=1))), device="meta", expert_weights="int4",
                          dense_weights="int4")


def test_loader_and_lora_refusals():
    _, args = moe_args()
    m = Transformer(args, expert_weights="int4").to(torch.bfloat16)
    assert m._megakernel_ok(1) is False
    for key in ("layers.0.feed_forward.experts.0.w1.weight_int4", "layers.0.feed_forward.experts.0.w2.weight_gscale",
                "layers.0.feed_forward.experts.0.w4.weight"):
        with pytest.raises(ValueError):  # a pre-quantised checkpoint key is not a format the loader reads
            m.load_state_dict({key: torch.zeros(1)}, strict=False)
    with pytest.raises(AssertionError):  # a bf16 expert weight of the wrong shape, before any kernel runs
        m.load_state_dict({"layers.0.feed_forward.experts.0.w1.weight": torch.zeros(args.dim, args.dim + 8, dtype=torch.bfloat16)}, strict=False)
    lora = {"layers.0.feed_forward.experts.2.w1.lora_A.weight": torch.zeros(4, args.dim, dtype=torch.bfloat16),
            "layers.0.feed_forward.experts.2.w1.lora_B.weight": torch.zeros(args.hidden_dim, 4, dtype=torch.bfloat16)}
    with pytest.raises(NotImplementedError, match="INT4 expert"):
        m._load_lora_state_dict(lora)


# ----------------------------------------------------------------------------- dense_weights="int4" on MoE models
@pytest.mark.parametrize("experts", ["fp8", "int4"])
def test_dense_int4_on_moe_quantises_the_attention_only(experts):
    p, args = moe_args()
    m = Transformer(args, dense_weights="int4", expert_weights=experts).to(torch.bfloat16)
    blk = m.layers["0"]
    att = blk.attention
    assert att.int4 and att.wqkv.dtype == torch.uint8 and att.wo_weight.dtype == torch.uint8
    cls = {"fp8": Fp8Expert, "int4": Int4Expert}[experts]
    assert all(type(e) is cls for e in blk.feed_forward.experts.values())
    assert blk.feed_forward.expert_weights == experts
    sd = m.state_dict()
    ref = set(synth.synth_state_dict(p, 1))
    att_keys = {k for k in ref if I4.is_dense_key(k) and ".attention." in k}
    ex_keys = {k for k in ref if ".experts." in k}
    ex_sfx = {"fp8": (".weight_e4m3", ".weight_scale"), "int4": (".weight_int4", ".weight_gscale")}[experts]
    want = (ref - att_keys - ex_keys) | {k[: -len(".weight")] + s for k in att_keys for s in (".weight_int4", ".weight_gscale")} \
        | {k[: -len(".weight")] + s for k in ex_keys for s in ex_sfx}
    assert set(sd) == want
    assert m._missing_keys(ref) == set()
    # a MoE block has no dense feed_forward.w1/w2/w3: such keys are not taken for INT4 Linears
    with pytest.raises(ValueError):
        m.load_state_dict({"layers.0.feed_forward.w1.weight": torch.zeros(args.hidden_dim, args.dim, dtype=torch.bfloat16)}, strict=False)
    with pytest.raises(NotImplementedError):
        m._load_lora_state_dict({"layers.0.attention.wo.lora_A.weight": torch.zeros(4, args.n_heads * args.head_dim, dtype=torch.bfloat16),
                                 "layers.0.attention.wo.lora_B.weight": torch.zeros(args.dim, 4, dtype=torch.bfloat16)})


def test_dense_int4_on_moe_needs_quantised_experts():
    _, args = moe_args()
    with pytest.raises(ValueError, match="quantised experts"):
        Transformer.empty(args, device="meta", dense_weights="int4")  # bf16 experts: refused before allocation
    with pytest.raises(ValueError, match="quantised experts"):
        Transformer.empty(args, device="meta", dense_weights="int4", expert_weights="bf16")
    Transformer.empty(args, device="meta", dense_weights="int4", expert_weights="int4")


def test_dense_int4_shape_checks_cover_the_attention_of_moe_models():
    # hidden_dim 320 is no dense Linear of a MoE model: only the attention shapes are checked (FP8 experts take any K % 8)
    _, args = moe_args(hidden_dim=320)
    Transformer.empty(args, device="meta", dense_weights="int4", expert_weights="fp8")
    # wo [dim, q_dim] with dim 320: N on neither 128 nor 192, and wqkv K = 320 splits a scale group
    _, args = moe_args(dim=320)
    with pytest.raises(ValueError, match="mma.sync"):
        Transformer.empty(args, device="meta", dense_weights="int4", expert_weights="fp8")
    _, args = moe_args()
    with pytest.raises(ValueError, match="dense model"):  # FP8 attention Linears on MoE models stay refused
        Transformer.empty(args, device="meta", dense_weights="fp8", expert_weights="fp8")
