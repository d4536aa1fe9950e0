"""FP8 (e4m3) expert weights without a GPU: the CPU restatement of the storage format (oracle/fp8.py) on hand-made rows, and the
host side of `Transformer(..., expert_weights="fp8")` -- storage, state-dict keys and refusals."""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200.moe import Fp8Expert
from mistral_inference_b200.transformer import Transformer
from oracle import fp8 as F8


def q_values(q: torch.Tensor) -> torch.Tensor:
    return q.view(torch.float8_e4m3fn).float()


def rows(*vals) -> torch.Tensor:
    return torch.tensor(vals, dtype=torch.float32).to(torch.bfloat16)


def test_scale_is_amax_over_448_and_one_for_zero_rows():
    w = torch.stack([rows(448.0, -3.0, 1.0, 0.0), rows(-7.0, 2.0, 0.5, 0.0), rows(0.0, 0.0, 0.0, 0.0), rows(-0.0, 0.0, -0.0, 0.0)])
    q, s = F8.quantize_rows(w)
    assert s.dtype == torch.float32 and q.dtype == torch.uint8
    assert s.tolist() == [1.0, (torch.tensor(7.0) / torch.tensor(448.0)).item(), 1.0, 1.0]
    # an all-zero row quantises to zeros and keeps the sign of negative zero
    assert q[2].tolist() == [0, 0, 0, 0]
    assert q[3].tolist() == [0x80, 0, 0x80, 0]
    wp = F8.fp8_weights(w)
    assert torch.equal(wp[3].view(torch.int16), w[3].view(torch.int16))
    # the row maximum maps to +-448 exactly and comes back exactly
    assert q_values(q[1])[0].item() == -448.0 and wp[1, 0].item() == -7.0 and wp[0, 0].item() == 448.0


def test_ties_round_to_even_and_saturate_at_448():
    # s = 1 (amax 448): q = e4m3(W) directly.  1.0625 and 1.1875 lie halfway between e4m3 neighbours (spacing 1/8 in [1, 2))
    w = rows(448.0, 1.0625, 1.1875, -1.0625, 3 * 2.0 ** -11, 2.0 ** -10, 400.0, -432.0)
    q, s = F8.quantize_rows(w[None])
    assert s.item() == 1.0
    # 2^-10 is halfway between 0 and the smallest subnormal 2^-9: ties to even -> 0; 400 lies halfway 384 / 416 -> 384 and 432
    # halfway 416 / 448 -> 448 (even mantissas)
    assert q_values(q[0]).tolist() == [448.0, 1.0, 1.25, -1.0, 2.0 ** -9, 0.0, 384.0, -448.0]


def test_values_past_448_clamp_to_448():
    # a row scale rounded down in fp32 can put amax / s a little above 448; the clamp (satfinite on the device) keeps it at 448
    x = torch.tensor([448.0 * (1 + 2.0 ** -20), 460.0, 500.0, -1e4, -448.5])
    assert x.clamp(-448, 448).to(torch.float8_e4m3fn).float().tolist() == [448.0, 448.0, 448.0, -448.0, -448.0]
    for a in torch.arange(1.0, 4.0, 1 / 64):  # every bf16 amax in [1, 4): q of the maximum is exactly +-448
        w = torch.tensor([[a.item(), -a.item() / 3]], dtype=torch.bfloat16)
        q, _ = F8.quantize_rows(w)
        assert q_values(q)[0, 0].item() == 448.0


def test_subnormal_results():
    # amax 448 * 2^-20 gives s = 2^-20; an entry of 2^-28 quantises to 2^-8 (e4m3 subnormal 2 * 2^-9), 2^-30 to 2^-10 -> 0 (tie to
    # even between 0 and 2^-9) and 3 * 2^-31 = 1.5 * 2^-10 to 2^-9
    w = rows(448 * 2.0 ** -20, 2.0 ** -28, 2.0 ** -30, 3 * 2.0 ** -31, -(2.0 ** -29))
    q, s = F8.quantize_rows(w[None])
    assert s.item() == 2.0 ** -20
    assert q_values(q[0]).tolist() == [448.0, 2.0 ** -8, 0.0, 2.0 ** -9, -(2.0 ** -9)]
    assert F8.fp8_weights(w[None])[0].float().tolist() == [448 * 2.0 ** -20, 2.0 ** -28, 0.0, 2.0 ** -29, -(2.0 ** -29)]


def test_error_within_the_e4m3_bound_per_row():
    g = torch.Generator().manual_seed(0)
    w = (torch.randn(64, 256, generator=g) * torch.logspace(-6, 6, 64)[:, None]).to(torch.bfloat16)
    q, s = F8.quantize_rows(w)
    wp = F8.dequantize_rows(q, s)
    err = (wp.float() - w.float()).abs()
    # e4m3: relative half-ulp 2^-4 for normals, absolute 2^-10 * s below 2^-6 * s; then one bf16 rounding (2^-9 relative)
    bound = torch.maximum(w.float().abs() * 2.0 ** -4, 2.0 ** -10 * s[:, None]) * (1 + 2.0 ** -7) + w.float().abs() * 2.0 ** -8
    assert (err <= bound).all()
    assert torch.equal(F8.dequantize_rows(q.view(torch.float8_e4m3fn), s), wp)


def test_fp8_checkpoint_replaces_expert_matrices_only():
    p = synth.shape("tiny-moe", n_layers=1)
    sd = synth.synth_state_dict(p, 3)
    out = F8.fp8_checkpoint(sd)
    assert set(out) == set(sd)
    for k, v in sd.items():
        if ".experts." in k:
            assert torch.equal(out[k], F8.fp8_weights(v)), k
        else:
            assert out[k] is v, k


# ----------------------------------------------------------------------------- host side of the model
def moe_args(n_layers: int = 1):
    p = synth.shape("tiny-moe", n_layers=n_layers)
    return p, mi.TransformerArgs.from_dict(dict(p))


def test_fp8_model_stores_uint8_experts_and_scales_that_survive_to_bf16():
    p, args = moe_args()
    m = Transformer(args, expert_weights="fp8")
    ff = m.layers["0"].feed_forward
    ex = ff.experts["0"]
    assert isinstance(ex, Fp8Expert)
    dim, hidden = args.dim, args.hidden_dim
    assert ex.w13_q.dtype == torch.uint8 and tuple(ex.w13_q.shape) == (2 * hidden, dim)
    assert ex.w2_q.dtype == torch.uint8 and tuple(ex.w2_q.shape) == (dim, hidden)
    with torch.no_grad():
        ex.w13_scale.copy_(torch.linspace(1e-30, 3e30, 2 * hidden))
        ex.w2_scale.copy_(torch.linspace(-5.0, 5.0, dim) * 1e-3)
    before = (ex.w13_scale.clone(), ex.w2_scale.clone())
    m = m.to(torch.bfloat16)
    ex = m.layers["0"].feed_forward.experts["0"]
    assert ex.w13_scale.dtype == torch.float32 and torch.equal(ex.w13_scale, before[0]) and torch.equal(ex.w2_scale, before[1])
    assert ex.w13_q.dtype == torch.uint8 and m.dtype == torch.bfloat16
    assert m.layers["0"].attention.wqkv.dtype == torch.bfloat16
    assert not hasattr(ex, "w13")  # no bf16 copy of the experts


def test_fp8_empty_allocates_the_fp8_layout():
    p, args = moe_args(2)
    m = Transformer.empty(args, device="cpu", expert_weights="fp8")
    ex = m.layers["1"].feed_forward.experts["7"]
    assert ex.w13_q.dtype == torch.uint8 and ex.w13_scale_bits.dtype == torch.int32 and ex.w13_q.device.type == "cpu"
    bf = Transformer.empty(args, device="cpu")
    expert_bytes = lambda mod: sum(t.numel() * t.element_size() for n, t in mod.named_parameters() if ".experts." in n)  # noqa: E731
    E, dim, hidden = args.moe.num_experts, args.dim, args.hidden_dim
    assert expert_bytes(m) == 2 * E * (3 * dim * hidden + (2 * hidden + dim) * 4)
    assert expert_bytes(bf) == 2 * E * 3 * dim * hidden * 2


def test_fp8_state_dict_keys_are_zero_copy_views():
    p, args = moe_args()
    m = Transformer(args, expert_weights="fp8").to(torch.bfloat16)
    sd = m.state_dict()
    ref = set(synth.synth_state_dict(p, 1))
    experts = {k for k in ref if ".experts." in k}
    want = (ref - experts) | {k[: -len(".weight")] + s for k in experts for s in (".weight_e4m3", ".weight_scale")}
    assert set(sd) == want
    ex = m.layers["0"].feed_forward.experts["3"]
    h, d = args.hidden_dim, args.dim
    w1, w3, w2 = (sd[f"layers.0.feed_forward.experts.3.{n}.weight_e4m3"] for n in ("w1", "w3", "w2"))
    assert w1.dtype == torch.float8_e4m3fn and tuple(w1.shape) == (h, d) and tuple(w2.shape) == (d, h)
    assert w1.data_ptr() == ex.w13_q.data_ptr() and w3.data_ptr() == ex.w13_q.data_ptr() + d and w2.data_ptr() == ex.w2_q.data_ptr()
    s1, s3 = sd["layers.0.feed_forward.experts.3.w1.weight_scale"], sd["layers.0.feed_forward.experts.3.w3.weight_scale"]
    assert s1.dtype == torch.float32 and s1.data_ptr() == ex.w13_scale_bits.data_ptr() and s3.data_ptr() == ex.w13_scale_bits.data_ptr() + 4
    assert s1.stride() == (2,) and w1.stride() == (2 * d, 1)
    # the missing-key check accepts the reference's bf16 expert keys for these entries
    assert m._missing_keys(ref) == set()


def test_fp8_refusals():
    with pytest.raises(ValueError):
        Transformer(mi.TransformerArgs.from_dict(dict(synth.shape("tiny"))), expert_weights="fp8")
    p, args = moe_args()
    with pytest.raises(ValueError):
        Transformer(args, expert_weights="int8")
    m = Transformer(args, expert_weights="fp8").to(torch.bfloat16)
    assert m._megakernel_ok(1) is False
    with pytest.raises(ValueError):  # a pre-quantised checkpoint key is not a format the loader reads
        m.load_state_dict({"layers.0.feed_forward.experts.0.w1.weight_e4m3": torch.zeros(1)}, strict=False)
    lora = {"layers.0.feed_forward.experts.2.w1.lora_A.weight": torch.zeros(4, args.dim, dtype=torch.bfloat16),
            "layers.0.feed_forward.experts.2.w1.lora_B.weight": torch.zeros(args.hidden_dim, 4, dtype=torch.bfloat16)}
    with pytest.raises(NotImplementedError):
        m._load_lora_state_dict(lora)


def test_fp8_merged_lora_on_other_linears_still_merges():
    p, args = moe_args()
    m = Transformer(args, expert_weights="fp8").to(torch.bfloat16)
    sd = synth.synth_state_dict(p, 2)
    with torch.no_grad():
        m.layers["0"].attention.wo_weight.copy_(sd["layers.0.attention.wo.weight"])
    g = torch.Generator().manual_seed(0)
    A = (torch.randn(4, args.n_heads * args.head_dim, generator=g) * 0.1).to(torch.bfloat16)
    B = (torch.randn(args.dim, 4, generator=g) * 0.1).to(torch.bfloat16)
    m._load_lora_state_dict({"layers.0.attention.wo.lora_A.weight": A, "layers.0.attention.wo.lora_B.weight": B}, scaling=2.0)
    want = sd["layers.0.attention.wo.weight"] + (B @ A) * 2.0
    assert torch.equal(m.layers["0"].attention.wo_weight, want)
