"""FP8 activations for FP8 dense weights without a GPU: the host side of `Transformer(..., prefill_compute="fp8")` -- keyword,
refusals, state dict, the layers' switch, the megakernel switch -- and the CPU restatement of the per-token quantiser
(tests/fp8_prefill_ref.py) at every edge of the format."""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer
from tests import fp8_prefill_ref as FP


def tiny_args(**overrides):
    p = synth.shape("tiny", **overrides)
    return p, mi.TransformerArgs.from_dict(dict(p))


def test_keyword_defaults_to_bf16_and_is_keyword_only():
    _, args = tiny_args()
    m = Transformer(args, dense_weights="fp8")
    assert m.prefill_compute == "bf16"
    assert not any(getattr(mod, "a8", False) for mod in m.modules())
    with pytest.raises(TypeError):
        Transformer(args, 0, 1, True, None, None, "bf16", "bf16", "fp8", 1, "fp8")
    m8 = Transformer(args, dense_weights="fp8", prefill_compute="fp8")
    assert m8.prefill_compute == "fp8"
    for blk in m8.layers.values():
        assert blk.attention.a8 and blk.feed_forward.a8


@pytest.mark.parametrize("kw", [dict(prefill_compute="int8", dense_weights="fp8"), dict(prefill_compute="FP8", dense_weights="fp8"),
                                dict(prefill_compute="fp8"), dict(prefill_compute="fp8", dense_weights="int4"),
                                dict(prefill_compute="fp8", dense_weights="bf16")])
def test_refusals(kw):
    _, args = tiny_args()
    with pytest.raises(ValueError):
        Transformer.empty(args, device="meta", **kw)


def test_refuses_shapes_the_fp8_kernel_cannot_tile():
    # dim 192: every FP8 dense Linear fits the A16 kernels (K % 64, N % 192), but K = 192 splits a 128-element k-block
    p = synth.shape("tiny", dim=192)
    args = mi.TransformerArgs.from_dict(dict(p))
    Transformer.empty(args, device="meta", dense_weights="fp8")
    with pytest.raises(ValueError):
        Transformer.empty(args, device="meta", dense_weights="fp8", prefill_compute="fp8")
    # the MoE refusal of dense_weights="fp8" comes first
    with pytest.raises(ValueError):
        Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape("tiny-moe"))), device="meta", dense_weights="fp8",
                          prefill_compute="fp8")
    for name in ("mistral-7b", "mistral-nemo-12b"):
        Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape(name, n_layers=1))), device="meta", dense_weights="fp8",
                          prefill_compute="fp8")


def test_state_dict_is_the_fp8_models():
    _, args = tiny_args()
    a = Transformer(args, dense_weights="fp8").to(torch.bfloat16).state_dict()
    b = Transformer(args, dense_weights="fp8", prefill_compute="fp8").to(torch.bfloat16).state_dict()
    assert list(a) == list(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k


def test_megakernel_switch_is_unchanged(monkeypatch):
    _, args = tiny_args()
    monkeypatch.setattr(_abi, "decode_step_fp8_unsupported", lambda *a, **k: None)
    monkeypatch.setattr(_abi, "decode_step_unsupported", lambda *a, **k: pytest.fail("the bf16 shape check was asked"))
    for kw in (dict(), dict(kv_cache="fp8")):
        m = Transformer(args, dense_weights="fp8", **kw).to(torch.bfloat16)
        m8 = Transformer(args, dense_weights="fp8", prefill_compute="fp8", **kw).to(torch.bfloat16)
        assert [m._megakernel_ok(b) for b in (1, 2, 8)] == [m8._megakernel_ok(b) for b in (1, 2, 8)]


# ----------------------------------------------------------------------------- the quantiser restatement
def e4m3(v: float) -> int:
    return int(torch.tensor([v]).to(torch.float8_e4m3fn).view(torch.uint8)[0])


def test_exponent_at_the_boundaries():
    a = torch.tensor([448.0, 450.0, 56.0, 57.0, 1.0, 3.0, 2.0 ** -133, 3 * 2.0 ** -133, 3.3895313892515355e38, 0.0], dtype=torch.float32)
    assert FP.act_exponent(a).tolist() == [0, 1, -3, -2, -8, -7, -141, -140, 120, 0]
    # the definition itself: a <= 448 * 2^e and a > 448 * 2^(e - 1)
    x = torch.tensor([2.0 ** k * m for k in range(-133, 128) for m in (1.0, 1.5, 1.75, 1.7578125, 1.9921875)], dtype=torch.float64)
    x = x[x < 3.39e38].float()
    e = FP.act_exponent(x).double()
    xd = x.double()
    assert bool((xd <= 448.0 * torch.pow(2.0, e)).all()) and bool((xd > 448.0 * torch.pow(2.0, e - 1)).all())


def test_quantiser_edges():
    rows = FP.edge_rows(16)
    q, e = FP.quantize_act(rows)
    assert e.dtype == torch.int32 and q.dtype == torch.uint8
    assert e.tolist() == [0, -3, 1, -40, 0, -7, 0, -6, -140, -141, -134, 0, 120, 0, 0, 0]
    assert q[0, :3].tolist() == [0x7E, e4m3(-1.0), e4m3(0.5)]          # 448 is the largest finite code
    assert q[1, :2].tolist() == [e4m3(-448.0), e4m3(24.0)]
    assert q[2, :2].tolist() == [e4m3(224.0), e4m3(0.5)]                 # 450 / 2 = 225 rounds to 224
    assert q[3, :2].tolist() == [0x7E, 0]                                # 2^-50 * 2^40 is below half the smallest subnormal
    assert q[4].tolist() == [0] * 16 and q[5].tolist() == [0] * 15 + [0x7C]  # 3 * 2^7 = 384
    assert q[6].tolist() == [0x80] * 16                                  # -0 keeps its sign
    assert q[7, :3].tolist() == [0x80, e4m3(5.0 * 2 ** 6), 0x80]
    assert q[8, :3].tolist() == [e4m3(2.0 ** 7), e4m3(-(2.0 ** 7)), e4m3(3 * 2.0 ** 7)]
    assert q[9, 0].item() == 0x7E - 0x06 and q[9, 1].item() == 0         # 2^-133 * 2^141 = 256
    assert q[11, :8].tolist() == [0x7E, 0x01, 0x02, 0x00, 0x02, 0x00, 0x04, 0x08]  # e4m3 subnormals and their ties to even
    assert q[12, 0].item() == e4m3(3.3895313892515355e38 * 2.0 ** -120)
    for r in (13, 14, 15):                                                # inf, -inf, NaN: the whole row is NaN
        assert q[r].tolist() == [FP.E4M3_NAN] * 16


def test_dequantised_rows_are_within_half_an_e4m3_step():
    g = torch.Generator().manual_seed(3)
    v = torch.cat([FP.edge_rows(256)[:13], (torch.randn(40, 256, generator=g) * torch.logspace(-30, 30, 40)[:, None]).to(torch.bfloat16)])
    q, e = FP.quantize_act(v)
    d = FP.dequantize_act(q, e)
    vd = v.double()
    # relative step 2^-3 for normal e4m3 codes, absolute 2^-9 * 2^e below them
    step = torch.maximum(vd.abs() * 2.0 ** -3, torch.pow(2.0, e.double() - 9)[:, None])
    assert bool(((d - vd).abs() <= step / 2).all())
    assert bool((q.view(torch.float8_e4m3fn).float().abs().amax(dim=1) <= 448).all())


def test_a8_linear_is_the_blockwise_contract():
    g = torch.Generator().manual_seed(5)
    T, N, K = 7, 64, 384
    v = (torch.randn(T, K, generator=g)).to(torch.bfloat16)
    wq = torch.randint(-4, 5, (N, K), generator=g).float().to(torch.float8_e4m3fn).view(torch.uint8)
    s = torch.rand(N, generator=g) + 0.5
    xq, e = FP.quantize_act(v)
    exact = FP.dequantize_act(xq, e) @ wq.view(torch.float8_e4m3fn).double().T
    y = FP.a8_linear(v, wq, s)
    # small-integer weights and e4m3 activations: every block sum and the fp32 total are exact, so only the output rounds
    want = ((exact * torch.pow(2.0, -e.double())[:, None]).float() * s[None, :]).double() * torch.pow(2.0, e.double())[:, None]
    assert torch.equal(y, want.float().to(torch.bfloat16))


def test_restatement_weight_switches_at_the_call_size():
    g = torch.Generator().manual_seed(9)
    w = (torch.randn(128, 256, generator=g) * 0.05).to(torch.bfloat16)
    pw = FP.fp8_prefill_checkpoint({"layers.0.feed_forward.w2.weight": w})["layers.0.feed_forward.w2.weight"]
    small, big = (torch.randn(T, 256, generator=g).to(torch.bfloat16) for T in (128, 129))
    from tests.fp8_dense_ref import dense_linear
    assert torch.equal(torch.nn.functional.linear(small, pw), dense_linear(small, pw.q, pw.s))
    assert torch.equal(torch.nn.functional.linear(big, pw), FP.a8_linear(big, pw.q, pw.s, FP.BLOCK_BITS))
