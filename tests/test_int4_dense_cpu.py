"""INT4 dense weights without a GPU: the format restated in tests/int4_dense_ref.py at its edges, the arithmetic of the bf16x2
dequantisation the kernels rely on (the subtraction of 136 is exact and q * s rounds once; the device instructions themselves are
held by the GPU tests) and the nibble selection of its device helper, restated, and the host side of `Transformer(..., dense_weights="int4")` -- storage, views, state-dict keys,
refusals before allocation, the megakernel switch -- plus the ratio-12 refusals of the FP8 cache and the megakernel."""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer
from mistral_inference_b200.build import build_library
from tests import int4_dense_ref as I4


@pytest.fixture(scope="module")
def built():
    return build_library()


def tiny_args(**overrides):
    p = synth.shape("tiny", **overrides)
    return p, mi.TransformerArgs.from_dict(dict(p))


def bf(vals):
    return torch.tensor(vals, dtype=torch.float32).to(torch.bfloat16)


def one_group(vals):
    """A [1, 128] weight whose first entries are `vals`, the rest zero."""
    w = torch.zeros(1, 128, dtype=torch.bfloat16)
    w[0, : len(vals)] = bf(vals)
    return w


# ----------------------------------------------------------------------------- the format at its edges
def test_amax_maps_to_plus_minus_seven_and_is_the_only_nonzero_value():
    for a in (7.0, 1.0, 0.3, 1e-20, 3e38):
        for sign in (1.0, -1.0):
            q, s = I4.quantize_codes(one_group([sign * a]))
            assert s.item() == bf([a / 7.0]).item()
            assert q[0, 0].item() == (7 if sign > 0 else -7) and (q[0, 1:] == 0).all()


def test_ties_round_half_to_even():
    # s = 1 (amax 7): x / s = k + 0.5 exactly rounds to the even neighbour
    q, s = I4.quantize_codes(one_group([7.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 3.5]))
    assert s.item() == 1.0
    assert q[0, :8].tolist() == [7, 0, 2, 2, 0, -2, -2, 4]


def test_scale_rounding_down_clamps_at_seven_and_minus_eight():
    # amax 7.0625: s = bf16(1.00892857) = 1.0078125, amax / s = 7.0078 -> 7; the clamp at +7 holds
    q, s = I4.quantize_codes(one_group([7.0625, -7.0625]))
    assert s.item() == 1.0078125 and q[0, :2].tolist() == [7, -7]
    # a subnormal scale has few bits: amax / 7 = 1.4 * 2^-133 rounds to 2^-133, amax / s = 9.8 -> clamp to 7 / -8
    tiny = 9.8 * 2.0 ** -133
    w = torch.tensor([[tiny, -tiny] + [0.0] * 126]).to(torch.bfloat16)
    q, s = I4.quantize_codes(w)
    assert s.view(torch.int16).item() == 1
    assert q[0, :2].tolist() == [7, -8]


def test_zero_groups_and_negative_zero():
    w = torch.zeros(2, 256, dtype=torch.bfloat16)
    w[0, :128] = -0.0
    w[1, 130] = -0.0
    w[1, 131] = 3.0
    codes, s = I4.quantize(w)
    assert s[0].tolist() == [1.0, 1.0] and s[1, 0].item() == 1.0  # all-zero groups (with -0) get s = 1
    wp = I4.dequantize(codes, s)
    assert torch.equal(wp[0].float(), torch.zeros(256))  # -0 comes back as +0: q = 0, 0 * s = +0
    assert not torch.signbit(wp[0].float()).any() and not torch.signbit(wp[1, 130].float())
    assert wp[1, 131].item() == 3.0


def test_tiny_amax_takes_the_smallest_positive_scale():
    # amax / 7 rounds to zero in bf16 (below 2^-134): s is raised to 2^-133, and the weight still gets a code
    x = 2.0 ** -133  # the smallest positive bf16
    q, s = I4.quantize_codes(one_group([x]))
    assert s.view(torch.int16).item() == 1 and q[0, 0].item() == 1
    assert I4.dequantize(I4.pack(q), s)[0, 0].item() == x


@pytest.mark.parametrize("K", [128, 28672])
def test_pack_unpack_roundtrip_and_w_prime(K):
    g = torch.Generator().manual_seed(K)
    w = (torch.randn(6, K, generator=g) * torch.logspace(-30, 30, 6)[:, None]).to(torch.bfloat16)
    codes, s = I4.quantize(w)
    assert codes.dtype == torch.uint8 and tuple(codes.shape) == (6, K // 2)
    assert s.dtype == torch.bfloat16 and tuple(s.shape) == (6, K // 128)
    q = I4.unpack(codes)
    assert int(q.min()) >= -8 and int(q.max()) <= 7 and torch.equal(I4.pack(q), codes)
    assert (codes & 0xF).tolist() == ((q[:, 0::2] + 8).to(torch.uint8)).tolist()  # low nibble = even k
    wp = I4.dequantize(codes, s)
    # W' = bf16_rn(q * s): the product is exact in fp32 (and in float64)
    exact = (q.double().view(6, K // 128, 128) * s.double()[..., None]).view(6, K)
    assert torch.equal(wp, exact.to(torch.bfloat16))
    # within half a step (plus W's bf16 rounding) of the weight: the clamp is never reached with a normal scale
    err = (wp.double() - w.double()).abs().view(6, K // 128, 128).amax(-1)
    assert (err <= (0.5 + 2 ** -7) * s.double() * 8 / 7).all()


def test_bf16x2_dequant_identity_over_all_codes_and_a_scale_sweep():
    # every positive finite bf16 scale the quantiser can produce (normal and subnormal), and their negatives for good measure.  This
    # holds the arithmetic (the restated bf16 operations, each one rounding of the exact result), not the device instructions
    bits = torch.arange(1, 0x7F80, dtype=torch.int32).to(torch.int16)
    s = bits.view(torch.bfloat16)
    s = torch.cat([s, -s])
    u = torch.arange(16)
    got = I4.bf16x2_dequant(u[:, None], s[None, :])
    want = ((u[:, None] - 8).float() * s[None, :].float()).to(torch.bfloat16)  # bf16_rn(fp32(q) * fp32(s))
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))
    # q * s is exact in fp32: the float64 product agrees
    assert torch.equal(((u[:, None] - 8).double() * s[None, :].double()).float(), (u[:, None] - 8).float() * s[None, :].float())
    # the subtraction is exact: (128 + u) - 136 = u - 8 in bf16
    biased = (torch.tensor(0x4300, dtype=torch.int16) + u.to(torch.int16)).view(torch.bfloat16)
    assert biased.float().tolist() == [128.0 + i for i in range(16)]


def _prmt(a: int, b: int, sel: int) -> int:
    """PTX prmt / __byte_perm without sign replication: byte i of the result is byte (sel >> 4i) & 7 of (b:a)."""
    src = (b << 32) | a
    return sum(((src >> (8 * ((sel >> (4 * i)) & 7))) & 0xFF) << (8 * i) for i in range(4))


def _int4x8_to_bf16x2(v: int, s: torch.Tensor, natural: bool):
    """The bit selection of int4x8_to_bf16x2 (csrc/int4.cuh) on one 32-bit word of codes, restated: the masks, the OR with 0x4300
    and, with NATURAL, the two byte permutes; then the two bf16 operations per half.  Returns the 8 bf16 values in word order."""
    t = [((v >> (4 * i)) & 0x000F000F) | 0x43004300 for i in range(4)]
    if natural:
        t = [_prmt(t[0], t[1], 0x5410), _prmt(t[2], t[3], 0x5410), _prmt(t[0], t[1], 0x7632), _prmt(t[2], t[3], 0x7632)]
    halves = torch.tensor([h for w in t for h in (w & 0xFFFF, w >> 16)], dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
    return I4.bf16x2_dequant(halves.view(torch.int16).to(torch.int32) - 0x4300, s)


def test_kernel_nibble_selection_gives_w_prime_in_both_orders():
    """The device helper's nibble masks and byte permutes, restated, put W' of the right k in each bf16 half: k order with NATURAL
    (the tile converter), (i, i + 4) pairs without (the GEMV).  The device's own sub / mul instructions, subnormal scales included,
    are held to W' by the GPU tests of every INT4 kernel."""
    g = torch.Generator().manual_seed(9)
    w = (torch.randn(4, 128, generator=g) * torch.tensor([1.0, 1e-3, 1e-38, 30.0])[:, None]).to(torch.bfloat16)
    codes, s = I4.quantize(w)
    wp = I4.dequantize(codes, s)
    for r in range(4):
        words = codes[r].view(-1, 4).to(torch.int64)
        for j in range(words.shape[0]):
            v = int(sum(int(words[j, b]) << (8 * b) for b in range(4)))
            k0 = 8 * j
            nat = _int4x8_to_bf16x2(v, s[r, 0], True)
            assert torch.equal(nat.view(torch.int16), wp[r, k0:k0 + 8].view(torch.int16)), (r, j)
            pairs = _int4x8_to_bf16x2(v, s[r, 0], False)
            order = [i + 4 * h for i in range(4) for h in range(2)]  # word i = (W'[i], W'[i + 4])
            assert torch.equal(pairs.view(torch.int16), wp[r, k0:k0 + 8][order].view(torch.int16)), (r, j)


def test_checkpoint_transform_replaces_only_the_layer_linears():
    p, _ = tiny_args()
    sd = synth.synth_state_dict(p, 1)
    ck = I4.int4_dense_checkpoint(sd)
    for k, v in sd.items():
        if I4.is_dense_key(k):
            assert torch.equal(ck[k], I4.dequantize(*I4.quantize(v)))
        else:
            assert ck[k] is v


# ----------------------------------------------------------------------------- the host side
def test_keyword_and_refusals_before_allocation():
    _, args = tiny_args()
    assert Transformer(args, dense_weights="int4").dense_weights == "int4"
    with pytest.raises(ValueError):
        Transformer(mi.TransformerArgs.from_dict(dict(synth.shape("tiny-moe"))), dense_weights="int4")
    with pytest.raises(NotImplementedError):
        Transformer(mi.TransformerArgs.from_dict(dict(synth.shape("tiny"), lora={"rank": 4, "scaling": 2.0})), dense_weights="int4")
    # K a multiple of 64 but not of 128 (dim 320 also puts wo on mma.sync), N on neither 128 nor 192 (hidden 544)
    for bad in (dict(dim=320), dict(dim=448, n_heads=4), dict(hidden_dim=544), dict(hidden_dim=576)):
        with pytest.raises(ValueError):
            Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape("tiny", **bad))), device="meta", dense_weights="int4")
    for name in ("mistral-7b", "mistral-nemo-12b", "mistral-large-2"):
        Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape(name, n_layers=1))), device="meta", dense_weights="int4")


def test_storage_dtypes_shapes_and_scales_that_survive_to_bf16():
    _, args = tiny_args()
    m = Transformer(args, dense_weights="int4")
    att, ff = m.layers["0"].attention, m.layers["0"].feed_forward
    dim, hidden, q_dim, kv_dim = args.dim, args.hidden_dim, args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    for t, (n, k) in ((att.wqkv, (q_dim + 2 * kv_dim, dim)), (att.wo_weight, (dim, q_dim)), (ff.w13, (2 * hidden, dim)),
                      (ff.w2_weight, (dim, hidden))):
        assert t.dtype == torch.uint8 and tuple(t.shape) == (n, k // 2)
    for bits, n, k in ((att.wqkv_gscale_bits, q_dim + 2 * kv_dim, dim), (att.wo_gscale_bits, dim, q_dim), (ff.w13_gscale_bits, 2 * hidden, dim),
                       (ff.w2_gscale_bits, dim, hidden)):
        assert bits.dtype == torch.int16 and tuple(bits.shape) == (n, k // 128)
    with torch.no_grad():
        ff.w13_gscale.copy_(torch.linspace(1e-30, 3e30, 2 * hidden * dim // 128).view(2 * hidden, -1))
    before = ff.w13_gscale.clone()
    m = m.to(torch.bfloat16)
    assert torch.equal(m.layers["0"].feed_forward.w13_gscale.view(torch.int16), before.view(torch.int16))
    assert m.dtype == torch.bfloat16 and m.tok_embeddings.weight.dtype == torch.bfloat16 and m.output_weight.dtype == torch.bfloat16


def test_layer_bytes_are_a_quarter_plus_the_scales():
    _, args = tiny_args()
    i4 = Transformer.empty(args, device="cpu", dense_weights="int4")
    layer_bytes = lambda mod: sum(t.numel() * t.element_size() for n, t in mod.named_parameters()  # noqa: E731
                                  if n.startswith("layers.") and "norm" not in n)
    q_dim, kv_dim = args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    mats = args.dim * (q_dim + 2 * kv_dim) + q_dim * args.dim + 3 * args.dim * args.hidden_dim
    assert layer_bytes(i4) == args.n_layers * (mats // 2 + 2 * mats // 128)


def test_views_are_zero_copy_with_the_packing_strides():
    _, args = tiny_args()
    m = Transformer(args, dense_weights="int4").to(torch.bfloat16)
    att, ff = m.layers["1"].attention, m.layers["1"].feed_forward
    dim, hidden, q_dim, kv_dim = args.dim, args.hidden_dim, args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    G = dim // 128
    for name, row0, rows in (("wq", 0, q_dim), ("wk", q_dim, kv_dim), ("wv", q_dim + kv_dim, kv_dim)):
        c, s = att.weight_int4(name), att.weight_gscale(name)
        assert c.dtype == torch.uint8 and tuple(c.shape) == (rows, dim // 2) and c.data_ptr() == att.wqkv.data_ptr() + row0 * dim // 2
        assert s.dtype == torch.bfloat16 and tuple(s.shape) == (rows, G) and s.data_ptr() == att.wqkv_gscale_bits.data_ptr() + 2 * row0 * G
    w1, w3 = ff.weight_int4("w1"), ff.weight_int4("w3")
    s1, s3 = ff.weight_gscale("w1"), ff.weight_gscale("w3")
    assert tuple(w1.shape) == (hidden, dim // 2) and w1.stride() == (dim, 1) and w3.data_ptr() == ff.w13.data_ptr() + dim // 2
    assert tuple(s1.shape) == (hidden, G) and s1.stride() == (2 * G, 1) and s3.data_ptr() == ff.w13_gscale_bits.data_ptr() + 2 * G
    assert ff.weight_int4("w2").data_ptr() == ff.w2_weight.data_ptr()


def test_state_dict_keys_and_loader_refusals():
    p, args = tiny_args()
    m = Transformer(args, dense_weights="int4").to(torch.bfloat16)
    sd = m.state_dict()
    ref = set(synth.synth_state_dict(p, 1))
    dense = {k for k in ref if I4.is_dense_key(k)}
    want = (ref - dense) | {k[: -len(".weight")] + s for k in dense for s in (".weight_int4", ".weight_gscale")}
    assert set(sd) == want
    assert sd["layers.0.feed_forward.w3.weight_int4"].data_ptr() == m.layers["0"].feed_forward.weight_int4("w3").data_ptr()
    assert m._missing_keys(ref) == set()
    assert m._missing_keys(ref - {"layers.1.attention.wv.weight"}) == {"layers.1.attention.wv.weight_int4",
                                                                       "layers.1.attention.wv.weight_gscale"}
    for key in ("layers.0.attention.wq.weight_int4", "layers.0.feed_forward.w2.weight_gscale"):
        with pytest.raises(ValueError):
            m.load_state_dict({key: torch.zeros(1)}, strict=False)
    with pytest.raises(AssertionError):  # a bf16 weight of the wrong shape, before any kernel runs
        m.load_state_dict({"layers.0.attention.wo.weight": torch.zeros(3, 128, dtype=torch.bfloat16)}, strict=False)
    lora = {"layers.0.attention.wo.lora_A.weight": torch.zeros(4, args.n_heads * args.head_dim, dtype=torch.bfloat16),
            "layers.0.attention.wo.lora_B.weight": torch.zeros(args.dim, 4, dtype=torch.bfloat16)}
    with pytest.raises(NotImplementedError):
        m._load_lora_state_dict(lora)


def test_megakernel_is_never_asked_for_int4(monkeypatch):
    _, args = tiny_args()
    m = Transformer(args, dense_weights="int4").to(torch.bfloat16)
    monkeypatch.setattr(_abi, "decode_step_fp8_unsupported", lambda *a, **k: pytest.fail("asked"))
    monkeypatch.setattr(_abi, "decode_step_unsupported", lambda *a, **k: pytest.fail("asked"))
    assert m._megakernel_ok(1) is False


# ----------------------------------------------------------------------------- head ratio 12
def test_fp8_cache_refuses_ratio_12_before_allocation():
    for name in ("mistral-large-2",):
        args = mi.TransformerArgs.from_dict(dict(synth.shape(name, n_layers=1)))
        with pytest.raises(ValueError, match="query heads per kv head"):
            Transformer.empty(args, device="meta", kv_cache="fp8")
        Transformer.empty(args, device="meta", kv_cache="bf16")
    # the ratios the FP8-cache kernels serve still construct
    Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape("mixtral-8x22b", n_layers=1))), device="meta", kv_cache="fp8")


def test_megakernel_plan_refuses_the_mistral_large_shape(built):
    p = synth.shape("mistral-large-2")
    why = _abi.decode_step_unsupported(p["dim"], p["hidden_dim"], p["n_heads"], p["n_kv_heads"], p["head_dim"], p["vocab_size"], 0, 0,
                                       smem_optin=227 * 1024)
    assert why is not None and "H/KV" in why
