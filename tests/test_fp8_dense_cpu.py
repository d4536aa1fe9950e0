"""FP8 (e4m3) dense weights without a GPU: the host side of `Transformer(..., dense_weights="fp8")` -- keyword, refusals,
storage and packing strides, state-dict keys, pipeline ranks, the megakernel switch -- the CPU restatement of the compute
(tests/fp8_dense_ref.py) and the decode megakernel's ring protocol under the e4m3 stage plan."""
import random

import pytest
import torch
import torch.nn.functional as F

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer
from oracle import fp8 as F8
from tests import fp8_dense_ref as FD
from tests.test_megakernel_protocol import WARPS, Mbar, simulate


def tiny_args(**overrides):
    p = synth.shape("tiny", **overrides)
    return p, mi.TransformerArgs.from_dict(dict(p))


def test_keyword_is_validated_and_defaults_to_bf16():
    _, args = tiny_args()
    assert Transformer(args).dense_weights == "bf16"
    with pytest.raises(ValueError):
        Transformer(args, dense_weights="int8")
    with pytest.raises(TypeError):  # keyword-only
        Transformer(args, 0, 1, True, None, None, "bf16", "fp8")


def test_refusals_come_before_allocation():
    p = synth.shape("tiny-moe")
    with pytest.raises(ValueError):
        Transformer(mi.TransformerArgs.from_dict(dict(p)), dense_weights="fp8")
    p = synth.shape("tiny")
    lora = mi.TransformerArgs.from_dict(dict(p, lora={"rank": 4, "scaling": 2.0}))
    with pytest.raises(NotImplementedError):
        Transformer(lora, dense_weights="fp8")
    # shapes that would put some Linear on the mma.sync GEMM: K not a multiple of 64 (dim 288), N a multiple of neither 128 nor
    # 192 (hidden 544 -> w13 N = 1088), wo N = dim = 320
    for bad in (dict(dim=288), dict(hidden_dim=544), dict(dim=320)):
        with pytest.raises(ValueError):
            Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape("tiny", **bad))), device="meta", dense_weights="fp8")
    # the 7B and Nemo shapes pass
    for name in ("mistral-7b", "mistral-nemo-12b"):
        Transformer.empty(mi.TransformerArgs.from_dict(dict(synth.shape(name, n_layers=1))), device="meta", dense_weights="fp8")


def test_storage_is_uint8_rows_and_int32_scales_that_survive_to_bf16():
    _, args = tiny_args()
    m = Transformer(args, dense_weights="fp8")
    att, ff = m.layers["0"].attention, m.layers["0"].feed_forward
    dim, hidden, q_dim, kv_dim = args.dim, args.hidden_dim, args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    assert att.wqkv.dtype == torch.uint8 and tuple(att.wqkv.shape) == (q_dim + 2 * kv_dim, dim)
    assert att.wo_weight.dtype == torch.uint8 and tuple(att.wo_weight.shape) == (dim, q_dim)
    assert ff.w13.dtype == torch.uint8 and tuple(ff.w13.shape) == (2 * hidden, dim)
    assert ff.w2_weight.dtype == torch.uint8 and tuple(ff.w2_weight.shape) == (dim, hidden)
    for bits in (att.wqkv_scale_bits, att.wo_scale_bits, ff.w13_scale_bits, ff.w2_scale_bits):
        assert bits.dtype == torch.int32
    with torch.no_grad():
        ff.w13_scale.copy_(torch.linspace(1e-30, 3e30, 2 * hidden))
        att.wo_scale.copy_(torch.linspace(-5.0, 5.0, dim) * 1e-3)
    before = (ff.w13_scale.clone(), att.wo_scale.clone())
    m = m.to(torch.bfloat16)
    att, ff = m.layers["0"].attention, m.layers["0"].feed_forward
    assert torch.equal(ff.w13_scale, before[0]) and torch.equal(att.wo_scale, before[1])
    assert ff.w13.dtype == torch.uint8 and m.dtype == torch.bfloat16
    # what stays bf16
    assert m.tok_embeddings.weight.dtype == torch.bfloat16 and m.output_weight.dtype == torch.bfloat16
    assert m.layers["0"].attention_norm.weight.dtype == torch.bfloat16


def test_empty_allocates_half_the_layer_bytes():
    _, args = tiny_args()
    fp8 = Transformer.empty(args, device="cpu", dense_weights="fp8")
    bf = Transformer.empty(args, device="cpu")
    layer_bytes = lambda mod: sum(t.numel() * t.element_size() for n, t in mod.named_parameters()  # noqa: E731
                                  if n.startswith("layers.") and "norm" not in n)
    q_dim, kv_dim = args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    N = q_dim + 2 * kv_dim + args.dim + 2 * args.hidden_dim + args.dim  # rows of wqkv, wo, w13, w2
    mats = args.dim * (q_dim + 2 * kv_dim) + q_dim * args.dim + 3 * args.dim * args.hidden_dim
    assert layer_bytes(bf) == args.n_layers * mats * 2
    assert layer_bytes(fp8) == args.n_layers * (mats + 4 * N)


def test_views_are_zero_copy_with_the_packing_strides():
    _, args = tiny_args()
    m = Transformer(args, dense_weights="fp8").to(torch.bfloat16)
    att, ff = m.layers["1"].attention, m.layers["1"].feed_forward
    dim, hidden, q_dim, kv_dim = args.dim, args.hidden_dim, args.n_heads * args.head_dim, args.n_kv_heads * args.head_dim
    # wqkv rows cat(q, k, v): row offsets 0, q_dim, q_dim + kv_dim
    for name, row0, rows in (("wq", 0, q_dim), ("wk", q_dim, kv_dim), ("wv", q_dim + kv_dim, kv_dim)):
        q, s = att.weight_e4m3(name), att.weight_scale(name)
        assert q.dtype == torch.float8_e4m3fn and tuple(q.shape) == (rows, dim) and q.stride() == (dim, 1)
        assert q.data_ptr() == att.wqkv.data_ptr() + row0 * dim
        assert s.dtype == torch.float32 and tuple(s.shape) == (rows,) and s.data_ptr() == att.wqkv_scale_bits.data_ptr() + 4 * row0
    assert att.weight_e4m3("wo").data_ptr() == att.wo_weight.data_ptr()
    # w13 rows interleave w1 / w3: row stride 2 * dim, scale stride 2, w3 one row and one scale later
    w1, w3 = ff.weight_e4m3("w1"), ff.weight_e4m3("w3")
    s1, s3 = ff.weight_scale("w1"), ff.weight_scale("w3")
    assert tuple(w1.shape) == (hidden, dim) and w1.stride() == (2 * dim, 1) and s1.stride() == (2,)
    assert w1.data_ptr() == ff.w13.data_ptr() and w3.data_ptr() == ff.w13.data_ptr() + dim
    assert s1.data_ptr() == ff.w13_scale_bits.data_ptr() and s3.data_ptr() == ff.w13_scale_bits.data_ptr() + 4
    assert ff.weight_e4m3("w2").data_ptr() == ff.w2_weight.data_ptr() and tuple(ff.weight_e4m3("w2").shape) == (dim, hidden)


def _fp8_keys(ref_keys, layers):
    dense = {k for k in ref_keys if FD.is_dense_key(k) and k.split(".")[1] in layers}
    return {k for k in ref_keys if not FD.is_dense_key(k) and (not k.startswith("layers.") or k.split(".")[1] in layers)} | \
        {k[: -len(".weight")] + s for k in dense for s in (".weight_e4m3", ".weight_scale")}


def test_state_dict_keys():
    p, args = tiny_args()
    m = Transformer(args, dense_weights="fp8").to(torch.bfloat16)
    sd = m.state_dict()
    ref = set(synth.synth_state_dict(p, 1))
    assert set(sd) == _fp8_keys(ref, {"0", "1"})
    assert sd["layers.0.attention.wk.weight_e4m3"].data_ptr() == m.layers["0"].attention.weight_e4m3("wk").data_ptr()
    assert m._missing_keys(ref) == set()  # the reference's bf16 keys set both the e4m3 rows and their scales
    assert m._missing_keys(ref - {"layers.1.feed_forward.w3.weight"}) == {"layers.1.feed_forward.w3.weight_e4m3",
                                                                          "layers.1.feed_forward.w3.weight_scale"}


def test_pipeline_rank_keys():
    p, args = tiny_args(n_layers=3)
    ref = set(synth.synth_state_dict(p, 1))
    for rank, layers in ((0, {"0", "1"}), (1, {"2"})):
        m = Transformer(args, pipeline_rank=rank, num_pipeline_ranks=2, dense_weights="fp8").to(torch.bfloat16)
        want = _fp8_keys(ref, layers)
        if rank == 0:
            want -= {"norm.weight", "output.weight"}
        else:
            want -= {"tok_embeddings.weight"}
        assert set(m.state_dict()) == want
        assert m.dtype == torch.bfloat16  # rank 1 holds no embedding: its first parameters are the e4m3 rows


def test_loader_refuses_pre_quantised_keys_and_lora_merges():
    p, args = tiny_args()
    m = Transformer(args, dense_weights="fp8").to(torch.bfloat16)
    for key in ("layers.0.attention.wq.weight_e4m3", "layers.0.feed_forward.w2.weight_scale"):
        with pytest.raises(ValueError):
            m.load_state_dict({key: torch.zeros(1)}, strict=False)
    lora = {"layers.0.attention.wo.lora_A.weight": torch.zeros(4, args.n_heads * args.head_dim, dtype=torch.bfloat16),
            "layers.0.attention.wo.lora_B.weight": torch.zeros(args.dim, 4, dtype=torch.bfloat16)}
    with pytest.raises(NotImplementedError):
        m._load_lora_state_dict(lora)


def test_megakernel_is_allowed_for_dense_fp8(monkeypatch):
    _, args = tiny_args()
    m = Transformer(args, dense_weights="fp8").to(torch.bfloat16)
    asked = []
    monkeypatch.setattr(_abi, "decode_step_fp8_unsupported", lambda *a, **k: asked.append(a) or None)
    monkeypatch.setattr(_abi, "decode_step_unsupported", lambda *a, **k: pytest.fail("the bf16 shape check was asked"))
    assert m._megakernel_ok(1) is True
    assert asked and m._megakernel_ok(2) is False
    # its existing conditions stay: an FP8 cache still takes the graph path
    m2 = Transformer(args, dense_weights="fp8", kv_cache="fp8").to(torch.bfloat16)
    assert m2._megakernel_ok(1) is False


# ----------------------------------------------------------------------------- the restatement
def test_dense_linear_is_one_scale_product_after_the_dot_product():
    g = torch.Generator().manual_seed(3)
    w = (torch.randn(64, 128, generator=g) * 0.02).to(torch.bfloat16)
    x = torch.randn(5, 128, generator=g).to(torch.bfloat16)
    q, s = F8.quantize_rows(w)
    y = FD.dense_linear(x, q, s)
    acc = x.double() @ q.view(torch.float8_e4m3fn).double().T  # exact here: 128 products of <= 8 + 4 significant bits
    want = (acc.float() * s[None, :]).to(torch.bfloat16)
    assert torch.equal(y, want)
    # the restatement model's F.linear computes it for a DenseFp8Weight, and nothing else changes
    dw = FD.DenseFp8Weight(q, s)
    assert dw.dtype == torch.bfloat16 and tuple(dw.shape) == (64, 128)
    assert torch.equal(F.linear(x, dw), y)
    sd = FD.fp8_dense_checkpoint({"layers.0.attention.wq.weight": w, "output.weight": w, "layers.0.attention_norm.weight": w[0]})
    assert isinstance(sd["layers.0.attention.wq.weight"], FD.DenseFp8Weight)
    assert sd["output.weight"] is w and sd["layers.0.attention_norm.weight"] is not None


def test_dense_definition_differs_from_the_expert_contract():
    # W' rounds every weight to bf16 after the scale; the dense definition scales the exact sum once.  Here they disagree.
    s = torch.tensor([3.0 / 448.0])
    q = torch.tensor([[448.0, 2.25, 104.0, 0.0]]).to(torch.float8_e4m3fn).view(torch.uint8)
    x = torch.tensor([[1.0, 1.0, 1.0, 0.0]], dtype=torch.bfloat16)
    assert FD.dense_linear(x, q, s).item() == 3.71875
    assert F.linear(x, F8.dequantize_rows(q, s)).item() == 3.703125


# ----------------------------------------------------------------------------- the megakernel's e4m3 stage plan
MK_WEIGHT_STAGE_BYTES = 16 * 1024


def cut(K: int, w8: bool):
    """cut_matrix (csrc/decode_megakernel.cuh): chunks per row and bytes per stage."""
    max_kc = MK_WEIGHT_STAGE_BYTES // 2 if w8 else MK_WEIGHT_STAGE_BYTES // 4
    nch = -(-K // max_kc)
    kc = K // nch
    return nch, 2 * kc * (1 if w8 else 2)


def test_e4m3_cut_keeps_stages_at_most_16_kb():
    for dim, hidden in ((4096, 14336), (5120, 14336)):
        for K in (dim, hidden, 4096):
            nch, stage = cut(K, True)
            assert stage <= MK_WEIGHT_STAGE_BYTES and (K // nch) % 16 == 0
            assert nch <= cut(K, False)[0]
    assert cut(4096, True) == (1, 8192) and cut(14336, True) == (2, 14336) and cut(5120, True) == (1, 10240)


def two_pairs(K: int) -> bool:
    """two_pairs_per_stage: an e4m3 matrix of one chunk whose four rows fit a 16 KB stage."""
    nch, _ = cut(K, True)
    return nch == 1 and 4 * K <= MK_WEIGHT_STAGE_BYTES


def test_two_pairs_per_stage_keep_7b_stages_at_16_kb():
    assert two_pairs(4096) and 4 * 4096 == MK_WEIGHT_STAGE_BYTES   # 7B: wqkv, wo, w13 (K = dim = q_dim = 4096)
    assert not two_pairs(14336) and not two_pairs(5120)           # 7B / Nemo w2: 2 x 7168; Nemo dim 5120: one pair, 10 KB
    assert two_pairs(1024) and not two_pairs(4112)


def simulate_w8(mats, n_stages: int, seed: int, max_steps: int = 400000, lone: int = WARPS) -> str:
    """The ring protocol of test_megakernel_protocol.simulate for the FP8 stage plan.  mats: per matrix (pairs, nch, two); two: the
    stages of a group are (g + 1) / 2, stage i read by warps 2i and 2i + 1, each arriving WARPS / 2 times on its empty barrier
    (WARPS when its pair is alone in the stage); nch == 0 marks K/V stages (every warp waits on each and arrives once)."""
    rng = random.Random(seed)
    full = [Mbar(1) for _ in range(n_stages)]
    empty = [Mbar(WARPS) for _ in range(n_stages)]
    slot_data = [None] * n_stages
    inflight, prod = [], []
    progs = [[] for _ in range(WARPS)]
    it = bar = 0
    for pairs, nch, two in mats:
        if nch == 0:
            for w in range(WARPS):
                progs[w] += [("kv", it + j, 1) for j in range(pairs)]
            prod += list(range(it, it + pairs))
            it += pairs
        else:
            for g0 in range(0, pairs, WARPS):
                g = min(WARPS, pairs - g0)
                n = (g + 1) // 2 if two else g * nch
                for w in range(g):
                    if two:
                        mine = [(it + w // 2, lone if (w == g - 1 and g % 2) else WARPS // 2)]
                    else:
                        mine = [(it + ch * g + w, WARPS) for ch in range(nch)]
                    for st, arr in mine:
                        progs[w] += [("prev", st, 0), ("stage", st, arr)]
                for w in range(WARPS):
                    progs[w].append(("bar", bar, 0))
                bar += 1
                prod += list(range(it, it + n))
                it += n
        for w in range(WARPS):
            progs[w].append(("bar", bar, 0))
        bar += 1
    pc, arrived, pi = [0] * WARPS, {}, 0
    for _ in range(max_steps):
        acts = ["land"] if inflight else []
        if pi < len(prod) and empty[prod[pi] % n_stages].test(((prod[pi] // n_stages) & 1) ^ 1):
            acts.append("prod")
        for w in range(WARPS):
            if pc[w] == len(progs[w]):
                continue
            kind, a, _ = progs[w][pc[w]]
            if kind == "prev" and empty[a % n_stages].test(((a // n_stages) & 1) ^ 1):
                acts.append(("go", w))
            elif kind in ("stage", "kv") and full[a % n_stages].test((a // n_stages) & 1):
                acts.append(("cons", w))
            elif kind == "bar" and (w not in arrived.setdefault(a, set()) or len(arrived[a]) == WARPS):
                acts.append(("bar", w))
        if not acts:
            return "ok" if pi == len(prod) and all(pc[w] == len(progs[w]) for w in range(WARPS)) else "deadlock"
        a = rng.choice(acts)
        if a == "land":
            slot, st = inflight.pop(rng.randrange(len(inflight)))
            slot_data[slot] = st
            full[slot].arrive()
        elif a == "prod":
            inflight.append((prod[pi] % n_stages, prod[pi]))
            pi += 1
        elif a[0] == "go":
            pc[a[1]] += 1
        elif a[0] == "cons":
            w = a[1]
            _, st, arr = progs[w][pc[w]]
            if slot_data[st % n_stages] != st:
                return "stale"
            for _k in range(arr):
                empty[st % n_stages].arrive()
            pc[w] += 1
        else:
            w = a[1]
            b = progs[w][pc[w]][1]
            if w not in arrived[b]:
                arrived[b].add(w)
            else:
                pc[w] += 1
    return "timeout"


# one CTA's slices with the e4m3 stage plan: 7B (QKV, [K/V], wo, gate/up two pairs per stage; down 2 chunks; bf16 lm head) and
# Nemo (dim 5120: one pair per stage; wo two pairs), odd and even pair counts, the smallest legal ring
W8_SHAPES = [
    ([(21, 1, True), (14, 1, True), (97, 1, True), (14, 2, False), (108, 1, False)], 12),
    ([(21, 1, True), (60, 0, False), (14, 1, True), (97, 1, True), (14, 2, False), (108, 1, False)], 12),
    ([(24, 1, False), (8, 0, False), (17, 1, True), (97, 1, False), (17, 2, False), (443, 2, False)], 9),
    ([(3, 1, True), (1, 1, True), (7, 1, True), (1, 1, False), (2, 1, False)], 9),
    ([(21, 1, True), (14, 1, True), (97, 1, True), (14, 2, False), (108, 1, False)], 9),
]


@pytest.mark.parametrize("mats,n_stages", W8_SHAPES)
def test_e4m3_stage_plan_keeps_the_ring_protocol(mats, n_stages):
    for seed in range(25):
        assert simulate_w8(mats, n_stages, seed) == "ok"


def test_e4m3_model_agrees_with_the_bf16_model_and_catches_a_wrong_arrival_count():
    """With every matrix one pair per stage the model is test_megakernel_protocol's; a lone pair arriving only WARPS / 2 times
    (its stage never frees) is caught."""
    mats = [(21, 1, False), (14, 1, False), (97, 1, False), (14, 4, False), (108, 1, False)]
    assert all(simulate_w8(mats, 12, s) == simulate([21, 14, 97, 14, 108], [1, 1, 1, 4, 1], 12, grouped=True, seed=s) == "ok"
               for s in range(5))
    odd = [(21, 1, True), (14, 1, True), (97, 1, True)]
    assert all(simulate_w8(odd, 12, s, lone=WARPS // 2) != "ok" for s in range(5))
