"""FP8 (e4m3) KV cache without a GPU: the CPU restatement of the format (tests/kv_fp8_ref.py) on hand-made rows, its projection
property, the integer rebuild of x' that the attention kernels run, and the host side of `BufferCache(kv_cache="fp8")` and
`Transformer(kv_cache=...)`."""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.transformer import Transformer
from oracle import restatement as R

from . import kv_fp8_ref as K
from .util import oracle_model

HD = 128
FINITE_CODES = [c for c in range(256) if c not in (0x7F, 0xFF)]  # 0x7f / 0xff are e4m3fn NaN


def row(*vals, fill: float = 0.0) -> torch.Tensor:
    """A bf16 row of 128 values: `vals` first, then `fill`."""
    return torch.tensor(list(vals) + [fill] * (HD - len(vals)), dtype=torch.float32).to(torch.bfloat16)


def q_values(q: torch.Tensor) -> torch.Tensor:
    return q.view(torch.float8_e4m3fn).float()


def bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int16)


# ----------------------------------------------------------------------------- the format on designed rows
def test_zero_and_negative_zero_rows():
    x = torch.stack([row(), row(-0.0, 0.0, -0.0, fill=-0.0)])
    q, e = K.quantize_kv_rows(x)
    assert e.dtype == torch.int8 and q.dtype == torch.uint8
    assert e.tolist() == [-124, -124]
    assert q[0].eq(0).all() and q[1].eq(0x80).sum().item() == HD - 1 and q[1, 1].item() == 0
    assert torch.equal(bits(K.kv_prime(x)), bits(x))  # -0 stays -0


def test_amax_exactly_448_times_2_pow_e_and_one_ulp_above():
    # 56 = 448 * 2^-3: e = -3 and q = 448; 56.25 (one bf16 ulp above) needs e = -2.  The same at 448 / 450 and 1.75 / 1.0
    x = torch.stack([row(56.0, -1.0), row(56.25, -1.0), row(448.0), row(450.0), row(1.75), row(1.0)])
    q, e = K.quantize_kv_rows(x)
    assert e.tolist() == [-3, -2, 0, 1, -8, -8]
    assert q_values(q[0])[:2].tolist() == [448.0, -8.0]
    assert q_values(q[1])[0].item() == 224.0  # 56.25 * 4 = 225 rounds to 224 (e4m3 spacing 16 in [128, 256))
    assert q_values(q[2])[0].item() == 448.0 and q_values(q[3])[0].item() == 224.0
    assert q_values(q[4])[0].item() == 448.0  # 1.75 = 448 * 2^-8
    assert q_values(q[5])[0].item() == 256.0  # 1.0 <= 448 * 2^-8 = 1.75, not <= 448 * 2^-9
    xp = K.kv_prime(x)
    assert xp[0, 0].item() == 56.0 and xp[1, 0].item() == 56.0 and xp[3, 0].item() == 448.0


def test_round_to_nearest_even_ties():
    # amax 448 -> e = 0, q = e4m3(x) directly.  1.0625 / 1.1875 lie halfway between neighbours (spacing 1/8 in [1, 2)); 2^-10 lies
    # halfway between 0 and the smallest subnormal 2^-9; 400 halfway between 384 and 416; 3 * 2^-10 halfway between 2^-9 and 2^-8
    x = row(448.0, 1.0625, 1.1875, -1.0625, 2.0 ** -10, 400.0, -432.0, 3 * 2.0 ** -10)
    q, e = K.quantize_kv_rows(x[None])
    assert e.item() == 0
    assert q_values(q[0])[:8].tolist() == [448.0, 1.0, 1.25, -1.0, 0.0, 384.0, -448.0, 2.0 ** -8]


def test_exponent_clamp_and_subnormal_results():
    # amax 2^-128 would want e = -136: the clamp keeps e = -124, so x * 2^124 = 2^-4 and the bf16 subnormals 2^-133 / 3 * 2^-133
    # become the e4m3 subnormals 2^-9 / 3 * 2^-9; every x' is the input (all are representable) -- bf16 subnormals included
    x = row(2.0 ** -128, 2.0 ** -133, -3 * 2.0 ** -133, 2.0 ** -130)
    assert x[1].item() == 2.0 ** -133 and x[2].item() == -3 * 2.0 ** -133
    q, e = K.quantize_kv_rows(x[None])
    assert e.item() == -124
    assert q_values(q[0])[:4].tolist() == [2.0 ** -4, 2.0 ** -9, -3 * 2.0 ** -9, 2.0 ** -6]
    assert torch.equal(bits(K.kv_prime(x[None])[0]), bits(x))
    # e = -118: 448 * 2^-118 is the amax; entries far below it round to (signed) zero
    y = row(448 * 2.0 ** -118, -(2.0 ** -130), 2.0 ** -127)
    q, e = K.quantize_kv_rows(y[None])
    assert e.item() == -118
    assert q[0, :3].tolist() == [0x7E, 0x80, 0x01]  # 448, -0 (2^-12 rounds to zero), 2^-9


def test_mixed_signs():
    x = row(-3.0, 2.5, -0.75, 0.3, -0.001, 0.0, -0.0, 6.0)
    q, e = K.quantize_kv_rows(x[None])
    assert e.item() == -6  # 6 <= 448 * 2^-6 = 7
    want = (x.float() * 64.0).to(torch.float8_e4m3fn).float()
    assert torch.equal(q_values(q[0]), want)
    assert torch.equal(torch.signbit(q_values(q[0])), torch.signbit(want))
    xp = K.kv_prime(x[None])[0]
    assert torch.equal(xp.float(), want / 64.0)


# ----------------------------------------------------------------------------- projection: dequant(quant(x')) == x'
def _code_rows(e: int) -> torch.Tensor:
    codes = torch.tensor(FINITE_CODES + [0] * (2 * HD - len(FINITE_CODES)), dtype=torch.uint8).view(2, HD)
    return K.dequant(codes, torch.full((2,), e, dtype=torch.int8))


@pytest.mark.parametrize("e", list(range(-124, 120)))
def test_projection_every_code_and_exponent(e):
    xp = _code_rows(e)
    assert torch.isfinite(xp.float()).all()
    again = K.kv_prime(xp)
    assert torch.equal(bits(again), bits(xp))
    # a row whose largest |q| is 224 re-quantises as (e - 1, 2q): other bytes, the same x'
    half = K.dequant(torch.tensor([[0x76] + [0x38] * (HD - 1)], dtype=torch.uint8), torch.tensor([e], dtype=torch.int8))  # 224, 1
    q2, e2 = K.quantize_kv_rows(half)
    assert e2.item() == max(-124, e - 1)
    assert torch.equal(bits(K.dequant(q2, e2)), bits(half))


def test_projection_random_rows():
    g = torch.Generator().manual_seed(0)
    scales = torch.pow(2.0, torch.randint(-120, 110, (512, 1), generator=g).float())
    x = (torch.randn(512, HD, generator=g) * scales).to(torch.bfloat16)
    xp = K.kv_prime(x)
    assert torch.equal(bits(K.kv_prime(xp)), bits(xp))
    # and x' is close to x: within half the largest e4m3 spacing of the row
    q, e = K.quantize_kv_rows(x)
    step = torch.ldexp(torch.ones(512), e.to(torch.int32) + 4)  # half the e4m3 spacing of [256, 512) is 16
    assert ((x.float() - xp.float()).abs() <= step[:, None]).all()


# ----------------------------------------------------------------------------- the kernels' integer rebuild of x'
def device_dequant_bits(code: int, e: int) -> int:
    """csrc/kv_fp8.cuh kv_dequant2 for one code and e >= -112: f16 bits of the e4m3 code (exact), exponent rebiased."""
    h = torch.tensor([code], dtype=torch.uint8).view(torch.float8_e4m3fn).to(torch.float16).view(torch.int16).item() & 0xFFFF
    mag = (h >> 3) & 0x0FFF
    return (h & 0x8000) | (((mag + ((112 + e) << 7)) & 0x7FFF) if mag else 0)


def test_integer_rebuild_matches_the_format():
    for e in list(range(-112, 120)):
        want = K.dequant(torch.tensor([FINITE_CODES], dtype=torch.uint8), torch.tensor([e], dtype=torch.int8))
        want = [b & 0xFFFF for b in bits(want)[0].tolist()]
        got = [device_dequant_bits(c, e) for c in FINITE_CODES]
        assert got == want, e


# ----------------------------------------------------------------------------- BufferCache(kv_cache="fp8")
def test_buffer_cache_fp8_storage():
    n_layers, B, L, KV = 4, 3, 100, 8
    c8 = BufferCache(n_layers, B, L, KV, HD, sliding_window=[16, None], kv_cache="fp8")
    cb = BufferCache(n_layers, B, L, KV, HD, sliding_window=[16, None]).to("cpu", torch.bfloat16)
    assert c8.kv_cache == "fp8" and cb.kv_cache == "bf16"
    assert c8.cache_sizes == cb.cache_sizes == [16, 100, 16, 100]
    for i, W in enumerate(c8.cache_sizes):
        assert c8.cache_k[i].dtype == c8.cache_v[i].dtype == torch.float8_e4m3fn
        assert c8.cache_k[i].shape == c8.cache_v[i].shape == (B, W, KV, HD)
        assert c8.cache_k_exp[i].dtype == c8.cache_v_exp[i].dtype == torch.int8
        assert c8.cache_k_exp[i].shape == c8.cache_v_exp[i].shape == (B, W, KV)
    assert cb.nbytes == 2 * 2 * B * (16 + 100) * 2 * KV * HD
    assert c8.nbytes * 2 * HD == cb.nbytes * (HD + 1)  # half the bf16 bytes, plus 1/128 of that for the exponents
    c8.to("cpu", torch.bfloat16)  # generate() passes the model dtype: the element format stays
    assert c8.cache_k[0].dtype == torch.float8_e4m3fn and c8.cache_v_exp[3].dtype == torch.int8
    c8.init_kvseqlens(B)
    md = c8.get_input_metadata([1, 1, 1])
    v = c8.get_view(1, md[1])
    assert v.fp8 and v.cache_k_exp is c8.cache_k_exp[1] and v.metadata.window == 100
    cb.init_kvseqlens(B)
    assert not cb.get_view(1, cb.get_input_metadata([1, 1, 1])[1]).fp8


def test_buffer_cache_refuses_unknown_formats_and_head_dims():
    with pytest.raises(ValueError):
        BufferCache(1, 1, 8, 1, HD, kv_cache="int8")
    with pytest.raises(ValueError):
        BufferCache(1, 1, 8, 1, 64, kv_cache="fp8")


# ----------------------------------------------------------------------------- Transformer(kv_cache=...)
def meta_model(**kw) -> Transformer:
    args = mi.TransformerArgs.from_dict(dict(synth.shape("tiny", **kw.pop("over", {}))))
    with torch.device("meta"):
        return Transformer(args, **kw)


def test_transformer_kv_cache_option():
    assert meta_model().kv_cache == "bf16"
    assert meta_model(kv_cache="fp8").kv_cache == "fp8"
    with pytest.raises(ValueError):
        meta_model(kv_cache="e5m2")
    with pytest.raises(ValueError):
        meta_model(kv_cache="fp8", over={"head_dim": 64})
    with pytest.raises(TypeError):  # keyword-only
        args = mi.TransformerArgs.from_dict(dict(synth.shape("tiny")))
        Transformer(args, 0, 1, True, None, None, "bf16", "fp8")


class _Stop(Exception):
    pass


@pytest.mark.parametrize("fmt", ["bf16", "fp8"])
def test_generate_builds_the_model_cache_format(fmt, monkeypatch):
    model = meta_model(kv_cache=fmt)
    seen = []

    def stop(ids, seqlens, cache, targets, images=None):
        seen.append(cache)
        raise _Stop

    monkeypatch.setattr(model, "forward_logprobs", stop)
    with pytest.raises(_Stop):
        mi.generate([[1, 2, 3]], model, max_tokens=2, temperature=0.0)
    (cache,) = seen
    assert cache.kv_cache == fmt
    want = torch.float8_e4m3fn if fmt == "fp8" else model.dtype
    assert cache.cache_k[0].dtype == want and (fmt == "bf16" or cache.cache_v_exp[0].dtype == torch.int8)


# ----------------------------------------------------------------------------- the hooked restatement
def _normalised_ast(fn, drop_hook: bool) -> str:
    """ast.dump of a function without its docstring; with drop_hook, also without the kv_hook argument and the statement that
    applies it, and with the module prefix `R.` of the restatement's helpers removed."""
    import ast
    import inspect
    import textwrap

    tree = ast.parse(textwrap.dedent(inspect.getsource(fn)))
    f = tree.body[0]
    f.body = [st for st in f.body if not (isinstance(st, ast.Expr) and isinstance(st.value, ast.Constant))]
    if drop_hook:
        f.args.args = [a for a in f.args.args if a.arg != "kv_hook"]
        f.args.defaults = []
        f.body = [st for st in f.body if "kv_hook" not in ast.dump(st) or isinstance(st, ast.If)]

        class Unprefix(ast.NodeTransformer):
            def visit_Attribute(self, node):
                self.generic_visit(node)
                if isinstance(node.value, ast.Name) and node.value.id == "R":
                    return ast.copy_location(ast.Name(id=node.attr, ctx=node.ctx), node)
                return node

        f = Unprefix().visit(f)
    f.name = "attention_forward"
    f.returns = None
    for a in f.args.args:
        a.annotation = None
    return ast.dump(f)


def test_hooked_attention_is_the_restatement_plus_the_hook():
    """tests/kv_fp8_ref.attention_forward is oracle/restatement.attention_forward with one added statement (the hook).  Any
    change to the restatement's attention makes this fail until the hooked copy follows it."""
    assert _normalised_ast(K.attention_forward, True) == _normalised_ast(R.attention_forward, False)


@pytest.mark.parametrize("shape,over,chunk", [("tiny", {"sliding_window": 12}, None), ("tiny", {"sliding_window": 12}, 5),
                                              ("tiny", {}, 3), ("tiny-moe", {"sliding_window": 3}, 5)])
def test_restatement_with_identity_hook_is_unchanged(shape, over, chunk):
    p = synth.shape(shape, **over)
    om = oracle_model(p, 2)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 7 + i) for i, n in enumerate((17, 16))]
    want = R.generate(prompts, om, max_tokens=4, chunk_size=chunk, return_logits=True)
    with K.hooked_attention(lambda t: t):
        got = R.generate(prompts, om, max_tokens=4, chunk_size=chunk, return_logits=True)
    assert got[0] == want[0] and got[1] == want[1]
    assert all(torch.equal(a, b) for a, b in zip(got[2], want[2]))
    # and the hook is live: the FP8-cache model computes other logits (k', v' are not k, v)
    with K.fp8_kv_cache():
        fp8 = R.generate(prompts, om, max_tokens=4, chunk_size=chunk, return_logits=True)
    assert not torch.equal(fp8[2][0], want[2][0])
