"""FP8 (e4m3) KV cache on the GPU.

* mb200_kv_quantize against the CPU restatement (tests/kv_fp8_ref.py), bit for bit on the e4m3 bytes, the exponents and the
  in-place x'.
* attn_decode_tma_fp8_kernel<REP> and attn_prefill_fp8_kernel against their bf16 kernels on a bf16 ring that holds x', bit for
  bit: the FP8 readers rebuild x' exactly and run the bf16 arithmetic.
* Models with kv_cache="fp8" against the FP8-cache restatement (the oracle with k <- k', v <- v' after RoPE), within the
  tolerances of tests/test_gpu_model.py, and the reference's decode == re-prefill property.
"""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.transformer import Transformer
from mistral_inference_b200.transformer_layers import decode_splits
from oracle import fp8 as F8
from oracle import restatement as R

from . import kv_fp8_ref as K
from .test_gpu_model import Contamination, check_rows, report
from .util import LOGPROB_TOL, RouterProbe, assert_launched, launched_kernels, oracle_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
HD = 128
ATTN = r"attn_\w+_kernel"


def bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int16)


def random_rows(shape, seed: int) -> torch.Tensor:
    """bf16 rows [..., 128] whose scales span the format: most near 1, some tiny (e < -112: the kernels' exact fp32 rebuild), some
    large."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(*shape, HD, generator=g)
    pick = torch.randint(0, 8, shape, generator=g)
    scale = torch.tensor([1.0, 1.0, 1.0, 4.0, 2.0 ** -3, 2.0 ** 6, 2.0 ** -113, 2.0 ** -120])[pick]
    return (x * scale[..., None]).to(torch.bfloat16)


def designed_rows() -> torch.Tensor:
    def row(*vals, fill=0.0):
        return torch.tensor(list(vals) + [fill] * (HD - len(vals)), dtype=torch.float32)
    rows = [row(), row(-0.0, fill=-0.0), row(56.0, -1.0), row(56.25, -1.0), row(448.0, 1.0625, 1.1875, -1.0625, 2.0 ** -10, 400.0, -432.0),
            row(2.0 ** -128, 2.0 ** -133, -3 * 2.0 ** -133, 2.0 ** -130), row(448 * 2.0 ** -118, -(2.0 ** -130), 2.0 ** -127),
            row(-3.0, 2.5, -0.75, 0.3, -0.001, 0.0, -0.0, 6.0), row(1.75, fill=-1.75), row(2.0 ** 100, -(2.0 ** 90))]
    return torch.stack(rows).to(torch.bfloat16)


# ----------------------------------------------------------------------------- the quantiser
@pytest.mark.parametrize("KV,B,max_batch,W,lens,seqpos", [
    (8, 3, 5, 16, [5, 20, 1], [3, 9, 30]),     # chunk longer than W: only its last W tokens are cached; ring wrap
    (1, 1, 2, 64, [64], [100]),
    (4, 2, 2, 1000, [37, 3], [2, 998]),
])
def test_quantize_kernel_matches_the_format(KV, B, max_batch, W, lens, seqpos):
    T = sum(lens)
    k = random_rows((T, KV), 1)
    v = random_rows((T, KV), 2)
    d = designed_rows()
    n = min(len(d), T * KV)
    k.view(-1, HD)[:n] = d[:n]
    v.view(-1, HD)[-n:] = d[:n]
    c = BufferCache(1, max_batch, W, KV, HD, kv_cache="fp8").to(DEV, torch.bfloat16)
    c.init_kvseqlens(B)
    c._kv_seqlens_host = list(seqpos)
    rows = c.get_input_metadata(lens)[0].cache_rows
    for t in (c.cache_k[0], c.cache_v[0]):
        t.view(torch.uint8).fill_(0x55)
    for t in (c.cache_k_exp[0], c.cache_v_exp[0]):
        t.fill_(99)
    kg, vg = k.view(T, KV * HD).to(DEV), v.view(T, KV * HD).to(DEV)
    assert_launched(lambda: _abi.kv_quantize(kg, vg, True, c.cache_k[0], c.cache_v[0], c.cache_k_exp[0], c.cache_v_exp[0], rows),
                    r"kv_quantize_kernel", r"kv_quantize", 1)
    for x, xg, ring, ex in ((k, kg, c.cache_k[0], c.cache_k_exp[0]), (v, vg, c.cache_v[0], c.cache_v_exp[0])):
        q, e = K.quantize_kv_rows(x)
        assert torch.equal(bits(xg.cpu().view(T, KV, HD)), bits(K.dequant(q, e)))  # in place: x'
        flat_q = ring.view(torch.uint8).view(-1, KV, HD).cpu()
        flat_e = ex.view(-1, KV).cpu()
        written = torch.zeros(flat_q.shape[0], dtype=torch.bool)
        for t, r in enumerate(rows.tolist()):
            if r >= 0:
                assert torch.equal(flat_q[r], q[t]) and torch.equal(flat_e[r], e[t]), (t, r)
                written[r] = True
        assert written.sum().item() == sum(min(n, W) for n in lens)
        assert flat_q[~written].eq(0x55).all() and flat_e[~written].eq(99).all()  # rows -1 and other rows untouched
    # ring only (decode), from the in-place k', v': the projection gives the same x' (bytes may differ at a largest |q| of 224)
    _abi.kv_quantize(kg, vg, False, c.cache_k[0], c.cache_v[0], c.cache_k_exp[0], c.cache_v_exp[0], rows)
    for xg, ring, ex in ((kg, c.cache_k[0], c.cache_k_exp[0]), (vg, c.cache_v[0], c.cache_v_exp[0])):
        for t, r in enumerate(rows.tolist()):
            if r >= 0:
                got = K.dequant(ring.view(torch.uint8).view(-1, KV, HD)[r].cpu(), ex.view(-1, KV)[r].cpu())
                assert torch.equal(bits(got), bits(xg[t].view(KV, HD).cpu()))


# ----------------------------------------------------------------------------- decode attention
def fp8_ring(x: torch.Tensor, lens, poison: bool):
    """(e4m3 ring, exponents, bf16 ring of x') of bf16 rows x [max_batch, W, KV, 128]; with `poison`, slots >= lens[b] hold NaN codes
    and extreme exponents (and NaN in the bf16 ring)."""
    q, e = K.quantize_kv_rows(x)
    xp = K.dequant(q, e)
    if poison:
        for b in range(x.shape[0]):
            n = lens[b] if b < len(lens) else 0
            q[b, n:] = torch.tensor([0x7F, 0xFF, 0x00, 0x80], dtype=torch.uint8).repeat(HD // 4)
            e[b, n:] = torch.tensor([127, -128], dtype=torch.int8).repeat(x.shape[2])[: x.shape[2]]
            xp[b, n:] = float("nan")
    return q.view(torch.float8_e4m3fn).to(DEV), e.to(DEV), xp.to(DEV)


def decode_lens(B: int, W: int, S: int):
    C = [1, 63, 64, 65, 128, 129, 64 * S, 64 * S + 1, W - 1, W] + [max(1, S * c - 1) for c in (64, 65, 128)]
    C = sorted(set(min(max(n, 1), W) for n in C))
    return [C[(3 * b) % len(C)] for b in range(B)] if B > 1 else [W]


@pytest.mark.parametrize("rep", [1, 2, 4, 6, 8])
@pytest.mark.parametrize("B,W", [(1, 300), (2, 4096), (32, 4096), (32, 300)])
def test_decode_attention_fp8_equals_bf16_on_x_prime(rep, B, W):
    KV = 2 if B < 32 else 8
    H = KV * rep
    max_batch = B + 1
    S = decode_splits(B, KV, W)
    lens = decode_lens(B, W, S)
    x_k = random_rows((max_batch, W, KV), 10 + rep)
    x_v = random_rows((max_batch, W, KV), 20 + rep)
    k8, ek, kb = fp8_ring(x_k, lens, True)
    v8, ev, vb = fp8_ring(x_v, lens, True)
    q = torch.randn(B, H * HD, generator=torch.Generator().manual_seed(rep)).to(torch.bfloat16).to(DEV)
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(B, H * HD, H, KV, HD, H * HD, 0, max_batch), torch.device(DEV))
    want = torch.full_like(q, float("nan"))
    got = torch.full_like(q, float("nan"))
    _abi.attn_decode(q, kb, vb, kv_len, want, H, KV, HD, S, ws)
    assert_launched(lambda: _abi.attn_decode_fp8(q, k8, v8, ek, ev, kv_len, got, H, KV, HD, S, ws), rf"attn_decode_tma_fp8_kernel<{rep}>", ATTN, 1)
    assert torch.isfinite(want.float()).all()
    assert torch.equal(bits(got), bits(want)), f"S={S} lens={lens}: {(got.float() - want.float()).abs().max().item()}"


# ----------------------------------------------------------------------------- chunked-prefill attention
@pytest.mark.parametrize("W,seqpos,lens", [
    (64, (70, 5, 200), (10, 64, 100)),      # chunks below, at and above W; ring wrapped
    (100, (1, 99, 300), (130, 1, 37)),      # int window, unequal sequences
    (16, (16, 17), (3, 40)),                # a short window layer of a list of windows ...
    (4096, (500, 33), (65, 200)),           # ... and its full-context layer
])
@pytest.mark.parametrize("rep", [1, 4, 6])
def test_prefill_attention_fp8_equals_bf16_on_x_prime(W, seqpos, lens, rep):
    KV = 2
    H = KV * rep
    B, T = len(lens), sum(lens)
    x_k = random_rows((B, W, KV), 30 + W)
    x_v = random_rows((B, W, KV), 40 + W)
    k8, ek, kb = fp8_ring(x_k, [W] * B, False)
    v8, ev, vb = fp8_ring(x_v, [W] * B, False)
    kn = K.kv_prime(random_rows((T, KV), 50)).view(T, KV * HD).to(DEV)
    vn = K.kv_prime(random_rows((T, KV), 60)).view(T, KV * HD).to(DEV)
    q = torch.randn(T, H * HD, generator=torch.Generator().manual_seed(W)).to(torch.bfloat16).to(DEV)
    q_start = torch.tensor([0] + list(torch.tensor(lens).cumsum(0).tolist()), dtype=torch.int32, device=DEV)
    sp = torch.tensor(seqpos, dtype=torch.int32, device=DEV)
    want, got = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    _abi.attn_prefill(q, kn, vn, kb, vb, q_start, sp, want, B, max(lens), W, H, KV, HD, causal=True)
    assert_launched(lambda: _abi.attn_prefill_fp8(q, kn, vn, k8, v8, ek, ev, q_start, sp, got, B, max(lens), W, H, KV, HD),
                    r"attn_prefill_fp8_kernel", ATTN, 1)
    assert torch.isfinite(want.float()).all()
    assert torch.equal(bits(got), bits(want))


# ----------------------------------------------------------------------------- models against the FP8-cache restatement
def fp8_model_and_oracle(p: dict, max_batch: int, seed: int = 1, **kw):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16, kv_cache="fp8", **kw)
    sd = synth.synth_state_dict(p, seed, torch.bfloat16, "cuda")
    m.load_state_dict(sd)
    osd = {k: v.cpu() for k, v in sd.items()}
    if kw.get("expert_weights") == "fp8":  # the oracle runs on the dequantised experts W' (oracle/fp8.py)
        osd = F8.fp8_checkpoint(osd)
    om = R.OracleTransformer(oracle_args(p, max_batch), osd)
    return m.eval(), om


def fp8_cache(m: Transformer, max_seq: int) -> BufferCache:
    a = m.args
    c = BufferCache(m.n_local_layers, a.max_batch_size, max_seq, a.n_kv_heads, a.head_dim, a.sliding_window, kv_cache="fp8")
    c.to(m.device, m.dtype)
    for i in c.cache_k:  # never-written slots: NaN codes and extreme exponents
        c.cache_k[i].view(torch.uint8).fill_(0x7F)
        c.cache_v[i].view(torch.uint8).fill_(0xFF)
        c.cache_k_exp[i].fill_(127)
        c.cache_v_exp[i].fill_(-128)
    c.reset()
    return c


@pytest.mark.parametrize("shape,over,lens,chunk", [
    ("tiny", {}, [11, 9, 10], 4),
    ("tiny", {"sliding_window": 5}, [11, 9, 10], 4),
    ("tiny", {"sliding_window": [4, None]}, [70, 68], 33),
    ("tiny-moe", {"sliding_window": 3}, [11, 12], 5),
    ("tiny", {}, [23], None),                                                  # batch 1: graph decode, not the megakernel
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096, "sliding_window": 64}, [70 - (b % 3) for b in range(32)], None),  # B = 32, wrap
    ("mistral-nemo-12b", {"n_layers": 2, "vocab_size": 4096}, [48 - (b % 3) for b in range(8)], None),
])
def test_model_vs_fp8_cache_oracle(shape, over, lens, chunk):
    p = synth.shape(shape, **over)
    m, om = fp8_model_and_oracle(p, len(lens) + 1 if len(lens) < 32 else len(lens))
    check_against_oracle(m, om, p, f"{shape}{over}", lens, chunk)


def check_against_oracle(m: Transformer, om: R.OracleTransformer, p: dict, tag: str, lens, chunk) -> None:
    """Prefill (in chunks) and 4 decode steps of `m` against the FP8-cache restatement `om`, teacher-forced on the oracle's picks;
    every decode step on the FP8 kernels, none on the megakernel."""
    moe = p.get("moe") is not None
    B, steps = len(lens), 4  # decode: eager warm-up, graph capture, replays
    prompts = [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate(lens)]
    cache, ocache = fp8_cache(m, max(lens) + steps + 2), om.new_cache(max(lens) + steps + 2)
    cont = Contamination(B, moe)
    step_chunk = chunk or max(lens)
    with RouterProbe() as probe, K.fp8_kv_cache():
        for s in range(0, max(lens), step_chunk):
            chunks = [pr[s:s + step_chunk] for pr in prompts]
            sl = [len(c) for c in chunks]
            flat = torch.tensor(sum(chunks, []))
            got = m.forward(flat.cuda(), sl, cache)
            want = om.forward(flat, sl, ocache)
            d = report(f"fp8 cache {tag} prefill @{s}", got, want)
            check_rows(d, want, cont.rows(probe.end_forward(), sl), f"fp8 cache {tag} prefill @{s}")
            nxt = want[torch.tensor(sl).cumsum(0) - 1].argmax(-1)
        for step in range(steps):
            out = {}
            names = launched_kernels(lambda: out.setdefault("logits", m.forward(nxt.cuda(), [1] * B, cache)))
            got = out["logits"]
            want = om.forward(nxt, [1] * B, ocache)
            assert not any(n.startswith("decode_megakernel") for n in names), names
            if step == 0:  # eager warm-up step: the FP8 decode kernels ran (later steps replay a graph and log nothing)
                assert any(n.startswith("attn_decode_tma_fp8_kernel") for n in names) and any(n == "kv_quantize_kernel" for n in names), names
            d = report(f"fp8 cache {tag} decode step {step}", got, want)
            check_rows(d, want, cont.rows(probe.end_forward(), [1] * B), f"fp8 cache {tag} decode step {step}")
            nxt = want.argmax(-1)


@pytest.mark.parametrize("shape,over,lens", [("tiny", {"sliding_window": 6}, [12, 10, 11]), ("tiny", {}, [17])])  # + 6 tokens: every chunk of 5 non-empty
def test_fp8_cache_decode_equals_reprefill(shape, over, lens):
    """The reference's self-consistency property on the FP8-cache model: generate, then re-prefill prompt + tokens with
    chunk_size=5 and without chunks; the log-probabilities agree."""
    p = synth.shape(shape, **over)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 90 + i) for i, n in enumerate(lens)]
    m, _ = fp8_model_and_oracle(p, len(lens))
    toks, lp = mi.generate(prompts, m, max_tokens=6, temperature=0.0)
    full = [pr + t for pr, t in zip(prompts, toks)]
    for chunk in (5, None):
        gen2, lp2 = mi.generate(full, m, max_tokens=0, temperature=0.0, chunk_size=chunk)
        assert gen2 == [] and all(len(x) == len(y) for x, y in zip(lp, lp2))
        worst = max(abs(a - b) for x, y in zip(lp, lp2) for a, b in zip(x, y))
        print(f"[parity] fp8 cache {shape}{over} decode vs re-prefill (chunk {chunk}): logprob max|d|={worst:.4f}")
        assert worst <= LOGPROB_TOL


@pytest.mark.parametrize("lens,chunk", [([12, 11, 14], 5), ([19], None)])
def test_fp8_cache_with_fp8_experts(lens, chunk):
    """Both storage formats at once against the restatement run on the dequantised experts W' with the k', v' hook."""
    p = synth.shape("tiny-moe")
    m, om = fp8_model_and_oracle(p, len(lens), expert_weights="fp8")
    assert m.kv_cache == "fp8" and m.expert_weights == "fp8"
    check_against_oracle(m, om, p, f"tiny-moe fp8 experts {lens}", lens, chunk)


def test_model_refuses_a_cache_of_the_other_format():
    p = synth.shape("tiny")
    m, _ = fp8_model_and_oracle(p, 1)
    a = m.args
    c = BufferCache(m.n_local_layers, 1, 16, a.n_kv_heads, a.head_dim).to(m.device, m.dtype)
    with pytest.raises(AssertionError):
        m.forward(torch.tensor([1, 2, 3], device=DEV), [3], c)
