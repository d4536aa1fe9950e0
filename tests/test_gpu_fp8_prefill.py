"""FP8 activations for FP8 dense weights on the GPU (prefill_compute="fp8", include/mistral_b200.h).

* The quantiser kernels (mb200_quantize_act_e4m3, with and without the fused RMSNorm) equal the restatement of
  tests/fp8_prefill_ref.py byte for byte, codes and exponents, on the edge rows and on rows spread over 60 binades.
* The three _fp8a8 entry points, bit for bit, on exact designs: small-integer activations times a power of two per row (for the
  normed entries: +-2^j per row with eps = 0, so the RMSNorm output is the small-integer norm weight), small-integer e4m3 weights
  and arbitrary fp32 row scales.  Every k-block sum is then exact in the tensor cores and the fp32 total exact, so
  bf16(fp32(fp32(s * acc) * 2^e)) is the _fp8 entry point's bf16(fp32(s * sum x * q)) on the same input: the A8 call must equal
  the A16 call bit for bit, in every mode (STORE, RESIDUAL, SWIGLU, QKV + RoPE with ring scatter), and STORE also equals the
  float64 product.  The launch log shows the quantiser and the A8 kernel with the expected tile width.
* The accumulator: one k-block whose exact sum needs 17 bits (measured and reported), and a K = 4096 row whose running sum needs
  24 bits across k-blocks (exact: the promotion is fp32).
* Below the threshold the _fp8a8 entry points are the _fp8 ones: same bits, same launches.
* Gaussian data at the 7B and Nemo shapes: every Linear within a bound derived from the e4m3 and bf16 roundings of the float64
  product, and within one bf16 step of the restatement.
* Models: a first prefill of >= 129 tokens against the CPU restatement (tests/fp8_dense_ref.py + tests/fp8_prefill_ref.py),
  chunked prefill at <= 128 tokens and decode (megakernel at batch 1, graph path at batch 8) bit for bit against the FP8 model,
  generate against the restatement, and from_folder.
"""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.rope import precompute_freqs_cis
from mistral_inference_b200.transformer import Transformer
from oracle import fp8 as F8
from oracle import restatement as R

from . import fp8_prefill_ref as FP
from .test_gpu_model import check_rows, report
from .util import LOGPROB_TOL, launched_kernels, oracle_args

pytestmark = pytest.mark.gpu
DEV = "cuda"


def ws_for(T, K, N):
    return _abi.Workspace(_abi.workspace_bytes(T, max(K, N), 32, 8, 128, max(K, N), 0, 64), torch.device(DEV))


def a8_expected(T: int, N: int, K: int, env=None) -> bool:
    env = env or {}
    sk = env.get("MB200_STREAMK", "1")[:1] != "0" and T <= 128 and N % 128 == 0 and K % 64 == 0
    return T >= 128 and not sk


# ----------------------------------------------------------------------------- quantiser kernels
@pytest.mark.parametrize("K", [128, 256, 4096, 5120, 14336, 28672])
@pytest.mark.parametrize("norm", [False, True])
def test_quantiser_kernel_is_the_restatement(K, norm):
    g = torch.Generator().manual_seed(K)
    edges = FP.edge_rows(K)
    spread = (torch.randn(61, K, generator=g) * torch.pow(2.0, torch.arange(-30, 31).double()).float()[:, None]).to(torch.bfloat16)
    x = torch.cat([edges, spread, edges[:5]]).to(DEV)  # T = 82: no multiple of any tile
    w = None
    if norm:
        w = (torch.randn(K, generator=g) * 2).to(torch.bfloat16).to(DEV)
    q, e = _abi.quantize_act_e4m3(x, w, 1e-5 if norm else 0.0)
    v = _abi.rmsnorm(x, w, 1e-5) if norm else x  # the bf16 values the A16 path feeds its GEMM
    wq, we = FP.quantize_act(v.cpu())
    assert torch.equal(e.cpu(), we)
    assert torch.equal(q.cpu(), wq)


# ----------------------------------------------------------------------------- exact designs
def exact_design(T, N, K, normed, seed):
    g = torch.Generator().manual_seed(seed)
    j = torch.randint(-20, 21, (T, 1), generator=g).double()
    if normed:  # +-2^j: mean square 4^j, so with eps = 0 the RMSNorm scale is exactly 2^-j and the output is +-norm_w
        sign = torch.randint(0, 2, (T, K), generator=g).double() * 2 - 1
        x = sign * torch.pow(2.0, j)
        norm_w = torch.randint(-4, 5, (K,), generator=g).double().to(torch.bfloat16).to(DEV)
    else:
        x = torch.randint(-4, 5, (T, K), generator=g).double() * torch.pow(2.0, j)
        norm_w = None
    x = x.to(torch.bfloat16).to(DEV)
    q = torch.randint(-4, 5, (N, K), generator=g).float().to(torch.float8_e4m3fn).view(torch.uint8).to(DEV)
    s = (torch.rand(N, generator=g) * 3 + 0.01).to(DEV)
    return x, norm_w, q, s


def run_entry(entry, a8, T, N, K, x, norm_w, q, s, seed=0):
    """Runs one _fp8 / _fp8a8 entry point; returns its outputs (and the kernels it launched)."""
    ws = ws_for(T, K, N)
    outs = {}

    def call():
        if entry in ("store", "residual"):
            res = torch.randn(T, N, generator=torch.Generator().manual_seed(seed)).to(torch.bfloat16).to(DEV) if entry == "residual" else None
            out = torch.full((T, N), float("nan"), dtype=torch.bfloat16, device=DEV)
            _abi.linear_residual_fp8(x, q, s, res, out, ws, a8=a8)
            outs["out"] = out
        elif entry == "swiglu":
            out = torch.full((T, N // 2), float("nan"), dtype=torch.bfloat16, device=DEV)
            _abi.ffn_gateup_fp8(x, norm_w, q, s, out, 0.0, ws, a8=a8)
            outs["out"] = out
        else:  # qkv: N = (H + 2 KV) * 128 with H = 4 KV
            hd, KV = 128, N // (6 * 128)
            H = 4 * KV
            rope = torch.view_as_real(precompute_freqs_cis(hd, T + 16, 1e6)).contiguous().to(DEV)
            pos = torch.arange(T, dtype=torch.int32, device=DEV) + 7
            rows = torch.randperm(T + 3, generator=torch.Generator().manual_seed(seed))[:T].to(torch.int32)
            rows[::5] = -1
            rows = rows.to(DEV)
            qo = torch.empty(T, H * hd, dtype=torch.bfloat16, device=DEV)
            ko = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
            vo = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
            ck = torch.zeros(T + 3, KV * hd, dtype=torch.bfloat16, device=DEV)
            cv = torch.zeros(T + 3, KV * hd, dtype=torch.bfloat16, device=DEV)
            _abi.attn_qkv_fp8(x, norm_w, q, s, rope, pos, qo, ko, vo, ck, cv, rows, H, KV, hd, 0.0, ws, a8=a8)
            outs.update(q=qo, k=ko, v=vo, ck=ck, cv=cv)

    names = launched_kernels(call)
    torch.cuda.synchronize()
    return outs, names


def check_a8_case(entry, T, N, K, env, monkeypatch, seed=1):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    x, norm_w, q, s = exact_design(T, N, K, entry in ("swiglu", "qkv"), seed)
    got, names8 = run_entry(entry, True, T, N, K, x, norm_w, q, s, seed)
    want, names16 = run_entry(entry, False, T, N, K, x, norm_w, q, s, seed)
    for k in want:
        assert torch.equal(got[k].view(torch.int16), want[k].view(torch.int16)), (entry, T, N, K, k)
    mode = {"store": 0, "residual": 1, "swiglu": 3, "qkv": 4}[entry] | 32 | 128
    if a8_expected(T, N, K, env):
        forced = int(env.get("MB200_GEMM_BN", "0"))
        bn = forced if forced in (64, 128) and N % forced == 0 else (128 if N % 128 == 0 else 64)
        gemms = [n for n in names8 if "gemm" in n or "skinny" in n]
        assert gemms == [f"gemm_wgmma_a8_kernel<{mode}, {bn}>"], names8
        assert f"quantize_act_e4m3_kernel<{'true' if entry in ('swiglu', 'qkv') else 'false'}>" in names8, names8
    else:
        assert names8 == names16, (names8, names16)
    if entry == "store":  # the float64 product
        qf = q.view(torch.float8_e4m3fn).double()
        exact = x.double() @ qf.T
        assert torch.equal(got["out"], (exact * s.double()[None, :]).float().to(torch.bfloat16))  # s * acc is exact in float64


# Inside one k-block the tensor cores keep 2^16 + 2^j for j >= KEEP_FROM (the measured width of their sum, include/mistral_b200.h)
KEEP_FROM = 3
T_EDGES = [128, 129, 255, 256, 257, 511, 512, 513, 4096]


@pytest.mark.parametrize("T", T_EDGES)
@pytest.mark.parametrize("entry,N,K", [("store", 4096, 4096), ("residual", 4096, 14336), ("swiglu", 28672, 4096), ("qkv", 6144, 4096)])
def test_a8_equals_a16_on_exact_designs_real_shapes(entry, N, K, T, monkeypatch):
    check_a8_case(entry, T, N, K, {}, monkeypatch)


@pytest.mark.parametrize("T", [128, 129, 257, 513])
@pytest.mark.parametrize("entry,N,K,env", [
    ("store", 192, 128, {}), ("store", 192, 256, {}), ("residual", 576, 384, {}), ("store", 128, 128, {}),  # BN 64 and 128 at tile edges
    ("residual", 1024, 256, {"MB200_GEMM_BN": "64"}), ("swiglu", 512, 128, {"MB200_GEMM_BN": "64"}),       # forced BN 64
    ("swiglu", 1152, 640, {}), ("qkv", 768, 128, {}), ("qkv", 1536, 384, {"MB200_GEMM_BN": "64"}),
    ("store", 4096, 512, {"MB200_STREAMK": "0"}),                                                           # T = 128 without stream-K
])
def test_a8_equals_a16_on_exact_designs_edges(entry, N, K, env, T, monkeypatch):
    check_a8_case(entry, T, N, K, env, monkeypatch)


# ----------------------------------------------------------------------------- the accumulator
def one_row_call(xrow, wrows, T=256):
    """y[0, :] of the A8 STORE entry for a designed first token row (other rows zero), e4m3 weight rows `wrows`, s = 1."""
    K = xrow.numel()
    x = torch.zeros(T, K, dtype=torch.float64)
    x[0] = xrow
    q = wrows.float().to(torch.float8_e4m3fn)
    assert torch.equal(q.double(), wrows.double())
    x = x.to(torch.bfloat16).to(DEV)
    N = wrows.shape[0]
    out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
    names = launched_kernels(lambda: _abi.linear_residual_fp8(x, q.view(torch.uint8).to(DEV), torch.ones(N, device=DEV), None, out,
                                                              ws_for(T, K, N), a8=True))
    assert any(n.startswith("gemm_wgmma_a8_kernel") for n in names), names
    return out[0].double().cpu()


def test_one_k_block_sum_of_17_bits():
    """Inside one k-block: x = [256, 2^j, 0, ...], w = [256, 1, 0, ...], so block 0 sums 2^16 + 2^j (17 significant bits for
    j = 0); block 1 adds 256 * -256.  The output is 2^j where the tensor cores' block sum kept the small product and 0 where they
    dropped it: a measurement of the hardware's accumulator inside one promotion interval, printed, and held to the contract of
    include/mistral_b200.h."""
    K = 256
    kept = []
    for j in range(9):
        x = torch.zeros(K, dtype=torch.float64)
        w = torch.zeros(K, dtype=torch.float64)
        x[0], x[1], x[128] = 256.0, 2.0 ** j, 256.0
        w[0], w[1], w[128] = 256.0, 1.0, -256.0
        y = one_row_call(x, torch.stack([w] * 128))[0].item()
        assert y in (0.0, 2.0 ** j), (j, y)
        kept.append(y == 2.0 ** j)
    print(f"\n[fp8 accumulator] 2^16 + 2^j in one k-block keeps 2^j for j in {[j for j, k in enumerate(kept) if k]}")
    assert kept == sorted(kept), kept  # once kept, every larger term is kept
    assert kept[KEEP_FROM:] == [True] * (9 - KEEP_FROM) and not any(kept[:KEEP_FROM]), kept


def test_promotion_keeps_24_bits_across_k_blocks():
    """K = 4096: block 0 sums 128 * 256 * 256 = 2^23, blocks 1..30 add 1 each, block 31 subtracts 2^23.  The running sum
    2^23 + 30 needs 24 significant bits; fp32 promotion keeps it, so the output is exactly 30."""
    K = 4096
    x = torch.zeros(K, dtype=torch.float64)
    w = torch.zeros(K, dtype=torch.float64)
    x[:128], w[:128] = 256.0, 256.0
    for b in range(1, 31):
        x[128 * b], w[128 * b] = 1.0, 1.0
    x[128 * 31:], w[128 * 31:] = 256.0, -256.0
    y = one_row_call(x, torch.stack([w] * 128))
    assert bool((y == 30.0).all()), y[:4]


# ----------------------------------------------------------------------------- below the threshold
@pytest.mark.parametrize("T", [1, 4, 5, 64, 100, 127, 128])
@pytest.mark.parametrize("entry,N,K,env", [("store", 4096, 4096, {}), ("swiglu", 28672, 4096, {}), ("qkv", 6144, 4096, {}),
                                           ("residual", 192, 256, {}), ("store", 4096, 512, {"MB200_STREAMK": "0"})])
def test_below_threshold_is_the_fp8_entry(entry, N, K, env, T, monkeypatch):
    if a8_expected(T, N, K, env):
        pytest.skip("in the FP8-activation regime")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    g = torch.Generator().manual_seed(T)
    x = torch.randn(T, K, generator=g).to(torch.bfloat16).to(DEV)
    norm_w = (torch.rand(K, generator=g) + 0.5).to(torch.bfloat16).to(DEV)
    q, s = F8.quantize_rows((torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16))
    got, n8 = run_entry(entry, True, T, N, K, x, norm_w, q.to(DEV), s.to(DEV))
    want, n16 = run_entry(entry, False, T, N, K, x, norm_w, q.to(DEV), s.to(DEV))
    assert n8 == n16
    for k in want:
        assert torch.equal(got[k].view(torch.int16), want[k].view(torch.int16)), k


# ----------------------------------------------------------------------------- Gaussian data at the real shapes
@pytest.mark.parametrize("shape", ["mistral-7b", "mistral-nemo-12b"])
@pytest.mark.parametrize("T", [256, 1024])
def test_gaussian_linears_within_the_rounding_bound(shape, T):
    p = synth.shape(shape)
    dim, hidden, H, KV, hd = p["dim"], p["hidden_dim"], p["n_heads"], p["n_kv_heads"], p["head_dim"]
    g = torch.Generator().manual_seed(T)
    for name, N, K in (("wqkv", (H + 2 * KV) * hd, dim), ("wo", dim, H * hd), ("w13", 2 * hidden, dim), ("w2", dim, hidden)):
        x = torch.randn(T, K, generator=g).to(torch.bfloat16).to(DEV)
        q, s = F8.quantize_rows((torch.randn(N, K, generator=g) * 0.02).to(torch.bfloat16))
        q, s = q.to(DEV), s.to(DEV)
        out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
        _abi.linear_residual_fp8(x, q, s, None, out, ws_for(T, K, N), a8=True)
        wd = q.view(torch.float8_e4m3fn).double() * s.double()[:, None]
        exact = x.double() @ wd.T
        xq, e = FP.quantize_act(x)
        # e4m3: relative half step 2^-4 of normal codes, absolute 2^-10 * 2^e below them; bf16 output: relative 2^-8 (+ fp32 slack)
        bound = 2.0 ** -4 * (x.double().abs() @ wd.abs().T) + torch.pow(2.0, e.double() - 10)[:, None] * wd.abs().sum(1)[None, :]
        bound = bound + 2.0 ** -8 * exact.abs() * (1 + 2.0 ** -4) + 1e-30
        err = (out.double() - exact).abs()
        assert bool((err <= bound).all()), (name, (err / bound).max().item())
        o = out.double()
        # against the restatement: its block sums are exact then rounded (24) or truncated to 14 bits; the tensor cores truncate each
        # of the <= 33 terms of a k32 step below 2^-13 of the largest, 4 steps per block: < 2^-6 of the block's largest term, so
        # < 2^-6 * sum_k |x q| * s * 2^e in all, plus two bf16 output steps
        absdot = (FP.dequantize_act(xq, e).abs() @ wd.abs().T)
        for bits in (24, 14):
            c = FP.a8_epilogue(FP.a8_accumulate(xq, q, bits), s, e).double()
            step = torch.pow(2.0, torch.floor(torch.log2(c.abs().clamp_min(1e-30))) - 7)
            d = (o - c).abs()
            print(f"\n[fp8 prefill] {shape} {name} T={T} vs restatement (block sums {bits} bits): exact {(o == c).double().mean().item():.4f}, "
                  f"max {(d / step).max().item():.0f} bf16 steps, max |d| / sum|xq w| {(d / absdot.clamp_min(1e-30)).max().item():.2e}")
            assert bool((d <= 2 * step + 2.0 ** -6 * absdot).all()), (name, bits)
        print(f"[fp8 prefill] {shape} {name} T={T}: max err / bound {(err / bound).max().item():.3f}, "
              f"rel rms vs float64 {((err ** 2).mean().sqrt() / exact.pow(2).mean().sqrt()).item():.4f}")


# ----------------------------------------------------------------------------- models
def models(p: dict, max_batch: int, seed: int = 1):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    sd = synth.synth_state_dict(p, seed, torch.bfloat16, DEV)
    m8 = Transformer.empty(args, DEV, torch.bfloat16, dense_weights="fp8", prefill_compute="fp8")
    m8.load_state_dict(sd)
    m = Transformer.empty(args, DEV, torch.bfloat16, dense_weights="fp8")
    m.load_state_dict(sd)
    return m8.eval(), m.eval(), sd


def new_cache(m, B, n):
    c = BufferCache(m.n_local_layers, m.args.max_batch_size, n, m.args.n_kv_heads, m.args.head_dim, m.args.sliding_window,
                    kv_cache=m.kv_cache).to(m.device, m.dtype)
    c.reset()
    return c


@pytest.mark.parametrize("shape,over,lens", [("tiny", {}, [150, 131]), ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [200, 140])])
def test_model_first_prefill_vs_restatement(shape, over, lens):
    p = synth.shape(shape, **over)
    m8, _, sd = models(p, len(lens))
    om = R.OracleTransformer(oracle_args(p, len(lens)), FP.fp8_prefill_checkpoint({k: v.cpu() for k, v in sd.items()}))
    prompts = [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate(lens)]
    flat = torch.tensor(sum(prompts, []))
    names = []
    got = {}
    names = launched_kernels(lambda: got.setdefault("l", m8.forward(flat.to(DEV), lens, new_cache(m8, len(lens), max(lens) + 4))))
    assert any(n.startswith("gemm_wgmma_a8_kernel") for n in names), names
    want = om.forward(flat, lens, om.new_cache(max(lens) + 4))
    check_rows(report(f"fp8 prefill {shape}", got["l"], want), want, None, f"fp8 prefill {shape}")


@pytest.mark.parametrize("shape,over,lens", [("tiny", {}, [300]), ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [260]),
                                             ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [60 + 7 * b for b in range(8)])])
def test_chunked_prefill_and_decode_equal_the_fp8_model(shape, over, lens):
    """Chunks of <= 128 tokens and every decode step (batch 1: the FP8 megakernel; batch 8: the graph path) never reach the A8
    regime: the logits are the FP8 model's bit for bit."""
    p = synth.shape(shape, **over)
    m8, m, _ = models(p, len(lens))
    B, steps = len(lens), 6
    prompts = [synth.synth_prompt(n, p["vocab_size"], 40 + i) for i, n in enumerate(lens)]
    c8, c = new_cache(m8, B, max(lens) + steps + 2), new_cache(m, B, max(lens) + steps + 2)
    chunk = 128 // B if B > 1 else 128
    for s0 in range(0, max(lens), chunk):
        chunks = [pr[s0:s0 + chunk] for pr in prompts]
        sl = [len(x) for x in chunks]
        flat = torch.tensor(sum(chunks, [])).to(DEV)
        a, b = m8.forward(flat, sl, c8), m.forward(flat, sl, c)
        assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a, b.view(torch.int16) if b.dtype == torch.bfloat16 else b)
        nxt = b[torch.tensor(sl).cumsum(0) - 1].argmax(-1)
    kinds = set()
    for _ in range(steps):
        out = {}
        kinds |= {n.split("<")[0] for n in launched_kernels(lambda: out.setdefault("a", m8.forward(nxt, [1] * B, c8)))}
        b = m.forward(nxt, [1] * B, c)
        assert torch.equal(out["a"], b)
        nxt = b.argmax(-1)
    assert "gemm_wgmma_a8_kernel" not in kinds
    if B == 1:
        assert "decode_megakernel" in kinds, kinds


def test_generate_vs_restatement():
    p = synth.shape("mistral-7b", n_layers=2, vocab_size=4096)
    m8, _, sd = models(p, 2)
    om = R.OracleTransformer(oracle_args(p, 2), FP.fp8_prefill_checkpoint({k: v.cpu() for k, v in sd.items()}))
    prompts = [synth.synth_prompt(n, p["vocab_size"], 5 + i) for i, n in enumerate((180, 150))]
    toks, lp = mi.generate(prompts, m8, max_tokens=5, temperature=0.0, chunk_size=512)
    full = [pr + t for pr, t in zip(prompts, toks)]
    _, olp = R.generate(full, om, max_tokens=0, chunk_size=512)
    worst = max(abs(a - b) for x, y in zip(lp, olp) for a, b in zip(x, y))
    print(f"\n[parity] fp8 prefill generate: logprob max|d|={worst:.4f}")
    assert worst <= LOGPROB_TOL


def test_from_folder_loads(tmp_path):
    p = synth.shape("tiny")
    synth.write_model_folder(str(tmp_path), p, seed=3)
    m8 = Transformer.from_folder(tmp_path, max_batch_size=1, dense_weights="fp8", prefill_compute="fp8")
    m = Transformer.from_folder(tmp_path, max_batch_size=1, dense_weights="fp8")
    assert m8.prefill_compute == "fp8"
    a, b = m8.state_dict(), m.state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    toks = torch.tensor(synth.synth_prompt(140, p["vocab_size"], 2)).to(DEV)
    names = launched_kernels(lambda: m8.forward(toks, [140], new_cache(m8, 1, 150)))
    assert any(n.startswith("gemm_wgmma_a8_kernel") for n in names), names
