"""FP8 (e4m3) dense weights on the GPU (include/mistral_b200.h).

* The three FP8 entry points (mb200_attn_qkv_fp8, mb200_ffn_gateup_fp8, mb200_linear_residual_fp8) bit for bit against an
  exact-by-construction float64 reference, in every regime their dispatch reaches -- GEMV (T <= 4), stream-K (TA 32 / 64 / 128),
  small wgmma (each BN), prefill wgmma (BN 128 / 192 / 256, the blocked walk past 16 m tiles) -- and every mode (STORE,
  RESIDUAL, SWIGLU, QKV + RoPE with ring scatter), at the T, N, K edges of tests/test_gpu_linear_edges.py.  q holds small
  integers (exact e4m3 codes) plus rows with the codes the quantiser produces at the format's ends (subnormals, +-448, all-zero
  rows); x is that file's design, so sum x * q is exact in fp32 in any order (`matmul_exact` proves it per output).  The row
  scales are arbitrary fp32 numbers and the one product y = bf16(fp32(s * acc)) is emulated in float32.  NaN guard rows stay
  NaN, every kernel switch gives the same bits, the launch log names the FP8 kernel, and a shape the bf16 path would give to
  mma.sync is refused.
* One case where the experts' W' contract and this definition round differently: the kernels give this definition.
* Models with dense_weights="fp8" (2-layer 7B and Nemo shapes, tiny) against the CPU restatement run with FP8 dense Linears
  (tests/fp8_dense_ref.py: fp8_dense_checkpoint) within the tolerance of tests/util.py: prefill, chunked prefill, graph decode at B = 2,
  8 and 32, the megakernel at B = 1, generate; the FP8 megakernel against the FP8 graph path over 64 greedy steps; with
  kv_cache="fp8"; tiny-pixtral with images.
"""
import re
from typing import Dict

import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.transformer import Transformer
from oracle import fp8 as F8
from oracle import restatement as R
from oracle import vision as V
from oracle.make_vision_pins import VISION_CASES, case_images, case_params

from . import fp8_dense_ref as FD
from . import kv_fp8_ref as K
from .test_gpu_linear_edges import (CASES, DEV, EPS, REAL, Case, Design, check_guards, check_values, design, exact_product, ints, qkv,
                                    reference, small_bn, variants)
from .test_gpu_model import check_rows, report
from .test_gpu_moe_edges import assert_same, env
from .util import LOGPROB_TOL, launched_kernels, oracle_args

WSCALE = 32  # EPI_WSCALE
MODES = {"store": 0, "residual": 1, "swiglu": 3, "qkv": 4}
NORMED = {"store": False, "residual": False, "swiglu": True, "qkv": True}
E4M3_NAN = 0x7F


# ----------------------------------------------------------------------------- the regime restatement
def fp8_regime(entry: str, T: int, N: int, K: int, envd: Dict[str, str], sms: int) -> str:
    """Regex of the one kernel run_linear_fp8 launches, or 'refused' where run_linear would pick gemm_mma_kernel."""
    mode = MODES[entry] | WSCALE
    if T <= 4:
        return rf"^skinny_linear_kernel<{T}, {mode}, {'true' if NORMED[entry] else 'false'}, true>$"
    ta = 32 if T <= 32 else (64 if T <= 64 else 128)
    if envd.get("MB200_STREAMK", "1")[:1] != "0" and T <= 128 and N % 128 == 0 and K % 64 == 0:
        return rf"^gemm_streamk_fp8_kernel<{mode}, {ta}>$"
    if K % 64 != 0 or not ((N % 128 == 0 or N % 192 == 0) if T >= 128 else N % 32 == 0):
        return "refused"
    if T < 128:
        return rf"^gemm_wgmma_fp8_kernel<{mode}, {small_bn(N, sms, envd)}, {ta}>$"
    pair = envd.get("MB200_GEMM_CLUSTER", "1")[:1] != "0" and T >= 512
    units, m_units = (sms // 2, -(-(-(-T // 128)) // 2)) if pair else (sms, -(-T // 128))
    bn = 256
    if N % 256 or m_units * (N // 256) < units:
        bn = 128 if N % 128 == 0 else 192
    forced = int(envd.get("MB200_GEMM_BN", "0") or 0)
    if forced in (128, 192, 256) and N % forced == 0:
        bn = forced
    return rf"^gemm_wgmma_fp8_kernel<{mode}, {bn}, 128>$"


def fp8_cases():
    fam = [c for c in CASES if c.entry in MODES]
    real = [c for c in REAL if c.entry in MODES and not c.name.startswith("mixtral")]
    return fam, real


FAM, REAL8 = fp8_cases()
OK_FAM = [c for c in FAM if fp8_regime(c.entry, c.T, c.N, c.K, dict(c.env), 132) != "refused"]
REFUSED = [c for c in FAM if fp8_regime(c.entry, c.T, c.N, c.K, dict(c.env), 132) == "refused"]


# ----------------------------------------------------------------------------- designed inputs
def fp8_design(c: Case, device, seed: int = 0):
    """(Design with w = the e4m3 values of q as float64, s fp32 [N]).  q: integers in [-7, 7] (exact e4m3 codes); rows 1, 2, 3 of
    every 97: +-448 mixed with small integers, subnormal codes (k * 2^-9), all zeros (scale 1, as the quantiser writes it)."""
    d = design(c, device, seed)
    N, K = c.N, c.K
    gen = torch.Generator(device=device).manual_seed(seed + 17 * N + K)
    q = ints(gen, (N, K), 7, device)
    rows = torch.arange(N, device=device)
    big, sub, zero = rows % 97 == 1, rows % 97 == 2, rows % 97 == 3
    cols = torch.arange(K, device=device)
    q[big[:, None] & (cols % 61 == 5)[None, :]] = 448.0
    q[big[:, None] & (cols % 61 == 30)[None, :]] = -448.0
    q[sub] = ints(gen, (int(sub.sum()), K), 7, device) * 2.0 ** -9
    q[zero] = 0.0
    if c.entry == "qkv":  # keep the code columns of the coded heads plain integers (their x holds the Hadamard codes)
        q[:, :8] = ints(gen, (N, 8), 7, device)
    # arbitrary fp32 scales around the bf16 design's magnitude: 2^-s times a random fp32 mantissa in [1, 2)
    # (SwiGLU: at most the bf16 design's magnitude -- its fp32 expf overflows for gate values below -88, as in the bf16 path)
    e = torch.randint(-3, 0 if c.entry == "swiglu" else 2, (N,), generator=gen, device=device).double()
    mant = 1 + torch.rand(N, generator=gen, device=device, dtype=torch.float64)
    s = mant * torch.pow(2.0, e) * (d.w.abs().amax(1).clamp_min(2.0 ** -20) / 7)
    # as the quantiser would scale them (s = amax / 448): the +-448 and the subnormal rows land in the other rows' range, where the
    # SwiGLU and RoPE epilogues are certified (fp32 expf overflows below -88, as in the bf16 path)
    s[big] /= 64
    s[sub] *= 2.0 ** 9
    s = s.float()
    s[zero] = 1.0
    return Design(d.x, d.nw, q, d.extra, d.positions), s


def e4m3_bytes(q: torch.Tensor) -> torch.Tensor:
    out = q.float().to(torch.float8_e4m3fn)
    assert torch.equal(out.double(), q), "a designed weight is not an e4m3 value"
    return out.view(torch.uint8)


class Run8:
    """NaN-padded inputs (e4m3 NaN guard rows after q) and NaN-filled outputs, as test_gpu_linear_edges.Run."""

    def __init__(self, c: Case, d: Design, s: torch.Tensor):
        from .test_gpu_linear_edges import Run

        self.base = Run(c, d)
        self.c = c
        self.qbuf = torch.full((c.N + 3, c.K), E4M3_NAN, dtype=torch.uint8, device=DEV)
        self.q = self.qbuf[:c.N]
        self.q.copy_(e4m3_bytes(d.w.to(DEV)))
        self.s = s.to(DEV).contiguous()
        self.extra = d.extra.to(torch.bfloat16).to(DEV).contiguous() if d.extra is not None else None

    def launch(self, envd: Dict[str, str]):
        c, b = self.c, self.base
        o = b.outputs()

        def call():
            if c.entry in ("store", "residual"):
                _abi.linear_residual_fp8(b.x, self.q, self.s, self.extra, o["out"][1], b.ws)
            elif c.entry == "swiglu":
                _abi.ffn_gateup_fp8(b.x, b.nw, self.q, self.s, o["out"][1], EPS, b.ws)
            else:
                H, KV, hd = c.heads
                _abi.attn_qkv_fp8(b.x, b.nw, self.q, self.s, b.rope, b.positions, o["q"][1], o["k"][1], o["v"][1], o["ck"][1], o["cv"][1],
                                  b.rows, H, KV, hd, EPS, b.ws)

        with env(**{"MB200_STREAMK": "1", "MB200_GEMM_CLUSTER": "1", "MB200_GEMM_BN": "0", **envd}):
            names = launched_kernels(call)
        torch.cuda.synchronize()
        return names, o


def fp8_want(c: Case, d: Design, s: torch.Tensor, dref):
    xn = d.x * d.nw if d.nw is not None else d.x
    acc = exact_product(xn.to(dref), d.w.to(dref))  # exact fp32 sums of x * q
    y = (acc.float() * s.to(dref)[None, :]).double()  # the one fp32 product
    return reference(c, Design(*(t.to(dref) if t is not None else None for t in d)), y)


def test_designs_are_exact_and_e4m3():
    """Host-side: every FP8 design is made of e4m3 codes and exact fp32 sums (no GPU needed)."""
    for c in [c for c in OK_FAM if c.T * c.N * c.K <= 2 ** 24][:12]:
        d, s = fp8_design(c, "cpu")
        e4m3_bytes(d.w)
        xn = d.x * d.nw if d.nw is not None else d.x
        exact_product(xn, d.w)
        assert s.dtype == torch.float32 and (s > 0).all()


def run_case8(c: Case):
    sms = _abi.device_info()[0]
    big = c.T * c.N * c.K > 2 ** 27
    dref = DEV if big else "cpu"
    d, s = fp8_design(c, DEV)
    want = fp8_want(c, d, s, dref)
    r = Run8(c, d, s)
    base = dict(c.env)
    names, o = r.launch(base)
    regime = fp8_regime(c.entry, c.T, c.N, c.K, base, sms)
    assert len(names) == 1 and re.search(regime, names[0]), f"{c.name}: launched {names}, expected {regime}"
    check_guards(c, r.base, o, c.name)
    check_values(c, want, o, c.name)
    first = {k: v[1].clone() for k, v in o.items()}
    seen = {regime}
    runs = []
    for e in variants(c, sms):
        reg = fp8_regime(c.entry, c.T, c.N, c.K, e, sms)
        if reg not in seen and reg != "refused":
            seen.add(reg)
            runs.append(e)
    if "streamk" in regime:
        runs.append(base)  # stream-K flags reset themselves on the same workspace
    for e in runs:
        names, o = r.launch(e)
        reg = fp8_regime(c.entry, c.T, c.N, c.K, e, sms)
        what = f"{c.name} {e}"
        assert len(names) == 1 and re.search(reg, names[0]), f"{what}: launched {names}, expected {reg}"
        assert not any("gemm_mma_kernel" in n for n in names)
        check_guards(c, r.base, o, what)
        for k, v in first.items():
            assert_same(o[k][1], v, f"{what}: {k} vs the base run")


@pytest.mark.gpu
@pytest.mark.parametrize("case", OK_FAM, ids=[c.name for c in OK_FAM])
def test_fp8_linear_regimes(case):
    run_case8(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", REAL8, ids=[c.name for c in REAL8])
def test_fp8_linear_real_shapes(case):
    run_case8(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", REFUSED, ids=[c.name for c in REFUSED])
def test_fp8_linear_refuses_the_mma_regime(case):
    d, s = fp8_design(case, DEV)
    r = Run8(case, d, s)
    with pytest.raises(_abi.Mb200Error, match="mma.sync"):
        r.launch({})


@pytest.mark.gpu
@pytest.mark.parametrize("T", [1, 8, 100, 256])
def test_fp8_linear_uses_this_definition_not_w_prime(T):
    """s = 3/448, q = (448, 2.25, 104): bf16(s * 554.25) = 3.71875, while W' = bf16(q * s) sums to 3.703125."""
    K, N = 256, 256
    q = torch.zeros(N, K, dtype=torch.float64)
    q[:, :3] = torch.tensor([448.0, 2.25, 104.0], dtype=torch.float64)
    s = torch.full((N,), 3.0 / 448.0, dtype=torch.float32)
    x = torch.zeros(T, K, dtype=torch.bfloat16)
    x[:, :3] = 1.0
    out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(T, K, 32, 8, 128, K, 0, 4), torch.device(DEV))
    _abi.linear_residual_fp8(x.to(DEV), e4m3_bytes(q).to(DEV), s.to(DEV), None, out, ws)
    assert (out.float() == 3.71875).all()
    qf, sf = e4m3_bytes(q), s
    assert FD.dense_linear(x[:1], qf, sf)[0, 0].item() == 3.71875
    assert torch.nn.functional.linear(x[:1], F8.dequantize_rows(qf, sf)).float()[0, 0].item() == 3.703125


# ----------------------------------------------------------------------------- models against the restatement
def fp8_model_and_oracle(p: dict, max_batch: int, seed: int = 1, **kw):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16, dense_weights="fp8", **kw)
    sd = synth.synth_state_dict(p, seed, torch.bfloat16, "cuda")
    m.load_state_dict(sd)
    om = R.OracleTransformer(oracle_args(p, max_batch), FD.fp8_dense_checkpoint({k: v.cpu() for k, v in sd.items()}))
    return m.eval(), om, sd


def test_quantised_storage_matches_the_restatement():
    """Host-only part of the loader check: the restatement's q and s are those of quantize_rows (tests/fp8_dense_ref.py)."""
    w = (torch.randn(256, 128, generator=torch.Generator().manual_seed(0)) * 0.02).to(torch.bfloat16)
    dw = FD.DenseFp8Weight(*F8.quantize_rows(w))
    q, s = F8.quantize_rows(w)
    assert torch.equal(dw.q, q) and torch.equal(dw.s, s)


@pytest.mark.gpu
def test_loader_quantises_like_the_restatement():
    p = synth.shape("tiny")
    m, _, sd = fp8_model_and_oracle(p, 1)
    msd = m.state_dict()
    for k, v in sd.items():
        if FD.is_dense_key(k):
            q, s = F8.quantize_rows(v.cpu())
            base = k[: -len(".weight")]
            assert torch.equal(msd[base + ".weight_e4m3"].view(torch.uint8).cpu(), q), k
            assert torch.equal(msd[base + ".weight_scale"].cpu(), s), k


def run_against_oracle(m, om, p, tag, lens, chunk, steps=4):
    """Prefill (in chunks) and `steps` decode steps of m against om, teacher-forced on the oracle's picks."""
    B = len(lens)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate(lens)]
    cache = BufferCache(m.n_local_layers, m.args.max_batch_size, max(lens) + steps + 2, m.args.n_kv_heads, m.args.head_dim,
                        m.args.sliding_window, kv_cache=m.kv_cache).to(m.device, m.dtype)
    cache.reset()
    ocache = om.new_cache(max(lens) + steps + 2)
    step_chunk = chunk or max(lens)
    for s0 in range(0, max(lens), step_chunk):
        chunks = [pr[s0:s0 + step_chunk] for pr in prompts]
        sl = [len(c) for c in chunks]
        flat = torch.tensor(sum(chunks, []))
        got = m.forward(flat.cuda(), sl, cache)
        want = om.forward(flat, sl, ocache)
        check_rows(report(f"fp8 dense {tag} prefill @{s0}", got, want), want, None, f"fp8 dense {tag} prefill @{s0}")
        nxt = want[torch.tensor(sl).cumsum(0) - 1].argmax(-1)
    kinds = set()
    for step in range(steps):
        out = {}
        names = launched_kernels(lambda: out.setdefault("logits", m.forward(nxt.cuda(), [1] * B, cache)))
        kinds |= {n.split("<")[0] for n in names}
        got = out["logits"]
        want = om.forward(nxt, [1] * B, ocache)
        check_rows(report(f"fp8 dense {tag} decode {step}", got, want), want, None, f"fp8 dense {tag} decode {step}")
        nxt = want.argmax(-1)
    # the layer Linears run the FP8 kernels (the bf16 lm head its own); nothing falls to mma.sync
    assert "gemm_mma_kernel" not in kinds and (kinds & {"decode_megakernel", "skinny_linear_kernel", "gemm_streamk_fp8_kernel",
                                                        "gemm_wgmma_fp8_kernel"}), kinds
    return kinds


@pytest.mark.gpu
@pytest.mark.parametrize("shape,over,lens,chunk", [
    ("tiny", {}, [11, 9], 4),                                                       # chunked prefill, graph decode B = 2
    ("tiny", {"sliding_window": 5}, [11, 9, 10, 7, 12, 8, 9, 10], None),          # B = 8
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096, "sliding_window": 64}, [70 - (b % 3) for b in range(32)], None),  # B = 32
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [200, 140], 128),           # prefill wgmma + chunks, B = 2
    ("mistral-nemo-12b", {"n_layers": 2, "vocab_size": 4096}, [48 - (b % 3) for b in range(8)], None),
    ("mistral-nemo-12b", {"n_layers": 2, "vocab_size": 4096}, [150], None),         # B = 1: the FP8 megakernel
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [300], None),               # B = 1: the FP8 megakernel
])
def test_fp8_model_vs_oracle(shape, over, lens, chunk):
    p = synth.shape(shape, **over)
    m, om, _ = fp8_model_and_oracle(p, len(lens))
    kinds = run_against_oracle(m, om, p, f"{shape}{over}", lens, chunk)
    if len(lens) == 1:
        assert "decode_megakernel" in kinds, kinds


@pytest.mark.gpu
def test_fp8_generate_vs_oracle():
    p = synth.shape("mistral-7b", n_layers=2, vocab_size=4096)
    m, om, _ = fp8_model_and_oracle(p, 3)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 5 + i) for i, n in enumerate((40, 33, 37))]
    for ps in (prompts, prompts[:1]):  # graph decode at B = 3, the megakernel at B = 1
        toks, lp = mi.generate(ps, m, max_tokens=6, temperature=0.0, chunk_size=16)
        full = [pr + t for pr, t in zip(ps, toks)]
        _, olp = R.generate(full, om, max_tokens=0, chunk_size=16)
        worst = max(abs(a - b) for x, y in zip(lp, olp) for a, b in zip(x, y))
        print(f"[parity] fp8 dense generate B={len(ps)}: logprob max|d|={worst:.4f}")
        assert worst <= LOGPROB_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["mistral-7b", "mistral-nemo-12b"])
def test_fp8_megakernel_vs_graph_path(shape, monkeypatch):
    """64 greedy steps at batch 1 on the FP8 megakernel and on the FP8 graph path: the same picks wherever the pick is decisive
    (top-2 logits more than 4 bf16 ulps apart on both paths); the runs are teacher-forced on the megakernel's picks."""
    p = synth.shape(shape, n_layers=2, vocab_size=4096)
    m, _, _ = fp8_model_and_oracle(p, 1)
    prompt = synth.synth_prompt(40, p["vocab_size"], 3)
    runs = {}
    forced = None
    for path in ("mk", "graph"):
        monkeypatch.setenv("MB200_MEGAKERNEL", "1" if path == "mk" else "0")
        cache = BufferCache(m.n_local_layers, 1, 128, m.args.n_kv_heads, m.args.head_dim).to(m.device, m.dtype)
        cache.reset()
        logits = m.forward(torch.tensor(prompt, device=DEV), [len(prompt)], cache)
        tok = logits[-1:].argmax(-1)
        rows = []
        for i in range(64):
            names = launched_kernels(lambda: rows.append(m.decode_static(tok, cache).clone()))
            if i == 0:
                assert any(n.startswith("decode_megakernel<4, true>") for n in names) == (path == "mk"), names
            tok = rows[-1].argmax(-1) if forced is None else forced[i:i + 1]
        runs[path] = torch.cat(rows)
        if forced is None:
            forced = runs[path].argmax(-1)
    a, b = runs["mk"], runs["graph"]
    top2a, top2b = a.topk(2, -1).values, b.topk(2, -1).values
    ulp = torch.tensor([2.0 ** (torch.frexp(v).exponent.item() - 8) for v in top2a[:, 0].abs().clamp_min(1e-3)])
    decisive = ((top2a[:, 0] - top2a[:, 1]).cpu() > 4 * ulp) & ((top2b[:, 0] - top2b[:, 1]).cpu() > 4 * ulp)
    assert decisive.sum() >= 32, int(decisive.sum())
    assert torch.equal(a.argmax(-1)[decisive.to(a.device)], b.argmax(-1)[decisive.to(b.device)])


@pytest.mark.gpu
@pytest.mark.parametrize("lens,chunk", [([12, 11, 14], 5), ([19], None)])
def test_fp8_dense_with_fp8_cache(lens, chunk):
    p = synth.shape("tiny")
    m, om, _ = fp8_model_and_oracle(p, len(lens), kv_cache="fp8")
    with K.fp8_kv_cache():
        run_against_oracle(m, om, p, f"tiny fp8 cache {lens}", lens, chunk)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(VISION_CASES))
def test_fp8_dense_pixtral_with_images(name):
    """The text layers in FP8, the vision tower and adapter in bf16: generate with images against the multimodal restatement run
    on the FP8 dense checkpoint."""
    p = case_params(name)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 3
    m = Transformer.empty(args, DEV, torch.bfloat16, dense_weights="fp8")
    sd = synth.synth_state_dict(p, 3)
    m.load_state_dict({k: v.to(DEV) for k, v in sd.items()})
    assert m.vision_encoder.transformer.layers[0].attention.wqkv.dtype == torch.bfloat16
    prompts, images = VISION_CASES[name][2], case_images(name)
    toks, lps = mi.generate(prompts, m.eval(), images=images, max_tokens=7, temperature=0.0)
    full = [pr + t for pr, t in zip(prompts, toks)]
    imgs = [torch.tensor(im, dtype=torch.bfloat16) for ims in images for im in ims]
    om = V.MultimodalOracle(R.OracleTransformer(oracle_args(p, len(prompts)), FD.fp8_dense_checkpoint(sd)), p["vision_encoder"], imgs)
    _, o_lp = R.generate(full, om, max_tokens=0)
    worst = max(abs(a - b) for x, y in zip(lps, o_lp) for a, b in zip(x, y))
    print(f"[parity] fp8 dense {name} with images: logprob max|d|={worst:.4f}")
    assert worst <= LOGPROB_TOL, worst


def test_fp8_dense_regime_restatement_covers_every_family():
    fams = set()
    for c in OK_FAM + REAL8:
        r = fp8_regime(c.entry, c.T, c.N, c.K, dict(c.env), 132)
        fams.add(r.split("<")[0].lstrip("^"))
        m = re.search(r"gemm_wgmma_fp8_kernel<\d+, (\d+), (\d+)>", r)
        if m:
            fams.add(f"wgmma bn{m.group(1)} ta{m.group(2)}")
        m = re.search(r"gemm_streamk_fp8_kernel<\d+, (\d+)>", r)
        if m:
            fams.add(f"sk ta{m.group(1)}")
    for want in ("skinny_linear_kernel", "sk ta32", "sk ta64", "sk ta128", "wgmma bn128 ta128", "wgmma bn192 ta128", "wgmma bn256 ta128"):
        assert want in fams, (want, sorted(fams))
    assert REFUSED


# ----------------------------------------------------------------------------- the FP8 megakernel, bit for bit
# tests/test_gpu_megakernel_phases.py's designed step (every accumulation exact, every phase checked against the oracle on the
# kernel's own input), with each layer matrix stored in the FP8 format: a power-of-two row scale s and, for every designed value v
# at column c, e4m3(v / s) at c plus the e4m3 remainder lo = v / s - e4m3(v / s), moved to another column c' as lo * x[c] / x[c']
# (the inputs are signed powers of two, so the product and its grid are unchanged).  The
# kernel's sum over q is then matvec(design) / s exactly, and y = bf16(s * acc) is the bf16 design's y: check_step applies as is.
# The lm head stays bf16.
from . import test_gpu_megakernel_phases as MP  # noqa: E402


def split_e4m3(d: "MP.Design", x: torch.Tensor, gen: torch.Generator):
    """(Design over e4m3 values, fp32 row scales) with matvec(result, x) * scale == matvec(d, x) exactly.  Every input of the
    designs is a power of two with a sign, so the remainder of column c can sit at any other column c' as lo * x[c] / x[c']."""
    N, m = d.idx.shape
    # s = 1, 1/2 or 1/4 at random, or larger where the row's largest value would pass 240 (e4m3 rounds 240 to at most 256 < 448)
    room = torch.floor(torch.log2(240.0 / d.val.abs().amax(1).clamp_min(2.0 ** -20)))
    scale = torch.pow(2.0, -torch.minimum(room, torch.randint(0, 3, (N,), generator=gen).double()))
    v = d.val / scale[:, None]
    hi = v.float().to(torch.float8_e4m3fn).double()
    lo = v - hi
    assert MP.is_pow2(x).all(), "an input is not a power of two"
    idx2 = torch.zeros_like(d.idx)
    lo2 = torch.zeros_like(lo)
    need = torch.ones(N, m, dtype=torch.bool)
    for _ in range(1000):  # entries whose moved remainder is not an e4m3 value, or whose column is taken, draw again
        if not need.any():
            break
        r, j = torch.nonzero(need, as_tuple=True)
        pick = torch.randint(x.numel(), (len(r),), generator=gen)
        cand = lo[r, j] * x[d.idx[r, j]] / x[pick]
        idx2[r, j], lo2[r, j] = pick, cand
        need[r, j] = ~((cand.float().to(torch.float8_e4m3fn).double() == cand) & (cand.abs() <= 448))
        both = torch.cat([d.idx, idx2], 1)
        need |= (idx2[:, :, None] == both[:, None, :]).sum(2) > 1
    assert not need.any(), "no second columns found"
    return MP.Design(torch.cat([d.idx, idx2], 1), torch.cat([hi, lo2], 1)), scale.float()


class Step8(MP.Step):
    """MP.Step with e4m3 layer matrices, launched through decode_step_fp8."""

    def __init__(self, s, n_layers, pos, W, gen, **kw):
        super().__init__(s, n_layers, pos, W, gen, **kw)
        H, KV = s.H, s.KV
        q_dim, kv_dim = H * HD8, KV * HD8
        rows = []
        for l, lay in enumerate(self.layers):
            x_in = self.x0 if l == 0 else self.x_out[l - 1]
            xn = R.rms_norm(MP.bf(x_in)[None], MP.bf(lay["an"]), MP.EPS)[0].double()
            y = MP.bf(MP.matvec(lay["qkv"], xn))
            attn = y[q_dim + kv_dim:].view(KV, HD8).repeat_interleave(H // KV, 0).reshape(-1).double()
            h = MP.bf(MP.bf(MP.matvec(lay["wo"], attn)).double() + MP.bf(x_in).double())
            hn = R.rms_norm(h[None], MP.bf(lay["fn"]), MP.EPS)[0].double()
            pre = MP.bf(MP.matvec(lay["w13"], hn)).view(-1, 2)
            g = MP.bf(torch.nn.functional.silu(pre[:, 0]) * pre[:, 1]).double()
            ptrs = []
            scales = []
            for key, x, K in (("qkv", xn, s.dim), ("wo", attn, q_dim), ("w13", hn, s.dim), ("w2", g, s.hidden)):
                d8, sc = split_e4m3(lay[key], x, gen)
                assert MP.accumulation_exact(MP.products(d8, x)).all(), f"{key}: the e4m3 design is not exact"
                assert torch.equal(MP.matvec(d8, x) * sc.double(), MP.matvec(lay[key], x)), key
                qd = torch.zeros(d8.idx.shape[0], K, dtype=torch.uint8, device=DEV)
                qd.scatter_(1, d8.idx.to(DEV), e4m3_bytes(d8.val).to(DEV))
                sd = sc.to(DEV)
                self._keep += [qd, sd]
                ptrs.append(qd.data_ptr())
                scales.append(sd.data_ptr())
            dev = lay["dev"]
            rows.append(ptrs + dev[4:8] + scales)
        self.desc8 = torch.tensor(rows, dtype=torch.int64, device=DEV)

    def launch(self):
        s = self.s
        for off, n in ((self.sc.x, 2 * s.dim), (self.sc.h, s.dim), (self.sc.q, s.H * HD8), (self.sc.attn, s.H * HD8), (self.sc.g, s.hidden)):
            self.buf(off, n).fill_(NAN8)
        self.logits.fill_(NAN8)
        _abi.decode_step_fp8(self.desc8, self.win, self.L, self.emb, self.fn_dev, self.w_out, self.rope_dev, self.token, self.pos, 0,
                             self.logits, self.next, s.dim, s.hidden, s.H, s.KV, HD8, s.vocab, MP.EPS, self.ws)


HD8 = 128
NAN8 = float("nan")


def fp8_chunk_shapes():
    """e4m3 rows are cut into chunks of up to 8192: one full chunk (dim 8192, a 16 KB stage), 2 x 4128, 2 x 7168 (14336), 2 x 8192,
    3 x 8192; q_dim 8192 and 6144."""
    return [MP.Shape("K8192-24576", 8192, 24576, 16, 8, 256), MP.Shape("K4096-8256", 4096, 8256, 64, 8, 256),
            MP.Shape("K5120-16384", 5120, 16384, 48, 8, 256), MP.Shape("K4096-14336", 4096, 14336, 32, 8, 256)]


def fp8_cut_ok(K: int) -> bool:
    """Both cuts of K work: bf16 chunks of 8-element multiples (the lm head) and e4m3 chunks of 16-byte multiples."""
    nch8 = -(-K // 8192)
    return MP.cut_ok(K) and K % (nch8 * 16) == 0


def fp8_pair_shapes(G: int):
    """MP.pair_shapes with dim and hidden at the nearest values both cuts accept: pair counts at G - 4, G, G + 4, 8G +- 4 for wo /
    down (P = dim / 2), gate/up (P = hidden) and QKV; the lm head also at G +- 1, 8G + 1."""
    out = []
    dims = [MP.nearest(2 * p, [d for d in range(16, 20000, 16) if fp8_cut_ok(d)]) for p in MP.pair_targets(G)]
    hiddens = [MP.nearest(p, [h for h in range(16, 20000, 16) if fp8_cut_ok(h)]) for p in MP.pair_targets(G)]
    heads = [MP.QKV_HEADS[MP.nearest(p, list(MP.QKV_HEADS))] for p in MP.pair_targets(G)]
    vocabs = [2 * p for p in MP.pair_targets(G, lm=True)]
    for i, v in enumerate(vocabs):
        H, KV = heads[i % len(heads)]
        out.append(MP.Shape(f"pairs{i}", dims[i % len(dims)], hiddens[(i + 2) % len(hiddens)], H, KV, v))
    H, KV = MP.QKV_HEADS[min(p for p in MP.QKV_HEADS if p > 8 * G)]
    out.append(MP.Shape("pairs-trailing", dims[0], 8 * G + 16, H, KV, vocabs[0]))  # gate/up P = hidden just above 8G, 16-byte rows
    return out


def run_step8(s, n_layers: int, seed: int, pos: int = 37, W: int = 64, **kw):
    st = Step8(s, n_layers, pos, W, torch.Generator().manual_seed(seed), **kw)
    names = launched_kernels(st.launch)
    assert names == [f"decode_megakernel<{s.H // s.KV}, true>"], names
    out = st.read()
    MP.check_step(st, out, f"fp8 {s.name} L={n_layers}")


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["pairs", "chunks", "reps"])
def test_fp8_megakernel_exact_at_edges(which):
    G = _abi.device_info()[0]
    shapes = {"pairs": fp8_pair_shapes(G), "chunks": fp8_chunk_shapes(), "reps": MP.rep_shapes()}[which]
    assert len(shapes) >= 3
    for i, s in enumerate(shapes):
        run_step8(s, 1 + i % 3, seed=300 + i)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mistral-7b", "nemo-12b"])
@pytest.mark.parametrize("n_layers", [1, 2])
def test_fp8_megakernel_exact_real(name, n_layers):
    run_step8(MP.REAL[name], n_layers, seed=n_layers, pos=1000, W=4096, probes=False)
