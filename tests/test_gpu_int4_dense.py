"""INT4 dense weights on the GPU (include/mistral_b200.h).

* mb200_quantize_int4_groups equals the restatement of tests/int4_dense_ref.py bit for bit, at the format's edges and through the
  strided rows the loader writes (w1 / w3 into the interleaved w13 rows).
* The three INT4 entry points (mb200_attn_qkv_int4, mb200_ffn_gateup_int4, mb200_linear_residual_int4) bit for bit against an
  exact-by-construction float64 reference, in every regime their dispatch reaches -- GEMV (T <= 4), stream-K (TA 32 / 64 / 128),
  small wgmma, prefill wgmma (BN 128 / 192 / 256, single CTAs where bf16 runs clusters, the blocked walk) -- and every mode they
  serve, at the T, N, K edges of tests/test_gpu_linear_edges.py and at the 7B, Nemo and Mistral Large shapes.  The weights are
  codes in [-8, 7] times power-of-two group scales (so W' is the designed weight and every fp32 sum is exact, `exact_product`
  proves it), with all-zero groups (scale 1) and, for the plain Linears, rows whose scales are bf16 subnormals.  Every kernel
  switch gives the same bits, the launch log names the INT4 kernel, and a shape the bf16 path would give to mma.sync is refused.
* From 5 tokens on (stream-K and wgmma keep the bf16 kernels' tiles and k order) the INT4 entry points equal the bf16 entry
  points run on W' bit for bit, on random, inexact data.
* Models with dense_weights="int4": a first prefill of >= 128 tokens per sequence gives the bf16 model's logits on W' bit for bit
  (tiny, 2-layer 7B, 2-layer Mistral Large); chunked prefill, graph decode at B = 1, 3 and 8 and generate against the CPU
  restatement run on the W' checkpoint within the tolerance of tests/util.py; from_folder's peak memory.
"""
import re
from typing import Dict

import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer
from oracle import restatement as R

from . import int4_dense_ref as I4
from .test_gpu_linear_edges import (DEV, EPS, Case, Design, check_guards, check_values, design, exact_product, ints, qkv, reference,
                                    small_bn, w_scale)
from .test_gpu_moe_edges import assert_same, env
from .util import LOGPROB_TOL, launched_kernels, oracle_args

MODES = {"store": 0, "residual": 1, "swiglu": 3, "qkv": 4}
NORMED = {"store": False, "residual": False, "swiglu": True, "qkv": True}
BF16_NAN = 0x7FC0


# ----------------------------------------------------------------------------- the regime restatement
def int4_regime(entry: str, T: int, N: int, K: int, envd: Dict[str, str], sms: int) -> str:
    """Regex of the one kernel run_linear_int4 launches, or 'refused'."""
    mode = MODES[entry]
    if K % 128:
        return "refused"
    if T <= 4:
        return rf"^skinny_linear_kernel<{T}, {mode}, {'true' if NORMED[entry] else 'false'}, false, true>$"
    ta = 32 if T <= 32 else (64 if T <= 64 else 128)
    if envd.get("MB200_STREAMK", "1")[:1] != "0" and T <= 128 and N % 128 == 0:
        return rf"^gemm_streamk_int4_kernel<{mode}, {ta}>$"
    if not ((N % 128 == 0 or N % 192 == 0) if T >= 128 else N % 32 == 0):
        return "refused"
    if T < 128:
        return rf"^gemm_wgmma_int4_kernel<{mode}, {small_bn(N, sms, envd)}, {ta}>$"
    pair = envd.get("MB200_GEMM_CLUSTER", "1")[:1] != "0" and T >= 512
    units, m_units = (sms // 2, -(-(-(-T // 128)) // 2)) if pair else (sms, -(-T // 128))
    bn = 256
    if N % 256 or m_units * (N // 256) < units:
        bn = 128 if N % 128 == 0 else 192
    forced = int(envd.get("MB200_GEMM_BN", "0") or 0)
    if forced in (128, 192, 256) and N % forced == 0:
        bn = forced
    return rf"^gemm_wgmma_int4_kernel<{mode}, {bn}, 128>$"


def family_cases():
    out = []
    heads = {1024: (4, 2, 128), 2048: (8, 4, 128)}
    for i, e in enumerate(MODES):
        def mk(name, T, N, K, _e=e):
            return qkv(name, T, K, *heads[N]) if _e == "qkv" else Case(name, _e, T, N, K)

        # GEMV: every T; K / 32 below one unrolled round (1152: tail loop only) and past it (4224: one round + tail); partial CTA
        for T, K in ((1 + i % 4, 1152), (1 + (i + 2) % 4, 4224), (1 + (i + 1) % 4, 128), (1 + (i + 3) % 4, 2048)):
            out.append(Case(f"{e}-gemv-t{T}-k{K}", e, T, 1000, K) if e != "qkv" else qkv(f"{e}-gemv-t{T}-k{K}", T, K, 6, 1, 128))
        # stream-K at TA edges; a tile split by every CTA; one scale group (two k-blocks); fewer k-blocks than ring stages
        out.append(mk(f"{e}-sk-t5", 5, 1024, 512))
        out.append(mk(f"{e}-sk-t32-n128-k4096", 32, 128, 4096) if e != "qkv" else mk(f"{e}-sk-t32-k4096", 32, 1024, 4096))
        out.append(mk(f"{e}-sk-t33-k128", 33, 1024, 128))
        out.append(mk(f"{e}-sk-t64-k256", 64, 1024, 256))
        out.append(mk(f"{e}-sk-t65", 65, 1024, 768))
        out.append(mk(f"{e}-sk-t127", 127, 2048, 512))
        out.append(mk(f"{e}-sk-t128", 128, 1024, 1024))
        # prefill wgmma: 129 rows; BN 192 (N % 192 only); 511 rows; 512 / 513 rows, which bf16 runs as clusters
        out.append(mk(f"{e}-pf-t129", 129, 1024, 512))
        out.append(Case(f"{e}-pf-t200-n960", e, 200, 960, 512) if e != "qkv" else qkv(f"{e}-pf-t200-hd64", 200, 512, 5, 5, 64))
        out.append(mk(f"{e}-pf-t511", 511, 1024, 256))
        out.append(mk(f"{e}-pf-t512", 512, 1024, 256))
        out.append(Case(f"{e}-pf-t513-n4608", e, 513, 4608, 128) if e != "qkv" else qkv(f"{e}-pf-t513-hd64", 513, 128, 24, 24, 64))
        if e != "qkv":  # small-batch wgmma (N % 128 != 0), and the mma.sync shapes, refused
            out.append(Case(f"{e}-small-t40-n480", e, 40, 480, 512))
            out.append(Case(f"{e}-mma-t5", e, 5, 1000, 256))
            out.append(Case(f"{e}-mma-t300", e, 300, 1000, 384))
            out.append(Case(f"{e}-k320", e, 20, 1024, 320))
        else:
            out.append(qkv(f"{e}-small-t40-hd64", 40, 512, 3, 3, 64))
    off = (("MB200_GEMM_CLUSTER", "0"),)
    out += [Case("store-walk-t4100", "store", 4100, 2304, 128), Case("residual-walk-t2049", "residual", 2049, 3072, 128, off),
            Case("swiglu-walk-t8200", "swiglu", 8200, 1792, 128), qkv("qkv-walk-t4200", 4200, 256, 8, 2, 128)]
    return out


def real_cases():
    out = []
    shapes = {"mistral-7b": (4096, 32, 8, 14336), "nemo-12b": (5120, 32, 8, 14336), "mistral-large-2": (12288, 96, 8, 28672)}
    for name, (dim, H, KV, hidden) in shapes.items():
        for T in (1, 2, 4, 32, 129) if name == "mistral-large-2" else (3, 32, 1024):  # T = 2: x of 48 KB plus the reduction array
            out += [qkv(f"{name}-qkv-t{T}", T, dim, H, KV, 128), Case(f"{name}-wo-t{T}", "residual", T, dim, H * 128),
                    Case(f"{name}-gateup-t{T}", "swiglu", T, 2 * hidden, dim), Case(f"{name}-down-t{T}", "residual", T, dim, hidden)]
    return out


FAM = family_cases()
REAL4 = real_cases()
OK_FAM = [c for c in FAM if int4_regime(c.entry, c.T, c.N, c.K, dict(c.env), 132) != "refused"]
REFUSED = [c for c in FAM if int4_regime(c.entry, c.T, c.N, c.K, dict(c.env), 132) == "refused"]


# ----------------------------------------------------------------------------- designed inputs
def int4_design(c: Case, device, seed: int = 0):
    """(Design whose w = q * s exactly, q int [N, K] in -8..7, s float64 [N, K/128] powers of two).  x, norm weights, residuals and
    positions are test_gpu_linear_edges' design; every 97 rows, row 3 is all zero (scale 1, as the quantiser writes it) and, for
    the plain Linears, row 2 has bf16-subnormal scales."""
    d = design(c, device, seed)
    N, K = c.N, c.K
    gen = torch.Generator(device=device).manual_seed(seed + 13 * N + K)
    normed = NORMED[c.entry]
    e0 = w_scale(K, 1.6 if normed else 1.2, 12.0 if c.entry == "swiglu" else 3.0)
    q = ints(gen, (N, K), 7, device)
    rows, cols = torch.arange(N, device=device), torch.arange(K, device=device)
    q[(rows % 5 == 1)[:, None] & (cols % 13 == 4)[None, :]] = -8.0
    # powers of two computed on the CPU, where pow(2, -k) is exact
    s = pow2(-(e0 + torch.randint(0, 3, (N, K // 128), generator=gen, device=device)), device)
    if c.entry in ("store", "residual"):
        s[rows % 97 == 2] = pow2(-(126 + torch.randint(0, 5, (int((rows % 97 == 2).sum()), K // 128), generator=gen, device=device)), device)
    zero = rows % 97 == 3
    q[zero] = 0.0
    s[zero] = 1.0
    w = q * s.repeat_interleave(128, 1)
    return Design(d.x, d.nw, w, d.extra, d.positions), q, s


def pow2(e: torch.Tensor, device) -> torch.Tensor:
    out = torch.pow(2.0, e.cpu().double()).to(device)
    assert torch.equal(torch.frexp(out.cpu())[0].abs(), torch.full_like(out.cpu(), 0.5)), "a scale is not a power of two"
    return out


def pack_codes(q: torch.Tensor) -> torch.Tensor:
    return I4.pack(q.to(torch.int8).cpu()).to(DEV)


class Run4:
    """test_gpu_linear_edges.Run's inputs and outputs, with the weight as codes and scales followed by three guard rows whose
    scales are NaN."""

    def __init__(self, c: Case, d: Design, q: torch.Tensor, s: torch.Tensor):
        from .test_gpu_linear_edges import Run

        self.base = Run(c, d)
        self.c = c
        G = c.K // 128
        self.cbuf = torch.full((c.N + 3, c.K // 2), 0x77, dtype=torch.uint8, device=DEV)
        self.codes = self.cbuf[:c.N]
        self.codes.copy_(pack_codes(q))
        self.sbuf = torch.full((c.N + 3, G), BF16_NAN, dtype=torch.int16, device=DEV).view(torch.bfloat16)
        self.scales = self.sbuf[:c.N]
        self.scales.copy_(s.to(DEV).to(torch.bfloat16))
        assert torch.equal(self.scales.double(), s.to(DEV)), "a designed scale is not a bf16 value"
        self.extra = d.extra.to(torch.bfloat16).to(DEV).contiguous() if d.extra is not None else None

    def launch(self, envd: Dict[str, str]):
        c, b = self.c, self.base
        o = b.outputs()

        def call():
            if c.entry in ("store", "residual"):
                _abi.linear_residual_int4(b.x, self.codes, self.scales, self.extra, o["out"][1], b.ws)
            elif c.entry == "swiglu":
                _abi.ffn_gateup_int4(b.x, b.nw, self.codes, self.scales, o["out"][1], EPS, b.ws)
            else:
                H, KV, hd = c.heads
                _abi.attn_qkv_int4(b.x, b.nw, self.codes, self.scales, b.rope, b.positions, o["q"][1], o["k"][1], o["v"][1], o["ck"][1],
                                   o["cv"][1], b.rows, H, KV, hd, EPS, b.ws)

        with env(**{"MB200_STREAMK": "1", "MB200_GEMM_CLUSTER": "1", "MB200_GEMM_BN": "0", **envd}):
            names = launched_kernels(call)
        torch.cuda.synchronize()
        return names, o


def int4_variants(c: Case, sms: int):
    base = dict(c.env)
    seen = {int4_regime(c.entry, c.T, c.N, c.K, base, sms)}
    out = []
    cands = [{"MB200_STREAMK": "0"}] + [{"MB200_STREAMK": "0", "MB200_GEMM_BN": str(b)} for b in (32, 64, 128, 192, 256)]
    cands += [{"MB200_GEMM_CLUSTER": "0", "MB200_GEMM_BN": str(b)} for b in ("0", 128, 192, 256)]
    for v in cands:
        e = {**base, **v}
        r = int4_regime(c.entry, c.T, c.N, c.K, e, sms)
        if r not in seen and r != "refused":
            seen.add(r)
            out.append(e)
    return out


def run_case4(c: Case):
    sms = _abi.device_info()[0]
    dref = DEV if c.T * c.N * c.K > 2 ** 27 else "cpu"
    d, q, s = int4_design(c, DEV)
    xn = d.x * d.nw if d.nw is not None else d.x
    acc = exact_product(xn.to(dref), d.w.to(dref))
    want = reference(c, Design(*(t.to(dref) if t is not None else None for t in d)), acc)
    r = Run4(c, d, q, s)
    base = dict(c.env)
    names, o = r.launch(base)
    regime = int4_regime(c.entry, c.T, c.N, c.K, base, sms)
    assert len(names) == 1 and re.search(regime, names[0]), f"{c.name}: launched {names}, expected {regime}"
    check_guards(c, r.base, o, c.name)
    check_values(c, want, o, c.name)
    first = {k: v[1].clone() for k, v in o.items()}
    runs = int4_variants(c, sms)
    if "streamk" in regime:
        runs.append(base)  # stream-K flags reset themselves on the same workspace
    for e in runs:
        names, o = r.launch(e)
        reg = int4_regime(c.entry, c.T, c.N, c.K, e, sms)
        what = f"{c.name} {e}"
        assert len(names) == 1 and re.search(reg, names[0]), f"{what}: launched {names}, expected {reg}"
        check_guards(c, r.base, o, what)
        for k, v in first.items():
            assert_same(o[k][1], v, f"{what}: {k} vs the base run")


def test_int4_designs_are_exact_and_representable():
    """Host-side: q in -8..7, bf16 power-of-two scales, exact fp32 sums."""
    for c in [c for c in OK_FAM if c.T * c.N * c.K <= 2 ** 24][:16]:
        d, q, s = int4_design(c, "cpu")
        assert int(q.min()) >= -8 and int(q.max()) <= 7
        assert torch.equal(s.to(torch.bfloat16).double(), s)
        xn = d.x * d.nw if d.nw is not None else d.x
        exact_product(xn, d.w)


def test_int4_regime_restatement_covers_every_family():
    fams = set()
    for c in OK_FAM + REAL4:
        r = int4_regime(c.entry, c.T, c.N, c.K, dict(c.env), 132)
        fams.add(r.split("<")[0].lstrip("^"))
        m = re.search(r"gemm_wgmma_int4_kernel<\d+, (\d+), (\d+)>", r)
        if m:
            fams.add(f"wgmma bn{m.group(1)} ta{m.group(2)}")
        m = re.search(r"gemm_streamk_int4_kernel<\d+, (\d+)>", r)
        if m:
            fams.add(f"sk ta{m.group(1)}")
    for want in ("skinny_linear_kernel", "sk ta32", "sk ta64", "sk ta128", "wgmma bn128 ta128", "wgmma bn192 ta128", "wgmma bn256 ta128",
                 "wgmma bn32 ta64"):
        assert want in fams, (want, sorted(fams))
    assert REFUSED


@pytest.mark.gpu
@pytest.mark.parametrize("case", OK_FAM, ids=[c.name for c in OK_FAM])
def test_int4_linear_regimes(case):
    run_case4(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", REAL4, ids=[c.name for c in REAL4])
def test_int4_linear_real_shapes(case):
    run_case4(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", REFUSED, ids=[c.name for c in REFUSED])
def test_int4_linear_refuses(case):
    """mma.sync shapes, and K that would split a scale group, are refused before any kernel runs."""
    if case.K % 128 == 0:
        d, q, s = int4_design(case, DEV)
        r = Run4(case, d, q, s)
        with pytest.raises(_abi.Mb200Error, match="mma.sync"):
            r.launch({})
        return
    T, N, K = case.T, case.N, case.K
    codes = torch.zeros(N, K // 2, dtype=torch.uint8, device=DEV)
    scales = torch.ones(N, K // 128, dtype=torch.bfloat16, device=DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(T, K, 32, 8, 128, K, 0, 4), torch.device(DEV))
    with pytest.raises(_abi.Mb200Error, match="multiple of 128"):
        launched_kernels(lambda: _abi.linear_residual_int4(torch.zeros(T, K, dtype=torch.bfloat16, device=DEV), codes, scales, None,
                                                           torch.empty(T, N, dtype=torch.bfloat16, device=DEV), ws))


# ----------------------------------------------------------------------------- the quantiser
def quantiser_input(N: int, K: int, seed: int) -> torch.Tensor:
    """Random rows at magnitudes from 1e-38 to 1e30, plus the edges: ties at .5 of the step, a lone amax, -8 clamps (subnormal
    scales), all-zero and -0 groups, subnormal weights."""
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(N, K, generator=g, dtype=torch.float64) * torch.logspace(-38, 30, N, dtype=torch.float64)[:, None]
    w = w.to(torch.bfloat16)
    if N >= 8 and K >= 256:
        w[0, :128] = torch.tensor([7.0, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 3.5] + [0.0] * 120, dtype=torch.bfloat16)
        w[1, :128] = 0
        w[1, 5] = -3.0  # a group whose amax is its only non-zero value
        w[2, :128] = -0.0
        w[3, :128] = 0
        w[3, 0], w[3, 1] = 9.8 * 2.0 ** -133, -9.8 * 2.0 ** -133  # subnormal scale: 7 and the -8 clamp
        w[4, :128] = torch.tensor([2.0 ** -133] + [0.0] * 127, dtype=torch.bfloat16)  # amax / 7 rounds to 0: the smallest scale
        w[5, 128:256] = (torch.arange(128, dtype=torch.float64) - 64).to(torch.bfloat16) * 2.0 ** -140  # subnormal weights
    return w


@pytest.mark.gpu
@pytest.mark.parametrize("N,K", [(16, 128), (16, 384), (12, 4096), (6, 28672)])
def test_quantiser_matches_the_restatement(N, K):
    w = quantiser_input(N, K, K)
    codes = torch.empty(N, K // 2, dtype=torch.uint8, device=DEV)
    s = torch.empty(N, K // 128, dtype=torch.bfloat16, device=DEV)
    names = launched_kernels(lambda: _abi.quantize_int4_groups(w.to(DEV), codes, s))
    assert names == ["quantize_int4_groups_kernel"], names
    rc, rs = I4.quantize(w)
    assert torch.equal(s.cpu().view(torch.int16), rs.view(torch.int16))
    assert torch.equal(codes.cpu(), rc)


@pytest.mark.gpu
def test_quantiser_strided_rows_fill_the_interleaved_w13():
    h, d = 96, 512
    w1, w3 = quantiser_input(h, d, 1), quantiser_input(h, d, 2)
    w13 = torch.full((2 * h, d // 2), 0xAB, dtype=torch.uint8, device=DEV)
    g13 = torch.full((2 * h, d // 128), 0x5555, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    for seg, w in ((0, w1), (1, w3)):
        _abi.quantize_int4_groups(w.to(DEV), w13.view(h, 2, d // 2)[:, seg], g13.view(h, 2, d // 128)[:, seg])
    for seg, w in ((0, w1), (1, w3)):
        rc, rs = I4.quantize(w)
        assert torch.equal(w13.view(h, 2, d // 2)[:, seg].cpu(), rc)
        assert torch.equal(g13.view(h, 2, d // 128)[:, seg].cpu().view(torch.int16), rs.view(torch.int16))


# ----------------------------------------------------------------------------- against the bf16 entry points on W'
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["residual", "swiglu", "qkv"])
@pytest.mark.parametrize("T", [5, 32, 100, 128, 129, 600, 4096])
def test_int4_equals_bf16_on_w_prime(entry, T):
    """Random bf16 data (no exactness): the INT4 entry point and the bf16 one on W' give the same bits wherever INT4 keeps the bf16
    tiles and k order (stream-K, small and prefill wgmma; the bf16 prefill's clusters and the INT4 single CTAs sum a tile alike)."""
    g = torch.Generator(device=DEV).manual_seed(T)
    dim, H, KV, hidden = 1024, 8, 2, 1536
    N, K = {"residual": (dim, hidden), "swiglu": (2 * hidden, dim), "qkv": ((H + 2 * KV) * 128, dim)}[entry]
    w = (torch.randn(N, K, generator=g, device=DEV) * 0.03).to(torch.bfloat16)
    codes = torch.empty(N, K // 2, dtype=torch.uint8, device=DEV)
    s = torch.empty(N, K // 128, dtype=torch.bfloat16, device=DEV)
    _abi.quantize_int4_groups(w, codes, s)
    wp = I4.dequantize(codes.cpu(), s.cpu()).to(DEV)
    x = torch.randn(T, K, generator=g, device=DEV).to(torch.bfloat16)
    nw = (1 + 0.1 * torch.randn(K, generator=g, device=DEV)).to(torch.bfloat16)
    ws = _abi.Workspace(_abi.workspace_bytes(T, K, 32, 8, 128, K, 0, 4), torch.device(DEV))
    outs = []
    for int4 in (True, False):
        if entry == "residual":
            res = torch.randn(T, N, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV).to(torch.bfloat16)
            out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
            if int4:
                _abi.linear_residual_int4(x, codes, s, res, out, ws)
            else:
                _abi.linear_residual(x, wp, res, out, ws)
            outs.append([out])
        elif entry == "swiglu":
            out = torch.empty(T, hidden, dtype=torch.bfloat16, device=DEV)
            if int4:
                _abi.ffn_gateup_int4(x, nw, codes, s, out, EPS, ws)
            else:
                _abi.ffn_gateup(x, nw, wp, out, EPS, ws)
            outs.append([out])
        else:
            from mistral_inference_b200.rope import precompute_freqs_cis
            rope = torch.view_as_real(precompute_freqs_cis(128, 4096, 1e6)).contiguous().to(DEV)
            pos = torch.arange(T, dtype=torch.int32, device=DEV) % 4096
            q = torch.empty(T, H * 128, dtype=torch.bfloat16, device=DEV)
            k = torch.empty(T, KV * 128, dtype=torch.bfloat16, device=DEV)
            v = torch.empty(T, KV * 128, dtype=torch.bfloat16, device=DEV)
            if int4:
                _abi.attn_qkv_int4(x, nw, codes, s, rope, pos, q, k, v, None, None, None, H, KV, 128, EPS, ws)
            else:
                _abi.attn_qkv(x, nw, wp, rope, pos, q, k, v, None, None, None, H, KV, 128, EPS, ws)
            outs.append([q, k, v])
    torch.cuda.synchronize()
    for a, b in zip(*outs):
        assert_same(a, b, f"{entry} T={T}: int4 vs bf16 on W'")


# ----------------------------------------------------------------------------- models
def int4_model(p: dict, max_batch: int, seed: int = 1, dense_weights: str = "int4"):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, DEV, torch.bfloat16, dense_weights=dense_weights)
    sd = synth.synth_state_dict(p, seed, torch.bfloat16, DEV)
    m.load_state_dict(sd if dense_weights == "int4" else I4.int4_dense_checkpoint({k: v.cpu() for k, v in sd.items()}))
    return m.eval(), sd


@pytest.mark.gpu
def test_loader_quantises_like_the_restatement():
    p = synth.shape("tiny")
    m, sd = int4_model(p, 1)
    msd = m.state_dict()
    for k, v in sd.items():
        if I4.is_dense_key(k):
            rc, rs = I4.quantize(v.cpu())
            base = k[: -len(".weight")]
            assert torch.equal(msd[base + ".weight_int4"].cpu(), rc), k
            assert torch.equal(msd[base + ".weight_gscale"].cpu().view(torch.int16), rs.view(torch.int16)), k


@pytest.mark.gpu
@pytest.mark.parametrize("shape,over,lens", [
    ("tiny", {}, [200, 130]),
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [300, 128]),
    ("mistral-large-2", {"n_layers": 2, "vocab_size": 4096}, [160]),
])
def test_first_prefill_equals_the_bf16_model_on_w_prime(shape, over, lens):
    """A first prefill of >= 128 tokens per sequence: every layer Linear runs a wgmma kernel whose tiles are W', so the INT4
    model's logits are the bf16 model's on the W' checkpoint, bit for bit."""
    p = synth.shape(shape, **over)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 7 + i) for i, n in enumerate(lens)]
    flat = torch.tensor(sum(prompts, []), device=DEV)
    logits = {}
    for fmt in ("int4", "bf16"):
        m, _ = int4_model(p, len(lens), dense_weights=fmt)
        from mistral_inference_b200.cache import BufferCache
        cache = BufferCache(m.n_local_layers, len(lens), max(lens) + 4, m.args.n_kv_heads, m.args.head_dim).to(m.device, m.dtype)
        cache.reset()
        names = launched_kernels(lambda: logits.setdefault(fmt, m.forward(flat, lens, cache)))
        if fmt == "int4":
            assert any(n.startswith("gemm_wgmma_int4_kernel") for n in names) and not any("skinny" in n or "streamk" in n for n in names)
        del m
        torch.cuda.empty_cache()
    assert torch.equal(logits["int4"], logits["bf16"])


def oracle_for(p: dict, sd, max_batch: int):
    return R.OracleTransformer(oracle_args(p, max_batch), I4.int4_dense_checkpoint({k: v.cpu() for k, v in sd.items()}))


def run_against_oracle(m, om, p, tag, lens, chunk, steps=4):
    """Prefill (in chunks) and `steps` decode steps of m against om, teacher-forced on the oracle's picks; returns the kernel
    families the decode steps launched."""
    from mistral_inference_b200.cache import BufferCache

    from .test_gpu_model import check_rows, report

    B = len(lens)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate(lens)]
    cache = BufferCache(m.n_local_layers, m.args.max_batch_size, max(lens) + steps + 2, m.args.n_kv_heads, m.args.head_dim,
                        m.args.sliding_window).to(m.device, m.dtype)
    cache.reset()
    ocache = om.new_cache(max(lens) + steps + 2)
    step_chunk = chunk or max(lens)
    for s0 in range(0, max(lens), step_chunk):
        chunks = [pr[s0:s0 + step_chunk] for pr in prompts]
        sl = [len(c) for c in chunks]
        flat = torch.tensor(sum(chunks, []))
        got = m.forward(flat.cuda(), sl, cache)
        want = om.forward(flat, sl, ocache)
        check_rows(report(f"{tag} prefill @{s0}", got, want), want, None, f"{tag} prefill @{s0}")
        nxt = want[torch.tensor(sl).cumsum(0) - 1].argmax(-1)
    kinds = set()
    for step in range(steps):
        out = {}
        names = launched_kernels(lambda: out.setdefault("logits", m.forward(nxt.cuda(), [1] * B, cache)))
        kinds |= {n.split("<")[0] for n in names}
        want = om.forward(nxt, [1] * B, ocache)
        check_rows(report(f"{tag} decode {step}", out["logits"], want), want, None, f"{tag} decode {step}")
        nxt = want.argmax(-1)
    return kinds


@pytest.mark.gpu
@pytest.mark.parametrize("shape,over,lens,chunk", [
    ("tiny", {}, [11, 9, 14], 4),                                                   # chunked prefill, graph decode B = 3
    ("tiny", {"sliding_window": 5}, [11, 9, 10, 7, 12, 8, 9, 10], None),           # B = 8
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [200], 128),                # B = 1: the graph path, no megakernel
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [40 - (b % 3) for b in range(8)], None),
    ("mistral-large-2", {"n_layers": 2, "vocab_size": 4096}, [150], 64),         # H/KV = 12: chunked prefill, B = 1 graph decode
    ("mistral-large-2", {"n_layers": 2, "vocab_size": 4096}, [20 - (b % 3) for b in range(8)], None),  # B = 8
])
def test_int4_model_vs_oracle(shape, over, lens, chunk):
    p = synth.shape(shape, **over)
    m, sd = int4_model(p, len(lens))
    kinds = run_against_oracle(m, oracle_for(p, sd, len(lens)), p, f"int4 {shape}{over}", lens, chunk)
    # the layer Linears run INT4 kernels (the lm head its bf16 one), batch 1 included: no megakernel, nothing on mma.sync
    assert "decode_megakernel" not in kinds and "gemm_mma_kernel" not in kinds, kinds
    assert kinds & {"skinny_linear_kernel", "gemm_streamk_int4_kernel", "gemm_wgmma_int4_kernel"}, kinds


@pytest.mark.gpu
def test_int4_generate_vs_oracle():
    p = synth.shape("mistral-7b", n_layers=2, vocab_size=4096)
    m, sd = int4_model(p, 3)
    om = oracle_for(p, sd, 3)
    prompts = [synth.synth_prompt(n, p["vocab_size"], 5 + i) for i, n in enumerate((40, 33, 37))]
    for ps in (prompts, prompts[:1]):
        toks, lp = mi.generate(ps, m, max_tokens=6, temperature=0.0, chunk_size=16)
        full = [pr + t for pr, t in zip(ps, toks)]
        _, olp = R.generate(full, om, max_tokens=0, chunk_size=16)
        worst = max(abs(a - b) for x, y in zip(lp, olp) for a, b in zip(x, y))
        print(f"[parity] int4 dense generate B={len(ps)}: logprob max|d|={worst:.4f}")
        assert worst <= LOGPROB_TOL


@pytest.mark.gpu
def test_from_folder_peak_is_the_int4_model_plus_one_tensor(tmp_path):
    p = synth.shape("mistral-7b", n_layers=8)
    synth.write_model_folder(tmp_path, p, seed=2)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = Transformer.from_folder(tmp_path, device=DEV, dense_weights="int4")
    torch.cuda.synchronize()
    held = torch.cuda.memory_allocated() - base
    peak = torch.cuda.max_memory_allocated() - base
    model = sum(t.numel() * t.element_size() for t in m.parameters())
    biggest = 2 * max(p["dim"] * p["hidden_dim"], p["vocab_size"] * p["dim"])  # one bf16 tensor of the checkpoint
    print(f"from_folder int4 8-layer 7B: model {model / 1e9:.3f} GB, held {held / 1e9:.3f} GB, peak {peak / 1e9:.3f} GB")
    assert held <= model * 1.01 + (64 << 20)
    assert peak <= model + biggest + (64 << 20), (peak, model, biggest)
    assert m.layers["0"].attention.wqkv.dtype == torch.uint8
