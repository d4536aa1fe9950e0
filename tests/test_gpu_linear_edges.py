"""The dense Linears outside the batch-1 megakernel (csrc/abi.cu: run_linear and the five entry points on it), bit for bit, in
every GEMM regime and pair epilogue, at the T, N, K and tile-walk edges.

Regimes (the host's own switches, restated by `dense_regime` below and asserted from the launch log in every GPU test):
  GEMV          T <= 4: skinny_linear_kernel<T, MODE, NORM> (RMSNorm in-kernel when the entry point norms)
  stream-K      5 <= T <= 128, N % 128 == 0, K % 64 == 0, MB200_STREAMK not 0: gemm_streamk_kernel<MODE, TA>, TA 32 / 64 / 128
  small wgmma   T < 128 otherwise, N % 32 == 0: gemm_wgmma_kernel<MODE, 1, BN, TA>, BN from the fill score or MB200_GEMM_BN
  prefill wgmma T >= 128, N % 128 == 0 or N % 192 == 0: gemm_wgmma_kernel<MODE, 1, BN, 128>, BN 128 / 192 / 256; m-fastest walk,
                or the 12 x 12 blocked walk past 16 m tiles
  2-CTA cluster the same with T >= 512 and MB200_GEMM_CLUSTER not 0: gemm_wgmma_kernel<MODE, 2, BN, 128>; 8 x 9 blocked walk past
                16 tile pairs
  mma.sync      anything else with K % 64 == 0: gemm_mma_kernel<MODE>
Normed entry points (lm_head, ffn_gateup, attn_qkv) run rmsnorm_kernel into the workspace first when T > 4.

Exact by construction.  x holds +-2^a (a in -1, 0, 1), or +-1 where the entry point norms (bf16(x * rsqrt(1 + eps)) = x, so the
GEMM sees x * norm_w exactly, norm_w small integers); W holds small integers * 2^-s.  `matmul_exact` proves on the host, for every
output, that the fp32 sum is exact in any order, so a correct kernel can differ from the float64 reference only at the rounding
points its epilogue declares (csrc/epilogue.cuh), and those are emulated in IEEE float32 (numpy on the host; torch float32
element-wise ops, one rounding per op, on the device for big shapes):
  STORE     bf16(acc)                       RESIDUAL  bf16(bf16(acc) + r)          F32   float(bf16(acc))
  BIAS      bf16(acc + b)                   BIAS+GELU bf16(gelu(bf16(acc + b)))    SWIGLU bf16(bf16(silu(bf16(a0))) * bf16(a1))
  QKV+RoPE  re = a*c - b*d, im = a*d + b*c with every product rounded (no FMA), cos/sin from the fp32 table, ring scatter
STORE, F32, RESIDUAL, BIAS and QKV must match on every element.  expf and erff are not correctly rounded, so SWIGLU and GELU are
certified as in test_gpu_moe_edges.py: an element whose float64 value is more than 2^-16 relative away from a bf16 rounding
boundary (and, for GELU, whose input is >= -2, where 1 + erf keeps erff's absolute error small in relative terms) must match
exactly, at least 99 % of the elements are certified, and the rest must be within one ulp.  In the QKV design the first four
tokens are coded by a 4 x 4 Hadamard sign pattern on eight columns that only the first q head and the first k head read, which
puts (y0, y1) = `fma_sensitive_pairs` of the token's position on every pair of those heads: a contracted multiply-add changes
their bits.

RMSNorm's own arithmetic is checked through *selection weights* (one power of two per W row): logits[t, n] is one normed input
element, so the norm's bits show in every regime; its float32 chain is emulated and tied to oracle.restatement.rms_norm.

Guards: every output (q / k / v, ring, g, logits, out) is NaN-filled with three guard rows, which must stay NaN, as must ring rows
that cache_rows does not name; x and W are views of NaN-padded buffers.  Every case also runs with every switch that changes its
kernel (MB200_STREAMK=0, each MB200_GEMM_BN, MB200_GEMM_CLUSTER=0): each variant must give the same bits.  A stream-K case runs
again after its variants on the same workspace, so its flags must have reset themselves.
"""
import math
import re
from functools import lru_cache
from typing import Dict, NamedTuple, Optional, Tuple

import numpy as np
import pytest
import torch

from mistral_inference_b200 import _abi
from mistral_inference_b200.rope import precompute_freqs_cis
from oracle import restatement as R

from .test_gpu_megakernel_phases import SILU_A, accumulation_exact, fma_sensitive_pairs, lsb_exponent
from .test_gpu_moe_edges import assert_same, bf16r, certain, env, matmul_exact, same
from .util import bf16_ulp_diff, launched_kernels

DEV = "cuda"
NAN = float("nan")
EPS = 1e-5
GUARD = 3                      # NaN rows after every output and input
SKINNY_MAX_T = 4               # MB200_SKINNY_MAX_T
KGM, KGN = {1: 12, 2: 8}, {1: 12, 2: 9}  # blocked walk: m units x n tiles per block, single CTA / cluster pair
ROPE_LEN = 4096
THETA = 1e6
# entry point -> (epilogue mode, norms its input)
ENTRIES = {"store": (0, False), "residual": (1, False), "f32": (2, True), "swiglu": (3, True), "qkv": (4, True), "bias": (6, False),
           "gelu": (7, False)}
GELU_MIN = -2.0                # GELU inputs below this are never certified
H4 = torch.tensor([[1, 1, 1, 1], [1, -1, 1, -1], [1, 1, -1, -1], [1, -1, -1, 1]], dtype=torch.float64)
CODE_POS = (ROPE_LEN - 1, 1, 2047, 333)  # positions of the four coded tokens (the table's last row first)


# ----------------------------------------------------------------------------- the regime restatement
def _off(envd: Dict[str, str], key: str) -> bool:
    return envd.get(key, "1")[:1] == "0"


def small_bn(N: int, sms: int, envd: Dict[str, str]) -> int:
    """wgmma_small_bn: MB200_GEMM_BN when it divides N, else the fullest rounds of N / BN tiles over the SMs (halved below half
    the SMs), wider tiles on ties."""
    forced = int(envd.get("MB200_GEMM_BN", "0") or 0)
    if forced in (32, 64, 128, 256) and N % forced == 0:
        return forced
    best, best_score = 0, -1.0
    for bn in (256, 128, 64, 32):
        if N % bn:
            continue
        tiles = N // bn
        score = tiles / (-(-tiles // sms) * sms)
        if tiles < sms // 2:
            score *= 0.5
        if score > best_score + 1e-9:
            best, best_score = bn, score
    return best


def dense_regime(entry: str, T: int, N: int, K: int, envd: Dict[str, str], sms: int) -> str:
    """Regex of the one kernel run_linear launches (rmsnorm_kernel, which the normed entry points run first for T > 4, is not
    in the launch log)."""
    mode, normed = ENTRIES[entry]
    if T <= SKINNY_MAX_T:
        return rf"^skinny_linear_kernel<{T}, {mode}, {'true' if normed else 'false'}>$"
    ta = 32 if T <= 32 else (64 if T <= 64 else 128)
    if not _off(envd, "MB200_STREAMK") and T <= 128 and N % 128 == 0 and K % 64 == 0:
        return rf"^gemm_streamk_kernel<{mode}, {ta}>$"
    wgmma = K % 64 == 0 and ((N % 128 == 0 or N % 192 == 0) if T >= 128 else N % 32 == 0)
    if not wgmma:
        return rf"^gemm_mma_kernel<{mode}>$"
    if T < 128:
        return rf"^gemm_wgmma_kernel<{mode}, 1, {small_bn(N, sms, envd)}, {ta}>$"
    pair = not _off(envd, "MB200_GEMM_CLUSTER") and T >= 512
    units = sms // 2 if pair else sms
    m_units = -(-(-(-T // 128)) // 2) if pair else -(-T // 128)
    bn = 256
    if N % 256 or m_units * (N // 256) < units:
        bn = 128 if N % 128 == 0 else 192
    forced = int(envd.get("MB200_GEMM_BN", "0") or 0)
    if forced in (128, 192, 256) and N % forced == 0:
        bn = forced
    return rf"^gemm_wgmma_kernel<{mode}, {2 if pair else 1}, {bn}, 128>$"


def family(regime: str) -> str:
    if regime.startswith("^skinny"):
        return "gemv"
    if regime.startswith("^gemm_streamk"):
        return "streamk"
    if regime.startswith("^gemm_mma"):
        return "mma"
    cl, ta = re.search(r"<\d+, (\d), \d+, (\d+)>", regime).groups()
    return "cluster" if cl == "2" else ("prefill" if ta == "128" else "small")


def walk(regime: str, T: int, N: int) -> str:
    """The tile walk of a prefill / cluster launch (tile_mn in gemm_wgmma.cuh): 'm-fastest', or 'blocked' (+ ' ragged' when
    the last m block or n block is partial)."""
    m = re.search(r"<\d+, (\d), (\d+), 128>", regime)
    if m is None:
        return "-"
    cl, bn = int(m.group(1)), int(m.group(2))
    num_m = -(-(-(-T // 128)) // cl)
    if num_m <= 16:
        return "m-fastest"
    return "blocked" + (" ragged" if num_m % KGM[cl] or (N // bn) % KGN[cl] else "")


# ----------------------------------------------------------------------------- the cases
class Case(NamedTuple):
    name: str
    entry: str
    T: int
    N: int                                  # the GEMM's N (2 hidden for swiglu, (H + 2 KV) hd for qkv)
    K: int
    env: Tuple[Tuple[str, str], ...] = ()
    heads: Optional[Tuple[int, int, int]] = None  # qkv: (H, KV, head_dim)
    bias: bool = True                       # bias / gelu: with the bias vector, or null


def qkv(name, T, K, H, KV, hd, envt=()):
    return Case(name, "qkv", T, (H + 2 * KV) * hd, K, envt, (H, KV, hd))


def family_cases():
    """Every family for every entry point that can reach it, at small shapes."""
    out = []
    qkv_heads = {1024: (4, 2, 128), 2048: (8, 4, 128), 128: (2, 2, 64), 1000: (6, 1, 128)}  # (H, KV, hd) -> N 1024, 2048, 384, 1024

    for i, e in enumerate(ENTRIES):
        def mk(name, T, N, K, _e=e):
            return qkv(name, T, K, *qkv_heads[N]) if _e == "qkv" else Case(name, _e, T, N, K)

        # GEMV: every T, K / 8 not a multiple of 128 (the tail loop), a partial last CTA (N / 16 not whole)
        for T, K in ((1 + i % 4, 1088), (1 + (i + 2) % 4, 4160)):
            out.append(mk(f"{e}-gemv-t{T}-k{K}", T, 1000, K))
        # stream-K: TA 32 / 64 / 128 at their edges; one 128-wide tile split by every CTA (qkv: three); one k-block; fewer
        # k-blocks than ring stages
        out.append(mk(f"{e}-sk-t5-n1024", 5, 1024, 512))
        out.append(mk(f"{e}-sk-t32-n128-k4096", 32, 128, 4096))
        out.append(mk(f"{e}-sk-t33-k64", 33, 1024, 64))
        out.append(mk(f"{e}-sk-t64-k128", 64, 1024, 128))
        out.append(mk(f"{e}-sk-t65", 65, 1024, 768))
        out.append(mk(f"{e}-sk-t127", 127, 2048, 512))
        out.append(mk(f"{e}-sk-t128", 128, 1024, 1024))
        # prefill wgmma (single CTA): N % 192 == 0 only (BN 192), odd / even m-tile counts, 511 rows
        out.append(mk(f"{e}-pf-t129", 129, 1024, 512))
        out.append(Case(f"{e}-pf-t200-n960", e, 200, 960, 512) if e != "qkv" else qkv(f"{e}-pf-t200-hd64", 200, 512, 5, 5, 64))
        out.append(mk(f"{e}-pf-t511", 511, 1024, 256))
        # 2-CTA cluster: 512 / 513 rows, a ragged pair
        out.append(mk(f"{e}-cl-t512", 512, 1024, 256))
        out.append(Case(f"{e}-cl-t513-n4608", e, 513, 4608, 128) if e != "qkv" else qkv(f"{e}-cl-t513-hd64", 513, 128, 24, 24, 64))
        # mma.sync: N % 32 != 0 below 128 rows, N % 128 != 0 and N % 192 != 0 above (n-tile tail)
        if e != "qkv":
            out.append(Case(f"{e}-mma-t5", e, 5, 1000, 256))
            out.append(Case(f"{e}-mma-t100", e, 100, 1000, 192))
            out.append(Case(f"{e}-mma-t300", e, 300, 1000, 320))
        else:  # head_dim 64 with H = KV odd: N % 128 == 64, the small-batch wgmma instead of stream-K
            out.append(qkv(f"{e}-small-t40-hd64", 40, 512, 3, 3, 64))
    # the blocked walks: single CTA at 2048 / 2049 / 3072 rows (cluster off), the cluster past 4096 rows, ragged and whole blocks
    off = (("MB200_GEMM_CLUSTER", "0"),)
    out += [Case("store-walk-t2048", "store", 2048, 3072, 128, off), Case("residual-walk-t2049", "residual", 2049, 3072, 128, off),
            Case("bias-walk-t3072", "bias", 3072, 3072, 64, off), Case("f32-walk-t2049-n2816", "f32", 2049, 2816, 128, off),
            Case("swiglu-walk-t2300", "swiglu", 2300, 2816, 64, off), Case("gelu-walk-t2100", "gelu", 2100, 1920, 64, off),
            qkv("qkv-walk-t2200", 2200, 128, 16, 4, 128, off),
            Case("residual-walk-t8200", "residual", 8200, 2560, 256), Case("store-walk-t8192", "store", 8192, 2304, 128),
            Case("swiglu-walk-t8200", "swiglu", 8200, 1792, 128), Case("f32-walk-t4224", "f32", 4224, 2304, 64),
            qkv("qkv-walk-t8200", 8200, 256, 8, 2, 128), Case("gelu-walk-t4500", "gelu", 4500, 1536, 64),
            Case("bias-walk-t5000-nobias", "bias", 5000, 2560, 64, bias=False)]
    out.append(Case("bias-sk-nobias", "bias", 20, 1024, 256, bias=False))
    out.append(Case("gelu-mma-nobias", "gelu", 300, 1000, 128, bias=False))
    return out


def real_cases():
    """Every dense Linear of the BASELINE configs at a decode batch and a prefill chunk (QKV, wo, gate/up, down, lm head at the
    row blocks forward_logprobs uses: max(128, 256 MiB / (4 V)))."""
    out = []
    shapes = {"mistral-7b": (4096, 32, 8, 14336, 32000), "nemo-12b": (5120, 32, 8, 14336, 131072)}
    for name, (dim, H, KV, hidden, V) in shapes.items():
        for T in (3, 32, 1024):
            out += [qkv(f"{name}-qkv-t{T}", T, dim, H, KV, 128), Case(f"{name}-wo-t{T}", "residual", T, dim, H * 128),
                    Case(f"{name}-gateup-t{T}", "swiglu", T, 2 * hidden, dim), Case(f"{name}-down-t{T}", "residual", T, dim, hidden)]
        out.append(Case(f"{name}-lm-t{max(128, (256 << 20) // (4 * V))}", "f32", max(128, (256 << 20) // (4 * V)), V, dim))
        out.append(Case(f"{name}-lm-t32", "f32", 32, V, dim))
    for T in (32, 1024):  # Mixtral-8x22B dense parts: dim 6144, QKV N 8192; an expert-shaped K = 16384 down projection
        out += [qkv(f"mixtral-8x22b-qkv-t{T}", T, 6144, 48, 8, 128), Case(f"mixtral-8x22b-wo-t{T}", "residual", T, 6144, 6144),
                Case(f"mixtral-8x22b-down-k16384-t{T}", "residual", T, 6144, 16384)]
    out.append(Case("mixtral-8x22b-lm-t2048", "f32", 2048, 32768, 6144))
    return out


CASES = family_cases()
REAL = real_cases()


def variants(c: Case, sms: int):
    """The switches that change this case's kernel, each once: MB200_STREAMK=0, every MB200_GEMM_BN (with stream-K off below 128
    rows), MB200_GEMM_CLUSTER=0 (with every BN)."""
    base = dict(c.env)
    seen = {dense_regime(c.entry, c.T, c.N, c.K, base, sms)}
    out = []
    cands = [{"MB200_STREAMK": "0"}] + [{"MB200_STREAMK": "0", "MB200_GEMM_BN": str(b)} for b in (32, 64, 128, 192, 256)]
    cands += [{"MB200_GEMM_CLUSTER": "0", "MB200_GEMM_BN": str(b)} for b in ("0", 128, 192, 256)]
    cands += [{"MB200_GEMM_BN": str(b)} for b in (128, 192, 256)]
    for v in cands:
        e = {**base, **v}
        r = dense_regime(c.entry, c.T, c.N, c.K, e, sms)
        if r not in seen:
            seen.add(r)
            out.append(e)
    return out


# ----------------------------------------------------------------------------- designed inputs
def ints(gen, shape, lim, device):
    return torch.randint(-lim, lim + 1, shape, generator=gen, device=device).double()


def pm_pow2(gen, shape, device):
    a = torch.randint(-1, 2, shape, generator=gen, device=device).double()
    s = torch.randint(0, 2, shape, generator=gen, device=device).double() * 2 - 1
    return s * torch.pow(2.0, a)


def w_scale(K: int, x_rms: float, target: float) -> int:
    """2^-s for integer weights in [-7, 7] (rms 4.32) that puts a K-long dot product near +-target."""
    return max(0, round(math.log2(math.sqrt(K) * x_rms * 4.32 / target)))


class Design(NamedTuple):
    x: torch.Tensor                # [T, K] float64: the entry point's input
    nw: Optional[torch.Tensor]     # [K] float64 norm weight (normed entry points)
    w: torch.Tensor                # [N, K] float64
    extra: Optional[torch.Tensor]  # residual [T, N] / bias [N] (float64), or None
    positions: Optional[torch.Tensor] = None  # qkv: [T] int64


@lru_cache(maxsize=None)
def rope_table(hd: int) -> torch.Tensor:
    return precompute_freqs_cis(hd, ROPE_LEN, THETA)


@lru_cache(maxsize=None)
def sensitive(hd: int, pos: int) -> Dict[int, Tuple[int, int]]:
    """fma_sensitive_pairs at a position of the hd-wide table (the helper walks 64 frequencies: a 64-wide table is doubled)."""
    tab = rope_table(hd)
    pairs = fma_sensitive_pairs(pos, tab if hd == 128 else torch.cat([tab, tab], 1))
    return {i: p for i, p in pairs.items() if i < hd // 2}


def code_targets(hd: int) -> torch.Tensor:
    """[4, hd]: row j holds (y0, y1) = the FMA-sensitive pair of every frequency at CODE_POS[j] ((3, -5) where there is none)."""
    y = torch.empty(4, hd, dtype=torch.float64)
    for j, pos in enumerate(CODE_POS):
        s = sensitive(hd, pos)
        for i in range(hd // 2):
            y[j, 2 * i], y[j, 2 * i + 1] = s.get(i, (3, -5))
    return y


def design(c: Case, device, seed: int = 0) -> Design:
    T, N, K = c.T, c.N, c.K
    gen = torch.Generator(device=device).manual_seed(seed + 7919 * T + 31 * N + K)
    mode, normed = ENTRIES[c.entry]
    if normed:
        x = torch.randint(0, 2, (T, K), generator=gen, device=device).double() * 2 - 1
        nw = torch.randint(1, 3, (K,), generator=gen, device=device).double() * (torch.randint(0, 2, (K,), generator=gen, device=device).double() * 2 - 1)
        x_rms = 1.6
    else:
        x, nw, x_rms = pm_pow2(gen, (T, K), device), None, 1.2
    # swiglu: a wide spread of gate values keeps 99 % certified; gelu: inputs mostly >= -2 (with the bias, or small without)
    target = {"gelu": 1.0 if c.bias else 0.5, "swiglu": 12.0}.get(c.entry, 3.0)
    w = ints(gen, (N, K), 7, device) * 2.0 ** -w_scale(K, x_rms, target)
    extra, positions = None, None
    if c.entry == "residual":
        extra = ints(gen, (T, N), 24, device) * 2.0 ** -3
    elif c.entry == "bias" and c.bias:
        extra = ints(gen, (N,), 16, device) * 2.0 ** -3
    elif c.entry == "gelu" and c.bias:
        extra = torch.randint(6, 13, (N,), generator=gen, device=device).double() * 2.0 ** -2  # 1.5 .. 3: inputs mostly >= -2
    if c.entry == "qkv":
        H, KV, hd = c.heads
        q_dim = H * hd
        positions = torch.randint(0, ROPE_LEN, (T,), generator=gen, device=device)
        positions[-1] = ROPE_LEN - 1
        ncode = min(T, 4)
        positions[:ncode] = torch.tensor(CODE_POS[:ncode], device=device)
        # the first q head and the first k head read only the eight code columns: the four coded tokens get code_targets
        u = H4.T @ code_targets(hd) / 4  # [4 codes, hd]
        hi = bf16r(u)
        lo = u - hi
        assert torch.equal(bf16r(lo), lo), "a code weight does not split into two bf16 values"
        rows = torch.cat([torch.arange(hd), torch.arange(q_dim, q_dim + hd)]).to(device)
        w[rows] = 0
        w[rows, 0:8:2] = torch.cat([hi.T, hi.T]).to(device)
        w[rows, 1:8:2] = torch.cat([lo.T, lo.T]).to(device)
        nw[:8] = 1
        x[:ncode, 0:8:2] = H4[:ncode].to(device)
        x[:ncode, 1:8:2] = H4[:ncode].to(device)
    return Design(x, nw, w, extra, positions)


def exact_product(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """a @ w.T in float64, after proving per output (in blocks of rows of w) that every fp32 sum of it is exact in any order."""
    out = torch.empty(a.shape[0], w.shape[0], dtype=torch.float64, device=a.device)
    for n0 in range(0, w.shape[0], 8192):
        blk = w[n0:n0 + 8192]
        assert matmul_exact(a, blk).all(), f"rows {n0}..: not an exact fp32 sum"
        out[:, n0:n0 + 8192] = a @ blk.T
    return out


# ----------------------------------------------------------------------------- the epilogues, emulated
def bf(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16)


def rope_f32(y: np.ndarray, cs: np.ndarray, fma: bool = False) -> np.ndarray:
    """y [T, heads, hd] float32 (bf16 values), cs [T, hd/2, 2] fp32 table rows: the rotated pairs, every product and sum
    rounded to float32 (fma=True: the first product of each component kept exact, as a contracted multiply-add would)."""
    a, b = y[..., 0::2], y[..., 1::2]
    c, d = cs[:, None, :, 0], cs[:, None, :, 1]
    if fma:
        re_ = (a.astype(np.float64) * c - (b * d)).astype(np.float32)
        im_ = (a.astype(np.float64) * d + (b * c)).astype(np.float32)
    else:
        re_, im_ = a * c - b * d, a * d + b * c
    out = np.empty_like(y)
    out[..., 0::2], out[..., 1::2] = re_, im_
    return out


def swiglu_parts(acc: torch.Tensor):
    """(g, certified) from the exact float64 accumulators: bf16(bf16(silu(bf16(a0))) * bf16(a1))."""
    y = bf16r(acc)
    y0, y1 = y[:, 0::2], y[:, 1::2]
    s = y0 / (1 + torch.exp(-y0))
    return bf16r(bf16r(s) * y1), certain(s) & (y0.abs() < 64)


def gelu_parts(v: torch.Tensor):
    """(out, certified) from v = bf16(acc + b) (float64): bf16(v * 0.5 * (1 + erf(v / sqrt 2)))."""
    g = v * 0.5 * (1 + torch.special.erf(v / math.sqrt(2.0)))
    return bf16r(g), certain(g) & (v >= GELU_MIN)


def gelu_f32_bounds(v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The kernel's float32 chain bf16(fp32(fp32(v * 0.5) * fp32(1 + erff(fp32(v * 0.70710678f))))) with erff anywhere within 3
    float32 ulps of erf: the bf16 results at both ends of that error (float64 [lo, hi]).  Below -2, where 1 + erf cancels, a
    correct kernel may be many bf16 ulps from the float64 GELU, but never outside these bounds."""
    vf = v.cpu().numpy().astype(np.float32)
    z = vf * np.float32(0.70710678118654752)
    e = torch.special.erf(torch.from_numpy(z).double()).numpy()
    ulp = np.spacing(np.abs(e).astype(np.float32)).astype(np.float64)
    ends = []
    for s in (-3, 3):
        ef = (e + s * ulp).astype(np.float32)
        g = (vf * np.float32(0.5)) * (np.float32(1) + ef)
        ends.append(bf(torch.from_numpy(g.astype(np.float32))).double())
    return torch.minimum(*ends).to(v.device), torch.maximum(*ends).to(v.device)


def reference(c: Case, d: Design, acc: torch.Tensor) -> Dict[str, Tuple[torch.Tensor, Optional[torch.Tensor]]]:
    """{output: (expected values, certified mask or None for 'every element')} from the exact accumulators acc [T, N]."""
    y32 = bf(acc.float())  # the exact sum is an fp32 number: one rounding to bf16
    if c.entry == "store":
        return {"out": (y32, None)}
    if c.entry == "f32":
        return {"out": (y32.float(), None)}
    if c.entry == "residual":
        return {"out": (bf(y32.float() + d.extra.float()), None)}
    if c.entry in ("bias", "gelu"):
        pre = bf(acc.float() + d.extra.float()) if d.extra is not None else y32
        if c.entry == "bias":
            return {"out": (pre, None)}
        g, cert = gelu_parts(pre.double())
        return {"out": (bf(g), cert), "bounds": gelu_f32_bounds(pre.double())}
    if c.entry == "swiglu":
        g, cert = swiglu_parts(acc)
        return {"out": (bf(g), cert)}
    H, KV, hd = c.heads
    q_dim, kv_dim = H * hd, KV * hd
    y = y32.float().cpu().numpy()
    cs = torch.view_as_real(rope_table(hd)).numpy()[d.positions.cpu().numpy()]
    T = c.T
    q = rope_f32(y[:, :q_dim].reshape(T, H, hd), cs).reshape(T, q_dim)
    k = rope_f32(y[:, q_dim:q_dim + kv_dim].reshape(T, KV, hd), cs).reshape(T, kv_dim)
    return {"q": (bf(torch.from_numpy(q)), None), "k": (bf(torch.from_numpy(k)), None), "v": (y32[:, q_dim + kv_dim:].cpu(), None)}


# ----------------------------------------------------------------------------- running one entry point
def nan_view(shape, dtype=torch.bfloat16):
    buf = torch.full((shape[0] + GUARD, *shape[1:]), NAN, dtype=dtype, device=DEV)
    return buf, buf[:shape[0]]


class Run:
    """The device side of one case: NaN-padded inputs and NaN-filled outputs with guard rows, and the ring for qkv."""

    def __init__(self, c: Case, d: Design):
        self.c = c
        T, N, K = c.T, c.N, c.K
        self.xbuf, self.x = nan_view((T, K))
        self.x.copy_(d.x)
        self.wbuf, self.w = nan_view((N, K))
        self.w.copy_(d.w)
        self.nw = bf(d.nw).to(DEV) if d.nw is not None else None
        self.extra = bf(d.extra).to(DEV).contiguous() if d.extra is not None else None
        self.ws = _abi.Workspace(_abi.workspace_bytes(T, K, 32, 8, 128, K, 0, 4), torch.device(DEV))
        if c.entry == "qkv":
            H, KV, hd = c.heads
            self.positions = d.positions.to(torch.int32).to(DEV)
            self.rope = torch.view_as_real(rope_table(hd)).contiguous().to(DEV)
            n_ring = T + 7
            perm = torch.randperm(n_ring, generator=torch.Generator().manual_seed(T))[:T].to(torch.int32)
            perm[torch.arange(T) % 5 == 3] = -1
            self.rows = perm.to(DEV)

    def outputs(self):
        c = self.c
        T = c.T
        if c.entry == "qkv":
            H, KV, hd = c.heads
            return {"q": nan_view((T, H * hd)), "k": nan_view((T, KV * hd)), "v": nan_view((T, KV * hd)),
                    "ck": (None, torch.full((T + 7, KV * hd), NAN, dtype=torch.bfloat16, device=DEV)),
                    "cv": (None, torch.full((T + 7, KV * hd), NAN, dtype=torch.bfloat16, device=DEV))}
        if c.entry == "f32":
            return {"out": nan_view((T, c.N), torch.float32)}
        return {"out": nan_view((T, c.N // 2 if c.entry == "swiglu" else c.N))}

    def launch(self, envd: Dict[str, str]):
        """NaN-filled outputs, one call under the switches of envd: (launch log, outputs)."""
        c, o = self.c, self.outputs()
        ws = self.ws

        def call():
            if c.entry in ("store", "residual"):
                _abi.linear_residual(self.x, self.w, self.extra, o["out"][1], ws)
            elif c.entry in ("bias", "gelu"):
                _abi.linear_bias(self.x, self.w, self.extra, o["out"][1], c.entry == "gelu", ws)
            elif c.entry == "f32":
                _abi.lm_head(self.x, self.nw, self.w, o["out"][1], EPS, ws)
            elif c.entry == "swiglu":
                _abi.ffn_gateup(self.x, self.nw, self.w, o["out"][1], EPS, ws)
            else:
                H, KV, hd = c.heads
                _abi.attn_qkv(self.x, self.nw, self.w, self.rope, self.positions, o["q"][1], o["k"][1], o["v"][1], o["ck"][1], o["cv"][1],
                              self.rows, H, KV, hd, EPS, ws)

        with env(**{"MB200_STREAMK": "1", "MB200_GEMM_CLUSTER": "1", "MB200_GEMM_BN": "0", **envd}):
            names = launched_kernels(call)
        torch.cuda.synchronize()
        return names, o


def check_guards(c: Case, r: Run, o, what: str):
    for k, (buf, view) in o.items():
        if buf is not None:
            assert torch.isnan(buf[view.shape[0]:].float()).all(), f"{what}: {k} guard rows were written"
            assert not torch.isnan(view.float()).any(), f"{what}: {k} has elements the kernel never wrote"
    if c.entry == "qkv":
        rows = r.rows.long()
        live = rows[rows >= 0]
        for ring, src in (("ck", "k"), ("cv", "v")):
            got = o[ring][1]
            assert_same(got[live].cpu(), o[src][1][rows >= 0].cpu(), f"{what}: ring {ring} rows named by cache_rows")
            rest = torch.ones(got.shape[0], dtype=torch.bool, device=DEV)
            rest[live] = False
            assert torch.isnan(got[rest].float()).all(), f"{what}: ring {ring} rows that cache_rows does not name were written"


def check_values(c: Case, want, o, what: str):
    """Every certified (or every) element exactly; uncertified ones within one ulp.  Returns (uncertified, total)."""
    unc = tot = 0
    for k, (ref, cert) in want.items():
        if k == "bounds":
            continue
        got = o[k][1]
        ref = ref.to(got.device)
        if cert is None:
            assert_same(got, ref, f"{what}: {k}")
            continue
        cert = cert.to(got.device)
        ok = same(got, ref)
        assert ok[cert].all(), f"{what}: {k} differs on {int((~ok & cert).sum())} certified elements"
        near = bf16_ulp_diff(got[~cert].cpu(), ref[~cert].cpu()) <= 1
        if "bounds" in want:  # GELU below -2: within the float32 chain's bounds for erff's error
            lo, hi = (b.to(got.device)[~cert].cpu() for b in want["bounds"])
            g = got[~cert].double().cpu()
            near |= (g >= lo) & (g <= hi)
        assert near.all(), f"{what}: {k}: an uncertified element is off by more than 1 ulp (and outside the erff bounds)"
        unc += int((~cert).sum())
        tot += cert.numel()
    return unc, tot


CERT_STATS: Dict[str, Tuple[int, int]] = {}


def run_case(c: Case):
    sms = _abi.device_info()[0]
    big = c.T * c.N * c.K > 2 ** 27
    dref = DEV if big else "cpu"
    d = design(c, DEV)
    xn = d.x * d.nw if d.nw is not None else d.x
    acc = exact_product(xn.to(dref), d.w.to(dref))
    want = reference(c, Design(*(t.to(dref) if t is not None else None for t in d)), acc)
    r = Run(c, d)
    base = dict(c.env)
    names, o = r.launch(base)
    regime = dense_regime(c.entry, c.T, c.N, c.K, base, sms)
    assert len(names) == 1 and re.search(regime, names[0]), f"{c.name}: launched {names}, expected {regime}"
    check_guards(c, r, o, c.name)
    unc, tot = check_values(c, want, o, c.name)
    if tot:
        # small cases are too few elements for a 1 % bound: they count in the file's total (test_certified_fraction_report)
        assert tot < 1 << 15 or unc <= 0.01 * tot, f"{c.name}: {unc} / {tot} elements uncertified"
        CERT_STATS[c.name] = (unc, tot)
        print(f"certified {c.entry} {c.name}: {1 - unc / tot:.5f} of {tot}")
    first = {k: v[1].clone() for k, v in o.items()}
    runs = [(e, "variant") for e in variants(c, sms)]
    if family(regime) == "streamk":
        runs.append((base, "stream-K again after another regime on the same workspace"))
    for e, why in runs:
        names, o = r.launch(e)
        reg = dense_regime(c.entry, c.T, c.N, c.K, e, sms)
        what = f"{c.name} {e} ({why})"
        assert len(names) == 1 and re.search(reg, names[0]), f"{what}: launched {names}, expected {reg}"
        check_guards(c, r, o, what)
        for k, v in first.items():
            assert_same(o[k][1], v, f"{what}: {k} vs the base run")


# ----------------------------------------------------------------------------- RMSNorm, emulated
def norm_inputs(T: int, K: int, seed: int, device="cpu"):
    """x: integers up to 2^floor(12 - log2(K)/2) times a per-token 2^-s (sum x^2 exact in fp32), norm weight: general bf16."""
    gen = torch.Generator(device=device).manual_seed(seed)
    lim = 2 ** int(12 - math.log2(K) / 2) - 1
    s = torch.randint(0, 12, (T, 1), generator=gen, device=device).double()
    x = ints(gen, (T, K), lim, device) * torch.pow(2.0, -s)
    x[:, 0] = torch.where(x[:, 0] == 0, torch.pow(2.0, -s[:, 0]), x[:, 0])  # no all-zero row
    nw = bf(torch.randn(K, generator=gen, device=device, dtype=torch.float64) * 0.5 + 1).double()
    return x, nw


def rms_norm_f32(x: torch.Tensor, nw: torch.Tensor) -> torch.Tensor:
    """The kernels' chain in numpy float32: r = 1 / sqrt_rn(tot / K + eps), bf16(bf16(x * r) * w)."""
    xs = x.cpu().numpy().astype(np.float32)
    tot = (x.double() ** 2).sum(1).cpu().numpy().astype(np.float32)  # exact (accumulation_exact)
    K = np.float32(x.shape[1])
    r = np.float32(1) / np.sqrt(tot / K + np.float32(EPS))
    xr = bf(torch.from_numpy((xs * r[:, None]).astype(np.float32))).float().numpy()
    return bf(torch.from_numpy(xr * nw.cpu().numpy().astype(np.float32)[None, :]))


def selection_weights(K: int, seed: int, device) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """[K, K]: row n holds 2^e[n] (e in -1..1) at column col[n] (a permutation), zero elsewhere."""
    gen = torch.Generator(device=device).manual_seed(seed)
    col = torch.randperm(K, generator=gen, device=device)
    e = torch.randint(-1, 2, (K,), generator=gen, device=device).double()
    w = torch.zeros(K, K, dtype=torch.float64, device=device)
    w[torch.arange(K, device=device), col] = torch.pow(2.0, e)
    return w, col, e


# ----------------------------------------------------------------------------- CPU: the design is exact, the checks are tight
def test_designs_are_exact():
    """Every entry point's design gives exact fp32 sums at the shortest and longest K used (64 .. 16384); the QKV code puts the
    sensitive pairs on the coded tokens' first q and k heads exactly; the norm inputs' sum of squares is exact."""
    for e in ENTRIES:
        for K in (64, 1088, 4096, 14336, 16384):
            c = qkv("x", 6, K, 2, 1, 128) if e == "qkv" else Case("x", e, 6, 256, K)
            d = design(c, "cpu")
            xn = d.x * d.nw if d.nw is not None else d.x
            assert matmul_exact(xn, d.w).all(), (e, K)
            assert torch.equal(bf16r(d.w), d.w) and torch.equal(bf16r(xn), xn)
            if d.extra is not None:
                assert torch.equal(bf16r(d.extra), d.extra)
            if e == "qkv":
                y = xn @ d.w.T
                tgt = code_targets(128)
                assert torch.equal(y[:4, :128], tgt) and torch.equal(y[:4, 256:384], tgt)
    for K in (1088, 4096, 5120, 14336):
        x, _ = norm_inputs(8, K, K)
        assert accumulation_exact(x * x).all() and torch.equal(bf16r(x), x), K
        assert (lsb_exponent(x[x != 0]) >= -11).all()  # integers times 2^-s, s <= 11


def test_fma_sensitive_code_pairs():
    """At each coded position, for head_dim 128 and 64, at least four frequencies have an FMA-sensitive pair, and the emulation
    really tells the fused form apart on them."""
    for hd in (128, 64):
        cs = torch.view_as_real(rope_table(hd)).numpy()
        for pos in CODE_POS:
            s = sensitive(hd, pos)
            assert len(s) >= 4, (hd, pos, len(s))
            y = code_targets(hd)[CODE_POS.index(pos)].float().numpy()[None, None, :]
            c1 = cs[[pos]]
            plain, fused = rope_f32(y, c1), rope_f32(y, c1, fma=True)
            differ = bf(torch.from_numpy(plain)) != bf(torch.from_numpy(fused))
            pairs = differ.view(hd // 2, 2).any(1)
            assert int(pairs.sum()) >= len(s), (hd, pos)


def _sample(entry: str, T: int = 64, N: int = 1024, K: int = 4096):
    c = Case("x", entry, T, N, K)
    d = design(c, "cpu")
    xn = d.x * d.nw if d.nw is not None else d.x
    return c, d, xn @ d.w.T


def test_certification_rates():
    """At least 99 % of SWIGLU and GELU elements are certified on the designed inputs (the GPU tests assert the same per case)."""
    for K in (256, 4096, 14336):
        _, _, acc = _sample("swiglu", K=K)
        assert swiglu_parts(acc)[1].float().mean() >= 0.99, K
        c, d, acc = _sample("gelu", K=K)
        v = bf16r(acc + d.extra)
        cert = gelu_parts(v)[1]
        assert cert.float().mean() >= 0.99 and (v < 0).float().mean() > 0.02, K  # the erf side of GELU is exercised
        lo, hi = gelu_f32_bounds(v)
        g = gelu_parts(v)[0]
        assert ((g >= lo) & (g <= hi)).all(), K  # the float64 GELU lies within the float32 chain's erff bounds


def test_residual_tightness():
    """bf16(bf16(acc) + r) differs from a single rounding bf16(acc + r) on at least 10 % of the elements."""
    _, d, acc = _sample("residual")
    right = bf16r(bf16r(acc) + d.extra)
    assert torch.equal(bf(bf(acc.float()).float() + d.extra.float()).double(), right)  # the fp32 add is exact here
    assert (right != bf16r(acc + d.extra)).float().mean() >= 0.10


def test_bias_tightness():
    """bf16(acc + b) differs from rounding before the bias, bf16(bf16(acc) + b), on at least 8 % of the elements, and so does
    GELU's input."""
    for e in ("bias", "gelu"):
        _, d, acc = _sample(e)
        assert (bf16r(acc + d.extra) != bf16r(bf16r(acc) + d.extra)).float().mean() >= 0.08, e


def test_swiglu_tightness():
    """Among certified elements, silu of the unrounded a0 changes at least 10 % of g, and an unrounded silu at least 10 %; the
    SILU_A gate values, certified powers of two, make g exact on every element."""
    _, _, acc = _sample("swiglu")
    g, cert = swiglu_parts(acc)
    a0, a1 = acc[:, 0::2], bf16r(acc[:, 1::2])
    y0 = bf16r(a0)
    unrounded_a0 = bf16r(bf16r(a0 / (1 + torch.exp(-a0))) * a1)
    unrounded_silu = bf16r(y0 / (1 + torch.exp(-y0)) * a1)
    assert (unrounded_a0 != g)[cert].float().mean() >= 0.10
    assert (unrounded_silu != g)[cert].float().mean() >= 0.10
    s = SILU_A / (1 + torch.exp(-SILU_A))
    assert certain(s).all()


def test_rope_tightness():
    """On the coded tokens of a QKV design, the fused (FMA) rotation changes at least 10 % of the first q head's elements; over the
    whole output it changes some, so the exact comparison sees a contraction."""
    for hd, heads in ((128, (4, 2, 128)), (64, (3, 3, 64))):
        c = qkv("x", 16, 512, *heads)
        d = design(c, "cpu")
        acc = (d.x * d.nw) @ d.w.T
        y = bf(acc.float()).float().numpy()
        cs = torch.view_as_real(rope_table(hd)).numpy()[d.positions.numpy()]
        H = heads[0]
        yq = y[:, :H * hd].reshape(16, H, hd)
        differ = bf(torch.from_numpy(rope_f32(yq, cs))) != bf(torch.from_numpy(rope_f32(yq, cs, fma=True)))
        assert differ[:4, 0].float().mean() >= 0.10, hd
        assert differ[4:, 1:].float().mean() < differ[:4, 0].float().mean()


def test_cases_reach_every_regime():
    """From the host's own switches at 132 SMs, the cases (with their variants) reach every family for every mode its entry points
    can take to it, every TA and BN, and both walks of both wgmma families, ragged blocks included."""
    sms = 132
    seen, walks = set(), set()
    for c in CASES + REAL:
        for e in [dict(c.env)] + variants(c, sms):
            r = dense_regime(c.entry, c.T, c.N, c.K, e, sms)
            seen.add(r)
            walks.add((family(r), walk(r, c.T, c.N)))
    modes = [m for m, _ in ENTRIES.values()]
    want = {rf"^skinny_linear_kernel<{1 + (i + j) % 4}, {m}, {'true' if n else 'false'}>$" for i, (m, n) in enumerate(ENTRIES.values())
            for j in (0, 2)}  # two T per mode, every T over the modes
    want |= {rf"^gemm_streamk_kernel<{m}, {ta}>$" for m in modes for ta in (32, 64, 128)}
    want |= {rf"^gemm_wgmma_kernel<{m}, 1, {bn}, {ta}>$" for m in modes for bn in (32, 64, 128, 256) for ta in (32, 64, 128)}
    want |= {rf"^gemm_wgmma_kernel<{m}, {cl}, {bn}, 128>$" for m in modes for cl in (1, 2) for bn in (128, 192, 256)}
    want |= {rf"^gemm_mma_kernel<{m}>$" for m in modes if m != 4}  # QKV's N = (H + 2 KV) hd always has a wgmma kernel
    assert want <= seen, sorted(want - seen)
    assert {T for c in CASES for T in (c.T,) if c.T <= 4} == {1, 2, 3, 4}
    assert {("prefill", "m-fastest"), ("prefill", "blocked"), ("prefill", "blocked ragged"), ("cluster", "m-fastest"),
            ("cluster", "blocked"), ("cluster", "blocked ragged")} <= walks, walks
    # edges of the table
    assert dense_regime("store", 4, 1024, 64, {}, sms).startswith("^skinny") and family(dense_regime("store", 5, 1024, 64, {}, sms)) == "streamk"
    assert family(dense_regime("store", 128, 1024, 64, {}, sms)) == "streamk" and family(dense_regime("store", 129, 1024, 64, {}, sms)) == "prefill"
    assert family(dense_regime("store", 511, 1024, 64, {}, sms)) == "prefill" and family(dense_regime("store", 512, 1024, 64, {}, sms)) == "cluster"
    assert walk(dense_regime("store", 2048, 3072, 64, {"MB200_GEMM_CLUSTER": "0"}, sms), 2048, 3072) == "m-fastest"
    assert walk(dense_regime("store", 2049, 3072, 64, {"MB200_GEMM_CLUSTER": "0"}, sms), 2049, 3072) == "blocked ragged"
    assert walk(dense_regime("store", 4096, 3072, 64, {}, sms), 4096, 3072) == "m-fastest"
    assert walk(dense_regime("residual", 8200, 2560, 64, {}, sms), 8200, 2560) == "blocked ragged"
    # stream-K: a single 128-wide tile split by every CTA, fewer k-blocks than ring stages
    assert any(c.N == 128 and family(dense_regime(c.entry, c.T, c.N, c.K, dict(c.env), sms)) == "streamk" for c in CASES)
    assert any(c.K == 64 and family(dense_regime(c.entry, c.T, c.N, c.K, dict(c.env), sms)) == "streamk" for c in CASES)
    # the GEMV tail loop (K / 8 not a multiple of 128) and N / 16 not whole
    assert all((c.K // 8) % 128 and c.N % 16 for c in CASES if c.T <= 4 and c.entry != "qkv")


def test_rmsnorm_emulation_matches_oracle():
    """oracle.restatement.rms_norm gives the bits of the float32 emulation on the norm inputs, with and without a general
    weight: kernel == emulation (GPU tests) and emulation == oracle here."""
    for K in (1088, 4096, 5120, 6144, 14336):
        x, nw = norm_inputs(16, K, K + 1)
        want = rms_norm_f32(x, nw)
        got = R.rms_norm(bf(x), bf(nw), EPS)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), K
        # the per-token scales differ: r is not the same power of two on every row
        assert len(set(bf(x.abs().max(1).values).tolist())) > 4


# ----------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_linear_regimes(case):
    """One entry point in one regime (asserted from the launch log), bit for bit against the emulated epilogue, guard rows and
    ring rows untouched; then every switch that changes the kernel gives the same bits."""
    run_case(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", REAL, ids=[c.name for c in REAL])
def test_linear_real_shapes(case):
    """Every dense Linear of Mistral-7B, Mistral-Nemo-12B and the Mixtral-8x22B dense parts, as test_linear_regimes."""
    run_case(case)
    torch.cuda.empty_cache()


NORM_CASES = [(T, K) for T, K in ((1, 4096), (2, 1088), (3, 5120), (4, 4160), (5, 4096), (64, 1088), (100, 1000 + 24), (200, 5120),
                                   (600, 4096), (2049, 1088))]


@pytest.mark.gpu
@pytest.mark.parametrize("T,K", NORM_CASES)
def test_rmsnorm_through_selection_weights(T, K):
    """lm_head with one power of two per weight row: logits[t, n] = 2^e[n] * xn[t, col[n]], so every bit of the in-kernel norm
    (T <= 4) or of rmsnorm_kernel (T > 4) shows, in the regime the shape selects; mb200_rmsnorm directly gives the same xn."""
    sms = _abi.device_info()[0]
    x, nw = norm_inputs(T, K, T * 7 + K)
    assert accumulation_exact(x * x).all()
    xn = rms_norm_f32(x, nw)
    w, col, e = selection_weights(K, T + K, "cpu")
    c = Case("norm", "f32", T, K, K)
    r = Run(c, Design(x, nw, w, None))
    names, o = r.launch({})
    reg = dense_regime("f32", T, K, K, {}, sms)
    assert len(names) == 1 and re.search(reg, names[0]), f"launched {names}, expected {reg}"
    check_guards(c, r, o, f"T={T} K={K}")
    want = (xn.double()[:, col] * torch.pow(2.0, e)[None, :]).float()
    assert_same(o["out"][1], want.to(DEV), f"T={T} K={K}: normed inputs through the lm head")
    direct = _abi.rmsnorm(r.x, r.nw, EPS)
    torch.cuda.synchronize()
    assert_same(direct.cpu(), xn, f"T={T} K={K}: mb200_rmsnorm")


@pytest.mark.gpu
def test_certified_fraction_report():
    """Runs last in the file: the SWIGLU and GELU certified fractions reached over the cases that ran."""
    if not CERT_STATS:
        pytest.skip("no certified case ran in this session")
    for entry in ("swiglu", "gelu"):
        unc = sum(u for k, (u, _) in CERT_STATS.items() if entry in k or ("gateup" in k and entry == "swiglu"))
        tot = sum(t for k, (_, t) in CERT_STATS.items() if entry in k or ("gateup" in k and entry == "swiglu"))
        if tot:
            print(f"certified fraction {entry}: {1 - unc / tot:.5f} of {tot} elements")
            assert unc <= 0.01 * tot
