"""The prefill / batched-decode mixture-of-experts path (csrc/moe.cuh: router, row plan, gather, grouped expert GEMMs, combine;
moe.py:MoeLayer.run) bit for bit, in every routing, plan and grouped-GEMM regime.

Regimes (the host's own switches, restated by `gemm_regime` below and asserted from the launch log in every GPU test):
  router      T <= 256: one CTA per token (8-warp fold), else one warp per token; E in {2, 4, 8, 16} are separate instantiations
  row plan    T * k <= 512: a thread per expert, no cluster pair list (plan[6] = 0); else the 1024-thread scan + pair list
  m tile      32 / 64 / 128 rows for T <= 32 / <= 64 / larger
  tile < 128  N % 128 == 0 and stream-K on: gemm_streamk_grouped_kernel<MODE, TA>; else gemm_wgmma_grouped_kernel<MODE, 1, BN, TA>
              with BN from the fill score or MB200_GEMM_BN
  tile 128    N % 256 == 0, cluster on and rows_cap >= 512 E: the 2-CTA cluster over tile pairs; else one CTA with BN 256 / 128 / 64;
              more than 16 m units: the GM x GN blocked tile walk, ragged last blocks included
  combine     k = 1..8 bf16 adds in ascending expert order, with or without the residual
  layer       MoeLayer.run in blocks of MOE_BLOCK_TOKENS tokens

Exact by construction.  Two families of inputs make every fp32 sum of the path exact in any order, proven on the host in the same
test (`matmul_exact`: every product on a common grid, sum |p| < 2^24 grid units):
  X  hn entries +-2^a (a in -1, 0, 1); gate, w1, w3 dense small integers * 2^-s.  Router logits and gate/up pre-activations are
     exact, so the bf16 logits are unique (and tie naturally at large T) and so are y0, y1.  What is left is expf inside the
     SiLU and the softmax: both are certified in float64 (`certain`: every value within 2^-16 relative of the float64 one rounds
     to the same bf16), and certified elements must match exactly.  g is bit-identical across all GEMM regimes on every element.
  Y  hn[:, 0] = 1; w1 row r holds a SILU_A value at column 0 only (bf16(silu) a certified power of two), w3 row r +-1 at one other
     column, so g is a token-dependent +- power of two; w2 dense small integers * 2^-s.  The down projection is exact, so yw, the
     combine and the layer output are bit-exact in every regime.
The float64 reference runs on the device for big shapes (cuBLAS DGEMM) and on the CPU for small ones; with exact sums both are
exact.  Each stage is checked on the kernel's own input read back from MoeBuffers, so a failure names its stage.  g, yw and out
are NaN-filled before every launch: every live row must be written, rows past the plan (or past T) must stay NaN.  Routing is
either natural (family X / Y gates, ties included) or designed: a code column per expert in hn (+-2) and the gate (16) pins
each token's k experts, so per-expert row counts -- empty experts, exact whole tiles, odd / even tile pairs -- are chosen.
"""
import contextlib
import ctypes
import math
import os
from typing import Dict, List, NamedTuple, Optional, Tuple

import pytest
import torch

from mistral_inference_b200 import _abi
from mistral_inference_b200.moe import MOE_BLOCK_TOKENS, MoeBuffers, MoeLayer
from oracle import restatement as R

from .test_gpu_megakernel_phases import SILU_A, SILU_S, accumulation_exact, lsb_exponent
from .util import launched_kernels

DEV = "cuda"
NAN = float("nan")
PLAN_HEADER = 64          # MOE_PLAN_HEADER
PAIR_SECOND = 1 << 30     # MOE_PAIR_SECOND
KGM, KGN = {1: 12, 2: 8}, {1: 12, 2: 9}  # blocked walk: m units x n tiles per block, single CTA / cluster pair
MARGIN = 2.0 ** -16       # relative distance from a bf16 rounding boundary that certifies an expf-based value
EPI_SWIGLU, EPI_MOE_SCALE = 3, 5
Y_SILU = torch.tensor([a for a, s in zip(SILU_A.tolist(), SILU_S.tolist()) if s in (-0.25, 0.5, 1.0)], dtype=torch.float64)


# ----------------------------------------------------------------------------- float64 helpers
def bf16r(v: torch.Tensor) -> torch.Tensor:
    """Round float64 to the nearest bf16 value (ties to even), exactly: 8 significant bits (normal range)."""
    m, e = torch.frexp(v)
    return torch.ldexp(torch.round(m * 256.0) / 256.0, e)


def certain(v: torch.Tensor, margin: float = MARGIN) -> torch.Tensor:
    """Values whose whole neighbourhood v * (1 +- margin) rounds to one bf16 value (rounding is monotone, so both ends suffice):
    any computation of v with a relative error below `margin` rounds to bf16r(v)."""
    lo, hi = bf16r(v * (1 - margin)), bf16r(v * (1 + margin))
    return ((lo == hi) & (v.abs() >= 2.0 ** -100)) | (v == 0)


def row_grid(a: torch.Tensor) -> torch.Tensor:
    """Exponent of the finest grid 2^e that every nonzero entry of each row lies on (0 for an all-zero row)."""
    nz = a != 0
    lsb = torch.where(nz, lsb_exponent(torch.where(nz, a, torch.ones_like(a))), torch.full_like(a, 1 << 20, dtype=torch.int64))
    e = lsb.min(1).values
    return torch.where(nz.any(1), e, torch.zeros_like(e))


def matmul_exact(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """[M, K] x [N, K]^T, float64 entries that are bf16 values: True per output where every product a[m, j] w[n, j] lies on the
    grid 2^(ea_m + ew_n) and the sum of |products| is below 2^24 grid units, so fp32 computes the dot product exactly in any
    order (the matrix form of accumulation_exact; the unit counts are integers below 2^53, exact in float64)."""
    ea, ew = row_grid(a), row_grid(w)
    units = (a.abs() * torch.pow(2.0, -ea.double())[:, None]) @ (w.abs() * torch.pow(2.0, -ew.double())[:, None]).T
    return units < 2.0 ** 24


def same(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """Element-wise identity of bf16 values (NaN == NaN; +0 == -0)."""
    got, want = got.double(), want.double()
    return (got == want) | (torch.isnan(got) & torch.isnan(want))


def assert_same(got: torch.Tensor, want: torch.Tensor, what: str):
    ok = same(got, want)
    if not ok.all():
        bad = (~ok).nonzero()[:5].tolist()
        raise AssertionError(f"{what}: {(~ok).sum().item()} / {ok.numel()} elements differ, first at {bad}: "
                             f"got {[got[tuple(i)].item() for i in bad]}, want {[want[tuple(i)].item() for i in bad]}")


# ----------------------------------------------------------------------------- designed inputs
def scale_exp(K: int, rms: float) -> int:
    """2^-s scale of integer weights that puts a K-long dot product with entries of this rms near +-3."""
    return max(0, round(math.log2(math.sqrt(K) * rms / 3.0)))


def ints(gen: torch.Generator, shape, lim: int, device) -> torch.Tensor:
    return torch.randint(-lim, lim + 1, shape, generator=gen, device=device).double()


def pm_pow2(gen: torch.Generator, shape, device, exps=(-1, 0, 1)) -> torch.Tensor:
    """Entries +-2^a with a drawn from `exps`."""
    a = torch.tensor(exps, dtype=torch.float64, device=device)[torch.randint(0, len(exps), shape, generator=gen, device=device)]
    s = torch.randint(0, 2, shape, generator=gen, device=device).double() * 2 - 1
    return s * torch.pow(2.0, a)


def assign_counts(T: int, counts: List[int]) -> torch.Tensor:
    """[T, k] experts with exactly counts[e] tokens per expert, k distinct experts per token: the list of experts, each repeated
    counts[e] times, read in k columns of T (an expert spans two positions T apart only if counts[e] > T)."""
    k = sum(counts) // T
    assert sum(counts) == T * k and max(counts) <= T, counts
    flat = torch.cat([torch.full((c,), e, dtype=torch.int64) for e, c in enumerate(counts)])
    a = flat.view(k, T).T
    assert (a.sort(1).values[:, 1:] != a.sort(1).values[:, :-1]).all()
    return a


def assign_random(T: int, E: int, k: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(T)])


class Design(NamedTuple):
    family: str
    hn: torch.Tensor           # [T, dim] bf16 on DEV
    gate: torch.Tensor         # [E, dim] bf16 on DEV
    w13: List[torch.Tensor]    # E x [2 hidden, dim] bf16 on DEV, rows 2i = w1[i], 2i + 1 = w3[i]
    w2: List[torch.Tensor]     # E x [dim, hidden] bf16 on DEV


def design_inputs(family: str, T: int, dim: int, E: int, seed: int, assign: Optional[torch.Tensor] = None, device=DEV):
    """hn and the gate of a family; with `assign` [T, k], code columns 1..E pin every token's experts (+2 in a chosen expert's
    column, -2 elsewhere, gate weight 16 on the expert's own column: chosen logits ~ +32, the others ~ -32)."""
    gen = torch.Generator(device=device).manual_seed(seed)
    hn = pm_pow2(gen, (T, dim), device)
    s = scale_exp(dim, 5.7)
    gate = ints(gen, (E, dim), 7, device) * 2.0 ** -s
    if family == "Y":
        hn[:, 0] = 1.0
    if assign is not None:
        code = torch.full((T, E), -2.0, dtype=torch.float64)
        code.scatter_(1, assign, 2.0)
        hn[:, 1:E + 1] = code.to(device)
        gate[:, 1:E + 1] = torch.eye(E, dtype=torch.float64, device=device) * 2.0 ** 4
    return hn.to(torch.bfloat16), gate.to(torch.bfloat16)


def design_experts(family: str, dim: int, hidden: int, E: int, seed: int, device=DEV):
    gen = torch.Generator(device=device).manual_seed(seed + 1)
    w13, w2 = [], []
    s2 = scale_exp(hidden, 4.3 * (0.7 if family == "Y" else 1.0))
    for _ in range(E):
        if family == "X":
            s = scale_exp(dim, 5.7)
            w = ints(gen, (2 * hidden, dim), 7, device) * 2.0 ** -s
        else:
            w = torch.zeros(2 * hidden, dim, dtype=torch.float64, device=device)
            pick = torch.randint(0, len(Y_SILU), (hidden,), generator=gen, device=device)
            w[0::2, 0] = Y_SILU.to(device)[pick]
            col = torch.randint(1, dim, (hidden,), generator=gen, device=device)
            sign = torch.randint(0, 2, (hidden,), generator=gen, device=device).double() * 2 - 1
            w[1::2].scatter_(1, col[:, None], sign[:, None])
        w13.append(w.to(torch.bfloat16))
        w2.append((ints(gen, (dim, hidden), 7, device) * 2.0 ** -s2).to(torch.bfloat16))
    return w13, w2


def make_design(family, T, dim, hidden, E, seed, assign=None, experts=None) -> Design:
    hn, gate = design_inputs(family, T, dim, E, seed, assign)
    w13, w2 = experts if experts is not None else design_experts(family, dim, hidden, E, seed)
    return Design(family, hn, gate, w13, w2)


# ----------------------------------------------------------------------------- host restatements
def route_rule(logits: torch.Tensor, k: int):
    """The documented rule on exact bf16 logits [T, E] (float64): stable sort by (-logit, index) -- ties to the lower index --,
    fp32 softmax of the k (float64 here, certified per weight), bf16; experts and weights in ascending expert order."""
    top = torch.sort(-logits, dim=1, stable=True).indices[:, :k]
    lv = logits.gather(1, top)
    ex = torch.exp(lv - lv[:, :1])
    w = ex / ex.sum(1, keepdim=True)
    asc = top.argsort(1)
    return top.gather(1, asc), bf16r(w).gather(1, asc), certain(w).gather(1, asc)


def router_logits(d: Design) -> torch.Tensor:
    hn, gate = d.hn.double().cpu(), d.gate.double().cpu()
    assert matmul_exact(hn, gate).all(), "router logits are not exact fp32 sums"
    return bf16r(hn @ gate.T)


def boundary_tie(logits: torch.Tensor, k: int) -> torch.Tensor:
    """Tokens whose k-th and (k+1)-th largest bf16 logits are equal (the tie rule decides the selection)."""
    if k >= logits.shape[1]:
        return torch.zeros(logits.shape[0], dtype=torch.bool)
    v = torch.sort(logits, dim=1, descending=True).values
    return v[:, k - 1] == v[:, k]


def tile_rows_of(T: int) -> int:
    return 32 if T <= 32 else (64 if T <= 64 else 128)


def plan_host(sel: torch.Tensor, E: int, shard=(0, 1), prev=(0, 0)) -> Tuple[Dict[int, int], torch.Tensor]:
    """Every word moe_plan_kernel writes ({index: value}) and the slot of every (token, expert) pair: per-expert segments padded
    to the m tile, token order inside a segment, this rank's tile list, the cluster pair list (scan path only; MOE_PAIR_SECOND
    on a pair with a second tile), and the statistics words accumulated onto `prev`."""
    T, k = sel.shape
    pairs, tr = T * k, tile_rows_of(T)
    cap = -(-pairs // tr) + E
    counts = torch.bincount(sel.reshape(-1), minlength=E).tolist()
    words: Dict[int, int] = {}
    rows = n = npairs = 0
    seg = []
    for e in range(E):
        seg.append(rows)
        words[8 + e] = rows
        m = -(-counts[e] // tr)
        if e % shard[1] == shard[0]:
            for i in range(m):
                if n < cap:
                    words[PLAN_HEADER + n], words[PLAN_HEADER + cap + n] = e, rows + i * tr
                    n += 1
            if pairs > 512:
                for i in range(0, m, 2):
                    if npairs < cap:
                        words[PLAN_HEADER + 2 * cap + npairs] = e
                        words[PLAN_HEADER + 3 * cap + npairs] = (rows + i * tr) | (PAIR_SECOND if i + 1 < m else 0)
                        npairs += 1
        rows += m * tr
    words.update({8 + E: rows, 0: n, 1: rows, 2: cap, 3: pairs, 4: prev[0] + sum(c > 0 for c in counts), 5: prev[1] + 1,
                  6: npairs if pairs > 512 else 0})
    flat = sel.reshape(-1).tolist()
    run = [0] * E
    slot = []
    for e in flat:
        slot.append(seg[e] + run[e])
        run[e] += 1
    return words, torch.tensor(slot, dtype=torch.int64)


def gemm_regime(mode: int, T: int, E: int, k: int, N: int, env: Dict[str, str]) -> str:
    """Regex of the grouped GEMM kernel launch_grouped (csrc/moe.cuh) picks for one projection."""
    tr = tile_rows_of(T)
    rows_cap = (-(-T * k // tr) + E) * tr
    if tr < 128 and env.get("MB200_STREAMK", "1")[0] != "0" and N % 128 == 0:
        return rf"^gemm_streamk_grouped_kernel<{mode}, {tr}>$"
    if tr == 128:
        if N % 256 == 0 and env.get("MB200_GEMM_CLUSTER", "1")[0] != "0" and rows_cap >= E * 512:
            return rf"^gemm_wgmma_grouped_kernel<{mode}, 2, 256, 128>$"
        bn = next(b for b in (256, 128, 64, 32) if N % b == 0)
        return rf"^gemm_wgmma_grouped_kernel<{mode}, 1, {bn}, 128>$"
    forced = int(env.get("MB200_GEMM_BN", "0"))
    bn = str(forced) if forced in (32, 64, 128, 256) and N % forced == 0 else r"(256|128|64|32)"
    return rf"^gemm_wgmma_grouped_kernel<{mode}, 1, {bn}, {tr}>$"


def walk(words: Dict[int, int], N: int, regime: str) -> str:
    """The tile walk a wgmma grouped launch takes: 'm-fastest', or 'blocked' (+ ' ragged' when a last block is partial)."""
    import re

    m = re.search(r"<\d+, (\d), (\d+|\(.*\)), 128>", regime)
    if m is None:
        return "-"
    cl, bn = int(m.group(1)), int(m.group(2))
    num_m, num_n = (words[6] if cl == 2 else words[0]), N // bn
    if num_m <= 16:
        return "m-fastest"
    return "blocked" + (" ragged" if num_m % KGM[cl] or num_n % KGN[cl] else "") + (" wide" if num_n >= KGN[cl] else "")


@contextlib.contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in kw}
    os.environ.update({k: str(v) for k, v in kw.items()})
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def assert_names(names: List[str], want: List[str], what: str):
    import re

    assert len(names) == len(want) and all(re.search(w, n) for n, w in zip(names, want)), f"{what}: launched {names}, expected {want}"


# ----------------------------------------------------------------------------- running the path
def workspace(T: int, dim: int, hidden: int) -> _abi.Workspace:
    return _abi.Workspace(_abi.workspace_bytes(max(T, 8), dim, 32, 8, 128, hidden, 0, 4), torch.device(DEV))


def nan_fill(b: MoeBuffers):
    for t in (b.xs, b.row_w, b.g, b.yw):
        t.fill_(NAN)
    b.sel.fill_(-1)
    b.slot.fill_(-1)
    b.wts.fill_(NAN)


def route(d: Design, E: int, k: int, b: MoeBuffers, shard=(0, 1)) -> List[str]:
    return launched_kernels(lambda: _abi.moe_route(d.hn, d.gate, E, k, shard[0], shard[1], b))


def weight_tables(d: Design, E: int, owned=None):
    w13, w2 = (ctypes.c_void_p * E)(), (ctypes.c_void_p * E)()
    for e in range(E):
        if owned is None or e in owned:
            w13[e], w2[e] = d.w13[e].data_ptr(), d.w2[e].data_ptr()
    return w13, w2


def ffn(d: Design, E: int, k: int, b: MoeBuffers, ws, residual: Optional[torch.Tensor], pad: int = 3):
    """NaN-filled g, yw and out, then one grouped FFN call; returns (launches, out [T + pad, dim] with the pad rows)."""
    T, dim = d.hn.shape
    hidden = d.w13[0].shape[0] // 2
    b.g.fill_(NAN)
    b.yw.fill_(NAN)
    out = torch.full((T + pad, dim), NAN, dtype=torch.bfloat16, device=DEV)
    w13, w2 = weight_tables(d, E)
    names = launched_kernels(lambda: _abi.moe_grouped_ffn(b, w13, w2, residual, out[:T], T, dim, hidden, E, k, None, ws))
    torch.cuda.synchronize()
    return names, out


def check_route(d: Design, E: int, k: int, b: MoeBuffers, names: List[str], what: str, shard=(0, 1), prev=(0, 0)):
    """sel / wts against the rule, every plan word, the slots, and the gathered rows + weights (other rows keep NaN)."""
    T = d.hn.shape[0]
    torch.cuda.synchronize()
    assert_names(names, [rf"^moe_route_kernel<{E}, {'true' if T <= 256 else 'false'}>$",
                         rf"^moe_plan_kernel<{'short' if T * k <= 512 else 'scan'}>$", r"^moe_gather_kernel$"], what)
    logits = router_logits(d)
    sel_ref, wts_ref, cert = route_rule(logits, k)
    sel, wts = b.sel.view(T, k).cpu().long(), b.wts.view(T, k).cpu().double()
    assert torch.equal(sel, sel_ref), f"{what}: selection differs on tokens {(sel != sel_ref).any(1).nonzero()[:5].view(-1).tolist()}"
    ok = same(wts, wts_ref)
    assert ok[cert].all(), f"{what}: certified routing weights differ on {(~ok & cert).sum().item()} pairs"
    near = (wts - wts_ref).abs() <= torch.pow(2.0, torch.floor(torch.log2(wts_ref.abs().clamp_min(1e-30))) - 7)
    assert near[~cert].all(), f"{what}: uncertified routing weights more than one ulp off"
    words, slot = plan_host(sel, E, shard, prev)
    plan = b.plan.cpu()
    want = plan_prefill(b.plan.numel(), prev)
    for i, v in words.items():
        want[i] = v
    bad = (plan != want).nonzero().view(-1)[:8].tolist()
    assert not bad, f"{what}: plan words {bad}: got {plan[bad].tolist()}, want {want[bad].tolist()}"
    assert torch.equal(b.slot.cpu().long(), slot), f"{what}: slots"
    owned = (sel.reshape(-1) % shard[1]) == shard[0]
    xs, row_w = b.xs.cpu(), b.row_w.cpu()
    rows = slot[owned]
    assert_same(xs[rows], d.hn.cpu()[torch.arange(T * k)[owned] // k], f"{what}: gathered rows")
    assert_same(row_w[rows], wts.reshape(-1)[owned], f"{what}: gathered routing weights")
    rest = torch.ones(xs.shape[0], dtype=torch.bool)
    rest[rows] = False
    assert torch.isnan(xs[rest].float()).all() and torch.isnan(row_w[rest].float()).all(), f"{what}: gather wrote rows it does not own"
    return logits, sel, wts, cert, words, slot


def plan_prefill(n: int, prev=(0, 0)) -> torch.Tensor:
    p = torch.full((n,), -7, dtype=torch.int32)
    p[4], p[5] = prev
    return p


def fresh_buffers(T, dim, hidden, E, k, prev=(0, 0)) -> MoeBuffers:
    b = MoeBuffers(T, dim, hidden, E, k, torch.device(DEV), torch.bfloat16)
    nan_fill(b)
    b.plan.copy_(plan_prefill(b.plan.numel(), prev))
    return b


def expert_rows(words: Dict[int, int], E: int):
    return [(e, words[8 + e], words[9 + e]) for e in range(E) if words[9 + e] > words[8 + e]]


def gateup_ref(d: Design, xs: torch.Tensor, rows: torch.Tensor, sel_rows_e: torch.Tensor, dev):
    """g of the live rows `rows` (expert of each in sel_rows_e) from the kernel's xs, float64 on `dev`: (g, certified)."""
    hidden = d.w13[0].shape[0] // 2
    g = torch.empty(len(rows), hidden, dtype=torch.float64, device=dev)
    cert = torch.empty(len(rows), hidden, dtype=torch.bool, device=dev)
    for e in sel_rows_e.unique().tolist():
        m = (sel_rows_e == e).to(dev)
        a = xs[rows[m.cpu()]].to(dev).double()
        w = d.w13[e].to(dev).double()
        assert matmul_exact(a, w).all(), f"gate/up of expert {e}: not an exact fp32 sum"
        y = bf16r(a @ w.T)
        y0, y1 = y[:, 0::2], y[:, 1::2]
        s64 = y0 / (1 + torch.exp(-y0))
        cert[m] = certain(s64) & (y0.abs() < 64)
        g[m] = bf16r(bf16r(s64) * y1)
    return g, cert


def down_ref(d: Design, g: torch.Tensor, row_w: torch.Tensor, rows: torch.Tensor, sel_rows_e: torch.Tensor, dev):
    """yw of the live rows from the kernel's g and row_w: bf16(w * bf16(g W2^T)), exact when the down sums are."""
    dim = d.w2[0].shape[0]
    yw = torch.empty(len(rows), dim, dtype=torch.float64, device=dev)
    for e in sel_rows_e.unique().tolist():
        m = (sel_rows_e == e).to(dev)
        a = g[rows[m.cpu()]].to(dev).double()
        w = d.w2[e].to(dev).double()
        assert matmul_exact(a, w).all(), f"down projection of expert {e}: not an exact fp32 sum"
        yw[m] = bf16r(row_w[rows[m.cpu()]].to(dev).double()[:, None] * bf16r(a @ w.T))
    return yw


def combine_ref(yw: torch.Tensor, slot: torch.Tensor, residual: Optional[torch.Tensor]) -> torch.Tensor:
    """out[t] = bf16(h[t] + r), r = yw[slot(t, 0)], then r = bf16(r + yw[slot(t, j)]) in ascending expert order.  Sums of two bf16
    values are exact in float64, so one rounding restates the kernel's fp32 add + bf16 rounding (two bf16 values whose exponents
    are more than 16 apart leave the larger unchanged either way)."""
    T, k = slot.shape
    r = yw[slot[:, 0]].double()
    for j in range(1, k):
        r = bf16r(r + yw[slot[:, j]].double())
    return bf16r(residual.double() + r) if residual is not None else r


def check_ffn(d: Design, E: int, k: int, b: MoeBuffers, names, out, residual, sel, slot, words, regimes, what: str):
    """Every stage of the grouped FFN on its own input: g from xs, yw from g and row_w, out from yw.  Returns the count of
    uncertified g elements (family X) and of elements.  The float64 products run on the device for big shapes."""
    T, dim = d.hn.shape
    dev = DEV if T * k * dim * d.w13[0].shape[0] > 2 ** 26 else "cpu"
    assert_names(names, regimes + [r"^moe_combine_kernel$"], what)
    xs, g, yw, row_w = b.xs.cpu(), b.g.cpu(), b.yw.cpu(), b.row_w.cpu()
    rows = slot.view(-1)
    sel_e = sel.reshape(-1)
    used = words[1]
    g_ref, cert = gateup_ref(d, xs, rows, sel_e, dev)
    g_live = g[rows].to(dev)
    ok = same(g_live, g_ref)
    assert ok[cert].all(), f"{what}: g differs on {(~ok & cert).sum().item()} certified elements"
    if d.family == "Y":
        assert cert.all(), f"{what}: family Y g must be certified everywhere"
    assert torch.isnan(g[used:].float()).all(), f"{what}: g rows past the plan were written"
    assert torch.isfinite(g[rows].float()).all(), f"{what}: live g rows not written"
    assert torch.isnan(yw[used:].float()).all(), f"{what}: yw rows past the plan were written"
    assert torch.isfinite(yw[rows].float()).all(), f"{what}: live yw rows not written"
    if d.family == "Y":
        assert_same(yw[rows].to(dev), down_ref(d, g, row_w, rows, sel_e, dev), f"{what}: yw")
    assert_same(out[:T].cpu(), combine_ref(yw, slot.view(T, k), residual.cpu() if residual is not None else None).to(torch.bfloat16),
                f"{what}: combine")
    assert torch.isnan(out[T:].float()).all(), f"{what}: out rows past T were written"
    return int((~cert).sum()), cert.numel()


# ----------------------------------------------------------------------------- the cases
E8 = 8


def counts_cluster(T: int) -> List[int]:
    """T * 2 pairs over 8 experts: empty experts 0 and 7, exactly 3 and 4 whole tiles, odd and even tile counts, a ragged tail."""
    c = [0, 3 * 128, 4 * 128, 5 * 128 - 1, 6 * 128 + 1, 0, 0, 0]
    c[5] = min(T, T * 2 - sum(c))
    c[6] = T * 2 - sum(c)
    return c


class GemmCase(NamedTuple):
    name: str
    T: int
    dim: int
    hidden: int
    env: Tuple[Tuple[str, str], ...] = ()
    counts: Optional[Tuple[int, ...]] = None  # per-expert rows (k = 2, E = 8); None: uniform random pairs


GEMM_CASES = [
    GemmCase("streamk-ta32", 16, 256, 256),
    GemmCase("streamk-ta64", 48, 256, 256),
    GemmCase("mixed-ta32", 16, 320, 256),
    GemmCase("mixed-ta64", 60, 448, 256),
    *[GemmCase(f"small-ta{ta}-bn{bn}", T, 256, 256, (("MB200_STREAMK", "0"), ("MB200_GEMM_BN", str(bn))))
      for ta, T in ((32, 30), (64, 64)) for bn in (256, 128, 64, 32)],
    GemmCase("t128-bn256", 200, 256, 256),
    GemmCase("t128-bn128", 129, 384, 192),
    GemmCase("t128-bn64", 300, 320, 256),
    GemmCase("cluster-odd-even", 2500, 256, 256, counts=tuple(counts_cluster(2500))),
    GemmCase("cluster-off", 2500, 256, 256, (("MB200_GEMM_CLUSTER", "0"),), counts=tuple(counts_cluster(2500))),
    GemmCase("blocked-single", 1200, 3328, 1664),
    GemmCase("blocked-cluster", 2400, 3328, 1664),
]


def case_assign(c: GemmCase, k: int = 2) -> torch.Tensor:
    return assign_counts(c.T, list(c.counts)) if c.counts is not None else assign_random(c.T, E8, k, seed=c.T)


def case_regimes(c: GemmCase, k: int = 2) -> List[str]:
    envd = dict(c.env)
    return [gemm_regime(EPI_SWIGLU, c.T, E8, k, 2 * c.hidden, envd), gemm_regime(EPI_MOE_SCALE, c.T, E8, k, c.dim, envd)]


# ----------------------------------------------------------------------------- CPU: the design is exact, the checks are tight
def test_families_are_exact():
    """X: router logits and gate/up pre-activations are exact fp32 sums at the largest K used; Y: g is a +- power of two whose
    SiLU factor is certified, and the down projection is exact at the Mixtral hidden size."""
    for dim in (256, 3328, 4096, 6144):
        hn, gate = design_inputs("X", 64, dim, 16, seed=dim, device="cpu")
        assert matmul_exact(hn.double(), gate.double()).all()
        w13, _ = design_experts("X", dim, 64, 1, seed=dim, device="cpu")
        assert matmul_exact(hn.double(), w13[0].double()).all()
    hn, gate = design_inputs("Y", 16, 4096, 8, seed=3, device="cpu")
    w13, w2 = design_experts("Y", 4096, 14336, 1, seed=3, device="cpu")
    y = hn.double() @ w13[0].double().T
    y0, y1 = y[:, 0::2], y[:, 1::2]
    s = y0 / (1 + torch.exp(-y0))
    assert certain(s).all() and (bf16r(s).abs().log2() % 1 == 0).all()
    g = bf16r(bf16r(s) * y1)
    assert (g.abs().log2() % 1 == 0).all() and g.abs().min() >= 2.0 ** -4 and g.abs().max() <= 2.0
    assert matmul_exact(g, w2[0].double()).all()
    assert len(Y_SILU) >= 3


def test_exactness_proof_is_tight():
    """matmul_exact agrees with accumulation_exact on rows at 2^24 - 1 and 2^24 grid units and one product on a finer grid."""
    unit = 2.0 ** -7
    a = torch.tensor([[unit, -(2.0 ** 23 - 1) * unit] + [2.0 ** 14 * unit] * 512], dtype=torch.float64)
    w = torch.ones(1, a.shape[1], dtype=torch.float64)
    ok = a.clone()
    ok[0, 2] -= unit
    finer = ok.clone()
    finer[0, 0] = unit / 2
    for row, want in ((ok, True), (a, False), (finer, False)):
        assert accumulation_exact(row * w).item() == want and matmul_exact(row, w).item() == want
    # the weight side's grid counts too: a weight of 1/2 halves the unit
    assert not matmul_exact(ok, torch.cat([torch.full((1, 1), 0.5, dtype=torch.float64), w[:, 1:]], 1)).any()


def test_certification_is_tight():
    """certain() accepts a value just over MARGIN from a bf16 rounding boundary and rejects one just inside, on both sides of a
    midpoint and at a power of two (where the spacing below is half the spacing above)."""
    for mid in (1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, 1 - 2.0 ** -9, 0.75 + 2.0 ** -9):
        for side in (-1, 1):
            far = torch.tensor([mid * (1 + side * MARGIN * 1.01)], dtype=torch.float64)
            near = torch.tensor([mid * (1 + side * MARGIN * 0.99)], dtype=torch.float64)
            assert certain(far).item() and not certain(near).item(), (mid, side)
    assert certain(torch.tensor([1.0, 0.0, 1 / 3], dtype=torch.float64)).all()
    assert bf16r(torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8], dtype=torch.float64)).tolist() == [1.0, 1 + 2 * 2.0 ** -7]


def test_family_x_batches_have_router_ties():
    """A realistic family-X batch (T = 1000, dim = 4096) has tokens whose k-th and (k+1)-th bf16 router logits are equal, for every
    E: the natural-routing GPU tests put the tie rule under load."""
    for E in (2, 4, 8, 16):
        hn, gate = design_inputs("X", 1000, 4096, E, seed=E, device="cpu")
        logits = bf16r(hn.double() @ gate.double().T)
        assert sum(int(boundary_tie(logits, k).sum()) for k in ks(E)) > 0, E


def test_cases_reach_every_regime():
    """From the host's own switches (gemm_regime, plan_host), the GEMM cases reach every grouped kernel instantiation the table
    lists, both tile walks with a partial last block and num_n >= GN, and cluster pairs with and without a second tile."""
    seen, walks, seconds = set(), set(), set()
    for c in GEMM_CASES:
        words, _ = plan_host(case_assign(c).sort(1).values, E8)
        for r, N in zip(case_regimes(c), (2 * c.hidden, c.dim)):
            seen.add(r)
            walks.add(walk(words, N, r))
        if words[6]:
            cap = words[2]
            seconds |= {bool(words[PLAN_HEADER + 3 * cap + i] & PAIR_SECOND) for i in range(words[6])}
    want = {rf"^gemm_streamk_grouped_kernel<{m}, {ta}>$" for m in (3, 5) for ta in (32, 64)}
    want |= {rf"^gemm_wgmma_grouped_kernel<3, 1, {bn}, {ta}>$" for bn in (256, 128, 64, 32) for ta in (32, 64)}
    want |= {rf"^gemm_wgmma_grouped_kernel<5, 1, (256|128|64|32), {ta}>$" for ta in (32, 64)}
    want |= {rf"^gemm_wgmma_grouped_kernel<{m}, 1, {bn}, 128>$" for m in (3, 5) for bn in (256, 128)}
    want |= {r"^gemm_wgmma_grouped_kernel<5, 1, 64, 128>$"} | {rf"^gemm_wgmma_grouped_kernel<{m}, 2, 256, 128>$" for m in (3, 5)}
    assert want <= seen, sorted(want - seen)
    assert {"m-fastest", "blocked ragged wide"} <= walks, walks
    assert seconds == {True, False}
    # the blocked walks run in both the single-CTA and the cluster kernel
    blocked = [c for c in GEMM_CASES if "blocked" in c.name]
    assert {case_regimes(c)[0] for c in blocked} == {r"^gemm_wgmma_grouped_kernel<3, 1, 256, 128>$", r"^gemm_wgmma_grouped_kernel<3, 2, 256, 128>$"}
    for c in blocked:
        words, _ = plan_host(case_assign(c).sort(1).values, E8)
        for r, N in zip(case_regimes(c), (2 * c.hidden, c.dim)):
            assert walk(words, N, r) == "blocked ragged wide", (c.name, r)
    # plan and router edges
    assert {p <= 512 for p in (128 * 4, 171 * 3)} == {True, False} and 128 * 4 == 512 and 171 * 3 == 513
    assert {tile_rows_of(T) for T in (32, 33, 64, 65, 128, 129)} == {32, 64, 128}


# ----------------------------------------------------------------------------- GPU: router
def ks(E: int) -> List[int]:
    return sorted({1, 2, E // 2, min(E, 8)})


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [256, 4096, 6144])
@pytest.mark.parametrize("E", [2, 4, 8, 16])
def test_router_exact(E, dim):
    """Natural family-X routing at T on both sides of 256: the selection (ties included) and certified weights exactly."""
    uncertain = total = ties = 0
    for T in (1, 5, 256, 257, 1000):
        d = make_design("X", T, dim, 64, E, seed=T + dim + E, experts=([], []))
        for k in ks(E):
            b = fresh_buffers(T, dim, 64, E, k)
            logits, _, _, cert, _, _ = check_route(d, E, k, b, route(d, E, k, b), f"E={E} dim={dim} T={T} k={k}")
            uncertain += int((~cert).sum())
            total += cert.numel()
            ties += int(boundary_tie(logits, k).sum())
    assert uncertain <= 0.01 * total, f"{uncertain} / {total} routing weights uncertified"
    if dim == 4096 and E >= 4:  # two experts tie rarely: E = 2 gets its ties from test_router_designed_ties
        assert ties > 0, "no router tie at the k boundary: the tie rule went unexercised"


@pytest.mark.gpu
@pytest.mark.parametrize("E", [2, 4, 8, 16])
def test_router_designed_ties(E):
    """Duplicate gate rows, an all-zero gate (experts 0..k-1 at bf16(1/k) each) and a tie straddling the k boundary (code columns:
    k-1 experts at +2, the tied ones at 0, the rest at -2), with both router variants."""
    dim = 256
    for T in (5, 300):
        for k in ks(E):
            # duplicate rows: every expert e >= E/2 copies expert e - E/2
            d = make_design("X", T, dim, 64, E, seed=E + T + k, experts=([], []))
            gate = d.gate.clone()
            gate[E // 2:] = gate[:E - E // 2]
            d = d._replace(gate=gate)
            b = fresh_buffers(T, dim, 64, E, k)
            check_route(d, E, k, b, route(d, E, k, b), f"duplicate rows E={E} T={T} k={k}")
            # all-zero gate
            d = d._replace(gate=torch.zeros_like(gate))
            b = fresh_buffers(T, dim, 64, E, k)
            check_route(d, E, k, b, route(d, E, k, b), f"zero gate E={E} T={T} k={k}")
            assert (b.sel.view(T, k).cpu() == torch.arange(k)).all()
            assert (b.wts.cpu().double() == bf16r(torch.tensor(1.0 / k, dtype=torch.float64))).all()
            if k == E:
                continue
            # tie at the boundary: k - 1 experts win, the next two-or-more tie at zero, the lower indices take the last slots
            gen = torch.Generator().manual_seed(T * k)
            hn = d.hn.clone()
            codes = torch.full((T, E), -2.0)
            for t in range(T):
                p = torch.randperm(E, generator=gen)
                codes[t, p[:k - 1]] = 2.0
                codes[t, p[k - 1:k + 1 + t % max(1, E - k - 1)]] = 0.0
            hn[:, 1:E + 1] = codes.to(torch.bfloat16).to(DEV)
            g2 = torch.zeros_like(gate)
            g2[:, 1:E + 1] = torch.eye(E, dtype=torch.bfloat16, device=DEV)
            d = d._replace(hn=hn, gate=g2)
            b = fresh_buffers(T, dim, 64, E, k)
            logits = check_route(d, E, k, b, route(d, E, k, b), f"boundary tie E={E} T={T} k={k}")[0]
            assert boundary_tie(logits, k).all()


@pytest.mark.gpu
@pytest.mark.parametrize("E", [3, 32])
def test_router_rejects_unsupported_expert_counts(E):
    """E outside {2, 4, 8, 16} is refused with an error before any kernel runs; the buffers stay as they were."""
    T, dim, k = 7, 256, 2
    d = make_design("X", T, dim, 64, min(E, 16), seed=E, experts=([], []))
    gate = torch.zeros(E, dim, dtype=torch.bfloat16, device=DEV)
    b = fresh_buffers(T, dim, 64, min(E, 16), k)
    _abi.launch_log(True)
    try:
        with pytest.raises(_abi.Mb200Error):
            _abi.moe_route(d.hn, gate, E, k, 0, 1, b)
    finally:
        names = _abi.launch_log(False)
    assert names == []
    torch.cuda.synchronize()
    assert (b.sel.cpu() == -1).all() and (b.plan.cpu()[6:].eq(-7)).all()


# ----------------------------------------------------------------------------- GPU: row plan and gather
PLAN_CASES = [
    # name, T, E, k, assignment, shard
    ("pairs-512", 128, 8, 4, "random", (0, 1)),
    ("pairs-513", 171, 8, 3, "random", (0, 1)),
    ("narrow-router-short-plan", 257, 8, 1, "random", (0, 1)),
    *[(f"tile-edge-T{T}", T, 8, 2, "random", (0, 1)) for T in (32, 33, 64, 65, 128, 129)],
    ("two-experts", 600, 8, 2, "two", (0, 1)),
    ("two-experts-short", 100, 4, 2, "two", (0, 1)),
    ("whole-tiles-empty-ends", 512, 8, 2, "whole", (0, 1)),
    ("whole-tiles-empty-ends-t32", 32, 16, 2, "whole", (0, 1)),
    *[(f"shard-{g}of{G}", T, 8, 2, "random", (g, G)) for g, G in ((0, 2), (1, 2), (3, 4)) for T in (40, 700)],
]


def plan_assign(kind: str, T: int, E: int, k: int) -> torch.Tensor:
    if kind == "random":
        return assign_random(T, E, k, seed=T * 31 + k)
    if kind == "two":
        c = [0] * E
        c[1] = c[E - 2] = T
        return assign_counts(T, c)
    tr = tile_rows_of(T)  # "whole": expert 1 fills exactly one tile, expert 2 exactly three, experts 0 and E - 1 empty
    c = [0] * E
    c[1], c[2] = tr, min(3 * tr, T)
    rest = T * k - c[1] - c[2]
    for e in range(3, E - 1):
        c[e] = min(T, rest - sum(c[3:e]) if e == E - 2 else rest // (E - 4))
    assert sum(c) == T * k
    return assign_counts(T, c)


@pytest.mark.gpu
@pytest.mark.parametrize("case", PLAN_CASES, ids=[c[0] for c in PLAN_CASES])
def test_plan_and_gather(case):
    """Every plan word (header, segment starts, tile list, cluster pair list with MOE_PAIR_SECOND, untouched words), the slots,
    and the gathered rows; a second call on the same buffers accumulates the statistics words [4] and [5]."""
    name, T, E, k, kind, shard = case
    dim = 256
    a = plan_assign(kind, T, E, k)
    d = make_design("X", T, dim, 64, E, seed=T + E, assign=a, experts=([], []))
    b = fresh_buffers(T, dim, 64, E, k, prev=(11, 3))
    sel = check_route(d, E, k, b, route(d, E, k, b, shard), name, shard, prev=(11, 3))[1]
    assert torch.equal(sel, a.sort(1).values), f"{name}: the code columns did not pin the routing"
    words, _ = plan_host(sel, E, shard, (11, 3))
    prev = (words[4], words[5])
    nan_fill(b)
    check_route(d, E, k, b, route(d, E, k, b, shard), f"{name} (second call)", shard, prev=prev)


# ----------------------------------------------------------------------------- GPU: grouped GEMMs and combine, small shapes
@pytest.mark.gpu
@pytest.mark.parametrize("case", GEMM_CASES, ids=[c.name for c in GEMM_CASES])
def test_grouped_ffn_regimes(case):
    """Family X (g certified exactly) and family Y (g, yw and out exactly) through the regime the case selects, asserted from the
    launch log; the same routing in every regime.  Family X's g must not depend on the regime: each case also runs with the
    stream-K / cluster switches flipped where that changes the kernel, and compares g bit for bit."""
    k = 2
    a = case_assign(case, k)
    ws = workspace(case.T, case.dim, case.hidden)
    want = case_regimes(case, k)
    h = torch.randn(case.T, case.dim, generator=torch.Generator().manual_seed(5)).to(torch.bfloat16).to(DEV)
    unc = tot = 0
    g_x = None
    for fam in ("X", "Y"):
        d = make_design(fam, case.T, case.dim, case.hidden, E8, seed=case.T + case.dim, assign=a)
        b = fresh_buffers(case.T, case.dim, case.hidden, E8, k)
        with env(**dict(case.env)):
            _, sel, _, _, words, slot = check_route(d, E8, k, b, route(d, E8, k, b), f"{case.name} {fam}")
            names, out = ffn(d, E8, k, b, ws, h)
        u, n = check_ffn(d, E8, k, b, names, out, h, sel, slot.view(case.T, k), words, want, f"{case.name} {fam}")
        unc, tot = unc + u, tot + n
        if fam == "X":
            g_x = b.g.clone()
            flip = {"MB200_STREAMK": "0", "MB200_GEMM_CLUSTER": "0"} if not case.env else {k_: "1" for k_, _ in case.env}
            flip.setdefault("MB200_GEMM_BN", "0")
            with env(**flip):
                names2, _ = ffn(d, E8, k, b, ws, h)
            rows = slot.view(-1)
            assert_same(b.g[rows].cpu(), g_x[rows].cpu(), f"{case.name}: g across regimes {names[:2]} vs {names2[:2]}")
        else:
            y1 = out.clone()
            names2, out2 = ffn(d, E8, k, b, ws, h)  # twice on the same buffers: same bits
            assert_same(out2.cpu(), y1.cpu(), f"{case.name}: second call")
    assert unc <= 0.01 * tot, f"{case.name}: {unc} / {tot} g elements uncertified"


@pytest.mark.gpu
@pytest.mark.parametrize("k", range(1, 9))
def test_combine_every_k(k):
    """k = 1..8 (E = 8, so k = 8 takes every expert), with and without the residual: out bit for bit from the kernel's own yw,
    and yw bit for bit (family Y)."""
    T, dim, hidden = 37, 256, 256
    a = assign_random(T, E8, k, seed=k)
    d = make_design("Y", T, dim, hidden, E8, seed=k, assign=a)
    ws = workspace(T, dim, hidden)
    h = torch.randn(T, dim, generator=torch.Generator().manual_seed(k)).to(torch.bfloat16).to(DEV)
    for residual in (h, None):
        b = fresh_buffers(T, dim, hidden, E8, k)
        _, sel, _, _, words, slot = check_route(d, E8, k, b, route(d, E8, k, b), f"k={k}")
        names, out = ffn(d, E8, k, b, ws, residual)
        check_ffn(d, E8, k, b, names, out, residual, sel, slot.view(T, k), words, case_regimes(GemmCase("", T, dim, hidden), k),
                  f"k={k} residual={residual is not None}")


# ----------------------------------------------------------------------------- GPU: the Mixtral-8x7B expert shape
MIX_DIM, MIX_HIDDEN = 4096, 14336
MIX_T = [16, 64, 300, 2048]
MIX_ENVS = {16: [{}, {"MB200_STREAMK": "0"}, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "128"}],
            64: [{}, {"MB200_STREAMK": "0"}, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "256"}],
            300: [{}],
            2048: [{}, {"MB200_GEMM_CLUSTER": "0"}]}


@pytest.fixture(scope="module")
def mixtral_experts():
    """Family X and family Y experts at 4096 / 14336, E = 8 (~4.7 GB), built once on the device."""
    x = design_experts("X", MIX_DIM, MIX_HIDDEN, E8, seed=77)
    y = design_experts("Y", MIX_DIM, MIX_HIDDEN, E8, seed=78)
    yield {"X": x, "Y": y}
    del x, y
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("T", MIX_T)
def test_mixtral_shape_every_regime(T, mixtral_experts):
    """The real expert shape (224 k blocks in the down projection: split tiles reduced across experts) with natural routing:
    family X g certified exactly, family Y g / yw / out exactly; then every forced regime reproduces g (X) and out (Y) bit for bit."""
    k = 2
    ws = workspace(T, MIX_DIM, MIX_HIDDEN)
    h = torch.randn(T, MIX_DIM, generator=torch.Generator().manual_seed(T)).to(torch.bfloat16).to(DEV)
    for fam in ("X", "Y"):
        d = make_design(fam, T, MIX_DIM, MIX_HIDDEN, E8, seed=T + 5, experts=mixtral_experts[fam])
        b = fresh_buffers(T, MIX_DIM, MIX_HIDDEN, E8, k)
        _, sel, _, cert_w, words, slot = check_route(d, E8, k, b, route(d, E8, k, b), f"mixtral T={T} {fam}")
        first = None
        for e in MIX_ENVS[T]:
            want = [gemm_regime(EPI_SWIGLU, T, E8, k, 2 * MIX_HIDDEN, e), gemm_regime(EPI_MOE_SCALE, T, E8, k, MIX_DIM, e)]
            with env(**e):
                names, out = ffn(d, E8, k, b, ws, h)
            what = f"mixtral T={T} {fam} {e}"
            if first is None:
                u, n = check_ffn(d, E8, k, b, names, out, h, sel, slot.view(T, k), words, want, what)
                assert u <= 0.01 * n, f"{what}: {u} / {n} g elements uncertified"
                first = (b.g.clone(), out.clone())
            else:
                assert_names(names, want + [r"^moe_combine_kernel$"], what)
                rows = slot.view(-1).to(DEV)
                assert_same(b.g[rows].cpu(), first[0][rows].cpu(), f"{what}: g across regimes")
                if fam == "Y":
                    assert_same(out.cpu(), first[1].cpu(), f"{what}: out across regimes")


# ----------------------------------------------------------------------------- GPU: the layer, in blocks
@pytest.mark.gpu
def test_layer_blocks_match_split_and_oracle():
    """MoeLayer.run at T = MOE_BLOCK_TOKENS + 37 (two blocks) equals the two blocks run separately, is the same on a second call,
    and equals the oracle's MoE (moe.py:24-32, family Y) on every token without a router tie at the k boundary whose weights
    are certified."""
    from mistral_inference_b200.args import MoeArgs
    from mistral_inference_b200.transformer_layers import FeedForward

    T, dim, hidden, k = MOE_BLOCK_TOKENS + 37, 256, 256, 2
    d = make_design("Y", T, dim, hidden, E8, seed=9)
    experts = {}
    for e in range(E8):
        ff = FeedForward(dim, hidden)
        ff.w13 = torch.nn.Parameter(d.w13[e], requires_grad=False)
        ff.w2_weight = torch.nn.Parameter(d.w2[e], requires_grad=False)
        experts[e] = ff
    layer = MoeLayer(experts, torch.nn.Parameter(d.gate, requires_grad=False), MoeArgs(num_experts=E8, num_experts_per_tok=k))
    ws = workspace(MOE_BLOCK_TOKENS, dim, hidden)
    h = torch.randn(T, dim, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).to(DEV)
    names = launched_kernels(lambda: layer.run(d.hn, h, ws))
    assert names.count("moe_combine_kernel") == 2 and names.count("moe_plan_kernel<scan>") == 1, names  # 37 tokens: short plan
    assert names.count("moe_plan_kernel<short>") == 1, names
    whole = layer.run(d.hn, h, ws)
    again = layer.run(d.hn, h, ws)
    split = torch.cat([layer.run(d.hn[:MOE_BLOCK_TOKENS], h[:MOE_BLOCK_TOKENS], ws), layer.run(d.hn[MOE_BLOCK_TOKENS:], h[MOE_BLOCK_TOKENS:], ws)])
    torch.cuda.synchronize()
    assert_same(again.cpu(), whole.cpu(), "second call")
    assert_same(split.cpu(), whole.cpu(), "blocks run separately")
    x, gate = d.hn.cpu(), d.gate.cpu()
    logits = router_logits(d)
    _, _, cert = route_rule(logits, k)
    ok = ~boundary_tie(logits, k) & cert.all(1)
    assert ok.float().mean() > 0.9
    oracle = [(d.w13[e][0::2].cpu(), d.w2[e].cpu(), d.w13[e][1::2].cpu()) for e in range(E8)]
    want = h.cpu() + R.moe_forward(x, gate, oracle, k)
    assert_same(whole.cpu()[ok], want[ok], "layer vs oracle")
