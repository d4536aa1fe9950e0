"""The decode megakernel's projections, MoE stage and lm head (csrc/decode_megakernel.cuh, phases 1, 3, 4, 5 and the final norm +
lm head + fused argmax), bit for bit, at the pair, group and K-chunk edges of the device the test runs on.

Each [N, K] matrix is dealt to the G CTAs (one per SM) as contiguous ranges of row pairs, CTA c owning pairs [c*P/G, (c+1)*P/G)
with P = N/2, taken in groups of up to 8 pairs (one per consumer warp); K is cut into nch = ceil(K / 4096) chunks of K/nch
elements.  `cta_pairs` and `n_chunks` restate that arithmetic and every grid below is built from G.

Exact by construction.  Every matrix row is *designed*: a target value at one column (two, when the target is not a bf16
number), plus cancelling pairs w*x[a] - w*x[a] whose members sit in different K chunks wherever there are several.  Activations
are powers of two with a sign (the residual stream is +-0.5, so each RMSNorm gives exactly +-norm_w), so every product lies on a
common grid 2^-e and `accumulation_exact` proves on the host, per output row, that sum |w x| < 2^(24 - e) grid units: every fp32
accumulation of the step is exact in any order and a correct kernel can only differ from the oracle in its rounding points.  A
dropped, duplicated or shifted chunk breaks a cancellation; a store the kernel never makes stays NaN (the x, h, q, attention and
g buffers and the logits are NaN-filled before each launch).  Every visible ring slot holds the fresh key and value, so every P
is exactly 1 and the attention output is exactly v, with q != 0 so that RoPE runs on real values; some q pairs are chosen
(`fma_sensitive_pairs`) so that a fused multiply-add in the RoPE epilogue would change their bits.

Each phase is compared with the oracle applied to the kernel's own input of that phase, read back from the workspace
(`_abi.decode_buffers`), so an error shows in the phase that makes it:
  q and the fresh K / V row      <- x_in (the embedding row, or the previous layer's output)
  attention output               <- the fresh V row
  h = x_in + wo(attn)            <- the kernel's attention output and x_in
  g = silu(w1 hn) * w3 hn        <- the kernel's h (per selected expert for MoE)
  x_out = h + w2 g (MoE: the     <- the kernel's g and h
          weighted bf16 += in ascending expert index)
  logits, next_token             <- the kernel's final residual (the ping-pong half the final norm reads)
The matrix products of the oracle (F.linear) are, with every accumulation exact, the exact sum rounded once to bf16, which is what
`matvec` computes from the sparse design.  The gate pre-activations are picked (float64, `silu_targets`) so that bf16(silu) is
a power of two at least 2^-12 relative away from a rounding boundary; the selected router logits are equal, so every routing
weight is exactly 1/k (the one case with distinct logits checks its weights on the host in float64 the same way).
"""
import math
from typing import List, NamedTuple, Optional

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.rope import precompute_freqs_cis
from oracle import restatement as R

from .test_gpu_megakernel_attention import G_PCIE, G_SXM, rope_fp32
from .util import assert_bf16_close, assert_launched, launched_kernels, oracle_args

DEV = "cuda"
HD = 128
EPS = 1e-5
MAX_KC = 4096          # MK_MAX_KC: elements of one row chunk
GROUP = 8              # pairs per group (consumer warps)
ROPE_LEN = 4096
MK = r"decode_megakernel"
NAN = float("nan")


# ----------------------------------------------------------------------------- the CTA partition (cut_matrix restated)
def n_chunks(K: int) -> int:
    return -(-K // MAX_KC)


def cut_ok(K: int) -> bool:
    return K % (n_chunks(K) * 8) == 0


def cta_pairs(P: int, G: int) -> np.ndarray:
    """Pairs of every CTA: CTA c owns [c*P/G, (c+1)*P/G)."""
    c = np.arange(G + 1, dtype=np.int64)
    b = c * P // G
    return b[1:] - b[:-1]


def cta_first_pair(P: int, G: int, c: int) -> int:
    return c * P // G


class Shape(NamedTuple):
    name: str
    dim: int
    hidden: int
    H: int
    KV: int
    vocab: int
    E: int = 0
    k: int = 0

    def matrices(self):
        """(kind, N, K) of every matrix the step streams."""
        q_dim = self.H * HD
        return [("qkv", q_dim + 2 * self.KV * HD, self.dim), ("wo", self.dim, q_dim), ("gateup", 2 * self.hidden, self.dim),
                ("down", self.dim, self.hidden), ("lm", self.vocab, self.dim)]


REAL = {
    "mistral-7b": Shape("mistral-7b", 4096, 14336, 32, 8, 32000),
    "nemo-12b": Shape("nemo-12b", 5120, 14336, 32, 8, 131072),
    "mixtral-8x7b": Shape("mixtral-8x7b", 4096, 14336, 32, 8, 32000, 8, 2),
    "mixtral-8x22b": Shape("mixtral-8x22b", 6144, 16384, 48, 8, 32768, 8, 2),
}


def nearest(target: int, allowed) -> int:
    return min(allowed, key=lambda v: (abs(v - target), v))


def pair_targets(G: int, lm: bool = False) -> List[int]:
    t = [G - 4, G, G + 4, 8 * G - 4, 8 * G + 4]
    return t + ([G - 1, G + 1, 8 * G + 1] if lm else [])


def pair_shapes(G: int) -> List[Shape]:
    """Small shapes whose pair counts sit at G - 4, G, G + 4, 8G +- 4 (lm head also G +- 1, 8G + 1) for every matrix kind, at the
    nearest value the shape rules allow: wo / down P = dim/2 with dim % 8 == 0; gate/up P = hidden with hidden % 8 == 0
    (and 16-byte chunks); QKV P = (H + 2KV) * 64."""
    out = []
    dims = [nearest(2 * p, [d for d in range(8, 20000, 8) if cut_ok(d)]) for p in pair_targets(G)]
    hiddens = [nearest(p, [h for h in range(8, 20000, 8) if cut_ok(h)]) for p in pair_targets(G)]
    heads = [QKV_HEADS[nearest(p, list(QKV_HEADS))] for p in pair_targets(G)]
    vocabs = [2 * p for p in pair_targets(G, lm=True)]
    for i, v in enumerate(vocabs):
        H, KV = heads[i % len(heads)]
        out.append(Shape(f"pairs{i}", dims[i % len(dims)], hiddens[(i + 2) % len(hiddens)], H, KV, v))
    # the nearest QKV P to 8G + 4 can fall below 8G: also the first one above, for a trailing group of one pair
    H, KV = QKV_HEADS[min(p for p in QKV_HEADS if p > 8 * G)]
    out.append(Shape("pairs-trailing", dims[0], 8 * G + 8, H, KV, vocabs[0]))  # and gate/up P = hidden just above 8G
    return out


# QKV pair count (H + 2 KV) * 64 -> (H, KV) for every compiled head ratio and KV <= 8
QKV_HEADS = {}
for _kv in range(8, 0, -1):
    for _rep in (8, 6, 4, 2, 1):
        QKV_HEADS[(_kv * _rep + 2 * _kv) * 64] = (_kv * _rep, _kv)


def chunk_shapes() -> List[Shape]:
    """dim / hidden / q_dim at one full chunk (4096), two chunks of 2056 (not a multiple of 32 lanes x 8), three chunks (8208),
    several full chunks (12288, 16384), four chunks of 3584 (14336); q_dim at 4096, 5120 (2 x 2560) and 8192."""
    return [Shape("K4112-4096", 4112, 4096, 32, 8, 256), Shape("K4096-4112", 4096, 4112, 40, 5, 256),
            Shape("K8208-14336", 8208, 14336, 64, 8, 256), Shape("K12288-8208", 12288, 8208, 8, 8, 256),
            Shape("K16384-12288", 16384, 12288, 16, 8, 256), Shape("K1024-16384", 1024, 16384, 8, 4, 256)]


def rep_shapes() -> List[Shape]:
    """Every compiled head ratio (1, 2, 4, 6, 8), with 8, 2 and 5 KV heads."""
    return [Shape(f"rep{r}-kv{kv}", 512, 1024, kv * r, kv, 1024) for kv, r in ((8, 1), (2, 2), (8, 4), (2, 6), (5, 8), (1, 8))]


def max_hidden_k4(dim: int = 1024) -> int:
    """The largest hidden (16-byte chunks) at which k = 4 experts still leave a ring of >= 9 stages on the current device."""
    best = None
    for h in range(8, 40000, 8):
        if cut_ok(h) and _abi.decode_step_unsupported(dim, h, 8, 8, HD, 256, 4, 4) is None:
            best = h
    return best


# ----------------------------------------------------------------------------- designed rows and the exactness check
class Design(NamedTuple):
    """A sparse [N, K] matrix: row n has values val[n] at columns idx[n] (distinct), zero elsewhere."""
    idx: torch.Tensor  # [N, m] int64
    val: torch.Tensor  # [N, m] float64, every value a bf16 number


def is_pow2(x: torch.Tensor) -> torch.Tensor:
    m, _ = torch.frexp(x.abs())
    return (x != 0) & (m == 0.5)


def design_rows(x: torch.Tensor, hi: torch.Tensor, lo: Optional[torch.Tensor], gen: torch.Generator, n_pairs: int = 3) -> Design:
    """Rows whose product with x (float64 [K], usable where x is +-2^a) is exactly hi + lo: hi at one column, lo at a second,
    and `n_pairs` cancelling pairs (w at column a, -w x[a] / x[b] at column b) with a and b in different K chunks (when K has
    several), the first pair always reaching into the last chunk."""
    K = x.numel()
    N = hi.numel()
    nch = n_chunks(K)
    kc = K // nch
    usable = [torch.nonzero(is_pow2(x[c * kc:(c + 1) * kc])).flatten() + c * kc for c in range(nch)]
    assert all(len(u) >= 2 * n_pairs + 2 for u in usable), "too few power-of-two columns in a chunk"
    slots = [(int(torch.randint(nch, (1,), generator=gen)), "hi"), (nch - 1, "lo")]
    for p in range(n_pairs):
        a = nch - 1 if p == 0 else int(torch.randint(nch, (1,), generator=gen))
        b = (a + 1 + int(torch.randint(max(nch - 1, 1), (1,), generator=gen))) % nch if nch > 1 else 0
        slots += [(a, "pa"), (b, "pb")]
    # distinct columns per row: slot s of chunk ch takes usable entry (u_row + j * stride) of that chunk
    per_chunk = {}
    cols = []
    for ch, _ in slots:
        j = per_chunk.get(ch, 0)
        per_chunk[ch] = j + 1
        u = usable[ch]
        stride = max(1, len(u) // (len(slots) + 1))
        start = torch.randint(len(u), (N,), generator=gen)
        cols.append((ch, j, stride, u))
    base = torch.randint(1 << 30, (N,), generator=gen)
    idx = torch.empty(N, len(slots), dtype=torch.long)
    for s, (ch, j, stride, u) in enumerate(cols):
        idx[:, s] = u[(base + j * stride) % len(u)]
    val = torch.zeros(N, len(slots), dtype=torch.float64)
    val[:, 0] = hi / x[idx[:, 0]]
    val[:, 1] = (lo if lo is not None else torch.zeros(N, dtype=torch.float64)) / x[idx[:, 1]]
    for p in range(n_pairs):
        a, b = 2 + 2 * p, 3 + 2 * p
        w = torch.where(torch.rand(N, generator=gen) < 0.5, -1.0, 1.0).double()
        val[:, a] = w
        val[:, b] = -w * x[idx[:, a]] / x[idx[:, b]]
    assert torch.equal(val.to(torch.bfloat16).double(), val), "a designed weight is not a bf16 number"
    srt = idx.sort(1).values
    assert (srt[:, 1:] != srt[:, :-1]).all(), "designed columns collide"
    return Design(idx, val)


def lsb_exponent(p: torch.Tensor) -> torch.Tensor:
    """Exponent of the lowest set bit of every nonzero float64 p (p = odd * 2^result)."""
    m, e = torch.frexp(p.abs())
    i = (m * 2.0 ** 53).to(torch.int64)
    tz = torch.log2((i & -i).double()).round().to(torch.int64)
    return e.to(torch.int64) - 53 + tz


def accumulation_exact(prod: torch.Tensor) -> torch.Tensor:
    """Per row of products [N, m] (float64, each exact): every product lies on the grid 2^-e of the row's finest one and
    sum |p| < 2^(24 - e), i.e. the sum has fewer than 24 significant bits in grid units and fp32 computes it exactly in any order."""
    nz = prod != 0
    lsb = torch.where(nz, lsb_exponent(torch.where(nz, prod, torch.ones_like(prod))), torch.full_like(prod, 1 << 20, dtype=torch.int64))
    e = -lsb.min(1).values
    units = prod.abs().sum(1) * torch.pow(2.0, e.double())
    return (units < 2.0 ** 24) | ~nz.any(1)


def products(d: Design, x: torch.Tensor) -> torch.Tensor:
    return d.val * x.double()[d.idx]


def matvec(d: Design, x: torch.Tensor) -> torch.Tensor:
    """The exact product of the designed matrix and x (float64; exact whenever accumulation_exact holds)."""
    return products(d, x).sum(1)


def dense(d: Design, K: int) -> torch.Tensor:
    w = torch.zeros(d.idx.shape[0], K, dtype=torch.bfloat16, device=DEV)
    w.scatter_(1, d.idx.to(DEV), d.val.to(torch.bfloat16).to(DEV))
    return w


def bf(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16)


def silu_targets():
    """bf16 gate pre-activations a with bf16(silu(a)) a power of two (positive or negative) and silu(a) at least 2^-12
    (relative) away from a bf16 rounding boundary, in float64."""
    a = torch.arange(-2048, 2048, dtype=torch.float64) / 256.0
    a = a[bf(a).double() == a]
    s = a / (1 + torch.exp(-a))
    r = bf(s).double()
    ulp = torch.pow(2.0, torch.floor(torch.log2(r.abs().clamp_min(1e-30))) - 7)
    margin = (ulp / 2 - (s - r).abs()) / r.abs().clamp_min(1e-30)
    ok = is_pow2(r) & (margin > 2.0 ** -12) & (r.abs() >= 2.0 ** -4)
    return a[ok], r[ok]


SILU_A, SILU_S = silu_targets()


def fma_sensitive_pairs(pos: int, table: torch.Tensor) -> dict:
    """{frequency i: (a, b)}: small integers whose RoPE product at `pos` rounds to different bf16 values when re = ac - bd or
    im = ad + bc is computed with a fused multiply-add instead of two rounded products (float64 emulates the fused form)."""
    cd = torch.view_as_real(table[pos]).numpy().astype(np.float32)
    v = np.arange(-127, 128, dtype=np.float32)
    a, b = np.meshgrid(v, v, indexing="ij")
    out = {}
    for i in range(HD // 2):
        c, d = cd[i, 0], cd[i, 1]
        plain = [np.float32(a * c) - np.float32(b * d), np.float32(a * d) + np.float32(b * c)]
        fused = [(a.astype(np.float64) * c - np.float32(b * d)).astype(np.float32), (a.astype(np.float64) * d + np.float32(b * c)).astype(np.float32)]
        diff = np.zeros(a.shape, dtype=bool)
        for x, y in zip(plain, fused):
            diff |= bf(torch.from_numpy(np.ascontiguousarray(x))).view(torch.int16).numpy() != bf(torch.from_numpy(np.ascontiguousarray(y))).view(torch.int16).numpy()
        hit = np.argwhere(diff)
        if len(hit):
            j, k = hit[len(hit) // 2]
            out[i] = (int(v[j]), int(v[k]))
    return out


# ----------------------------------------------------------------------------- the synthetic model
class Step:
    """One decode step of a designed model on the device: weights, ring caches, pointers; `launch()` runs decode_step once."""

    def __init__(self, s: Shape, n_layers: int, pos: int, W: int, gen: torch.Generator, routes=None, probes: bool = True,
                 lm_targets: Optional[torch.Tensor] = None, router_logits=None):
        self.s, self.L, self.pos, self.W = s, n_layers, pos, W
        self.gen = gen
        dim, hidden, H, KV = s.dim, s.hidden, s.H, s.KV
        q_dim, kv_dim = H * HD, KV * HD
        self.table = precompute_freqs_cis(HD, ROPE_LEN, 1e6)
        self.rope_dev = torch.view_as_real(self.table).contiguous().to(DEV)
        sign = lambda n: torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0).double()  # noqa: E731
        pow2 = lambda n: torch.pow(2.0, torch.randint(-1, 2, (n,), generator=gen).double())  # noqa: E731
        self.x0 = 0.5 * sign(dim)
        self.emb = bf(self.x0)[None].to(DEV)
        self.layers, self.x_out = [], []
        # probes (rows whose down sum is not a bf16 number) keep the final norm's sum of squares exact only while dim < 4096
        probes = probes and dim < 4096
        self.routes = routes or [None] * n_layers
        self.router_logits = router_logits
        self.expert_ptr_w13, self.expert_ptr_w2, self.gates = [], [], []
        self._keep = []
        nan_w13 = torch.full((2 * hidden, dim), NAN, dtype=torch.bfloat16, device=DEV) if s.E else None
        nan_w2 = torch.full((dim, hidden), NAN, dtype=torch.bfloat16, device=DEV) if s.E else None
        x = self.x0
        n = min(pos + 1, W)
        for l in range(n_layers):
            last = l == n_layers - 1
            an, fn = pow2(dim), pow2(dim)
            xn = torch.sign(x) * an  # rms of +-0.5 is 0.5: the normed input is exactly +-1 * norm weight
            qk_t = torch.randint(-12, 13, (q_dim + kv_dim,), generator=gen).double()
            sens = fma_sensitive_pairs(pos, self.table)
            assert sens, f"no q pair at position {pos} whose RoPE result depends on FMA contraction"
            for i, (a, b) in sens.items():  # in every q head: a fused multiply-add in the RoPE epilogue changes these bits
                qk_t[torch.arange(H) * HD + 2 * i] = float(a)
                qk_t[torch.arange(H) * HD + 2 * i + 1] = float(b)
            v_t = sign(kv_dim) * pow2(kv_dim)
            d_qkv = design_rows(xn, torch.cat([qk_t, v_t]), None, gen)
            qkv = bf(torch.cat([qk_t, v_t]))
            k_rot = rope_fp32(qkv[q_dim:q_dim + kv_dim], pos, self.table)
            v = qkv[q_dim + kv_dim:]
            attn = v.view(KV, HD).repeat_interleave(H // KV, 0).reshape(-1).double()
            ck = torch.full((1, W, KV, HD), NAN, dtype=torch.bfloat16)
            cv = ck.clone()
            ck[0, :n] = k_rot.view(KV, HD)
            cv[0, :n] = v.view(KV, HD)
            ck[0, pos % W] = NAN
            cv[0, pos % W] = NAN
            h_t = 0.5 * sign(dim)
            d_wo = design_rows(attn, h_t - x, None, gen)
            h = h_t
            hn = torch.sign(h) * fn
            layer = {"qkv": d_qkv, "wo": d_wo, "an": an, "fn": fn, "ck": ck.to(DEV), "cv": cv.to(DEV)}
            x_t = 0.5 * sign(dim)
            if s.E == 0:
                d_w13, g = self._gateup(hn, gen)
                lo = None
                t = x_t - h
                if last and probes:
                    # rounding probes: bf16(bf16(t) + h) != bf16(t + h); x_out = +-0.5078125 there
                    rows = torch.randperm(dim, generator=gen)[:8]
                    t[rows] = -torch.sign(h[rows]) * 1.0
                    lo = torch.zeros(dim, dtype=torch.float64)
                    lo[rows] = -torch.sign(h[rows]) * 5 * 2.0 ** -10
                d_w2 = design_rows(g, t, lo, gen)
                layer.update({"w13": d_w13, "w2": d_w2})
                w13_dev, w2_dev = dense(d_w13, dim), dense(d_w2, hidden)
            else:
                sel = self.routes[l]
                k = s.k
                logits_t = torch.full((s.E,), -1.0, dtype=torch.float64)
                logits_t[torch.arange(s.E)] = -1.0 - torch.arange(s.E).double() / 16  # distinct, all below the selected
                if router_logits is not None and router_logits[l] is not None:
                    logits_t = router_logits[l].double()
                else:
                    logits_t[list(sel)] = 1.0
                d_gate = design_rows(hn, logits_t, None, gen, n_pairs=2)
                w = 1.0 / k
                d_w13s, d_w2s, gs = {}, {}, {}
                ys = []
                t = x_t - h  # res must equal t: sum_j bf16(w * y_j) in ascending index, every partial sum exact
                for j, e in enumerate(sorted(sel)):
                    d13, g = self._gateup(hn, gen)
                    gs[e] = g
                    d_w13s[e] = d13
                    if j < k - 1:
                        y = sign(dim) * torch.pow(2.0, torch.randint(0, 3, (dim,), generator=gen).double())
                    else:
                        y = (t - w * sum(ys)) / w if ys else t / w
                    ys.append(y)
                    d_w2s[e] = design_rows(g, y, None, gen)
                layer.update({"gate": d_gate, "w13s": d_w13s, "w2s": d_w2s})
                gate_dev = dense(d_gate, dim)
                p13 = [nan_w13.data_ptr()] * s.E
                p2 = [nan_w2.data_ptr()] * s.E
                for e in sel:
                    a, b = dense(d_w13s[e], dim), dense(d_w2s[e], hidden)
                    self._keep += [a, b]
                    p13[e], p2[e] = a.data_ptr(), b.data_ptr()
                self.gates.append(gate_dev)
                self.expert_ptr_w13 += p13
                self.expert_ptr_w2 += p2
                w13_dev = w2_dev = None
            qkv_dev, wo_dev = dense(d_qkv, dim), dense(d_wo, q_dim)
            an_dev, fn_dev = bf(an).to(DEV), bf(fn).to(DEV)
            self._keep += [qkv_dev, wo_dev, an_dev, fn_dev, w13_dev, w2_dev]
            layer["dev"] = [qkv_dev.data_ptr(), wo_dev.data_ptr(), w13_dev.data_ptr() if w13_dev is not None else 0,
                            w2_dev.data_ptr() if w2_dev is not None else 0, an_dev.data_ptr(), fn_dev.data_ptr(),
                            layer["ck"].data_ptr(), layer["cv"].data_ptr()]
            self.layers.append(layer)
            x = x_t.clone()
            if s.E == 0 and last and probes:
                x[rows] = torch.where(h[rows] < 0, 0.5078125, -0.5078125).double()
            self.x_out.append(x)
        self._keep += [nan_w13, nan_w2]
        # final norm + lm head: designed on the normed final residual, at its power-of-two columns
        self.final_norm = pow2(dim)
        xf = R.rms_norm(bf(x)[None], bf(self.final_norm), EPS)[0].double()
        if lm_targets is None:
            lm_targets = torch.randint(-64, 64, (s.vocab,), generator=gen).double() / 4
        self.d_lm = design_rows(xf, lm_targets, None, gen, n_pairs=2)
        self.w_out = dense(self.d_lm, dim)
        self.fn_dev = bf(self.final_norm).to(DEV)
        self.desc = torch.tensor([l["dev"] for l in self.layers], dtype=torch.int64, device=DEV)
        self.win = torch.tensor([W] * n_layers, dtype=torch.int32, device=DEV)
        self.token = torch.zeros(1, dtype=torch.long, device=DEV)
        self.logits = torch.full((s.vocab,), NAN, dtype=torch.float32, device=DEV)
        self.next = torch.full((1,), -1, dtype=torch.long, device=DEV)
        self.ws = _abi.Workspace(_abi.workspace_bytes(1, dim, H, KV, HD, hidden, s.vocab, 1), torch.device(DEV))
        self.sc = _abi.decode_buffers(dim, hidden, H, KV, HD, s.E, s.k)
        if s.E:
            self.gate_tab = torch.tensor([g.data_ptr() for g in self.gates], dtype=torch.int64, device=DEV)
            self.w13_tab = torch.tensor(self.expert_ptr_w13, dtype=torch.int64, device=DEV)
            self.w2_tab = torch.tensor(self.expert_ptr_w2, dtype=torch.int64, device=DEV)

    def _gateup(self, hn: torch.Tensor, gen: torch.Generator):
        """Interleaved w1 / w3 rows: gate pre-activations from SILU_TARGETS, up values +-1 or +-0.5; g = bf16(silu) * up."""
        hidden = self.s.hidden
        pick = torch.randint(len(SILU_A), (hidden,), generator=gen)
        up = torch.where(torch.rand(hidden, generator=gen) < 0.5, -1.0, 1.0).double() * torch.pow(2.0, -torch.randint(0, 2, (hidden,), generator=gen).double())
        t = torch.stack([SILU_A[pick], up], 1).reshape(-1)
        return design_rows(hn, t, None, gen), SILU_S[pick] * up

    def buf(self, off: int, n: int) -> torch.Tensor:
        return self.ws.buf[off:off + 2 * n].view(torch.bfloat16)

    def launch(self):
        s = self.s
        for off, n in ((self.sc.x, 2 * s.dim), (self.sc.h, s.dim), (self.sc.q, s.H * HD), (self.sc.attn, s.H * HD),
                       (self.sc.g, (s.k if s.E else 1) * s.hidden)):
            self.buf(off, n).fill_(NAN)
        self.logits.fill_(NAN)
        kw = {}
        if s.E:
            kw = dict(n_experts=s.E, top_k=s.k, moe_gate=self.gate_tab, moe_w13=self.w13_tab, moe_w2=self.w2_tab)
        _abi.decode_step(self.desc, self.win, self.L, self.emb, self.fn_dev, self.w_out, self.rope_dev, self.token, self.pos, 0,
                         self.logits, self.next, s.dim, s.hidden, s.H, s.KV, HD, s.vocab, EPS, self.ws, **kw)

    def read(self):
        s = self.s
        torch.cuda.synchronize()
        x = self.buf(self.sc.x, 2 * s.dim).cpu().view(2, s.dim)
        return {"x": x, "h": self.buf(self.sc.h, s.dim).cpu(), "q": self.buf(self.sc.q, s.H * HD).cpu(),
                "attn": self.buf(self.sc.attn, s.H * HD).cpu(), "g": self.buf(self.sc.g, (s.k if s.E else 1) * s.hidden).cpu().view(-1, s.hidden),
                "logits": self.logits.cpu(), "next": int(self.next.item()),
                "ck": [l["ck"][0, self.pos % self.W].cpu() for l in self.layers],
                "cv": [l["cv"][0, self.pos % self.W].cpu() for l in self.layers]}


# ----------------------------------------------------------------------------- the oracle, phase by phase, on the kernel's inputs
def same_bits(got: torch.Tensor, want: torch.Tensor, what: str):
    got, want = bf(got.float()).reshape(-1), bf(want.float()).reshape(-1)
    bad = got.view(torch.int16) != want.view(torch.int16)
    if bad.any():
        i = int(torch.nonzero(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at {i}: got {got[i].item()!r}, want {want[i].item()!r}")


def check_exact(d: Design, x: torch.Tensor, what: str):
    ok = accumulation_exact(products(d, x))
    assert ok.all(), f"{what}: the design is not exact on {int((~ok).sum())} rows"


def check_step(st: Step, out, what: str):
    s, L = st.s, st.L
    q_dim, kv_dim = s.H * HD, s.KV * HD
    if L >= 2:  # the other ping-pong half: layer L-2's output, the last layer's input
        same_bits(out["x"][(L - 1) & 1], st.x_out[L - 2], f"{what} x_out of layer {L - 2}")
    for l in range(L):  # the ring row of every layer; q / attention / h / g of the last
        lay = st.layers[l]
        last = l == L - 1
        # the input of a middle layer is overwritten before the step ends: its design stands in for it
        x_in = st.x0 if l == 0 else (out["x"][(L - 1) & 1].double() if last else st.x_out[l - 1])
        assert accumulation_exact((bf(x_in).double() ** 2)[None]).all(), f"{what} L{l}: the attention norm's sum of squares is not exact"
        xn = R.rms_norm(bf(x_in)[None], bf(lay["an"]), EPS)[0].double()
        check_exact(lay["qkv"], xn, f"{what} L{l} qkv")
        y = bf(matvec(lay["qkv"], xn))
        same_bits(out["ck"][l].reshape(-1), rope_fp32(y[q_dim:q_dim + kv_dim], st.pos, st.table), f"{what} L{l} k row")
        same_bits(out["cv"][l].reshape(-1), y[q_dim + kv_dim:], f"{what} L{l} v row")
        if not last:
            continue
        same_bits(out["q"], rope_fp32(y[:q_dim], st.pos, st.table), f"{what} q")
        v = out["cv"][l].reshape(s.KV, HD)
        same_bits(out["attn"], v.repeat_interleave(s.H // s.KV, 0), f"{what} attention output")
        a = out["attn"].double()
        check_exact(lay["wo"], a, f"{what} wo")
        h = bf(bf(matvec(lay["wo"], a)).double() + bf(x_in).double())
        same_bits(out["h"], h, f"{what} h")
        hk = out["h"].double()
        assert accumulation_exact((hk ** 2)[None]).all(), f"{what}: the ffn norm's sum of squares is not exact"
        hn = R.rms_norm(bf(hk)[None], bf(lay["fn"]), EPS)[0]
        if s.E == 0:
            check_exact(lay["w13"], hn.double(), f"{what} w13")
            pre = bf(matvec(lay["w13"], hn.double())).view(-1, 2)
            g = bf(F.silu(pre[:, 0]) * pre[:, 1])
            same_bits(out["g"][0], g, f"{what} g")
            gk = out["g"][0].double()
            check_exact(lay["w2"], gk, f"{what} w2")
            xo = bf(bf(matvec(lay["w2"], gk)).double() + hk)
        else:
            logits = bf(matvec(lay["gate"], hn.double()))
            sel, wts = route_rule(logits, s.k)
            assert sel == sorted(st.routes[l]), f"{what}: the designed route {st.routes[l]} is not the rule's {sel}"
            res = None
            for j, e in enumerate(sel):
                pre = bf(matvec(lay["w13s"][e], hn.double())).view(-1, 2)
                g = bf(F.silu(pre[:, 0]) * pre[:, 1])
                same_bits(out["g"][j], g, f"{what} g of expert {e} (slot {j})")
                y = bf(matvec(lay["w2s"][e], out["g"][j].double()))
                t = bf(wts[j] * y)
                res = t if res is None else bf(res + t)  # moe.py:29-31, ascending expert index
            xo = bf(hk + res.double())
        same_bits(out["x"][L & 1], xo, f"{what} x_out of layer {L - 1}")
    xf = out["x"][L & 1].double()
    assert accumulation_exact((xf ** 2)[None]).all(), f"{what}: the final norm's sum of squares is not exact"
    xfn = R.rms_norm(bf(xf)[None], bf(st.final_norm), EPS)[0].double()
    check_exact(st.d_lm, xfn, f"{what} lm head")
    want = bf(matvec(st.d_lm, xfn)).float()
    same_bits(out["logits"], want, f"{what} logits")
    assert out["next"] == int(want.argmax()), f"{what}: next_token {out['next']} != argmax {int(want.argmax())}"


def route_rule(logits: torch.Tensor, k: int):
    """The documented routing rule: top-k of the bf16 logits, ties to the lower expert index; fp32 softmax over the k, rounded to
    bf16; returned in ascending expert index."""
    order = sorted(range(logits.numel()), key=lambda e: (-float(logits[e]), e))[:k]
    w = bf(torch.softmax(logits[order].float(), 0))
    pairs = sorted(zip(order, w.tolist()))
    return [e for e, _ in pairs], [torch.tensor(v, dtype=torch.bfloat16) for _, v in pairs]


def run_case(s: Shape, n_layers: int, seed: int, pos: int = 37, W: int = 64, **kw):
    st = Step(s, n_layers, pos, W, torch.Generator().manual_seed(seed), **kw)
    rep = s.H // s.KV
    assert_launched(st.launch, rf"decode_megakernel<{rep}>", MK, 1)
    out = st.read()
    check_step(st, out, f"{s.name} L={n_layers}")
    return st, out


# ----------------------------------------------------------------------------- CPU: the grid reaches every edge, the check is tight
@pytest.mark.parametrize("G", [G_SXM, G_PCIE])
def test_grid_reaches_pair_and_chunk_edges(G):
    """For G = 132 and 114: every matrix kind has P at G - 4, G, G + 4 and 8G +- 4 (lm head also G +- 1, 8G + 1), or the nearest
    P the shape rules allow, so the grid has CTAs with no pair (P < G), exactly one group and a trailing group of one pair; and
    dim, hidden and q_dim reach one full chunk, 2 x 2056, 3 chunks, several full chunks and 4 x 3584."""
    shapes = pair_shapes(G) + chunk_shapes() + list(REAL.values())
    P = {kind: set() for kind in ("qkv", "wo", "gateup", "down", "lm")}
    for s in shapes:
        for kind, N, K in s.matrices():
            assert cut_ok(K) and N % 2 == 0, (s, kind)
            P[kind].add(N // 2)
    for kind, ps in P.items():
        allowed = {"qkv": list(QKV_HEADS), "wo": range(4, 20000, 4), "down": range(4, 20000, 4), "gateup": range(8, 20000, 8),
                   "lm": range(1, 200000)}[kind]
        allowed = [p for p in allowed if kind in ("qkv", "lm") or cut_ok(2 * p if kind in ("wo", "down") else p)]
        for t in pair_targets(G, lm=kind == "lm"):
            assert nearest(t, allowed) in ps, f"G={G}: {kind} misses P = {nearest(t, allowed)} (target {t})"
    counts = {kind: [cta_pairs(p, G) for p in ps] for kind, ps in P.items()}
    for kind, cs in counts.items():
        if kind != "qkv":  # (H + 2 KV) * 64 >= 192 > G: every CTA has a QKV pair
            assert any((c == 0).any() for c in cs), f"G={G}: {kind}: no CTA without pairs"
        assert any((c == GROUP).any() for c in cs), f"G={G}: {kind}: no CTA with exactly one group"
        assert any(((c % GROUP == 1) & (c > GROUP)).any() for c in cs), f"G={G}: {kind}: no trailing group of one pair"
    Ks = {K for s in shapes for _, _, K in s.matrices()}
    assert {4096, 4112, 8208, 14336} <= Ks and (12288 in Ks or 16384 in Ks)
    assert {n_chunks(K) for K in Ks} >= {1, 2, 3, 4}
    assert 4112 // 2 % (32 * 8) != 0 and 14336 // n_chunks(14336) == 3584


def test_exactness_check_is_tight():
    """A row of products on the grid 2^-e passes at sum |p| = 2^24 - 1 grid units and is rejected one unit wider."""
    unit = 2.0 ** -7
    base = torch.tensor([[unit, -(2.0 ** 23 - 1) * unit] + [2.0 ** 14 * unit] * 512], dtype=torch.float64)  # 1 + (2^23 - 1) + 2^23
    ok = base.clone()
    ok[0, 2] -= unit  # 2^24 - 1 units
    assert (ok.abs().sum() / unit).item() == 2.0 ** 24 - 1 and accumulation_exact(ok).all()
    assert (base.abs().sum() / unit).item() == 2.0 ** 24 and not accumulation_exact(base).any()
    finer = ok.clone()
    finer[0, 0] = unit / 2  # one product on a finer grid doubles the unit count
    assert not accumulation_exact(finer).any()


def test_silu_targets_are_robust():
    assert len(SILU_A) >= 4 and (SILU_S > 0).any() and (SILU_S < 0).any()


def test_design_rows_cancel_across_chunks():
    gen = torch.Generator().manual_seed(0)
    for K in (256, 4112, 8208, 14336):
        x = torch.where(torch.rand(K, generator=gen) < 0.5, -1.0, 1.0).double() * torch.pow(2.0, torch.randint(-1, 2, (K,), generator=gen).double())
        t = torch.randint(-12, 13, (64,), generator=gen).double()
        d = design_rows(x, t, None, gen)
        assert torch.equal(matvec(d, x), t) and accumulation_exact(products(d, x)).all()
        if n_chunks(K) > 1:
            kc = K // n_chunks(K)
            last = x.clone()
            last[(n_chunks(K) - 1) * kc:] = 0  # the last chunk read as zero
            assert (matvec(d, last) != t).float().mean() > 0.75  # broken halves of two pairs can cancel each other


# ----------------------------------------------------------------------------- GPU: the exact family
@pytest.mark.gpu
@pytest.mark.parametrize("which", ["pairs", "chunks", "reps"])
def test_phases_exact_at_edges(which):
    """Every phase bit for bit, on shapes whose pair counts and K chunks sit on the edges of this device's partition."""
    G = _abi.device_info()[0]
    shapes = {"pairs": pair_shapes(G), "chunks": chunk_shapes(), "reps": rep_shapes()}[which]
    for i, s in enumerate(shapes):
        run_case(s, 1 + i % 3, seed=100 + i)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mistral-7b", "nemo-12b"])
@pytest.mark.parametrize("n_layers", [1, 2, 3])
def test_phases_exact_real_dense(name, n_layers):
    """Real dense shapes at their real vocabulary, 1 to 3 layers: both halves of the residual ping-pong feed the final norm."""
    run_case(REAL[name], n_layers, seed=n_layers, pos=1000, W=4096, probes=False)


def moe_routes(E: int, k: int, n_layers: int):
    """Per layer a different selection, together covering expert 0 and expert E - 1."""
    out = []
    for l in range(n_layers):
        start = [0, E - k, (E - k) // 2][l % 3]
        out.append(list(range(start, start + k)) if l != 2 else sorted({0, E - 1} | set(range(1, k - 1)))[:k])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("E,k", [(2, 1), (2, 2), (8, 2), (8, 4), (16, 1), (16, 4), (4, 4)])
def test_moe_phases_exact(E, k):
    """In-kernel router, top-k, softmax over the k (equal selected logits: every weight exactly 1/k), the selected experts'
    gate/up and the bf16 += in ascending expert index, over 3 layers that select different experts (expert 0 and E - 1 among
    them), so the producers' route barrier reuses a parity."""
    s = Shape(f"moe-E{E}-k{k}", 1024, 2056, 8, 8, 512, E, k)
    routes = moe_routes(E, k, 3)
    assert any(0 in r for r in routes) and any(E - 1 in r for r in routes)
    run_case(s, 3, seed=E * 10 + k, routes=routes)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["mixtral-8x7b", "mixtral-8x22b"])
def test_moe_phases_exact_real(name):
    s = REAL[name]
    run_case(s, 3, seed=7, pos=500, W=1024, routes=moe_routes(s.E, s.k, 3))


@pytest.mark.gpu
def test_moe_widest_hidden_at_k4():
    """The largest hidden at which four experts' g still leave a ring of 9 stages on this device."""
    hidden = max_hidden_k4(1024)
    assert hidden is not None and _abi.decode_step_unsupported(1024, hidden + 8 * n_chunks(hidden + 8), 8, 8, HD, 256, 8, 4) is not None
    s = Shape(f"moe-k4-hidden{hidden}", 1024, hidden, 8, 8, 512, 8, 4)
    run_case(s, 2, seed=3, routes=[[0, 2, 5, 7], [1, 3, 4, 6]])


@pytest.mark.gpu
def test_moe_distinct_weights_ascending_order():
    """Distinct selected logits (weights off the 1/k grid, checked on the host in float64) and expert outputs chosen so that the
    bf16 += gives a different result in route-weight order than in ascending expert index."""
    E, k = 8, 4
    sel = [1, 3, 4, 6]
    logits = torch.full((E,), -4.0, dtype=torch.float64)
    logits[sel] = torch.tensor([0.0, 1.0, 2.0, 0.5], dtype=torch.float64)  # weight order 4, 3, 6, 1: not ascending
    s = Shape("moe-distinct", 64, 256, 8, 8, 512, E, k)
    gen = torch.Generator().manual_seed(5)
    st = Step(s, 1, 20, 64, gen, routes=[sel], router_logits=[logits])
    # expected weights, each well inside its bf16 rounding interval
    p = torch.softmax(logits[sel], 0)
    r = bf(p).double()
    ulp = torch.pow(2.0, torch.floor(torch.log2(r)) - 7)
    assert ((ulp / 2 - (p - r).abs()) / ulp > 2.0 ** -8).all()
    assert_launched(st.launch, r"decode_megakernel<1>", MK, 1)
    out = st.read()
    # the designed y of this case do not keep the residual stream on +-0.5: compare the combine itself, then the logits on
    # the kernel's x within the ops tolerance (the final norm is no longer exact)
    lay = st.layers[0]
    hk = out["h"].double()
    hn = R.rms_norm(bf(hk)[None], bf(lay["fn"]), EPS)[0].double()
    got_sel, wts = route_rule(bf(matvec(lay["gate"], hn)), k)
    assert got_sel == sel
    ts = [bf(wts[j] * bf(matvec(lay["w2s"][e], out["g"][j].double()))) for j, e in enumerate(sel)]
    asc = ts[0]
    for t in ts[1:]:
        asc = bf(asc + t)
    by_weight = [ts[j] for j in sorted(range(k), key=lambda j: -float(wts[j]))]
    alt = by_weight[0]
    for t in by_weight[1:]:
        alt = bf(alt + t)
    assert not torch.equal(asc, alt), "the design does not tell the two orders apart"
    same_bits(out["x"][1], bf(hk + asc.double()), "x_out (ascending expert index)")


@pytest.mark.gpu
@pytest.mark.parametrize("E,k", [(8, 2), (16, 4), (2, 1)])
def test_router_ties_lower_index_wins(E, k):
    """Router logits tied across the k / k+1 boundary: the kernel selects the lower expert index, and mb200_moe_route makes the
    same choice on the same input.  (torch.topk's order among ties is unspecified and not asserted.)"""
    s = Shape(f"tie-E{E}-k{k}", 256, 256, 8, 8, 512, E, k)
    logits = torch.full((E,), -1.0, dtype=torch.float64)
    tied = list(range(E - 1, E - 2 - k, -1))  # k + 1 experts at the top, equal; the lower k indices must win
    logits[tied] = 1.0
    want = sorted(tied)[:k]
    st, out = run_case(s, 1, seed=E + k, routes=[want], router_logits=[logits])
    lay = st.layers[0]
    hn = R.rms_norm(bf(out["h"].double())[None], bf(lay["fn"]), EPS)[0]
    from mistral_inference_b200.moe import MoeBuffers

    b = MoeBuffers(1, s.dim, s.hidden, E, k, torch.device(DEV), torch.bfloat16)
    _abi.moe_route(hn[None].to(DEV), st.gates[0], E, k, 0, 1, b)
    torch.cuda.synchronize()
    assert sorted(b.sel.cpu().reshape(-1).tolist()) == want


# ----------------------------------------------------------------------------- GPU: fused argmax at real vocabularies
@pytest.mark.gpu
@pytest.mark.parametrize("vocab", [32000, 131072])
@pytest.mark.parametrize("where", ["first-pair", "last-pair", "tie-across-ctas"])
def test_argmax_real_vocab(vocab, where):
    G = _abi.device_info()[0]
    P = vocab // 2
    c = G // 3
    first = 2 * cta_first_pair(P, G, c)
    last = 2 * cta_first_pair(P, G, c + 1) - 1
    t = torch.randint(-64, 64, (vocab,), generator=torch.Generator().manual_seed(vocab)).double() / 4
    top = 40.0
    want = {"first-pair": first, "last-pair": last, "tie-across-ctas": last}[where]
    t[want] = top
    if where == "tie-across-ctas":
        t[last + 1] = top  # first row of CTA c + 1
    s = Shape(f"argmax-{vocab}", 1024, 1024, 8, 8, vocab)
    st, out = run_case(s, 1, seed=1, lm_targets=t)
    assert out["next"] == want


# ----------------------------------------------------------------------------- GPU: random data on the real shapes
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REAL))
def test_phases_random_real_shapes(name):
    """Random weights and input on each real shape (1 layer): q, h, g and the logits against the oracle on the kernel's own
    inputs, within test_gpu_ops.py's model (<= 1 bf16 ulp and >= 97 % bit-exact; g, after three chained roundings, <= 4 ulps and
    >= 96 %, as test_ffn_gateup allows).  This covers general RoPE and SiLU values."""
    s = REAL[name]
    gen = torch.Generator(device=DEV).manual_seed(11)
    dim, hidden, H, KV = s.dim, s.hidden, s.H, s.KV
    q_dim, kv_dim = H * HD, KV * HD
    r = lambda *shape, sc=1.0: (torch.randn(*shape, generator=gen, device=DEV) * sc).to(torch.bfloat16)  # noqa: E731
    emb, an, fn, final = r(1, dim), 1 + r(dim, sc=0.1), 1 + r(dim, sc=0.1), 1 + r(dim, sc=0.1)
    an, fn, final = an.to(torch.bfloat16), fn.to(torch.bfloat16), final.to(torch.bfloat16)
    wqkv, wo = r(q_dim + 2 * kv_dim, dim, sc=dim ** -0.5), r(dim, q_dim, sc=q_dim ** -0.5)
    w_out = r(s.vocab, dim, sc=dim ** -0.5)
    pos, W = 300, 512
    ck = torch.zeros(1, W, KV, HD, dtype=torch.bfloat16, device=DEV)
    cv = r(1, W, KV, HD)
    ck[0, :pos] = r(pos, KV, HD)
    experts = s.E
    if experts:
        gate = r(experts, dim, sc=dim ** -0.5)
        w13 = [r(2 * hidden, dim, sc=dim ** -0.5) for _ in range(experts)]
        w2 = [r(dim, hidden, sc=hidden ** -0.5) for _ in range(experts)]
        w13p = w2p = 0
    else:
        w13, w2 = r(2 * hidden, dim, sc=dim ** -0.5), r(dim, hidden, sc=hidden ** -0.5)
        w13p, w2p = w13.data_ptr(), w2.data_ptr()
    desc = torch.tensor([[wqkv.data_ptr(), wo.data_ptr(), w13p, w2p, an.data_ptr(), fn.data_ptr(), ck.data_ptr(), cv.data_ptr()]],
                        dtype=torch.int64, device=DEV)
    table = precompute_freqs_cis(HD, ROPE_LEN, 1e6)
    rope_dev = torch.view_as_real(table).contiguous().to(DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(1, dim, H, KV, HD, hidden, s.vocab, 1), torch.device(DEV))
    sc = _abi.decode_buffers(dim, hidden, H, KV, HD, s.E, s.k)
    logits = torch.empty(s.vocab, dtype=torch.float32, device=DEV)
    nxt = torch.zeros(1, dtype=torch.long, device=DEV)
    tok = torch.zeros(1, dtype=torch.long, device=DEV)
    kw = {}
    if experts:
        kw = dict(n_experts=s.E, top_k=s.k, moe_gate=torch.tensor([gate.data_ptr()], dtype=torch.int64, device=DEV),
                  moe_w13=torch.tensor([w.data_ptr() for w in w13], dtype=torch.int64, device=DEV),
                  moe_w2=torch.tensor([w.data_ptr() for w in w2], dtype=torch.int64, device=DEV))
    win = torch.tensor([W], dtype=torch.int32, device=DEV)
    assert_launched(lambda: _abi.decode_step(desc, win, 1, emb, final, w_out, rope_dev, tok, pos, 0, logits, nxt, dim, hidden, H, KV, HD,
                                             s.vocab, EPS, ws, **kw), rf"decode_megakernel<{H // KV}>", MK, 1)
    torch.cuda.synchronize()
    buf = lambda off, n: ws.buf[off:off + 2 * n].view(torch.bfloat16).cpu()  # noqa: E731
    x_in = emb[0].cpu()
    xn = R.rms_norm(x_in[None], an.cpu(), EPS)
    y = F.linear(xn, wqkv.cpu())
    q_ref, k_ref = R.apply_rope(y[:, :q_dim].view(1, H, HD), y[:, q_dim:q_dim + kv_dim].view(1, KV, HD), table[[pos]])
    assert_bf16_close(buf(sc.q, q_dim)[None], q_ref.reshape(1, -1), what=f"{name} q")
    assert_bf16_close(ck[0, pos].cpu().reshape(1, -1), k_ref.reshape(1, -1), what=f"{name} k row")
    attn = buf(sc.attn, q_dim)
    h_ref = x_in + F.linear(attn[None], wo.cpu())[0]
    assert_bf16_close(buf(sc.h, dim)[None], h_ref[None], what=f"{name} h")
    h = buf(sc.h, dim)
    hn = R.rms_norm(h[None], fn.cpu(), EPS)
    if experts:
        gl = F.linear(hn, gate.cpu())
        top = gl.float().topk(s.k + 1).values[0]
        assert top[s.k - 1] > top[s.k], "random router logits tied at the k-th place"
        sel = sorted(gl[0].float().topk(s.k).indices.tolist())
        g = buf(sc.g, s.k * hidden).view(s.k, hidden)
        for j, e in enumerate(sel):
            w1, w3 = w13[e].cpu()[0::2], w13[e].cpu()[1::2]
            assert_bf16_close(g[j][None], F.silu(F.linear(hn, w1)) * F.linear(hn, w3), max_ulp=4, min_exact=0.96, what=f"{name} g of expert {e}")
        # moe.py:24-32 on the kernel's own g: bf16(w * w2_e g_e) summed with bf16 += in ascending expert index
        _, wts = route_rule(gl[0], s.k)
        res = None
        for j, e in enumerate(sel):
            t = bf(wts[j] * F.linear(g[j][None], w2[e].cpu())[0])
            res = t if res is None else res + t
        x_ref = h + res
    else:
        w1, w3 = w13.cpu()[0::2], w13.cpu()[1::2]
        g = buf(sc.g, hidden)
        assert_bf16_close(g[None], F.silu(F.linear(hn, w1)) * F.linear(hn, w3), max_ulp=4, min_exact=0.96, what=f"{name} g")
        x_ref = h + F.linear(g[None], w2.cpu())[0]
    x_out = buf(sc.x, 2 * dim).view(2, dim)[1]
    assert_bf16_close(x_out[None], x_ref[None], what=f"{name} x_out")
    want = F.linear(R.rms_norm(x_out[None], final.cpu(), EPS), w_out.cpu()).float()
    assert_bf16_close(logits.cpu()[None], want, what=f"{name} logits")
    assert int(nxt.item()) == int(logits.argmax().item())


# ----------------------------------------------------------------------------- GPU: shapes the step refuses take the per-layer path
@pytest.mark.gpu
@pytest.mark.parametrize("n_layers", [1, 2])
def test_unsupported_moe_falls_back_to_per_layer_path(n_layers):
    """A Mixtral-8x7B-shaped model with k = 3 leaves the megakernel fewer than 9 ring stages: batch-1 generate runs on the
    per-layer path (no decode_megakernel launch) and matches the oracle; the k = 2 shape still takes the megakernel."""
    p = synth.shape("mixtral-8x7b", n_layers=n_layers, vocab_size=32000, moe=dict(num_experts=8, num_experts_per_tok=3))
    assert _abi.decode_step_unsupported(4096, 14336, 32, 8, HD, 32000, 8, 3) is not None
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 1
    from mistral_inference_b200.transformer import Transformer

    m = Transformer.empty(args, "cuda", torch.bfloat16)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, "cuda")
    m.load_state_dict(sd)
    prompt = synth.synth_prompt(7, 32000, 5)
    names = launched_kernels(lambda: mi.generate([prompt], m, max_tokens=4, temperature=0.0))
    assert not any("decode_megakernel" in n for n in names)
    assert not m._megakernel_ok(1)
    om = R.OracleTransformer(oracle_args(p, 1), {k: v.cpu() for k, v in sd.items()})
    from mistral_inference_b200.cache import BufferCache

    cache = BufferCache(m.n_local_layers, 1, 16, 8, HD, None)
    cache.to(m.device, m.dtype)
    cache.reset()
    got = [m.forward(torch.tensor(prompt, device=DEV), [7], cache)[-1:].float().cpu()]
    names = launched_kernels(lambda: got.append(m.forward(torch.tensor([prompt[0]], device=DEV), [1], cache).float().cpu()))
    assert not any("decode_megakernel" in n for n in names)
    oc = om.new_cache(16)
    want = [om.forward(torch.tensor(prompt), [7], oc)[-1:], om.forward(torch.tensor([prompt[0]]), [1], oc)]
    for gth, w in zip(got, want):
        tol = 2 * 2.0 ** (math.floor(math.log2(w.abs().max().item())) - 7)
        assert (gth - w).abs().max().item() <= tol


@pytest.mark.gpu
@pytest.mark.parametrize("name,k", [("mixtral-8x7b", 2), ("mixtral-8x22b", 2), ("mistral-7b", 0), ("nemo-12b", 0)])
def test_supported_real_shapes_take_the_megakernel(name, k):
    s = REAL[name]
    assert _abi.decode_step_unsupported(s.dim, s.hidden, s.H, s.KV, HD, s.vocab, s.E, k) is None
    p = synth.shape({"nemo-12b": "mistral-nemo-12b"}.get(name, name), n_layers=1)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 1
    from mistral_inference_b200.transformer import Transformer

    m = Transformer.empty(args, "cuda", torch.bfloat16)  # shapes only: the query needs no weights
    assert m._megakernel_ok(1)
    assert not m._megakernel_ok(2)


def test_rope_fma_probes_exist():
    """At every position the exact family decodes at, some q pairs round differently under a fused multiply-add (CPU)."""
    table = precompute_freqs_cis(HD, ROPE_LEN, 1e6)
    for pos in (37, 1000, 500, 20):
        assert len(fma_sensitive_pairs(pos, table)) >= 8
