"""Attention kernels at tile, window and split edges: which keys each query sees, and how they are weighted.

Three kernels are checked against tables computed here from the mask definition of oracle/attention_ref.py (query at absolute
position P sees keys in (P - W, P], bottom-right aligned; a ring slot holds position pos % W; decode sees slots [0, kv_len)):
attn_prefill_wgmma_kernel (first prefill), attn_prefill_kernel (ring + chunk, the cache-less mode, and first prefill under
MB200_ATTN=mma) and attn_decode_tma_kernel<REP> (decode), every compiled head ratio REP = H / KV of 1, 2, 4, 6, 8.  The readers
of the FP8 (e4m3) KV cache run the same tables as one more kernel each: attn_prefill_fp8_kernel ("mma_fp8", ring + chunk) and
attn_decode_tma_fp8_kernel<REP> ("tma_fp8").  Their e4m3 ring and exponents are written from the same bf16 K / V by the library's
own quantiser (mb200_kv_quantize); the position codes of V are exact in e4m3, so V' == V and the tables are unchanged.  Every GPU
test asserts, from the library's launch log, which kernel ran.

Most grids use KV = 2, which keeps the larger head ratios cheap.  The production decode grid uses KV = 8 (Mistral-7B, Nemo): at
batch 1 the model runs S = 33 splits, so from about 2.1k keys every split holds two or more 64-key tiles, and at a 32k ring
about 16.

Visible sets (exact).  With q = 0 every score is 0 and every P is exactly 1 in all three kernels (exp2 of 0), so l counts the
visible keys and P.V sums exact integers in fp32.  V encodes the key's absolute position: dims 0..63 hold
one-hot((j + a) mod 64), dims 64..127 one-hot((j div 64 + c) mod 64), both scaled by s = 1 or 2, where a, c and s depend on the
KV head g and the sequence b.  The output is then O[i, h, d] = count_d / n_i, and the kernel's count * fl(1 / n) (or fl(count / n))
must be within one bf16 ulp of the correctly rounded count / n, and exactly 0 where the count is 0.  Adding, dropping or moving one
key changes some bucket count by one; a bucket holds at most ~64 keys at n <= 4096, so that output moves by >= 1/64 relative,
which is >= 2 bf16 ulps.  Reading the neighbouring head's or sequence's V shifts the histograms and doubles or halves s (the scale
is what tells two heads apart when a whole 4096-slot ring is visible and both histograms are flat).  A ring longer than 4096 slots
(W = 32768) would put 512 keys in every bucket of that code, and one key in 512 is below a bf16 ulp; there dims 64..127 code the
64-key block only for the first and the last 2048 slots of the ring (32 buckets each) and stay zero in between, so the keys at both
ends of a full ring, and the ones just past them, sit in buckets of at most 65 keys.
test_comparator_rejects_every_single_key_change keeps this claim true for every configuration of the grids below, on the CPU.

Softmax weighting (bounded).  Against a float64 reference, every element satisfies
    |O - O64| <= 2^-8 * sum_j p_j |v_j| + ulp_bf16(O64):
rounding P to bf16 for the tensor-core P.V product moves each p_j by at most 2^-9 relative (the denominator l sums the unrounded
fp32 P), which moves O by at most 2^-9 * sum_j p_j |v_j|; the final rounding to bf16 adds half an ulp; fp32 accumulation, the fp32
score scale and ex2.approx contribute less than 2^-20 relative.  The bound leaves a factor of two of headroom on each term.
"""
import functools
from typing import NamedTuple, Optional, Tuple

import numpy as np
import pytest
import torch

from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer_layers import decode_splits

from .util import assert_launched, bf16_ulp_diff

DEV = "cuda"
HD = 128
KV = 2  # the default KV of a Case: small KV counts keep the larger head ratios cheap
REPS = [1, 2, 4, 6, 8]
ATTN = r"attn_\w+_kernel"
KERNEL = {"wgmma": r"attn_prefill_wgmma_kernel\b", "mma": r"attn_prefill_kernel\b", "tma": r"attn_decode_tma_kernel<{rep}>",
          "mma_fp8": r"attn_prefill_fp8_kernel\b", "tma_fp8": r"attn_decode_tma_fp8_kernel<{rep}>"}


class Case(NamedTuple):
    kind: str          # "prefill" (causal, ring + chunk), "nocache" (causal=0, one block over the flattened batch), "decode"
    seqpos: Tuple      # prefill: positions already in the ring per sequence; decode: kv_len per sequence
    lens: Tuple        # prefill: chunk length per sequence; nocache: (T,); decode: unused
    W: int             # window = ring size
    S: int = 1         # decode: KV splits
    KV: int = KV       # kv heads


# ----------------------------------------------------------------------------- grids
FIRST_SEQLENS = [(128,), (129,), (127, 129), (256,), (257, 1), (1, 300, 5, 128), (1000,)]
FIRST_WINDOWS = [1, 2, 127, 128, 129, 255, 256, 257, 4096]  # 4096: longer than every sequence
RING_WINDOWS = [16, 64, 100, 128]
NOCACHE_T = [1, 64, 65, 200]
DECODE_WINDOWS = [100, 300, 4096]
DECODE_SPLITS = [64, 7, 1, 2]  # in this order on one workspace: S = 7 right after S = 64
DECODE_B = 5
PROD_KV = 8                        # Mistral-7B / Nemo
PROD_LONG_WINDOWS = [4096, 32768]  # batch 1: kv_len 65, 2113, 4000, W at S = 64, 33 (the model's S at B = 1), 7, 1
PROD_FORCED_S = {2: 64, 4: 33, 8: 7}  # batches 2, 4, 8 on a 4096 ring: the model's S and this one
LONG_RING = 4096                   # rings longer than this take the edge code in dims 64..127 (module docstring)


def first_prefill_cases():
    return [Case("prefill", (0,) * len(s), s, W) for s in FIRST_SEQLENS for W in FIRST_WINDOWS]


def ring_cases():
    out = []
    for k, W in enumerate(RING_WINDOWS):
        lens = [1, 63, 64, 65, 130]
        lens = lens[k:] + lens[:k]
        out.append(Case("prefill", (1, W - 1, W, W + 1, 3 * W + 5), tuple(lens), W))
        out.append(Case("prefill", (W + 1, 0, 3 * W + 5), (lens[0], lens[1], lens[2]), W))  # one first-time sequence in the batch
    return out


def nocache_cases():
    return [Case("nocache", (0,), (T,), 0) for T in NOCACHE_T]


def decode_cases():
    out = []
    for W in DECODE_WINDOWS:
        lens = [min(n, W) for n in (1, 63, 64, 65, 127, 128, 129, W)]
        for k, S in enumerate(DECODE_SPLITS):
            out.append(Case("decode", tuple(lens[(5 * k + i) % len(lens)] for i in range(DECODE_B)), (), W, S))
    return out


def production_long_cases(W: int):
    """Batch 1 at KV = 8: splits of one tile up to 512 (2113 keys over 33 splits: 2 tiles each; 4000 over 7: 9; 32768 over 33: 16;
    over 7: 74), and empty splits (65 keys over 64)."""
    return [Case("decode", (n,), (), W, S, PROD_KV) for S in (64, 33, 7, 1) for n in (65, 2113, 4000, W)]


def production_batch_cases():
    """Batches 2, 4, 8 at KV = 8 on a 4096 ring, ragged kv_len around the tile, at 320 / 321 and at W, under the model's S
    (decode_splits: 16, 8, 4) and a forced one."""
    W, lens = 4096, (1, 63, 64, 65, 320, 321, 4096)
    out = []
    for B, forced in PROD_FORCED_S.items():
        for k, S in enumerate((decode_splits(B, PROD_KV, W), forced)):
            out.append(Case("decode", tuple(lens[(3 * k + B + i) % len(lens)] for i in range(B)), (), W, S, PROD_KV))
    return out


def production_cases():
    return [c for W in PROD_LONG_WINDOWS for c in production_long_cases(W)] + production_batch_cases()


# ----------------------------------------------------------------------------- position codes and the visible sets
def code_params(g: int, b: int):
    """(a, c, s) of KV head g in sequence b: neighbouring heads and sequences differ in all three."""
    return (7 * g + 13 * b + 1) % 64, (5 * g + 11 * b + 3) % 64, float(2 ** ((g + b) % 2))


def codes(pos: np.ndarray, g: int, b: int, W: int = 0) -> np.ndarray:
    """[n, 128] V rows of the keys at absolute positions `pos` (decode: ring slots) of a ring of W slots."""
    a, c, s = code_params(g, b)
    v = np.zeros((len(pos), HD))
    r = np.arange(len(pos))
    v[r, (pos + a) % 64] = s
    if W <= LONG_RING:
        v[r, 64 + (pos // 64 + c) % 64] = s
    else:  # the first 2048 slots (and position -1) in dims 64..95, the last 2048 (and position W) in dims 96..127
        head, tail = pos < 2048, pos >= W - 2048
        v[r[head], 64 + (pos[head] // 64 + c) % 32] = s
        v[r[tail], 96 + ((pos[tail] - (W - 2048)) // 64 + c) % 32] = s
    return v


def n_seqs(case: Case) -> int:
    return len(case.seqpos)


def n_positions(case: Case, b: int) -> int:
    """Key positions of sequence b that exist: prefill [0, seqpos + len), nocache [0, T), decode the W ring slots."""
    if case.kind == "decode":
        return case.W
    return case.seqpos[b] + case.lens[b]


def visible_mask(case: Case, b: int) -> np.ndarray:
    """bool [queries of sequence b, n_positions]: the mask of oracle/attention_ref.py restated over absolute positions."""
    j = np.arange(n_positions(case, b))[None, :]
    if case.kind == "decode":  # one query; the ring's first kv_len slots, in any order
        return j < case.seqpos[b]
    if case.kind == "nocache":
        return np.ones((case.lens[0], case.lens[0]), dtype=bool)
    P = case.seqpos[b] + np.arange(case.lens[b])[:, None]
    return (j <= P) & (j > P - case.W)


class Table(NamedTuple):
    counts: np.ndarray  # [rows, KV, 128] float64: sum of the visible keys' codes
    n: np.ndarray       # [rows] visible keys
    seq: np.ndarray     # [rows] sequence of the row
    lo: np.ndarray      # [rows] lowest / highest visible position (the sets are contiguous ranges)
    hi: np.ndarray


@functools.lru_cache(maxsize=None)
def expected(case: Case) -> Table:
    counts, n, seq, lo, hi = [], [], [], [], []
    for b in range(n_seqs(case)):
        m = visible_mask(case, b)
        pos = np.arange(m.shape[1])
        counts.append(np.stack([m.astype(np.float64) @ codes(pos, g, b, case.W) for g in range(case.KV)], 1))
        n.append(m.sum(1))
        seq.append(np.full(m.shape[0], b))
        lo.append(m.argmax(1))
        hi.append(m.shape[1] - 1 - m[:, ::-1].argmax(1))
    return Table(*(np.concatenate(x) for x in (counts, n, seq, lo, hi)))


def bf16_round(x: np.ndarray) -> torch.Tensor:
    """Nearest bf16 of float64 values.  Through fp32: count / n with n <= 4096 is never within 2^-24 of a bf16 tie without being
    one, so the double rounding is exact here."""
    return torch.from_numpy(x).float().to(torch.bfloat16)


def rows_off(got: torch.Tensor, counts: np.ndarray, n: np.ndarray) -> np.ndarray:
    """Per row of `got` [rows, X, 128] against the visible-set table (counts [rows, X, 128], n [rows]): True where some element is
    more than one bf16 ulp from count / n, is not exactly 0 where the count is 0, or is not finite."""
    got = got.float().cpu()
    want = bf16_round(counts / n[:, None, None])
    bad = (bf16_ulp_diff(got, want) > 1) | (torch.from_numpy(counts == 0) & (got != 0)) | ~torch.isfinite(got)
    return bad.flatten(1).any(1).numpy()


def assert_visible_sets(got: torch.Tensor, case: Case, rep: int):
    """got [rows, H, 128] against the table of `case` (query head h reads KV head h // rep)."""
    t = expected(case)
    counts = np.repeat(t.counts, rep, axis=1)
    off = rows_off(got, counts, t.n)
    if off.any():
        i = int(np.flatnonzero(off)[0])
        g = got.float().cpu()[i].reshape(case.KV, rep, HD)[:, 0]
        raise AssertionError(f"{case}: {int(off.sum())} of {len(off)} query rows see the wrong keys; first: row {i} (sequence "
                             f"{t.seq[i]}, keys {t.lo[i]}..{t.hi[i]}, n = {t.n[i]}); got n * O[head 0] = "
                             f"{(g[0] * float(t.n[i])).tolist()}, want the counts {t.counts[i, 0].tolist()}")


def range_counts(lo: np.ndarray, hi: np.ndarray, g: int, b: int, W: int = 0) -> np.ndarray:
    """Code sums of the key ranges [lo, hi] (may reach position -1) of one head and sequence, by prefix sums."""
    base = -64
    pos = np.arange(base, int(hi.max()) + 2)
    pre = np.concatenate([np.zeros((1, HD)), np.cumsum(codes(pos, g, b, W), 0)])
    return pre[hi + 1 - base] - pre[lo - base]


def single_key_changes(case: Case):
    """(name, counts [rows, KV, 128], n [rows], applies [rows]) for each single-key change of every row's visible set."""
    t = expected(case)
    lo, hi, seq = t.lo, t.hi, t.seq
    B = n_seqs(case) + (1 if case.kind == "decode" else 0)  # decode: the cache holds one more sequence

    def over(lo_, hi_, seq_of_row):
        out = np.zeros_like(t.counts)
        for b in np.unique(seq):
            r = seq == b
            for g in range(case.KV):
                out[r, g] = range_counts(lo_[r], hi_[r], g, seq_of_row(b), case.W)
        return out

    same = lambda b: b  # noqa: E731
    ok = t.n > 1
    yield "drop the lowest key", over(lo + 1, hi, same), t.n - 1, ok
    yield "drop the highest key", over(lo, hi - 1, same), t.n - 1, ok
    yield "add key lo - 1", over(lo - 1, hi, same), t.n + 1, np.ones_like(ok)
    yield "add key hi + 1", over(lo, hi + 1, same), t.n + 1, np.ones_like(ok)
    if case.KV > 1:
        yield "the neighbouring KV head's keys", np.roll(t.counts, -1, axis=1), t.n, np.ones_like(ok)
    if B > 1:
        yield "the neighbouring sequence's keys", over(lo, hi, lambda b: b + 1 if b + 1 < B else b - 1), t.n, np.ones_like(ok)


ALL_CASES = first_prefill_cases() + ring_cases() + nocache_cases() + decode_cases() + production_cases()


def test_table_matches_contiguous_ranges():
    """The tables come from the mask; the single-key changes below assume every visible set is one contiguous range."""
    for case in ALL_CASES:
        t = expected(case)
        assert (t.n == t.hi - t.lo + 1).all(), case
        for b in np.unique(t.seq):
            r = t.seq == b
            for g in range(case.KV):
                assert np.array_equal(range_counts(t.lo[r], t.hi[r], g, int(b), case.W), t.counts[r, g]), (case, b, g)


def case_id(c: Case) -> str:
    return f"{c.kind}-pos{'_'.join(map(str, c.seqpos))}-len{'_'.join(map(str, c.lens))}-W{c.W}-S{c.S}" + (f"-KV{c.KV}" if c.KV != KV else "")


@pytest.mark.parametrize("case", ALL_CASES, ids=case_id)
def test_comparator_rejects_every_single_key_change(case):
    """CPU check of the comparator, not of a kernel: for every row of every configuration the GPU tests run, a kernel that saw
    one key more, one key fewer, or the keys of the neighbouring KV head or sequence would be caught, even if it rounded
    perfectly -- and the correct table itself passes."""
    t = expected(case)
    assert not rows_off(bf16_round(t.counts / t.n[:, None, None]), t.counts, t.n).any()
    for what, counts, n, applies in single_key_changes(case):
        wrong = bf16_round(counts[applies] / n[applies][:, None, None])
        caught = rows_off(wrong, t.counts[applies], t.n[applies])
        assert caught.all(), f"{case}: '{what}' not detected on {int((~caught).sum())} rows, e.g. row {int(np.flatnonzero(~caught)[0])}"




# ----------------------------------------------------------------------------- running the kernels
def partial_bytes(cases, rep: int = 8) -> int:
    """Split partials of the largest decode launch among `cases` (at head ratio `rep`)."""
    return max([n_seqs(c) * c.KV * c.S * rep * (HD + 2) * 4 for c in cases if c.kind == "decode"] + [0])


@pytest.fixture(scope="module")
def ws():
    need = partial_bytes(decode_cases() + production_cases() + list(SOFTMAX_CASES.values()) + [SOFTMAX_PROD_CASE])
    return _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + need, torch.device(DEV))


def select_kernel(kernel: str, monkeypatch):
    monkeypatch.delenv("MB200_ATTN", raising=False)
    if kernel == "mma":
        monkeypatch.setenv("MB200_ATTN", "mma")  # first prefill would take the wgmma kernel


def kv_prime(K, V):
    """(K', V'): x' of every row of the per-sequence bf16 K / V [n, KV, 128], from the library's quantiser (write-back only)."""
    Kp, Vp = [], []
    for k, v in zip(K, V):
        kd, vd = k.reshape(k.shape[0], -1).to(DEV), v.reshape(v.shape[0], -1).to(DEV)
        _abi.kv_quantize(kd, vd, True)
        Kp.append(kd.cpu().view(k.shape))
        Vp.append(vd.cpu().view(v.shape))
    return Kp, Vp


def fp8_ring(k_rows: torch.Tensor, v_rows: torch.Tensor, rows: torch.Tensor, n_rows: int, KV: int):
    """(e4m3 K ring, e4m3 V ring, exp_k, exp_v) of n_rows rows, written by the library's quantiser from the bf16 rows k_rows / v_rows
    [T, KV*128] into ring rows `rows` [T] (-1: not cached).  Every other row holds NaN codes (0x7F, 0xFF) and extreme exponents
    (127, -128), which a reader must never use."""
    k8 = torch.tensor([0x7F, 0xFF, 0x00, 0x80], dtype=torch.uint8, device=DEV).repeat(n_rows * KV * HD // 4).view(n_rows, KV, HD)
    v8 = k8.clone()
    ek = torch.tensor([127, -128], dtype=torch.int8, device=DEV).repeat(n_rows * KV)[: n_rows * KV].view(n_rows, KV).contiguous()
    ev = ek.clone()
    if k_rows.shape[0] > 0:
        _abi.kv_quantize(k_rows.contiguous(), v_rows.contiguous(), False, k8, v8, ek, ev, rows.to(torch.int32).contiguous())
    return k8, v8, ek, ev


def run(case: Case, q: torch.Tensor, K, V, rep: int, ws, fp8: bool = False) -> torch.Tensor:
    """One launch.  q [rows, H, 128] bf16 (rows in table order), K / V: per sequence [n_positions, KV, 128] bf16 on the CPU,
    indexed by absolute position (decode: ring slot; one extra sequence fills the cache row past B).  Returns out [rows, H, 128].
    With `fp8` the ring is e4m3, quantised from K / V by the library, and the chunk rows are the library's K', V'."""
    KV = case.KV
    H = KV * rep
    qd = q.reshape(q.shape[0], H * HD).to(DEV)
    out = torch.full_like(qd, float("nan"))
    B = n_seqs(case)
    if case.kind == "decode":
        ck = torch.stack([k.clone() for k in K]).to(DEV)  # [max_batch, W, KV, 128]
        cv = torch.stack([v.clone() for v in V]).to(DEV)
        kv_len = torch.tensor(case.seqpos, dtype=torch.int32, device=DEV)
        if fp8:
            MB, W = ck.shape[:2]
            rows = torch.arange(MB * W, dtype=torch.int32, device=DEV).view(MB, W)
            for b, n in enumerate(case.seqpos):  # slots >= kv_len are never written
                rows[b, n:] = -1
            k8, v8, ek, ev = fp8_ring(ck.view(MB * W, -1), cv.view(MB * W, -1), rows.view(-1), MB * W, KV)
            del ck, cv
            _abi.attn_decode_fp8(qd, k8.view(MB, W, KV, HD), v8.view(MB, W, KV, HD), ek, ev, kv_len, out, H, KV, HD, case.S, ws)
            return out.view(-1, H, HD)
        for b, n in enumerate(case.seqpos):  # slots >= kv_len are uninitialised memory in the reference (cache.py:166)
            ck[b, n:] = float("nan")
            cv[b, n:] = float("nan")
        _abi.attn_decode(qd, ck, cv, kv_len, out, H, KV, HD, case.S, ws)
        return out.view(-1, H, HD)
    if case.kind == "nocache":
        k, v = K[0].reshape(-1, KV * HD).to(DEV), V[0].reshape(-1, KV * HD).to(DEV)
        _abi.attn_prefill(qd, k, v, None, None, None, None, out, 1, case.lens[0], 0, H, KV, HD, causal=False)
        return out.view(-1, H, HD)
    W = case.W
    k_new = torch.cat([K[b][p:p + s] for b, (p, s) in enumerate(zip(case.seqpos, case.lens))]).reshape(-1, KV * HD).to(DEV)
    v_new = torch.cat([V[b][p:p + s] for b, (p, s) in enumerate(zip(case.seqpos, case.lens))]).reshape(-1, KV * HD).to(DEV)
    q_start = torch.tensor([0] + np.cumsum(case.lens).tolist(), dtype=torch.int32, device=DEV)
    seqpos = torch.tensor(case.seqpos, dtype=torch.int32, device=DEV)
    first = all(p == 0 for p in case.seqpos)
    if fp8:
        _abi.kv_quantize(k_new, v_new, True)  # the model attends over the chunk's k', v'
        pos = [torch.arange(max(0, p - W), p) for p in case.seqpos]  # ring slot pos % W holds position pos
        rows = torch.cat([b * W + pos[b] % W for b in range(B)])
        kr = torch.cat([K[b][pos[b]] for b in range(B)]).reshape(-1, KV * HD).to(DEV)
        vr = torch.cat([V[b][pos[b]] for b in range(B)]).reshape(-1, KV * HD).to(DEV)
        k8, v8, ek, ev = fp8_ring(kr, vr, rows.to(DEV), B * W, KV)
        _abi.attn_prefill_fp8(qd, k_new, v_new, k8.view(B, W, KV, HD), v8.view(B, W, KV, HD), ek, ev, q_start, seqpos, out, B,
                              max(case.lens), W, H, KV, HD, first_prefill=first)
        return out.view(-1, H, HD)
    ck = torch.full((B, W, KV, HD), float("nan"), dtype=torch.bfloat16, device=DEV)  # never-written slots must not be read
    cv = ck.clone()
    for b, p in enumerate(case.seqpos):  # ring slot pos % W holds position pos, for the last W positions before the chunk
        pos = torch.arange(max(0, p - W), p)
        ck[b, (pos % W).to(DEV)] = K[b][pos].to(DEV)
        cv[b, (pos % W).to(DEV)] = V[b][pos].to(DEV)
    _abi.attn_prefill(qd, k_new, v_new, ck, cv, q_start, seqpos, out, B, max(case.lens), W, H, KV, HD, causal=True, first_prefill=first)
    return out.view(-1, H, HD)


@functools.lru_cache(maxsize=2)
def _code_inputs(ns: Tuple[int, ...], W: int, KV: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    K, V = [], []
    for b, n in enumerate(ns):
        K.append(torch.randn(n, KV, HD, generator=g).to(torch.bfloat16))
        V.append(torch.from_numpy(np.stack([codes(np.arange(n), gg, b, W) for gg in range(KV)], 1)).to(torch.bfloat16))
    return K, V


def code_inputs(case: Case, seed: int):
    """q = 0, K random where a key exists, V = position codes; decode fills one more cache row (max_batch = B + 1).  Decode inputs
    depend on (B, W, KV, seed) only, so cases that share them share one (cached) ring."""
    B = n_seqs(case) + (1 if case.kind == "decode" else 0)
    return _code_inputs(tuple(n_positions(case, b) for b in range(B)), case.W, case.KV, seed)


def check_visible_sets(cases, kernel: str, rep: int, ws, monkeypatch, seed: Optional[int] = None):
    """Every case of `cases` on `kernel`, each with its own inputs (seed = its index) or all with those of `seed`."""
    select_kernel(kernel, monkeypatch)
    fp8 = kernel.endswith("_fp8")
    outs, exact = [], set()

    def launches():
        for i, case in enumerate(cases):
            K, V = code_inputs(case, seed=i if seed is None else seed)
            if fp8 and id(V) not in exact:  # the codes are exact in e4m3 (values 0 and s = 1 or 2), so the tables hold for x'
                assert all(torch.equal(vp.view(torch.int16), v.view(torch.int16)) for v, vp in zip(V, kv_prime(V, V)[1])), f"{case}: V' != V"
                exact.add(id(V))
            rows = len(expected(case).n)
            outs.append(run(case, torch.zeros(rows, case.KV * rep, HD, dtype=torch.bfloat16), K, V, rep, ws, fp8))

    assert_launched(launches, KERNEL[kernel].format(rep=rep), ATTN, len(cases))
    for case, out in zip(cases, outs):
        assert_visible_sets(out, case, rep)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("kernel", ["wgmma", "mma"])
def test_first_prefill_visible_sets(kernel, rep, ws, monkeypatch):
    """First prefill (T >= 128, max_seqlen >= 128, seqpos 0): windows at and one away from the 128-key tiles, sequences at and one
    away from them, 128-row TMA boxes that run into the next sequence or past T; the same table for the mma kernel."""
    check_visible_sets(first_prefill_cases(), kernel, rep, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
def test_ring_prefill_visible_sets(rep, ws, monkeypatch):
    """Chunks on top of the ring (seqpos > 0, attn_prefill_kernel): before, at and after the first wrap, several wraps, chunks
    around the 64-key tile, and a batch in which one sequence has nothing cached yet."""
    check_visible_sets(ring_cases(), "mma", rep, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
def test_ring_prefill_visible_sets_fp8(rep, ws, monkeypatch):
    """The same chunks on an e4m3 ring (attn_prefill_fp8_kernel): the old keys come from the ring's codes and exponents, wrapped
    or not, the chunk's from its bf16 k', v'."""
    check_visible_sets(ring_cases(), "mma_fp8", rep, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
def test_cacheless_visible_sets(rep, ws, monkeypatch):
    """causal = 0 (attn_prefill_kernel): every query sees all T keys."""
    check_visible_sets(nocache_cases(), "mma", rep, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("kernel", ["tma", "tma_fp8"])
def test_decode_visible_sets(kernel, rep, ws, monkeypatch):
    """The decode kernel: kv_len around the 64-key tile and at the window, more splits than keys, B = 5 on a cache with
    max_batch 6, and on one workspace S = 64 then S = 7 (the split counters reset themselves between launches)."""
    check_visible_sets(decode_cases(), kernel, rep, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("kernel", ["tma", "tma_fp8"])
@pytest.mark.parametrize("W", PROD_LONG_WINDOWS)
def test_production_decode_visible_sets(W, kernel, rep, ws, monkeypatch):
    """KV = 8, batch 1, on a 4096 and a 32768 ring: splits holding up to 16 tiles (so the FP8 reader's one-tile-ahead exponent
    loads and its 5-stage ring run inside a split with k_begin > 0), at S = 64, 33, 7, 1 on one workspace."""
    check_visible_sets(production_long_cases(W), kernel, rep, ws, monkeypatch, seed=W)


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("kernel", ["tma", "tma_fp8"])
def test_production_batch_decode_visible_sets(kernel, rep, ws, monkeypatch):
    """KV = 8, batches 2, 4, 8 on a 4096 ring with ragged kv_len, at the model's S and a forced one."""
    check_visible_sets(production_batch_cases(), kernel, rep, ws, monkeypatch)


# ----------------------------------------------------------------------------- softmax weighting against float64
SOFTMAX_CASES = {
    "wgmma": Case("prefill", (0, 0), (300, 129), 200),
    "mma": Case("prefill", (150, 37), (130, 65), 200),
    "tma": Case("decode", (300, 129, 64, 1, 200), (), 300, 7),
    "mma_fp8": Case("prefill", (150, 37), (130, 65), 200),
    "tma_fp8": Case("decode", (300, 129, 64, 1, 200), (), 300, 7),
}
SOFTMAX_PROD_CASE = Case("decode", (4000,), (), 4096, 7, PROD_KV)  # 572 keys per split: 9 tiles, the last one partial
LOG2E = 1.4426950408889634
SCORE_LOG2_PER_UNIT = HD * HD ** -0.5 * LOG2E  # q = k = all-ones vectors: score in log2 units
DOMINANT = [0, 63, 64, 127, 128, 199, 255, 256, 299]  # first, 64/128-key tile edges, window lower edges, last keys


def softmax_inputs(case: Case, pattern: str, rep: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    KV = case.KV
    H = KV * rep
    rows = len(expected(case).n)
    B = n_seqs(case) + (1 if case.kind == "decode" else 0)
    K, V = [], []
    u = torch.sign(torch.randn(HD, generator=g))  # the direction the dominant keys share with every query
    for b in range(B):
        n = n_positions(case, b)
        V.append(torch.randn(n, KV, HD, generator=g).to(torch.bfloat16))
        if pattern == "rising":  # score rises by 0.07 log2 units per position: the running max grows in every tile and split
            K.append((torch.arange(n, dtype=torch.float64) * (0.07 / SCORE_LOG2_PER_UNIT))[:, None, None].expand(n, KV, HD).to(torch.bfloat16))
        elif pattern == "dominant":  # scores within about +-1.5 log2 units, and keys 18..34 units above them at the DOMINANT positions
            k = torch.randn(n, KV, HD, generator=g) * 0.25
            for i, j in enumerate(p for p in DOMINANT if p < n):
                k[j] = u * (18 + 2 * i) / SCORE_LOG2_PER_UNIT
            K.append(k.to(torch.bfloat16))
        else:  # "wide": scores ~ N(0, 20^2) log2 units, spanning about +-60
            K.append((torch.randn(n, KV, HD, generator=g) * 3.7).to(torch.bfloat16))
    if pattern == "rising":
        q = torch.ones(rows, H, HD)
    elif pattern == "dominant":
        q = u + 0.3 * torch.randn(rows, H, HD, generator=g)
    else:
        q = torch.randn(rows, H, HD, generator=g) * 3.7
    return q.to(torch.bfloat16), K, V


def reference64(case: Case, q: torch.Tensor, K, V, rep: int):
    """(O64, sum_j p_j |v_j|), both [rows, H, 128] float64, straight from the mask and a float64 softmax."""
    outs, mags, r0 = [], [], 0
    for b in range(n_seqs(case)):
        m = torch.from_numpy(visible_mask(case, b))
        qb = q[r0:r0 + m.shape[0]].double()
        r0 += m.shape[0]
        kb = K[b].double().repeat_interleave(rep, 1)  # [n, H, 128]
        vb = V[b].double().repeat_interleave(rep, 1)
        s =torch.einsum("ihd,jhd->hij", qb, kb) * HD ** -0.5
        p = torch.softmax(s.masked_fill(~m[None], float("-inf")), -1)
        outs.append(torch.einsum("hij,jhd->ihd", p, vb))
        mags.append(torch.einsum("hij,jhd->ihd", p, vb.abs()))
    return torch.cat(outs), torch.cat(mags)


def check_softmax(case: Case, kernel: str, rep: int, pattern: str, ws, monkeypatch):
    """One launch of `kernel` on softmax_inputs against reference64, within the bound of the module docstring.  The FP8 readers
    see K', V' (the chunk's and the ring's), so their reference is computed on K', V'."""
    select_kernel(kernel, monkeypatch)
    fp8 = kernel.endswith("_fp8")
    q, K, V = softmax_inputs(case, pattern, rep, seed=rep)
    outs = []
    assert_launched(lambda: outs.append(run(case, q, K, V, rep, ws, fp8)), KERNEL[kernel].format(rep=rep), ATTN, 1)
    got = outs[0].double().cpu()
    o64, mag = reference64(case, q, *(kv_prime(K, V) if fp8 else (K, V)), rep)
    ulp = torch.exp2(torch.floor(torch.log2(o64.abs().clamp_min(2.0 ** -126))) - 7)
    bound = 2.0 ** -8 * mag + ulp
    err = (got - o64).abs()
    assert torch.isfinite(got).all(), "non-finite output"
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"{(err > bound).sum().item()} elements beyond the bound; worst err / bound = {worst:.2f}"


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["rising", "dominant", "wide"])
@pytest.mark.parametrize("rep", [1, 4, 8])
@pytest.mark.parametrize("kernel", ["wgmma", "mma", "tma", "mma_fp8", "tma_fp8"])
def test_softmax_weighting_vs_float64(kernel, rep, pattern, ws, monkeypatch):
    """Online softmax under stress: maxima that grow in every key tile and split, one dominant key at the first / last / tile-edge
    / window-edge position, and scores spanning +-60 in log2 units.  Bound derived in the module docstring."""
    check_softmax(SOFTMAX_CASES[kernel], kernel, rep, pattern, ws, monkeypatch)


@pytest.mark.gpu
@pytest.mark.parametrize("pattern", ["rising", "dominant", "wide"])
@pytest.mark.parametrize("rep", REPS)
@pytest.mark.parametrize("kernel", ["tma", "tma_fp8"])
def test_softmax_weighting_production_decode(kernel, rep, pattern, ws, monkeypatch):
    """The same bound at KV = 8, batch 1, 4000 keys over 7 splits of 9 tiles each: the running max and the exponents of V change
    from tile to tile inside a split."""
    check_softmax(SOFTMAX_PROD_CASE, kernel, rep, pattern, ws, monkeypatch)
