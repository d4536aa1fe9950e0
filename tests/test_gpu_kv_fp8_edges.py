"""The FP8 (e4m3) KV cache at exponent, code, split and capacity edges.

The format (include/mistral_b200.h, FP8 KV cache) stores each (slot, kv head) row as 128 e4m3 codes q and one int8 exponent e, and
x' = q * 2^e.  Each reader rebuilds the bf16 bits of x' and runs its bf16 kernel's arithmetic, so it is bit-identical to that
kernel on a bf16 ring holding x'.  The tests here apply that oracle, and exact tables where the design allows, where the suite did
not reach before:

* Exponent sweep.  Rings built directly from (code, e): one (sequence, kv head) per exponent e in [-124, 120] (31 sequences x 8 kv
  heads), and its rows hold every finite e4m3 code, so every (code, e) pair a ring can hold goes through both rebuild paths of
  kv_dequant2 (the integer rebias for e >= -112, the exact fp32 product below) in the decode reader's V and K tiles and the
  prefill reader's ring rows.  The quantiser writes e = 120 only for amax > 1.75 * 2^127, where no code above 256 occurs; code 256
  under e = 120 is x' = +-inf.
* The quantiser on every finite bf16 amax below 2^127, both signs: codes, exponent, write-back and ring rows against the CPU
  restatement (tests/kv_fp8_ref.py), the projection property, and the rows at and above 2^127 that lie outside the format.
* Decode with several tiles per split (the production case: S = 33 at batch 1 and KV = 8) on rows whose exponents change from key
  to key, and a 2-layer model with 32 query heads over 8 kv heads against the FP8-cache restatement at S > 1.
* The counter block of the split merge: B * KV = 2048 fills it, 2049 is refused before any launch, and the FP8 and bf16 decode
  kernels alternate on one workspace with different S.
"""
import math

import pytest
import torch

import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer_layers import decode_splits

from . import kv_fp8_ref as K
from .test_gpu_kv_fp8 import check_against_oracle, fp8_model_and_oracle, random_rows
from .util import assert_launched, launched_kernels

DEV = "cuda"
HD = 128
ATTN = r"attn_\w+_kernel"
REPS = [1, 2, 4, 6, 8]
E_MIN, E_MAX = K.EXP_MIN, 120       # the exponents the quantiser writes (2^-e is a normal fp32 for all of them)
E_SPLIT = -112                      # kv_dequant2: the integer rebias from here up, the exact fp32 product below
SEQS, KVH = 31, 8                   # 248 (sequence, kv head) rows, one exponent each
LAYOUT_EXPS = list(range(E_MIN, E_MAX + 1)) + [E_SPLIT - 1, E_SPLIT, E_MAX - 1]  # the last three: the path switch and the top again
CODE_256 = 0x78                     # e4m3 magnitude code of 256; 0x79..0x7E are 288..448


def bits(x: torch.Tensor) -> torch.Tensor:
    return x.contiguous().view(torch.int16)


def e4m3_value(codes: torch.Tensor) -> torch.Tensor:
    return codes.to(torch.uint8).view(torch.float8_e4m3fn).double()


def holdable(code: int, e: int) -> bool:
    """Can a quantised ring hold `code` under `e`?  Every finite code under e < 120; under e = 120 (amax > 1.75 * 2^127, and
    amax <= 255 * 2^120) only codes up to 256."""
    return (code & 0x7F) != 0x7F and E_MIN <= e <= E_MAX and (e < E_MAX or (code & 0x7F) <= CODE_256)


def code_row(e: int, half: int, roll: int, key: bool = False) -> torch.Tensor:
    """128 e4m3 codes: the 127 finite codes of one sign (half 0: 0x00..0x7E, half 1: 0x80..0xFE) rotated by `roll`, then the zero of
    that sign.  Under e = 120 codes above 256 become that zero; in a key (`key`) so does 256, whose x' is infinite and would make
    every score of the row infinite."""
    row = torch.roll(torch.arange(127) + 128 * half, roll)
    if e == E_MAX:
        top = CODE_256 if key else CODE_256 + 1
        row = torch.where((row & 0x7F) >= top, row & 0x80, row)
    return torch.cat([row, torch.tensor([128 * half])]).to(torch.uint8)


def exps_grid() -> torch.Tensor:
    return torch.tensor(LAYOUT_EXPS, dtype=torch.int8).view(SEQS, KVH)


def poisoned_ring(B: int, W: int, KV: int):
    """(q, e) of a ring whose every row holds NaN codes and extreme exponents, and the bf16 ring of NaN that stands for it."""
    q = torch.tensor([0x7F, 0xFF, 0x00, 0x80], dtype=torch.uint8).repeat(B * W * KV * HD // 4).view(B, W, KV, HD)
    e = torch.tensor([127, -128], dtype=torch.int8).repeat(B * W * KV)[: B * W * KV].view(B, W, KV).contiguous()
    return q, e


def xprime_ring(q: torch.Tensor, e: torch.Tensor, written: torch.Tensor) -> torch.Tensor:
    """bf16 ring of x' where `written` [B, W] is set, NaN elsewhere."""
    xp = K.dequant(q, e)
    xp[~written] = float("nan")
    return xp


def sweep_v_rows(half: int) -> torch.Tensor:
    """[SEQS, KVH, 128] codes of the V rows of launch `half`."""
    E = exps_grid()
    return torch.stack([torch.stack([code_row(int(E[b, g]), half, (7 * b + g) % 127) for g in range(KVH)]) for b in range(SEQS)])


def sweep_k_rows(half: int, slot: int) -> torch.Tensor:
    E = exps_grid()
    return torch.stack([torch.stack([code_row(int(E[b, g]), (half + slot) % 2, (31 * slot + 5 * b + g) % 127, key=True) for g in range(KVH)])
                        for b in range(SEQS)])


PREFILL_W = 16
PREFILL_SEQPOS = [10 if b % 2 == 0 else 37 for b in range(SEQS)]  # slots 0..9 written / every slot written, the ring wrapped twice
PREFILL_LENS = [1 if (b // 2) % 2 == 0 else 3 for b in range(SEQS)]


def prefill_ring_rows(pos: int, key: bool) -> torch.Tensor:
    """[SEQS, KVH, 128] codes of the ring rows at absolute position `pos` (in slot pos % W)."""
    E = exps_grid()
    return torch.stack([torch.stack([code_row(int(E[b, g]), pos % 2, (8 * pos + 3 * key + b + g) % 127, key=key) for g in range(KVH)])
                        for b in range(SEQS)])


def prefill_visible(b: int) -> range:
    """Ring positions every query of sequence b sees (the chunk's first query sees (p - W, p])."""
    p = PREFILL_SEQPOS[b]
    return range(max(0, p - PREFILL_W + 1), p)


def scaled_queries(n: int, rep: int, seed: int) -> torch.Tensor:
    """[n, SEQS, KVH * rep, 128] bf16: 8 non-zero dims of +-[1, 2) per head, times 2^(-6 - e) of the head's group, so that q . x'
    does not depend on e and the softmax weights every key of the sweep rows (checked on the CPU)."""
    g = torch.Generator().manual_seed(seed)
    u = (1 + torch.rand(n, SEQS, KVH * rep, HD, generator=g)) * torch.sign(torch.randn(n, SEQS, KVH * rep, HD, generator=g))
    keep = torch.rand(n, SEQS, KVH * rep, HD, generator=g).argsort(-1) < 8
    scale = torch.ldexp(torch.ones(SEQS, KVH), -6 - exps_grid().to(torch.int32)).repeat_interleave(rep, 1)
    return (u * keep * scale[None, :, :, None]).to(torch.bfloat16)


# ----------------------------------------------------------------------------- CPU checks of the designs
def test_sweep_layout_covers_every_holdable_pair():
    """V launches hold every (code, e) pair a ring can hold; K and prefill-key rows every one but +-256 under e = 120; the design
    puts one exponent per (sequence, kv head), e4m3 values are what the table says, and x' is exact in bf16."""
    E = exps_grid()
    want = {(c, e) for e in range(E_MIN, E_MAX + 1) for c in range(256) if holdable(c, e)}
    assert sorted(set(E.flatten().tolist())) == list(range(E_MIN, E_MAX + 1))
    no_inf = {(CODE_256, E_MAX), (CODE_256 | 0x80, E_MAX)}
    visible = sorted(set(p for b in range(SEQS) for p in prefill_visible(b)))
    for name, rows_of_seq, excluded in (  # rows_of_seq(b): the code rows [n, KVH, 128] sequence b's queries read
            ("decode V", lambda b: torch.stack([sweep_v_rows(h)[b] for h in (0, 1)]), set()),
            ("decode K", lambda b: torch.stack([sweep_k_rows(h, s)[b] for h in (0, 1) for s in range(4)]), no_inf),
            ("prefill K", lambda b: torch.stack([prefill_rows[True][p][b] for p in prefill_visible(b)]), no_inf),
            ("prefill V", lambda b: torch.stack([prefill_rows[False][p][b] for p in prefill_visible(b)]), set())):
        if name == "prefill K":
            prefill_rows = {key: {p: prefill_ring_rows(p, key) for p in visible} for key in (True, False)}
        got = set()
        for b in range(SEQS):
            rows = rows_of_seq(b)
            for g in range(KVH):
                got |= {(c, int(E[b, g])) for c in rows[:, g].flatten().tolist()}
        assert all(holdable(c, e) for c, e in got), name
        assert got == want - excluded, f"{name}: missing {sorted(want - excluded - got)[:8]}"
    # e4m3 values: 254 finite, 0x7F / 0xFF NaN, and x' = q * 2^e is the exact product (or +-inf for 256 * 2^120)
    v = e4m3_value(torch.arange(256))
    assert int(torch.isnan(v).sum()) == 2 and v[0x7E] == 448 and v[CODE_256] == 256 and v[1] == 2.0 ** -9
    for e in (E_MIN, E_SPLIT - 1, E_SPLIT, 0, E_MAX):
        codes = torch.tensor([c for c in range(256) if holdable(c, e)])
        xp = K.dequant(codes.to(torch.uint8), torch.tensor(e, dtype=torch.int8)).double()
        exact = e4m3_value(codes) * 2.0 ** e
        assert torch.equal(xp, torch.where(exact.abs() >= 2.0 ** 128, exact.sign() * math.inf, exact)), e


def test_scaled_queries_weight_every_key():
    """In the K sweeps every one of a row's keys gets a softmax weight of at least 2^-16 (float64, on the exact x')."""
    E = exps_grid().to(torch.int32)
    for rep in (1, 8):
        q = scaled_queries(1, rep, seed=rep)[0].double()  # [SEQS, H, 128]
        for h in (0, 1):
            keys = torch.stack([e4m3_value(sweep_k_rows(h, s)) * torch.ldexp(torch.ones(SEQS, KVH), E).double()[..., None]
                                for s in range(4)], 2)  # [SEQS, KVH, 4, 128]
            s = torch.einsum("bhd,bhjd->bhj", q, keys.repeat_interleave(rep, 1)) * HD ** -0.5
            p = torch.softmax(s, -1)
            assert p.min() >= 2.0 ** -16, (rep, h, p.min().item())


# ----------------------------------------------------------------------------- exponent sweep: decode reader
def decode_pair(q, k8, ek, v8, ev, xk, xv, kv_len, KV, rep, S):
    """(FP8 decode out, bf16 decode out on x'), each on a fresh workspace."""
    B = q.shape[0]
    H = KV * rep
    ws = _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + B * KV * S * rep * (HD + 2) * 4, torch.device(DEV))
    want, got = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    _abi.attn_decode(q, xk, xv, kv_len, want, H, KV, HD, S, ws)
    assert_launched(lambda: _abi.attn_decode_fp8(q, k8, v8, ek, ev, kv_len, got, H, KV, HD, S, ws),
                    rf"attn_decode_tma_fp8_kernel<{rep}>", ATTN, 1)
    return got, want


@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
def test_decode_v_rows_every_code_and_exponent(rep):
    """kv_len = 1, S = 1: the output is the V row.  It equals x' bit for bit where x' is a normal bf16, and the bf16 kernel on x'
    everywhere (zeros, bf16 subnormals and +-inf included)."""
    W, E = 64, exps_grid()
    for half in (0, 1):
        qk, ek = poisoned_ring(SEQS + 1, W, KVH)
        qv, ev = qk.clone(), ek.clone()
        qk[:, 0], ek[:, 0] = K.quantize_kv_rows(random_rows((SEQS + 1, KVH), 70 + half))
        qv[:SEQS, 0], ev[:SEQS, 0] = sweep_v_rows(half), E
        written = torch.zeros(SEQS + 1, W, dtype=torch.bool)
        written[:, 0] = True
        xk, xv = xprime_ring(qk, ek, written), xprime_ring(qv, ev, written)
        q = torch.randn(SEQS, KVH * rep * HD, generator=torch.Generator().manual_seed(rep)).to(torch.bfloat16).to(DEV)
        kv_len = torch.ones(SEQS, dtype=torch.int32, device=DEV)
        dev = [t.to(DEV) for t in (qk, ek, qv, ev, xk, xv)]
        got, want = decode_pair(q, dev[0].view(torch.float8_e4m3fn), dev[1], dev[2].view(torch.float8_e4m3fn), dev[3], dev[4], dev[5],
                                kv_len, KVH, rep, 1)
        got, want = got.cpu().view(SEQS, KVH, rep, HD), want.cpu().view(SEQS, KVH, rep, HD)
        assert torch.equal(bits(got), bits(want)), f"half {half}: FP8 != bf16 on x' at exponents " \
            f"{sorted(set(E[(bits(got) != bits(want)).flatten(2).any(-1)].tolist()))[:8]}"
        xp = xv[:SEQS, 0][:, :, None, :].expand(SEQS, KVH, rep, HD)
        exp_field = bits(xp) & 0x7F80
        normal = (exp_field != 0) & (exp_field != 0x7F80)
        off = normal & (bits(got) != bits(xp))
        assert not off.any(), f"half {half}: output != x' at exponents {sorted(set(E[off.flatten(2).any(-1)].tolist()))[:8]}"
        assert int(normal.sum()) > 0.8 * normal.numel()


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 4])
@pytest.mark.parametrize("rep", REPS)
def test_decode_k_rows_every_code_and_exponent(rep, S):
    """kv_len = 4: four key rows of codes under the group's exponent, queries scaled by 2^-e so that all four keys carry weight;
    the output equals the bf16 kernel on x' bit for bit (S = 4: one key per split)."""
    W, E = 64, exps_grid()
    for half in (0, 1):
        qk, ek = poisoned_ring(SEQS + 1, W, KVH)
        qv, ev = qk.clone(), ek.clone()
        for s in range(4):
            qk[:SEQS, s], ek[:SEQS, s] = sweep_k_rows(half, s), E
        qv[:, :4], ev[:, :4] = K.quantize_kv_rows(random_rows((SEQS + 1, 4, KVH), 80 + half))
        qk[SEQS, :4], ek[SEQS, :4] = K.quantize_kv_rows(random_rows((4, KVH), 90 + half))
        written = torch.zeros(SEQS + 1, W, dtype=torch.bool)
        written[:, :4] = True
        xk, xv = xprime_ring(qk, ek, written), xprime_ring(qv, ev, written)
        q = scaled_queries(1, rep, seed=rep + 10 * half)[0].reshape(SEQS, -1).to(DEV)
        kv_len = torch.full((SEQS,), 4, dtype=torch.int32, device=DEV)
        dev = [t.to(DEV) for t in (qk, ek, qv, ev, xk, xv)]
        got, want = decode_pair(q, dev[0].view(torch.float8_e4m3fn), dev[1], dev[2].view(torch.float8_e4m3fn), dev[3], dev[4], dev[5],
                                kv_len, KVH, rep, S)
        got, want = got.cpu().view(SEQS, KVH, rep * HD), want.cpu().view(SEQS, KVH, rep * HD)
        assert torch.isfinite(want.float()).all()
        bad = (bits(got) != bits(want)).any(-1)
        assert not bad.any(), f"half {half}: FP8 != bf16 on x' at exponents {sorted(set(E[bad].tolist()))[:8]}"


# ----------------------------------------------------------------------------- exponent sweep: prefill reader
@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
def test_prefill_ring_rows_every_code_and_exponent(rep):
    """Chunks of 1 and 3 tokens on a 16-slot ring whose K and V rows hold the sweep codes under each group's exponent: sequences at
    position 10 (slots 0..9 written, none wrapped) and 37 (every slot written, wrapped twice).  attn_prefill_fp8_kernel equals
    attn_prefill_kernel on x' bit for bit."""
    W, E, seqpos, lens = PREFILL_W, exps_grid(), PREFILL_SEQPOS, PREFILL_LENS
    T = sum(lens)
    qk, ek = poisoned_ring(SEQS, W, KVH)
    qv, ev = qk.clone(), ek.clone()
    written = torch.zeros(SEQS, W, dtype=torch.bool)
    rows_at = {pos: (prefill_ring_rows(pos, True), prefill_ring_rows(pos, False)) for pos in range(max(seqpos))}
    for b, p in enumerate(seqpos):
        for pos in range(max(0, p - W), p):
            slot = pos % W
            qk[b, slot], qv[b, slot] = rows_at[pos][0][b], rows_at[pos][1][b]
            ek[b, slot], ev[b, slot] = E[b], E[b]
            written[b, slot] = True
    xk, xv = xprime_ring(qk, ek, written), xprime_ring(qv, ev, written)
    g = torch.Generator().manual_seed(100 + rep)
    seq_of_tok = torch.repeat_interleave(torch.arange(SEQS), torch.tensor(lens))
    scale = torch.ldexp(torch.ones(SEQS, KVH), E.to(torch.int32))[seq_of_tok]  # chunk keys at the group's scale too
    kn = K.kv_prime(((torch.randn(T, KVH, HD, generator=g) * 16).clamp(-200, 200) * scale[..., None]).to(torch.bfloat16))
    vn = K.kv_prime(torch.randn(T, KVH, HD, generator=g).to(torch.bfloat16))
    qs = scaled_queries(3, rep, seed=rep)  # [3, SEQS, H, 128]
    q = torch.cat([qs[:n, b] for b, n in enumerate(lens)]).reshape(T, -1)
    q_start = torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32, device=DEV)
    sp = torch.tensor(seqpos, dtype=torch.int32, device=DEV)
    H = KVH * rep
    qd, knd, vnd = q.to(DEV), kn.reshape(T, -1).to(DEV), vn.reshape(T, -1).to(DEV)
    want, got = torch.full_like(qd, float("nan")), torch.full_like(qd, float("nan"))
    _abi.attn_prefill(qd, knd, vnd, xk.to(DEV), xv.to(DEV), q_start, sp, want, SEQS, max(lens), W, H, KVH, HD, causal=True)
    assert_launched(lambda: _abi.attn_prefill_fp8(qd, knd, vnd, qk.to(DEV).view(torch.float8_e4m3fn), qv.to(DEV).view(torch.float8_e4m3fn),
                                                  ek.to(DEV), ev.to(DEV), q_start, sp, got, SEQS, max(lens), W, H, KVH, HD),
                    r"attn_prefill_fp8_kernel\b", ATTN, 1)
    got, want = got.cpu().view(T, KVH, rep * HD), want.cpu().view(T, KVH, rep * HD)
    finite_groups = E[seq_of_tok] <= 100  # higher up, sums of up to 18 weighted V rows near 2^127 may overflow fp32 in both kernels
    assert torch.isfinite(want.float())[finite_groups].all()
    bad = (bits(got) != bits(want)).any(-1)
    assert not bad.any(), f"FP8 != bf16 on x' at exponents {sorted(set(E[seq_of_tok][bad].tolist()))[:8]}"


# ----------------------------------------------------------------------------- several tiles per split
@pytest.mark.gpu
@pytest.mark.parametrize("rep", REPS)
def test_decode_multi_tile_splits_equal_bf16_on_x_prime(rep):
    """KV = 8 at batch 1 on a 16384-slot ring, rows whose scales (hence exponents) change from key to key: 2113 keys over 33 splits
    (2 tiles each, as the model decodes from 2.1k keys), 16384 over 33 (8) and over 7 (37: the 5-stage ring turns over 7 times
    inside one split), 4000 over 64; one workspace.  Bit for bit against the bf16 kernel on x'."""
    W, KV = 16384, 8
    H = KV * rep
    q8, e8 = K.quantize_kv_rows(random_rows((2, W, KV), 110 + rep))
    v8, f8 = K.quantize_kv_rows(random_rows((2, W, KV), 120 + rep))
    q = torch.randn(1, H * HD, generator=torch.Generator().manual_seed(rep)).to(torch.bfloat16).to(DEV)
    ws = _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + KV * 64 * rep * (HD + 2) * 4, torch.device(DEV))
    for n, S in ((2113, 33), (W, 33), (W, 7), (4000, 64)):
        written = torch.zeros(2, W, dtype=torch.bool)
        written[0, :n] = written[1] = True
        k8, ek = poisoned_ring(2, W, KV)
        vv, ev = k8.clone(), ek.clone()
        k8[written], ek[written], vv[written], ev[written] = q8[written], e8[written], v8[written], f8[written]
        xk, xv = xprime_ring(k8, ek, written).to(DEV), xprime_ring(vv, ev, written).to(DEV)
        kv_len = torch.tensor([n], dtype=torch.int32, device=DEV)
        want, got = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
        _abi.attn_decode(q, xk, xv, kv_len, want, H, KV, HD, S, ws)
        del xk, xv
        assert_launched(lambda: _abi.attn_decode_fp8(q, k8.to(DEV).view(torch.float8_e4m3fn), vv.to(DEV).view(torch.float8_e4m3fn), ek.to(DEV),
                                                     ev.to(DEV), kv_len, got, H, KV, HD, S, ws),
                        rf"attn_decode_tma_fp8_kernel<{rep}>", ATTN, 1)
        assert torch.isfinite(want.float()).all()
        assert torch.equal(bits(got), bits(want)), f"kv_len {n}, S {S}: max |d| {(got.float() - want.float()).abs().max().item()}"


# ----------------------------------------------------------------------------- the quantiser, exhaustively
def amax_rows(lo_bits: int, hi_bits: int, seed: int) -> torch.Tensor:
    """One row per bf16 magnitude with bit pattern in [lo_bits, hi_bits), both signs: that value at a rotating position, the other
    127 elements at or below it -- the 63 bf16 values just below it (down to 0) and 64 fractions of it -- with random signs."""
    mag = torch.arange(lo_bits, hi_bits, dtype=torch.int32)
    amax = torch.cat([mag, mag]).to(torch.int16).view(torch.bfloat16).float()
    amax[len(mag):] *= -1
    n = len(amax)
    a = amax.abs()[:, None]
    below = (torch.cat([mag, mag])[:, None] - torch.arange(1, 64)).clamp_min(0).to(torch.int16).view(torch.bfloat16).float()
    fracs = torch.cat([torch.tensor([0.0, 1.0, 0.5, 0.75]), torch.linspace(0.001, 0.999, 60)])
    row = torch.cat([amax[:, None], below, (a * fracs).to(torch.bfloat16).float()], 1)  # [n, 128]
    g = torch.Generator().manual_seed(seed)
    sign = torch.where(torch.rand(n, HD, generator=g) < 0.5, -1.0, 1.0)
    sign[:, 0] = 1.0
    row = row * sign
    shift = torch.arange(n)[:, None]
    row = torch.gather(row, 1, (torch.arange(HD)[None, :] - shift) % HD)  # amax lands at position n % 128
    return row.to(torch.bfloat16)


def test_amax_rows_design():
    """Each row's largest magnitude is its designed amax, and the rows hit every exponent of the format."""
    rows = amax_rows(0, 254 * 128, 1)
    mag = torch.arange(0, 254 * 128, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).float()
    assert torch.equal(rows.float().abs().amax(1), torch.cat([mag, mag]))
    _, e = K.quantize_kv_rows(rows)
    assert sorted(set(e.tolist())) == list(range(E_MIN, E_MAX))  # e = 120 only from amax > 1.75 * 2^127, outside these rows
    top = amax_rows(254 * 128, 254 * 128 + 128, 2)
    assert set(K.quantize_kv_rows(top)[1].tolist()) == {E_MAX - 1, E_MAX}


def quantize_on_device(x: torch.Tensor, rows: torch.Tensor, n_rows: int):
    """mb200_kv_quantize of x [T, KV, 128] as K and of x reversed along T as V, with write-back, into a ring of n_rows rows
    pre-filled with 0x55 codes and exponent 99.  Returns (k', v', ring q k, ring q v, ring e k, ring e v) on the CPU."""
    T, KV, _ = x.shape
    kd, vd = x.reshape(T, -1).to(DEV), x.flip(0).reshape(T, -1).contiguous().to(DEV)
    ck = torch.full((n_rows, KV, HD), 0x55, dtype=torch.uint8, device=DEV)
    cv = ck.clone()
    ek = torch.full((n_rows, KV), 99, dtype=torch.int8, device=DEV)
    ev = ek.clone()
    assert_launched(lambda: _abi.kv_quantize(kd, vd, True, ck, cv, ek, ev, rows.to(DEV)), r"kv_quantize_kernel", r"kv_quantize", 1)
    return [t.cpu() for t in (kd.view(T, KV, HD), vd.view(T, KV, HD), ck, cv, ek, ev)]


def check_ring(ring_q, ring_e, q, e, rows, n_rows):
    written = torch.zeros(n_rows, dtype=torch.bool)
    r = rows[rows >= 0].long()
    written[r] = True
    assert torch.equal(ring_q[r], q[rows >= 0]) and torch.equal(ring_e[r], e[rows >= 0])
    assert ring_q[~written].eq(0x55).all() and ring_e[~written].eq(99).all()  # tokens with row -1 and unused rows: untouched


@pytest.mark.gpu
def test_quantizer_every_amax():
    """Every finite bf16 amax below 2^127, both signs (65024 rows as K, the same rows in reverse order as V): e, the codes, the
    in-place x' and the ring rows (a permutation, every fifth token uncached) bit for bit against the CPU restatement.  Then the
    projection: quantising x' returns x', and the stored bytes differ only where a row's largest |q| is 224, as (e - 1, 2q)."""
    x = amax_rows(0, 254 * 128, 3).view(-1, 8, HD)  # [8128 tokens, 8 kv heads, 128]
    T, n_rows = x.shape[0], x.shape[0] + 7
    rows = torch.randperm(n_rows, generator=torch.Generator().manual_seed(4))[:T].to(torch.int32)
    rows[::5] = -1
    kp, vp, ck, cv, ek, ev = quantize_on_device(x, rows, n_rows)
    for xs, xp, ring_q, ring_e in ((x, kp, ck, ek), (x.flip(0), vp, cv, ev)):
        q, e = K.quantize_kv_rows(xs)
        assert torch.equal(bits(xp), bits(K.dequant(q, e))), "write-back x'"
        check_ring(ring_q, ring_e, q, e, rows, n_rows)
    # projection: x' -> x' (write-back of x' again), bytes only as documented
    all_rows = torch.arange(T, dtype=torch.int32)
    kpp, _, ck2, _, ek2, _ = quantize_on_device(kp, all_rows, T)
    assert torch.equal(bits(kpp), bits(kp)), "quantising x' again changed x'"
    q1, e1 = ck[rows[rows >= 0].long()], ek[rows[rows >= 0].long()]  # (q, e) of the cached tokens, from the first pass
    q2, e2 = ck2[(rows >= 0).nonzero().flatten()], ek2[(rows >= 0).nonzero().flatten()]
    v1, v2 = e4m3_value(q1), e4m3_value(q2)
    differ = (q1 != q2).any(-1) | (e1 != e2)
    doc = (v1.abs().amax(-1) == 224) & (e1.to(torch.int32) > E_MIN)
    assert torch.equal(differ, doc), f"{int((differ & ~doc).sum())} rows differ other than documented, {int((doc & ~differ).sum())} do not differ"
    assert torch.equal(e2[doc].to(torch.int32), e1[doc].to(torch.int32) - 1) and torch.equal(v2[doc], 2 * v1[doc])


@pytest.mark.gpu
def test_quantizer_outside_the_format():
    """Rows with amax >= 2^127 are outside the format.  The device does what the restatement does there: amax up to 1.75 * 2^127
    takes e = 119 with finite x'; above it e = 120, where 1.9375 * 2^127 and up round to code 256 and x' = +-inf."""
    x = amax_rows(254 * 128, 254 * 128 + 128, 5).view(-1, 8, HD)  # 256 rows
    T = x.shape[0]
    rows = torch.arange(T, dtype=torch.int32)
    kp, _, ck, _, ek, _ = quantize_on_device(x, rows, T)
    q, e = K.quantize_kv_rows(x)
    assert torch.equal(ck, q) and torch.equal(ek, e)
    assert torch.equal(bits(kp), bits(K.dequant(q, e)))
    amax = x.float().abs().amax(-1)
    pos = x.float().abs() == amax[..., None]
    assert (kp.float()[pos & (amax[..., None] >= 1.9375 * 2.0 ** 127)].abs() == math.inf).all()
    assert torch.isfinite(kp.float()[(amax <= 1.75 * 2.0 ** 127)]).all()


# ----------------------------------------------------------------------------- model at the production decode shape
def recording_splits(monkeypatch):
    """Records (B, kv heads, ring size, S) of every attn_decode_fp8 call the model makes (eager and graph-captured steps)."""
    calls = []
    orig = _abi.attn_decode_fp8

    def spy(q, cache_k, cache_v, exp_k, exp_v, kv_len, out, n_heads, n_kv_heads, head_dim, n_splits, ws):
        calls.append((q.shape[0], n_kv_heads, cache_k.shape[1], n_splits))
        return orig(q, cache_k, cache_v, exp_k, exp_v, kv_len, out, n_heads, n_kv_heads, head_dim, n_splits, ws)

    monkeypatch.setattr(_abi, "attn_decode_fp8", spy)
    return calls


@pytest.mark.gpu
@pytest.mark.parametrize("over,lens,chunk,tiles", [
    ({}, [2300], None, 2),                         # batch 1: S = 33, 70 keys per split on the per-layer graph path
    ({"sliding_window": 1024}, [2100, 1800, 1500], 700, 2),  # chunks read a wrapped e4m3 ring; decode over 1024 slots at S = 11
])
def test_model_production_decode_shape(over, lens, chunk, tiles, monkeypatch):
    """2 layers, 32 query heads over 8 kv heads of 128, kv_cache="fp8", against the FP8-cache restatement; the FP8 decode kernel
    runs with S > 1 and at least `tiles` 64-key tiles in a split."""
    p = synth.shape("mistral-7b", n_layers=2, dim=256, hidden_dim=512, vocab_size=512, sliding_window=over.get("sliding_window"))
    m, om = fp8_model_and_oracle(p, len(lens))
    calls = recording_splits(monkeypatch)
    check_against_oracle(m, om, p, f"32/8 heads {over}", lens, chunk)
    assert calls, "no FP8 decode launch"
    for B, KV, W, S in calls:
        assert (B, KV) == (len(lens), 8) and S == decode_splits(B, KV, W) and S > 1, (B, KV, W, S)
        first_len = min(min(lens) + 1, W)  # the shortest kv_len of the first decode step
        keys_per_split = math.ceil(first_len / S)
        assert math.ceil(keys_per_split / 64) >= tiles, (first_len, S)


# ----------------------------------------------------------------------------- the split counters
def small_rings(B: int, W: int, KV: int, seed: int):
    k8, ek = K.quantize_kv_rows(random_rows((B, W, KV), seed))
    v8, ev = K.quantize_kv_rows(random_rows((B, W, KV), seed + 1))
    return [t.to(DEV) for t in (k8, ek, v8, ev, K.dequant(k8, ek), K.dequant(v8, ev))]


@pytest.mark.gpu
@pytest.mark.parametrize("B,KV", [(256, 8), (2048, 1)])
def test_counter_block_full(B, KV):
    """B * KV = 2048 fills the 8 KB counter block: both decode kernels run at S = 2, agree bit for bit, and leave every counter 0."""
    W, rep, S = 64, 1, 2
    H = KV * rep
    k8, ek, v8, ev, xk, xv = small_rings(B, W, KV, 7)
    kv_len = torch.randint(1, W + 1, (B,), generator=torch.Generator().manual_seed(8), dtype=torch.int32).to(DEV)
    q = torch.randn(B, H * HD, generator=torch.Generator().manual_seed(9)).to(torch.bfloat16).to(DEV)
    ws = _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + B * KV * S * rep * (HD + 2) * 4, torch.device(DEV))
    want, got = torch.full_like(q, float("nan")), torch.full_like(q, float("nan"))
    _abi.attn_decode(q, xk, xv, kv_len, want, H, KV, HD, S, ws)
    assert ws.buf[:8192].eq(0).all()
    _abi.attn_decode_fp8(q, k8.view(torch.float8_e4m3fn), v8.view(torch.float8_e4m3fn), ek, ev, kv_len, got, H, KV, HD, S, ws)
    assert ws.buf[:8192].eq(0).all()
    assert torch.isfinite(want.float()).all() and torch.equal(bits(got), bits(want))


@pytest.mark.gpu
@pytest.mark.parametrize("B,KV", [(2049, 1), (683, 3)])
def test_counter_block_overflow_is_refused(B, KV):
    """B * KV = 2049 returns MB200_E_INVALID from both decode entry points, before any launch."""
    W, S = 4, 2
    q = torch.zeros(B, KV * HD, dtype=torch.bfloat16, device=DEV)
    ring = torch.zeros(B, W, KV, HD, dtype=torch.bfloat16, device=DEV)
    ring8 = torch.zeros(B, W, KV, HD, dtype=torch.uint8, device=DEV)
    ex = torch.zeros(B, W, KV, dtype=torch.int8, device=DEV)
    kv_len = torch.ones(B, dtype=torch.int32, device=DEV)
    ws = _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + B * KV * S * (HD + 2) * 4, torch.device(DEV))
    for call in (lambda out: _abi.attn_decode(q, ring, ring, kv_len, out, KV, KV, HD, S, ws),
                 lambda out: _abi.attn_decode_fp8(q, ring8, ring8, ex, ex, kv_len, out, KV, KV, HD, S, ws)):
        out = torch.full_like(q, float("nan"))
        errs = []

        def attempt():
            try:
                call(out)
            except _abi.Mb200Error as err:
                errs.append(str(err))

        assert not [n for n in launched_kernels(attempt) if n.startswith("attn_")]
        assert errs and "failed (-1)" in errs[0], errs
        torch.cuda.synchronize()
        assert torch.isnan(out.float()).all()


@pytest.mark.gpu
def test_fp8_and_bf16_decode_alternate_on_one_workspace():
    """The FP8 and bf16 decode kernels alternate on one workspace with different S (KV = 8, B = 4, ragged kv_len).  Each launch
    equals the same kernel at the same S on a fresh workspace, bit for bit, and leaves the counters 0."""
    B, W, KV, rep = 4, 4096, 8, 4
    H = KV * rep
    k8, ek, v8, ev, xk, xv = small_rings(B, W, KV, 11)
    kv_len = torch.tensor([4096, 65, 2113, 1], dtype=torch.int32, device=DEV)
    q = torch.randn(B, H * HD, generator=torch.Generator().manual_seed(12)).to(torch.bfloat16).to(DEV)
    part = B * KV * 64 * rep * (HD + 2) * 4
    shared = _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + part, torch.device(DEV))

    def launch(fp8, S, ws):
        out = torch.full_like(q, float("nan"))
        if fp8:
            _abi.attn_decode_fp8(q, k8.view(torch.float8_e4m3fn), v8.view(torch.float8_e4m3fn), ek, ev, kv_len, out, H, KV, HD, S, ws)
        else:
            _abi.attn_decode(q, xk, xv, kv_len, out, H, KV, HD, S, ws)
        return out

    for fp8, S in ((True, 64), (False, 7), (True, 33), (False, 64), (True, 2), (False, 33), (True, 7), (False, 2), (True, 64)):
        got = launch(fp8, S, shared)
        assert shared.buf[:8192].eq(0).all(), (fp8, S)
        fresh = launch(fp8, S, _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + part, torch.device(DEV)))
        assert torch.equal(bits(got), bits(fresh)), (fp8, S)
        if fp8:
            assert torch.equal(bits(got), bits(launch(False, S, _abi.Workspace(_abi.WORKSPACE_HEADER_BYTES + part, torch.device(DEV))))), S
