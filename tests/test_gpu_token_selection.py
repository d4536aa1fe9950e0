"""Token selection and speculative acceptance on the GPU (csrc/sampling.cuh, csrc/speculative.cuh), exactly, at tie, signed-zero,
NaN, vocabulary-tail and draw-boundary edges.

Every expected value is a float64 or exact-integer restatement on the host (tests/spec_ref.py, torch.argmax on the CPU copy of the
same fp32 rows).  Vocabulary sizes cover per = ceil(V / 1024) = 1, 2, 32, 128 and 129, partial last chunks and threads without
elements.  Where the kernel decides in fp32 what the reference decides in float64, an input is used only when it is decisive: at
least a relative 1e-5 from the decision's edge.  The kernels' fp32 errors stay far below that: a nucleus probability is one
expf (2 ulp) and two products, a prefix or block sum has at most per + 10 roundings (per sequential adds, then 5 shuffle and
5 cross-warp levels), so even at per = 129 the bound is (129 + 10 + 4) * 2^-24 < 9e-6.
"""
import math

import numpy as np
import pytest
import torch

from mistral_inference_b200 import _abi

from . import spec_ref as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
VS = [1, 31, 1000, 1024, 1025, 32000, 32768, 131072, 131073]
MARGIN = 1e-5
NAN_PAYLOADS = (0x7FC00000, 0x7FC12345, 0x7F800001)


def _f32(bits):
    return float(np.array([bits], dtype=np.uint32).view(np.float32)[0])


# ---------------------------------------------------------------------------------------------------------- argmax rows
def _argmax_rows(V: int, seed: int):
    """>= 64 distinct fp32 rows of V logits: seeded random rows, then each designed edge on a random row of its own.  Returns the
    rows [T, V] and per row the index the sign-bit-only key would have picked where that differs from torch's (or -1)."""
    g = torch.Generator().manual_seed(seed)
    rows, decoy = [], []

    def base():
        return torch.randn(V, generator=g) - 8.0  # every random logit < -1: a designed 0 or NaN is the maximum

    def add(r, d=-1):
        rows.append(r)
        decoy.append(d)

    i, j = int(torch.randint(0, V, (1,), generator=g)), V - 1
    for _ in range(16):
        add(torch.randn(V, generator=g) * 3)
    for _ in range(8):
        add((torch.randn(V, generator=g) * 2).to(torch.bfloat16).float())  # many exact ties
    r = base(); r[i] = r[min(i + 1024, V - 1)] = 5.0; add(r, min(i + 1024, V - 1))  # same thread's stride
    r = base(); a, b = 7 % V, (5 * 32 * 1 + 3) % V; r[a] = r[b] = 4.0; add(r, b)  # across warps (per = 1 lanes)
    r = base(); a, b = 3 % V, (V * 5) // 7; r[a] = r[b] = 4.0; add(r, b)  # across warps at any per
    r = base(); r[0] = r[j] = 6.0; add(r, j)  # first and last element
    r = base(); r[0] = 9.0; add(r)
    r = base(); r[j] = 9.0; add(r)
    add(torch.full((V,), -math.inf))
    r = base(); r[0] = -math.inf; r[j] = -math.inf; add(r)
    # signed zeros: -0.0 before +0.0, +0.0 before -0.0, and a row of zeros starting with -0.0
    r = base(); r[i] = -0.0; r[j] = 0.0; add(r, j if i != j else -1)
    r = base(); r[i] = 0.0; r[j] = -0.0; add(r)
    r = torch.zeros(V); r[::2] = -0.0; add(r, 1 if V > 1 else -1)
    r = torch.full((V,), -0.0); r[j] = 0.0; add(r, j)
    # NaN: positive, negative, different payloads, and NaN after +inf
    for bits in NAN_PAYLOADS:
        r = base(); r[i] = _f32(bits); add(r)
    r = base(); r[i] = _f32(0xFFC00000); r[j] = 3.0; add(r, j if i != j else -1)  # a negative NaN is still the maximum
    r = base(); r[0] = _f32(0x7FC00000); r[j] = _f32(0x7FC12345); add(r, j)  # the larger payload later
    r = base(); r[0] = math.inf; r[j] = _f32(0x7FC00000); add(r)
    r = base(); r[i] = _f32(0xFFC00000); r[j] = _f32(0x7FC00000); add(r, j if i != j else -1)
    while len(rows) < 64:
        add(torch.randn(V, generator=g))
    return torch.stack(rows), decoy


@pytest.mark.parametrize("V", VS)
def test_argmax_rows_exact(V):
    """mb200_argmax_rows == torch.argmax on the CPU, index for index, including -0.0/+0.0 ties (the first index wins) and NaN
    (the first NaN wins, whatever its sign or payload)."""
    rows, decoy = _argmax_rows(V, 100 + V)
    got = _abi.argmax_rows(rows.to(DEV)).cpu()
    want = rows.argmax(-1)
    bad = [(t, int(got[t]), int(want[t])) for t in range(rows.shape[0]) if got[t] != want[t]]
    assert not bad, f"V={V}: (row, kernel, torch) {bad}"
    assert len(set(map(tuple, rows.view(torch.int32).tolist()))) == rows.shape[0] or V <= 31  # the rows are all different


@pytest.mark.parametrize("k", [1, 4, 8])
def test_accept_greedy_exact(k):
    """B = 64 sequences at V = 131072 with their own rows, each row j a designed argmax row: out, n, the -1 tail and the seqpos
    advance equal spec_ref.accept_greedy, and the picks equal mb200_argmax_rows on every row the kernel reads.  Sequence b
    proposes the target's argmax up to j = b % (k + 1) and there the index a wrong key would pick (or argmax + 1)."""
    V, B, S = 131072, 64, k + 1
    designed, decoy = _argmax_rows(V, 7 + k)
    n_rows = designed.shape[0]
    pick = [(b * S + j * 13 + b // n_rows) % n_rows for b in range(B) for j in range(S)]
    logits = designed[pick].clone()
    # a distinct per-sequence perturbation of the random tail so that no two sequences share a row
    logits[:, -2] = torch.where(torch.isfinite(logits[:, -2]) & (logits[:, -2] < -1), -1.5 - torch.arange(B * S) * 1e-3, logits[:, -2])
    amax = logits.argmax(-1).view(B, S)
    dec = torch.tensor([decoy[p] for p in pick]).view(B, S)
    tokens = torch.zeros(B, S, dtype=torch.long)
    tokens[:, 0] = torch.arange(B) + 11
    for b in range(B):
        r = b % (k + 1)
        for j in range(k):
            a = int(amax[b, j])
            if j < r:
                tokens[b, j + 1] = a
            elif j == r:
                tokens[b, j + 1] = int(dec[b, j]) if int(dec[b, j]) not in (-1, a) else (a + 1) % V
            else:
                tokens[b, j + 1] = (a + 3) % V
    dl = logits.to(DEV)
    out = torch.full((B, S), -5, dtype=torch.long, device=DEV)
    n = torch.full((B,), -9, dtype=torch.int32, device=DEV)
    seqpos = torch.arange(B, dtype=torch.int32, device=DEV) * 3 + 100
    _abi.spec_accept_greedy(dl, tokens.to(DEV), out, n, seqpos)
    per_row = _abi.argmax_rows(dl).cpu().view(B, S)
    out, n, seqpos = out.cpu(), n.cpu(), seqpos.cpu()
    L = logits.view(B, S, V)
    for b in range(B):
        want, wn = ref.accept_greedy(L[b].numpy(), tokens[b].tolist())
        want[-1] = int(amax[b, wn])  # the reference is torch.argmax's index
        assert wn == b % (k + 1)
        assert int(n[b]) == wn and out[b].tolist() == want + [-1] * (S - len(want)), (b, out[b].tolist(), want)
        assert int(seqpos[b]) == b * 3 + 100 + wn + 1
        assert per_row[b, :wn + 1].tolist() == amax[b, :wn + 1].tolist() and int(out[b, wn]) == int(per_row[b, wn])


# ------------------------------------------------------------------------------------------------------- logprob_gather
def _logprob_tol(row: np.ndarray, t: int, lse_m: float) -> float:
    """The kernel's own error budget, from its operations: out = fl(fl(x_t - m) - logf(s)), s = sum of expf(fl(x_i - m)).
      x_t - m                  0.5 ulp of the difference
      each term of s           its argument's rounding, 2^-24 |x_i - m| relative, plus expf's 2 ulp; s is a sum of positive
                               terms, so its relative error is at most the softmax-weighted mean of these
      the sum                  per sequential adds plus log2(1024) = 10 tree levels, 2^-24 relative each
      logf                     1 ulp of log(s), plus the error of s carried through log: d(log s) = ds / s
      the final subtraction    0.5 ulp of the result"""
    V = row.size
    per = -(-V // 1024)
    m = row.max()
    d = row - m
    w = np.exp(d)  # softmax weights (unnormalised), float64
    w_mean_arg = float((w * np.abs(np.where(np.isfinite(d), d, 0.0))).sum() / w.sum())
    eps = 2.0 ** -24
    rel_s = w_mean_arg * eps + 2 * 2 * eps + (per + 10) * eps
    ulp = lambda x: float(np.spacing(np.float32(abs(x))))
    diff = float(row[t] - m)
    return 0.5 * ulp(diff) + rel_s * 1.01 + ulp(lse_m) + 0.5 * ulp(diff - lse_m)


@pytest.mark.parametrize("V", VS)
def test_logprob_gather_exact_budget(V):
    """log_softmax(row)[t] against float64 within the kernel's derived error budget, for logit spreads up to 1e4, targets at
    0, V - 1 and the argmax; a -inf logit gives exactly -inf; rows with target < 0 keep their sentinel."""
    g = torch.Generator().manual_seed(200 + V)
    rows, tgts = [], []
    for scale in (0.1, 1.0, 10.0, 300.0, 1e4 / 4):
        for t in ("zero", "last", "argmax", "random"):
            r = torch.randn(V, generator=g) * scale
            rows.append(r.clamp(-5e3, 5e3))
            tgts.append({"zero": 0, "last": V - 1, "argmax": int(r.argmax()), "random": int(torch.randint(0, V, (1,), generator=g))}[t])
    r = torch.randn(V, generator=g); r[0] = -1e4 / 2; r[-1] = 1e4 / 2; rows.append(r); tgts.append(0)  # spread 1e4
    if V > 1:
        r = torch.randn(V, generator=g); r[V // 2] = -math.inf; rows.append(r); tgts.append(V // 2)  # exactly -inf
    r = torch.randn(V, generator=g); rows.append(r); tgts.append(-1)
    r = torch.randn(V, generator=g); rows.append(r); tgts.append(-7)
    rows_t = torch.stack(rows)
    tgt = torch.tensor(tgts)
    out = torch.full((len(rows),), 123.25, device=DEV)
    _abi.logprob_gather(rows_t.to(DEV), tgt.to(DEV), out=out)
    out = out.cpu().double().numpy()
    for n, (r, t) in enumerate(zip(rows_t.numpy(), tgts)):
        if t < 0:
            assert out[n] == 123.25, n
            continue
        x = r.astype(np.float64)
        m = x.max()
        lse_m = float(np.log(np.exp(x - m).sum()))
        want = float(x[t] - m - lse_m)
        if not np.isfinite(x[t]):
            assert out[n] == -math.inf, (n, out[n])
            continue
        tol = _logprob_tol(x, t, lse_m)
        assert abs(out[n] - want) <= tol, (V, n, t, out[n], want, tol)


# ------------------------------------------------------------------------------------------------- sample_top_p, exact
TEMPS = [0.05, 0.7, 1.0, 4.0]
U_FIXED = [0.0, 2.0 ** -24, 0.5, float(np.nextafter(np.float32(1), np.float32(0)))]


def _top_p_rows(V: int, temp: float, seed: int):
    """Seeded random rows whose scaled logits spread ~5 nats at any temperature (a nucleus of a few to a few hundred tokens), and
    the designed rows.  Returns rows [R, V] and their names."""
    g = torch.Generator().manual_seed(seed)
    rows, names = [], []
    for n in range(6):
        rows.append(torch.randn(V, generator=g) * (4.0 * temp + 0.5))
        names.append(f"random{n}")
    # bf16 logits with an exact tie group straddling the cut at 0.8 (0.70 before it, 4 x 0.06 in it) and a tied top group (top_p = 0)
    p = np.full(V, 0.06 / max(V - 5, 1))
    if V >= 8:
        idx = torch.randperm(V, generator=g)[:5].tolist()
        p[idx[0]] = 0.70
        p[idx[1:]] = 0.06
        p /= p.sum()
        rows.append(torch.from_numpy(np.log(p) * temp).float().to(torch.bfloat16).float())
        names.append("bf16-tie-at-cut")
        q = np.full(V, 0.1 / (V - 3))
        idx = torch.randperm(V, generator=g)[:3].tolist()
        q[idx] = 0.3
        rows.append(torch.from_numpy(np.log(q / q.sum()) * temp).float().to(torch.bfloat16).float())
        names.append("bf16-tied-top")
    # -inf entries everywhere but a few; the only finite tokens at 0, at V - 1, inside the last thread's partial chunk
    per = -(-V // 1024)
    last_t = (V - 1) // per
    for name, where in (("first", [0]), ("last", [V - 1]), ("partial-chunk", list(range(last_t * per, V))[-3:]),
                        ("scattered", torch.randperm(V, generator=g)[:5].tolist())):
        r = torch.full((V,), -math.inf)
        r[where] = torch.randn(len(where), generator=g) * temp
        rows.append(r)
        names.append(f"inf-but-{name}")
    # one token at probability 1 at temperature 0.05 (a 6-logit gap is 120 nats there)
    r = torch.randn(V, generator=g).clamp(-3, 3)
    r[int(torch.randint(0, V, (1,), generator=g))] = 9.0
    rows.append(r)
    names.append("one-certain")
    return torch.stack(rows), names


@pytest.mark.parametrize("V", VS)
def test_sample_top_p_exact_picks(V):
    """For every decisive row and uniform, mb200_sample_top_p picks exactly the float64 inverse-CDF token of the float64 nucleus
    (kept iff the mass strictly above is <= top_p, ties kept together), at temperatures 0.05..4 and top_p 0 and 0.8.  Every
    row returns a valid index, never -1, and never a token the float64 nucleus drops."""
    n_u = len(U_FIXED) + 256
    checked = refused_rows = 0
    for ti, temp in enumerate(TEMPS):
        rows, names = _top_p_rows(V, temp, 300 + 17 * V + ti)
        R = rows.shape[0]
        ug = torch.Generator().manual_seed(400 + V + ti)
        us = torch.cat([torch.tensor(U_FIXED).expand(R, -1), torch.rand(R, 256, generator=ug)], 1).float()  # [R, n_u]
        dev_rows = rows.to(DEV).repeat_interleave(n_u, 0)
        for top_p in (0.0, 0.8):
            picks = _abi.sample_top_p(dev_rows, us.reshape(-1).to(DEV).contiguous(), temp, top_p).cpu().view(R, n_u).numpy()
            assert (picks >= 0).all() and (picks < V).all(), "an invalid index"
            nucs = ref.nuclei(ref.scaled_logits(rows.numpy(), temp), top_p, MARGIN)
            for r, nuc in enumerate(nucs):
                assert nuc.keeps(picks[r]).all(), (names[r], temp, top_p, "a token outside the float64 nucleus")
                if names[r].startswith(("bf16", "inf-but")) or (names[r] == "one-certain" and temp == 0.05):
                    assert nuc.decisive, (names[r], temp, top_p)
                if names[r] == "bf16-tie-at-cut" and top_p == 0.8:
                    assert nuc.idx.size == 5  # the whole tied group straddling the cut is kept
                if names[r] == "bf16-tied-top" and top_p == 0.0:
                    assert nuc.idx.size == 3  # top_p = 0 keeps exactly the maximum-probability group
                if names[r] == "one-certain" and temp == 0.05:
                    assert nuc.idx.size == 1 and (picks[r] == int(rows[r].argmax())).all()
                if not nuc.decisive:
                    refused_rows += 1
                    continue
                want, ok = ref.inverse_cdf(nuc.dense(), us[r].double().numpy(), MARGIN)
                bad = np.nonzero(ok & (picks[r] != want))[0]
                assert bad.size == 0, (names[r], temp, top_p, [(float(us[r, i]), int(picks[r, i]), int(want[i])) for i in bad[:5]])
                checked += int(ok.sum())
    print(f"\n[top-p] V={V}: {checked} decisive picks exact; {refused_rows} random rows refused as fixtures (cut within {MARGIN})")
    assert refused_rows <= 2 * len(TEMPS) * 3  # at most half the random rows
    assert checked > 0


# ------------------------------------------------------------------------------------------------- the draw's boundaries
def test_draw_boundary_sweep():
    """V = 32768 (one 32-token chunk per thread), top_p = 1: the finite tokens sit in three adjacent lanes of several warps, each
    followed by zero-mass lanes, with unequal probabilities so the scan's sums are inexact.  Around every weighted -> zero-mass
    lane boundary the uniform sweeps 513 consecutive fp32 values centred on the host's estimate of the boundary in u.  The picks
    must be non-decreasing in u and each must be the float64 inverse-CDF token or its kept neighbour across that boundary."""
    V, rows_n, half = 32768, 32, 256
    g = torch.Generator().manual_seed(500)
    rows, sweeps = [], []  # sweeps: (row, u values [513], token below, token above)
    gap_rows = 0
    for r in range(rows_n):
        row = torch.full((V,), -math.inf)
        warps = sorted(torch.randperm(32, generator=g)[:5].tolist())
        for w in warps:
            lane0 = int(torch.randint(0, 26, (1,), generator=g))
            for lane in range(lane0, lane0 + 3):
                row[(w * 32 + lane) * 32 + int(torch.randint(0, 32, (1,), generator=g))] = float(torch.randn(1, generator=g))
        rows.append(row)
        x = row.numpy()
        e = np.exp((x - x.max()).astype(np.float32)).astype(np.float32)
        wts = (e * (np.float32(1) / e.sum(dtype=np.float32))).astype(np.float32)  # the host's estimate of the kernel's weights
        d = ref.BlockDraw(wts)
        kept = np.nonzero(wts)[0]
        t_w = kept // 32
        gap_rows += d.orphans(rule="interval").size > 0
        for i, tok in enumerate(kept[:-1]):
            t = tok // 32
            if t_w[i + 1] == t + 1:
                continue  # the next lane is weighted: no zero-mass lane follows
            u_b = np.float32(d.upper[t] / d.total)
            us = [u_b]
            for _ in range(half):
                us.insert(0, np.nextafter(us[0], np.float32(0)))
                us.append(np.nextafter(us[-1], np.float32(1)))
            sweeps.append((r, np.array(us, dtype=np.float32), int(tok), int(kept[i + 1])))
    assert len(sweeps) >= rows_n * 4
    rows = torch.stack(rows)
    dev_rows = rows.to(DEV)
    picks = []
    for c in range(0, len(sweeps), 32):  # 32 sweeps (2 GB of rows) per launch
        part = sweeps[c:c + 32]
        ridx = torch.tensor([s[0] for s in part]).repeat_interleave(2 * half + 1)
        u = torch.from_numpy(np.concatenate([s[1] for s in part]))
        picks.append(_abi.sample_top_p(dev_rows[ridx.to(DEV)].contiguous(), u.to(DEV), 1.0, 1.0).cpu().view(len(part), -1).numpy())
    picks = np.concatenate(picks)
    nucs = ref.nuclei(rows.double().numpy(), 1.0)
    bad = []
    for n, (r, us, lo_tok, hi_tok) in enumerate(sweeps):
        p = picks[n]
        want, _ = ref.inverse_cdf(nucs[r].dense(), us.astype(np.float64))
        ok_tok = np.isin(p, [lo_tok, hi_tok]) & np.isin(want, [lo_tok, hi_tok])
        if not ((np.diff(p) >= 0).all() and ok_tok.all()):
            bad.append((n, r, lo_tok, hi_tok, sorted(set(p.tolist()))))
    print(f"\n[draw] {len(sweeps)} boundaries swept in {rows_n} rows; the host's fp32 model sees an unclaimed interval under the "
          f"replaced claim rule in {gap_rows} rows; {len(bad)} sweeps broken")
    assert not bad, bad[:5]


# ------------------------------------------------------------------------------------------ spec_accept_sample, exact
TEMP, TOP_P = 0.7, 0.8


def _nuclei(rows: torch.Tensor):
    return ref.nuclei(ref.scaled_logits(rows.numpy(), TEMP), TOP_P, MARGIN)


def _residual_decisive(p: np.ndarray, q: np.ndarray, u: float) -> bool:
    """Whether the kernel's fp32 draw from max(0, P - Q) must pick the float64 token at u.  The residual's prefix sums carry
    cancellation error relative to the prefix of P + Q (not of the residual), so the margin scales with that prefix."""
    r = np.maximum(p - q, 0.0)
    R = r.sum()
    if R < 1e3 * MARGIN:
        return False
    nz = np.nonzero(r)[0]
    edges = np.cumsum(r)[nz[:-1]] / R
    scale = MARGIN * (np.cumsum(p + q)[nz[:-1]] + u * 2.0) / R
    return bool((np.abs(u - edges) >= scale).all())


def _expected_round(P, Q, d, u):
    """spec_ref.accept_sample on the float64 nuclei, or None where a decision it makes is not decisive for the fp32 kernel."""
    k = len(d)
    Pd, Qd = [x.dense() for x in P], [x.dense() for x in Q]
    for j in range(k):
        if not (P[j].decisive and Q[j].decisive):
            return None
        p, q = Pd[j][d[j]], Qd[j][d[j]]
        if not (p == 0 or u[j] == 0 or abs(u[j] * q - p) >= MARGIN * max(p, u[j] * q)):
            return None
        if u[j] * q < p:
            continue
        if not _residual_decisive(Pd[j], Qd[j], u[k]):
            return None
        break
    else:
        if not P[k].decisive or not ref.inverse_cdf(Pd[k], np.array([u[k]]), MARGIN)[1][0]:
            return None
    return ref.accept_sample(Pd, Qd, d, u)


def _run_accept(logits, draft, tokens, u):
    B, S = tokens.shape
    out = torch.full((B, S), -5, dtype=torch.long, device=DEV)
    n = torch.full((B,), -9, dtype=torch.int32, device=DEV)
    seqpos = torch.arange(B, dtype=torch.int32, device=DEV) * 5 + 40
    _abi.spec_accept_sample(logits.to(DEV), draft.to(DEV), tokens.to(DEV), u.to(DEV), out, n, seqpos, TEMP, TOP_P)
    out, n, seqpos = out.cpu(), n.cpu(), seqpos.cpu()
    assert torch.equal(seqpos, torch.arange(B, dtype=torch.int32) * 5 + 40 + n + 1)
    assert ((out == -1) == (torch.arange(S)[None, :] > n[:, None].long())).all()
    return out, n


def _check_rounds(out, n, P, Q, tokens, u, min_decisive=0.9, what=""):
    B, S = tokens.shape
    k = S - 1
    decisive = 0
    for b in range(B):
        d = tokens[b, 1:].tolist()
        want = _expected_round(P[b], Q[b], d, u[b].double().tolist())
        if want is None:
            continue
        decisive += 1
        toks, wn = want
        assert int(n[b]) == wn and out[b, :wn + 1].tolist() == toks, (what, b, out[b].tolist(), toks, wn)
    assert decisive >= min_decisive * B, f"{what}: only {decisive} of {B} sequences decisive: the fixture is wrong"
    return decisive


def _proposals(draft: torch.Tensor, B: int, k: int, V: int, seed: int):
    """d_{j+1} drawn by mb200_sample_top_p from sequence b's own draft row b * k + j."""
    g = torch.Generator().manual_seed(seed)
    tokens = torch.zeros(B, k + 1, dtype=torch.long)
    tokens[:, 0] = torch.randint(0, V, (B,), generator=g)
    uq = torch.rand(B * k, generator=g)
    tokens[:, 1:] = _abi.sample_top_p(draft.to(DEV), uq.to(DEV), TEMP, TOP_P).cpu().view(B, k)
    return tokens


@pytest.mark.parametrize("V", [512, 32768, 131072])
@pytest.mark.parametrize("k", [1, 4, 8])
def test_accept_sample_exact_per_sequence(V, k):
    """B = 256 sequences with their own target and draft rows: for every sequence whose decisions are decisive, out, n, the -1
    tail and seqpos equal spec_ref.accept_sample on the float64 nuclei exactly.  Sequence b must read its own draft rows."""
    B, S = 256, k + 1
    g = torch.Generator().manual_seed(600 + 7 * V + k)
    scale = 2.5 if V == 512 else 4.0  # a nucleus of tens to hundreds of tokens
    target = torch.randn(B * S, V, generator=g) * scale
    # a draft close enough to the target that rounds accept several proposals, far enough that they also reject
    draft = (target.view(B, S, V)[:, :k] + 0.15 * scale * torch.randn(B, k, V, generator=g)).reshape(B * k, V).contiguous()
    tokens = _proposals(draft, B, k, V, 700 + V + k)
    u = torch.rand(B, S, generator=g)
    out, n = _run_accept(target, draft, tokens, u)
    P = [_nuclei(target[b * S:(b + 1) * S]) for b in range(B)]
    Q = [_nuclei(draft[b * k:(b + 1) * k]) for b in range(B)]
    for b in range(B):
        for j in range(k):
            if Q[b][j].decisive:
                assert Q[b][j].keeps(int(tokens[b, j + 1])), "a proposal outside its own draft row's nucleus"
    got = _check_rounds(out, n, P, Q, tokens, u, what=f"V={V} k={k}")
    accepted = int(n.sum())
    print(f"\n[spec-exact] V={V} k={k}: {got}/{B} sequences decisive and exact; mean accepted {accepted / B:.2f}")
    assert 0 < accepted < B * k  # both outcomes occur


@pytest.mark.parametrize("V", [512, 32768])
def test_accept_sample_designed(V):
    """u = 0 accepts exactly where P_j(d) > 0; a draft nucleus disjoint from the target's at every j rejects at 0 and draws from
    P_0; P == Q accepts everything for u < 1, and at u = 1 (a probability-zero rejection) the residual is all zero and the
    kernel draws from P_0."""
    k, B = 4, 64
    S = k + 1
    g = torch.Generator().manual_seed(800 + V)
    target = torch.randn(B * S, V, generator=g) * 4.0
    P = [_nuclei(target[b * S:(b + 1) * S]) for b in range(B)]

    # u = 0: accept iff P_j(d) > 0.  Proposals alternate between the target's kept tokens and tokens it drops.
    draft = (0.5 * target.view(B, S, V)[:, :k] + 3.0 * torch.randn(B, k, V, generator=g)).reshape(B * k, V).contiguous()
    tokens = _proposals(draft, B, k, V, 900 + V)
    u = torch.rand(B, S, generator=g)
    u[:, :k] = 0.0
    out, n = _run_accept(target, draft, tokens, u)
    Q = [_nuclei(draft[b * k:(b + 1) * k]) for b in range(B)]
    for b in range(B):
        first_zero = next((j for j in range(k) if not P[b][j].keeps(int(tokens[b, j + 1]))), k)
        assert int(n[b]) == first_zero, (b, int(n[b]), first_zero)
    assert 0 < int(n.sum()) < B * k
    _check_rounds(out, n, P, Q, tokens, u, what="u=0")

    # disjoint nuclei at every j: the draft's nucleus is the target's least likely tokens
    far = torch.full((B * k, V), -40.0)
    for b in range(B):
        for j in range(k):
            far[b * k + j, target[b * S + j].argsort()[:3]] = 10.0 * TEMP
    tokens = _proposals(far, B, k, V, 1000 + V)
    u = torch.rand(B, S, generator=g)
    out, n = _run_accept(target, far, tokens, u)
    assert (n == 0).all()
    Q = [_nuclei(far[b * k:(b + 1) * k]) for b in range(B)]
    _check_rounds(out, n, P, Q, tokens, u, what="disjoint")

    # P == Q: the draft rows are the target's own rows
    same = target.view(B, S, V)[:, :k].reshape(B * k, V).contiguous()
    tokens = _proposals(same, B, k, V, 1100 + V)
    u = torch.rand(B, S, generator=g)
    out, n = _run_accept(target, same, tokens, u)
    assert (n == k).all()
    _check_rounds(out, n, P, [p[:k] for p in P], tokens, u, what="P == Q")
    u[:, 0] = 1.0
    out, n = _run_accept(target, same, tokens, u)
    assert (n == 0).all()
    for b in range(B):
        want, ok = ref.inverse_cdf(P[b][0].dense(), np.array([float(u[b, k])]), MARGIN)
        if ok[0]:
            assert int(out[b, 0]) == int(want[0]), b


# ----------------------------------------------------------------------------------------- joint distribution of a round
def test_accept_sample_round_distribution():
    """V = 24, k = 3, 2^20 seeded rounds with the target and draft rows fixed per j: the emitted tuple, with its length, follows
    spec_ref.round_distribution (chi-square below the 1 - 1e-6 quantile, bins under 5 expected pooled) and no tuple outside its
    support appears.  This covers tokens 2 .. k + 1 of a round and the bonus token."""
    from scipy.stats import chi2

    V, k, N, batch = 24, 3, 1 << 20, 1 << 18
    S = k + 1
    g = torch.Generator().manual_seed(1200)
    t_rows = torch.randn(S, V, generator=g)  # nuclei of 6 to 14 tokens: 1810 tuples, every length of round
    d_rows = 0.6 * t_rows[:k] + 0.5 * torch.randn(k, V, generator=g)
    P, Q = _nuclei(t_rows), _nuclei(d_rows)
    assert all(x.decisive for x in P + Q)
    Pd, Qd = [x.dense() for x in P], [x.dense() for x in Q]
    dist = ref.round_distribution(lambda pre: Pd[len(pre)], lambda pre: Qd[len(pre)], k)
    counts = {}
    gen = torch.Generator(device=DEV).manual_seed(1201)
    logits = t_rows.to(DEV).repeat(batch, 1).contiguous()
    draft = d_rows.to(DEV).repeat(batch, 1).contiguous()
    for _ in range(N // batch):
        uq = torch.rand(batch * k, generator=gen, device=DEV)
        tokens = torch.zeros(batch, S, dtype=torch.long, device=DEV)
        tokens[:, 1:] = _abi.sample_top_p(draft, uq, TEMP, TOP_P).view(batch, k)
        uni = torch.rand(batch, S, generator=gen, device=DEV)
        out = torch.empty(batch, S, dtype=torch.long, device=DEV)
        n = torch.empty(batch, dtype=torch.int32, device=DEV)
        seqpos = torch.zeros(batch, dtype=torch.int32, device=DEV)
        _abi.spec_accept_sample(logits, draft, tokens, uni, out, n, seqpos, TEMP, TOP_P)
        o, nn = out.cpu(), n.cpu()
        # encode (length, tokens) as one integer per round
        code = (nn.long() + 1)
        for j in range(S):
            code = code * (V + 1) + torch.where(o[:, j] >= 0, o[:, j] + 1, torch.zeros_like(o[:, j]))
        vals, cnt = torch.unique(code, return_counts=True)
        for v, c in zip(vals.tolist(), cnt.tolist()):
            counts[v] = counts.get(v, 0) + c

    def encode(seq):
        c = len(seq)
        for j in range(S):
            c = c * (V + 1) + (seq[j] + 1 if j < len(seq) else 0)
        return c

    expect = {encode(s): m * N for s, m in dist.items()}
    outside = {c: v for c, v in counts.items() if c not in expect}
    assert not outside, f"{len(outside)} emitted tuples outside the support"
    obs = np.array([counts.get(c, 0) for c in expect], dtype=np.float64)
    exp = np.array(list(expect.values()))
    small = exp < 5
    obs = np.concatenate([obs[~small], [obs[small].sum()]]) if small.any() else obs
    exp = np.concatenate([exp[~small], [exp[small].sum()]]) if small.any() else exp
    stat = float(((obs - exp) ** 2 / exp).sum())
    limit = float(chi2.ppf(1 - 1e-6, exp.size - 1))
    lengths = np.bincount([len(s) for s in dist], minlength=S + 1)
    assert (lengths[1:] > 0).all()  # rounds of every length, the bonus token included
    print(f"\n[spec-round] {len(dist)} tuples in the support (by length {lengths[1:].tolist()}), chi2 {stat:.1f} < {limit:.1f} over "
          f"{exp.size} bins")
    assert stat < limit
