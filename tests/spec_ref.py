"""Float64 restatement of speculative decoding's acceptance rules (csrc/speculative.cuh).

Distributions are the nucleus distributions mb200_sample_top_p draws from: softmax(logits / temperature), token i kept iff the
mass of the tokens with a strictly larger probability is <= top_p (equal probabilities at the cut are kept together), then
renormalised.  `round_distribution` enumerates one round exactly: every proposal path of the draft, its acceptance and the final
draw, so the CPU tests can check that the emitted tokens are distributed as the target's own nucleus samples.
"""
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch


def nucleus(logits: Sequence[float], temperature: float, top_p: float) -> np.ndarray:
    z = np.asarray(logits, dtype=np.float64) / temperature
    p = np.exp(z - z.max())
    p /= p.sum()
    before = np.array([p[p > x].sum() for x in p])  # mass ranked strictly before each token
    kept = np.where(before <= top_p, p, 0.0)
    return kept / kept.sum()


def residual(p: np.ndarray, q: np.ndarray) -> np.ndarray:
    """max(0, p - q) renormalised; p itself when p == q (a rejection then has probability 0)."""
    r = np.maximum(p - q, 0.0)
    return r / r.sum() if r.sum() > 0 else p


def accept_greedy(logits: np.ndarray, tokens: Sequence[int]) -> Tuple[List[int], int]:
    """logits [S, V] of one sequence's verify rows, tokens [S] = [last, d_1 .. d_k] -> (emitted tokens, n accepted)."""
    S = len(tokens)
    for j in range(S):
        a = int(np.argmax(logits[j]))  # first index on ties
        if j == S - 1 or a != tokens[j + 1]:
            return [int(t) for t in tokens[1:j + 1]] + [a], j
    raise AssertionError("unreachable")


def accept_sample(p_rows: Sequence[np.ndarray], q_rows: Sequence[np.ndarray], proposals: Sequence[int], u: Sequence[float]
                  ) -> Tuple[List[int], int]:
    """One sequence, given distributions: p_rows [k + 1], q_rows [k], proposals d_1 .. d_k, uniforms u [k + 1] ->
    (emitted tokens, n accepted).  The final draw is the inverse CDF in index order, like the kernel's."""
    k = len(proposals)
    for j in range(k):
        d = proposals[j]
        if u[j] * q_rows[j][d] < p_rows[j][d]:
            continue
        return list(proposals[:j]) + [_draw(residual(p_rows[j], q_rows[j]), u[k])], j
    return list(proposals) + [_draw(p_rows[k], u[k])], k


def _draw(w: np.ndarray, u: float) -> int:
    c = np.cumsum(w)
    return int(min(np.searchsorted(c, u * c[-1], side="right"), len(w) - 1))


Dist = Callable[[Tuple[int, ...]], np.ndarray]


def round_distribution(p_of: Dist, q_of: Dist, k: int) -> Dict[Tuple[int, ...], float]:
    """Exact distribution of the tokens one round emits, by enumeration.  p_of(prefix) / q_of(prefix): the target's / draft's
    next-token distribution after the round's emitted prefix (a tuple of token ids; () is the round's start)."""
    out: Dict[Tuple[int, ...], float] = {}

    def walk(prefix: Tuple[int, ...], mass: float) -> None:
        p = p_of(prefix)
        if len(prefix) == k:  # every proposal accepted: the bonus token
            for x in np.nonzero(p)[0]:
                out[prefix + (int(x),)] = out.get(prefix + (int(x),), 0.0) + mass * p[x]
            return
        q = q_of(prefix)
        reject = 0.0
        for d in np.nonzero(q)[0]:
            a = min(1.0, p[d] / q[d])
            if a > 0:
                walk(prefix + (int(d),), mass * q[d] * a)
            reject += q[d] * (1.0 - a)
        if reject > 0:
            r = residual(p, q)
            for x in np.nonzero(r)[0]:
                out[prefix + (int(x),)] = out.get(prefix + (int(x),), 0.0) + mass * reject * r[x]

    walk((), 1.0)
    return out


def next_token_given_prefix(dist: Dict[Tuple[int, ...], float], prefix: Tuple[int, ...], V: int) -> Optional[np.ndarray]:
    """P(emitted[len(prefix)] = x | emitted starts with prefix and is longer than it), or None when that never happens."""
    i = len(prefix)
    w = np.zeros(V)
    for seq, m in dist.items():
        if len(seq) > i and seq[:i] == prefix:
            w[seq[i]] += m
    return w / w.sum() if w.sum() > 0 else None


def acceptance_rate(p: np.ndarray, q: np.ndarray) -> float:
    """Probability that one proposal drawn from q is accepted: sum(min(p, q))."""
    return float(np.minimum(p, q).sum())


# ---------------------------------------------------------------------------- token selection at the kernels' own inputs
def scaled_logits(logits: np.ndarray, temperature: float) -> np.ndarray:
    """logits / temperature as the kernels form it: the fp32 product with inv_t = fp32(1 / fp32(temperature)), widened exactly."""
    inv_t = np.float32(1.0) / np.float32(temperature)
    return (np.asarray(logits, dtype=np.float32) * inv_t).astype(np.float64)


class Nucleus:
    """The float64 nucleus of one row, stored sparsely: the kept token ids in index order (`idx`) and their renormalised
    probabilities (`w`), and `decisive`: whether the fp32 kernel must reach the same kept set.  It must when every cut decision is
    at least `margin` from top_p (the top group's mass before it is exactly 0 in fp32 as well) and the smallest kept probability
    is at least `margin` (relative) above the largest dropped one, so rounding cannot reorder the two across the cut."""

    def __init__(self, V: int, idx: np.ndarray, w: np.ndarray, decisive: bool):
        self.V, self.idx, self.w, self.decisive = V, idx, w, decisive

    def dense(self) -> np.ndarray:
        p = np.zeros(self.V)
        p[self.idx] = self.w
        return p

    def keeps(self, tokens) -> np.ndarray:
        return np.isin(np.asarray(tokens), self.idx)


def nuclei(z: np.ndarray, top_p: float, margin: float = 1e-5, cand: int = 4096) -> List[Nucleus]:
    """Nucleus of each row of scaled logits z [R, V]: probs = softmax(z), token i kept iff the mass of the strictly larger
    probabilities is <= top_p (equal probabilities share that mass, so ties at the cut are kept together).  The ranking is taken
    over the `cand` largest probabilities when those already hold more than top_p + margin and their smallest is dropped (every
    token outside them is then dropped too), else over the whole row."""
    zt = torch.as_tensor(np.atleast_2d(np.asarray(z, dtype=np.float64)))
    R, V = zt.shape
    e = torch.exp(zt - zt.max(-1, keepdim=True).values)
    probs = (e / e.sum(-1, keepdim=True)).numpy()
    K = min(cand, V)
    top, tid = (x.numpy() for x in torch.from_numpy(probs).topk(K, -1))
    out = []
    for r in range(R):
        t, i = top[r], tid[r]
        for full in (False, True):
            if full:
                i = np.argsort(-probs[r], kind="stable")
                t = probs[r][i]
            excl = np.concatenate([[0.0], np.cumsum(t)[:-1]])
            start = np.concatenate([[True], t[1:] != t[:-1]])
            before = excl[np.maximum.accumulate(np.where(start, np.arange(t.size), 0))]
            kept = (before <= top_p) & (t > 0)
            if full or (t.sum() > top_p + margin and not kept[-1]):
                break
        cut = before[(before > 0) & (t > 0)]
        dropped = t[~kept & (t > 0)]
        near_cut = cut.size > 0 and np.abs(cut - top_p).min() < margin
        near_tie = dropped.size > 0 and t[kept].min() * (1 - margin) <= dropped.max()
        idx = np.sort(i[kept])
        w = probs[r][idx]
        out.append(Nucleus(V, idx, w / w.sum(), not (near_cut or near_tie)))
    return out


def inverse_cdf(w: np.ndarray, u: np.ndarray, margin: float = 1e-5) -> Tuple[np.ndarray, np.ndarray]:
    """The inverse-CDF token in index order of the weights w >= 0 at each uniform u, and whether u is decisive: at least `margin`
    (relative) from every CDF edge that separates two tokens.  The last edge (the total) is not such an edge: the kernel sends a
    target that rounds onto it to the last weighted token, which is the token below it anyway."""
    w = np.asarray(w, dtype=np.float64)
    c = np.cumsum(w) / w.sum()
    nz = np.nonzero(w)[0]
    u = np.asarray(u, dtype=np.float64)
    tok = np.minimum(np.searchsorted(c, u, side="right"), nz[-1])
    edges = c[nz[:-1]]
    if edges.size == 0:
        return tok, np.ones(u.shape, dtype=bool)
    j = np.searchsorted(edges, u)
    lo, hi = edges[np.clip(j - 1, 0, edges.size - 1)], edges[np.clip(j, 0, edges.size - 1)]
    return tok, np.minimum(np.abs(u - lo) / lo, np.abs(u - hi) / hi) >= margin


# ------------------------------------------------------------- block_draw (csrc/sampling.cuh) in the kernel's fp32 arithmetic
SP_THREADS = 1024


class BlockDraw:
    """block_draw's fp32 arithmetic on the host, for the weights w (fp32): thread t sums its contiguous chunk of
    per = ceil(V / 1024) weights sequentially, a Hillis-Steele scan (shfl_up by 1, 2, 4, 8, 16) gives each lane its inclusive
    sum within the warp, each thread adds the warp totals before its warp sequentially, upper(t) = before + incl, and
    target = fp32(u * upper(1023)).  `claimants(target, rule)` lists the threads that claim a target; `resolve` applies the
    lowest-claimant rule, the winner's walk from upper(t - 1) and the row-wide fallback to the last weighted token."""

    def __init__(self, w: np.ndarray):
        w = np.asarray(w, dtype=np.float32)
        self.w, V = w, w.size
        self.per = per = -(-V // SP_THREADS)
        pad = np.zeros(SP_THREADS * per, dtype=np.float32)
        pad[:V] = w
        chunks = pad.reshape(SP_THREADS, per)
        mine = np.zeros(SP_THREADS, dtype=np.float32)
        for c in range(per):
            mine = mine + chunks[:, c]
        self.mine = mine
        incl = mine.reshape(32, 32).copy()
        lane = np.arange(32)
        o = 1
        while o < 32:
            up = np.concatenate([incl[:, :o], incl[:, :-o]], axis=1)
            incl = np.where(lane[None, :] >= o, incl + up, incl).astype(np.float32)
            o <<= 1
        before = np.zeros(32, dtype=np.float32)
        for wp in range(1, 32):
            before[wp] = before[wp - 1] + incl[wp - 1, 31]
        self.upper = (before[:, None] + incl).astype(np.float32).reshape(-1)
        self.lower = np.concatenate([np.zeros(1, dtype=np.float32), self.upper[:-1]])
        self.total = self.upper[-1]
        # the winner's running sum: run(t, c) = fp32(run(t, c - 1) + w) from lower(t) (adding a zero weight is exact, so the walk's
        # skipping of zero weights needs no special case)
        run = np.empty_like(chunks)
        acc = self.lower.copy()
        for c in range(per):
            acc = acc + chunks[:, c]
            run[:, c] = acc
        self.run, self.chunks = run, chunks
        nz = np.nonzero(w)[0]
        self.last = int(nz[-1]) if nz.size else -1

    def edge_targets(self) -> np.ndarray:
        """0, every upper(t) and the fp32 value just below each, below the total: the claims are constant between these, so they
        stand for every target in [0, total)."""
        ups = np.unique(self.upper[(self.upper > 0) & (self.upper <= self.total)])
        below = np.nextafter(ups, np.float32(-np.inf), dtype=np.float32)
        t = np.unique(np.concatenate([[np.float32(0)], ups, below]).astype(np.float32))
        return t[t < self.total]

    def orphans(self, rule: str = "lowest_upper") -> np.ndarray:
        """The edge targets below the last weighted upper(t) that no thread claims."""
        t = self.edge_targets()
        t = t[t < self.upper[self.mine > 0].max()]
        return t[~self.claimants(t, rule).any(axis=1)]

    def target(self, u) -> np.ndarray:
        return (np.asarray(u, dtype=np.float32) * self.total).astype(np.float32)

    def claimants(self, target: np.ndarray, rule: str = "lowest_upper") -> np.ndarray:
        """[n, 1024] claims.  'lowest_upper' (the kernel's rule): weighted and target < upper(t).  'interval' (the rule it
        replaced): weighted and upper(t - 1) <= target < upper(t)."""
        t = np.asarray(target, dtype=np.float32)[:, None]
        c = (self.mine > 0)[None, :] & (t < self.upper[None, :])
        if rule == "interval":
            c &= t >= self.lower[None, :]
        return c

    def resolve(self, target: np.ndarray, rule: str = "lowest_upper") -> np.ndarray:
        target = np.asarray(target, dtype=np.float32)
        c = self.claimants(target, rule)
        any_claim = c.any(axis=1)
        tid = np.argmax(c, axis=1)
        V = self.w.size
        out = np.full(target.size, self.last, dtype=np.int64)
        for n in np.nonzero(any_claim)[0]:
            t = tid[n]
            weighted = self.chunks[t] > 0
            hit = weighted & (target[n] < self.run[t])
            k = int(np.argmax(hit)) if hit.any() else int(np.nonzero(weighted)[0][-1])
            out[n] = min(t * self.per + k, V - 1)
        return out
