"""Float64 restatement of speculative decoding's acceptance rules (csrc/speculative.cuh).

Distributions are the nucleus distributions mb200_sample_top_p draws from: softmax(logits / temperature), token i kept iff the
mass of the tokens with a strictly larger probability is <= top_p (equal probabilities at the cut are kept together), then
renormalised.  `round_distribution` enumerates one round exactly: every proposal path of the draft, its acceptance and the final
draw, so the CPU tests can check that the emitted tokens are distributed as the target's own nucleus samples.
"""
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np


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
