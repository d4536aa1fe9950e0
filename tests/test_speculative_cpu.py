"""Speculative decoding without a GPU: the acceptance rule restated in float64 (tests/spec_ref.py) keeps the target's nucleus
distribution exactly, and generate(..., draft=...) refuses what it cannot run before it allocates anything."""
import itertools

import numpy as np
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import speculative
from mistral_inference_b200.transformer import Transformer

from . import spec_ref as ref

TEMP, TOP_P = 0.7, 0.8


def _dist_of(seed: int, V: int, scale: float = 2.0):
    """A next-token nucleus distribution per prefix, from seeded random logits."""
    cache = {}

    def f(prefix):
        if prefix not in cache:
            rng = np.random.default_rng([seed, *prefix])
            cache[prefix] = ref.nucleus(rng.normal(0, scale, V), TEMP, TOP_P)
        return cache[prefix]

    return f


def _check_round(p_of, q_of, k: int, V: int):
    dist = ref.round_distribution(p_of, q_of, k)
    assert abs(sum(dist.values()) - 1.0) < 1e-12
    assert all(1 <= len(s) <= k + 1 for s in dist)
    # every emitted position is distributed as the target's nucleus sample after the emitted prefix
    checked = 0
    for i in range(k + 1):
        for prefix in itertools.product(range(V), repeat=i):
            got = ref.next_token_given_prefix(dist, prefix, V)
            if got is None:
                continue
            np.testing.assert_allclose(got, p_of(prefix), rtol=0, atol=1e-12)
            checked += 1
    assert checked >= 1
    return dist


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("seeds", [(1, 2), (3, 4), (5, 6)])
def test_emitted_tokens_follow_the_target_nucleus(k, seeds):
    V = 5
    p_of, q_of = _dist_of(seeds[0], V), _dist_of(seeds[1], V)
    dist = _check_round(p_of, q_of, k, V)
    accepted_first = sum(m for s, m in dist.items() if len(s) >= 2)
    assert abs(accepted_first - ref.acceptance_rate(p_of(()), q_of(()))) < 1e-12


@pytest.mark.parametrize("k", [1, 3])
def test_draft_equal_to_target_accepts_everything(k):
    V = 5
    p_of = _dist_of(7, V)
    dist = _check_round(p_of, p_of, k, V)
    assert all(len(s) == k + 1 for s in dist)


def test_disjoint_nuclei_reject_at_row_zero():
    V = 6
    p = lambda prefix: np.array([0.5, 0.3, 0.2, 0, 0, 0], dtype=np.float64)  # noqa: E731
    q = lambda prefix: np.array([0, 0, 0, 0.6, 0.4, 0], dtype=np.float64)  # noqa: E731
    dist = _check_round(p, q, 3, V)
    assert all(len(s) == 1 for s in dist)
    assert ref.acceptance_rate(p(()), q(())) == 0.0


def test_tokens_outside_the_draft_nucleus():
    """q(d) = 0 for tokens outside the draft's nucleus: they are never proposed, and the residual max(0, p - q) emits them."""
    V = 6
    p_of = lambda prefix: ref.nucleus([1.0, 0.9, 0.8, 0.7, -3, -3], TEMP, TOP_P)  # noqa: E731
    q_of = lambda prefix: ref.nucleus([4.0, 0.0, -2, -2, -2, -2], TEMP, TOP_P)  # noqa: E731
    assert (q_of(())[1:] == 0).all() and (p_of(())[1:4] > 0).all()
    _check_round(p_of, q_of, 2, V)


def test_nucleus_matches_the_sorted_rule():
    """Kept iff the mass ranked strictly before a token is <= top_p (generate.py:161-170), equal probabilities together."""
    rng = np.random.default_rng(0)
    for _ in range(50):
        lg = rng.normal(0, 2, 40)
        p = np.exp(lg / TEMP - (lg / TEMP).max())
        p /= p.sum()
        order = np.argsort(-p, kind="stable")
        before = np.cumsum(p[order]) - p[order]
        kept = np.zeros(40, dtype=bool)
        kept[order[before <= TOP_P]] = True
        assert ((ref.nucleus(lg, TEMP, TOP_P) > 0) == kept).all()


def test_sample_rule_draws():
    """accept_sample, the kernel's per-sequence procedure, on fixed draws."""
    p = [np.array([0.5, 0.5, 0, 0]), np.array([0, 0, 1.0, 0])]
    q = [np.array([0.25, 0.75, 0, 0])]
    assert ref.accept_sample(p, q, [0], [0.99, 0.1]) == ([0, 2], 1)  # p/q = 2: accepted whatever u
    assert ref.accept_sample(p, q, [1], [0.5, 0.1]) == ([1, 2], 1)   # 0.5 * 0.75 < 0.5
    assert ref.accept_sample(p, q, [1], [0.7, 0.1]) == ([0], 0)      # 0.7 * 0.75 >= 0.5: residual = [1, 0, 0, 0]


def test_greedy_rule():
    lg = np.array([[0, 3, 1, 3], [5, 0, 0, 0], [0, 0, 9, 0]], dtype=np.float64)
    assert ref.accept_greedy(lg, [7, 1, 0]) == ([1, 0, 2], 2)
    assert ref.accept_greedy(lg, [7, 3, 0]) == ([1], 0)  # ties pick the first index
    assert ref.accept_greedy(lg, [7, 1, 2]) == ([1, 0], 1)


# ----------------------------------------------------------------------------------------------------- refusals, on meta models
def _meta(name: str, max_batch: int = 2, **kw) -> Transformer:
    over = {k: v for k, v in kw.items() if k in ("sliding_window", "vocab_size", "n_layers")}
    args = mi.TransformerArgs.from_dict(synth.shape(name, **over))
    args.max_batch_size = max_batch
    with torch.device("meta"):
        return Transformer(args, **{k: v for k, v in kw.items() if k not in over})


@pytest.fixture
def no_allocation(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("allocated a KV cache before refusing")

    monkeypatch.setattr(speculative, "BufferCache", refuse)
    monkeypatch.setattr(speculative, "_PromptPlan", refuse)


PROMPTS = [[1, 2, 3], [4, 5]]


@pytest.mark.parametrize("case", ["vocab", "draft_tokens", "pipeline", "expert_parallel", "images", "window", "draft_window", "batch"])
def test_refusals_before_allocation(case, no_allocation):
    target, draft = _meta("tiny"), _meta("tiny")
    kw = dict(max_tokens=8, temperature=0.0, draft=draft)
    match = None
    if case == "vocab":
        kw["draft"] = _meta("tiny", vocab_size=256)
        match = "vocabulary"
    elif case == "draft_tokens":
        kw["draft_tokens"] = 0
        match = "draft_tokens"
    elif case == "pipeline":
        target = _meta("tiny", pipeline_rank=0, num_pipeline_ranks=2)
        match = "pipeline"
    elif case == "expert_parallel":
        kw["draft"] = _meta("tiny-moe", expert_parallel=(0, 2))
        match = "expert parallelism"
    elif case == "images":
        kw["images"] = [[np.zeros((3, 16, 16))], []]
        match = "images"
    elif case == "window":
        target = _meta("tiny", sliding_window=[12, None])
        match = "sliding window of 12 tokens would wrap"
    elif case == "draft_window":
        kw["draft"] = _meta("tiny", sliding_window=14)
        match = "roll back"
    elif case == "batch":
        kw["draft"] = _meta("tiny", max_batch=1)
        match = "max_batch_size"
    with pytest.raises(ValueError, match=match):
        mi.generate(PROMPTS, target, **kw)


def test_window_that_holds_the_generation_is_accepted():
    """3 + 8 + 4 = 15 positions fit a 15-token window: no refusal."""
    speculative.check_draft(_meta("tiny", sliding_window=15), _meta("tiny", sliding_window=[None, 15]), [], PROMPTS, 8, 4)
    with pytest.raises(ValueError):
        speculative.check_draft(_meta("tiny", sliding_window=15), _meta("tiny"), [], PROMPTS, 8, 5)
