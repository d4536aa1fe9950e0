"""CPU model-check of token selection's integer and fp32 decisions (csrc/sampling.cuh, csrc/common.cuh).

block_draw's inverse-CDF draw is restated in the kernel's own fp32 arithmetic (tests/spec_ref.BlockDraw): thread-contiguous
chunk sums, the warp Hillis-Steele scan, the sequential warp prefix, the claim rule, the winner's walk and the fallback.  Each
lane's scan associates its additions differently, so a zero-mass thread's upper bound can sit an ulp above its weighted
predecessor's.  Under the kernel's rule (the lowest weighted thread with target < upper(t) wins) every target below the last
weighted upper(t) has a claimant, the rest fall back to the last kept token, and every target resolves to the inverse-CDF token or its kept neighbour across an ulp; under the rule it replaced (weighted and
upper(t - 1) <= target < upper(t)) such an interval belongs to nobody and the draw falls through to the row's last kept token.

The claims only change where the target crosses some upper(t), so checking 0, every upper(t) and the fp32 value just below each
upper(t) (BlockDraw.edge_targets) covers every target in [0, total).

argmax_key is restated bit for bit and checked against torch.argmax's order on strata of all 2^32 fp32 patterns."""
import numpy as np
import pytest
import torch

from . import spec_ref as ref


def _check_fixed_rule(w: np.ndarray) -> None:
    d = ref.BlockDraw(w)
    t = d.edge_targets()
    # every target below the largest weighted upper(t) has a claimant; above it (the zero-mass threads after the last weighted one
    # may round the total an ulp higher) the fallback's last weighted token is the inverse CDF's token
    reach = d.upper[d.mine > 0].max()
    claimed = d.claimants(t).any(axis=1)
    assert claimed[t < reach].all() and not claimed[t >= reach].any(), "a target below the last weighted bound has no claimant"
    picks = d.resolve(t)
    assert (np.diff(picks) >= 0).all(), "the draw is not monotone in the target"
    kept = np.nonzero(w)[0]
    assert np.isin(picks, kept).all()
    # float64 inverse CDF of the same fp32 weights at the same fp32 targets: the pick is that token or its kept neighbour
    c = np.cumsum(w.astype(np.float64))
    want = np.minimum(np.searchsorted(c, t.astype(np.float64), side="right"), kept[-1])
    pos = np.searchsorted(kept, want)
    got = np.searchsorted(kept, picks)
    assert (np.abs(got - pos) <= 1).all(), "a pick is not the inverse-CDF token or its kept neighbour"
    # u in [0, 1) maps to a target in [0, total]; the largest u lands on the last kept token
    assert d.resolve(d.target([np.nextafter(np.float32(1), np.float32(0))]))[0] == kept[-1]
    assert d.resolve(d.target([0.0]))[0] == kept[0]


def _nucleus_like(seed: int, V: int = 131072, kept: int = 150) -> np.ndarray:
    """A row's kept weights after the nucleus filter: ~150 tokens scattered over the vocabulary, unequal probabilities."""
    rng = np.random.default_rng(seed)
    w = np.zeros(V, dtype=np.float32)
    idx = rng.choice(V, kept, replace=False)
    p = np.exp(rng.normal(0, 1.5, kept))
    w[idx] = (p / p.sum()).astype(np.float32)
    return w


def _designed():
    rows = {}
    for V in (1, 31, 1000, 1024, 1025, 32768, 131072, 131073):
        w = np.zeros(V, dtype=np.float32)
        w[0] = 1
        rows[f"first-only-V{V}"] = w
        w = np.zeros(V, dtype=np.float32)
        w[V - 1] = 0.25
        rows[f"last-only-V{V}"] = w
        rng = np.random.default_rng(V)
        w = (0.5 + 0.5 * rng.random(V)).astype(np.float32)  # every token weighted, each well above the prefix sums' rounding
        rows[f"dense-V{V}"] = w
    # V = 131073: per = 129, thread 1016 holds the partial last chunk [131064, 131073), threads 1017.. hold nothing
    w = np.zeros(131073, dtype=np.float32)
    w[[131064, 131070, 131072]] = [0.3, 0.5, 0.2]
    rows["partial-chunk"] = w
    # V = 32768 (one token per thread): three adjacent weighted lanes then zero lanes, in several warps (the GPU sweep's rows)
    w = np.zeros(32768, dtype=np.float32)
    rng = np.random.default_rng(7)
    for warp in (0, 5, 17, 31):
        for lane in (3, 4, 5):
            w[(warp * 32 + lane) * 32 + 11] = rng.random() + 0.1
    rows["adjacent-lanes"] = w
    return rows


@pytest.mark.parametrize("name", list(_designed()))
def test_block_draw_designed_rows(name):
    _check_fixed_rule(_designed()[name])


def test_block_draw_nucleus_rows():
    """200 seeded nucleus-like rows at V = 131072: no target goes unclaimed, every pick is the inverse CDF's token or its
    neighbour.  The same rows under the replaced 'interval' rule have unclaimed targets, and there the draw falls through to the
    row's last kept token -- a token far from the inverse CDF's."""
    gaps = 0
    for seed in range(200):
        w = _nucleus_like(seed)
        _check_fixed_rule(w)
        d = ref.BlockDraw(w)
        assert d.orphans().size == 0
        orphan = d.orphans(rule="interval")
        if orphan.size:
            gaps += 1
            kept = np.nonzero(w)[0]
            c = np.cumsum(w.astype(np.float64))
            want = np.searchsorted(c, orphan.astype(np.float64), side="right")
            old = d.resolve(orphan, rule="interval")
            assert (old == kept[-1]).all()
            assert (np.searchsorted(kept, old) - np.searchsorted(kept, np.minimum(want, kept[-1])) > 1).any()
    print(f"\n[draw] the replaced claim rule leaves unclaimed targets in {gaps} of 200 rows; the kernel's rule in none")
    assert gaps > 0


# ------------------------------------------------------------------------------------------------------------ argmax_key
def _key_hi(bits: np.ndarray) -> np.ndarray:
    """argmax_key's high word (csrc/common.cuh): -0.0 -> +0.0, every NaN -> 0x7f800001 (one above +inf), then the sign flip."""
    bits = bits.astype(np.uint32)
    v = bits.view(np.float32)
    u = np.where(np.isnan(v), np.uint32(0x7F800001), np.where(v == 0, np.uint32(0), bits)).astype(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def _old_key_hi(bits: np.ndarray) -> np.ndarray:
    bits = bits.astype(np.uint32)
    return np.where(bits & np.uint32(0x80000000), ~bits, bits | np.uint32(0x80000000)).astype(np.uint32)


def _argmax_by_key(key_hi, row: np.ndarray) -> int:
    k = key_hi(row.view(np.uint32)).astype(np.uint64) << np.uint64(32)
    k |= (np.uint64(0x7FFFFFFF) - np.arange(row.size, dtype=np.uint64))
    return int(0x7FFFFFFF - int(k.max() & np.uint64(0xFFFFFFFF)))


def _strata() -> np.ndarray:
    """Every high half-word with a spread of low half-words (both ends, the middle, seeded random), plus the specials."""
    hi = np.arange(1 << 16, dtype=np.uint32) << np.uint32(16)
    lows = np.concatenate([np.array([0, 1, 0x7FFF, 0x8000, 0xFFFE, 0xFFFF], dtype=np.uint32),
                           np.random.default_rng(3).integers(0, 1 << 16, 10, dtype=np.uint32)])
    special = np.array([0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7F800001, 0x7FC00000, 0x7FFFFFFF, 0xFFC00000, 0xFF800001,
                        0xFFFFFFFF, 0x00000001, 0x80000001, 0x7F7FFFFF, 0xFF7FFFFF], dtype=np.uint32)
    return np.unique(np.concatenate([(hi[:, None] | lows[None, :]).reshape(-1), special]))


def test_argmax_key_orders_like_torch():
    """Over ~1.1M fp32 patterns: keys ordered by value with -0.0 == +0.0 and every NaN above +inf and equal to each other;
    equal keys exactly for equal values."""
    bits = _strata()
    with np.errstate(invalid="ignore"):
        v = bits.view(np.float32).astype(np.float64)
    key = _key_hi(bits)
    nan = np.isnan(v)
    assert (key[nan] == 0xFF800001).all() and key[nan].min() > key[~nan].max()
    order = np.argsort(key[~nan], kind="stable")
    ks, vs = key[~nan][order], v[~nan][order]
    assert (np.diff(vs) >= 0).all(), "the key is not monotone in the value"
    assert ((np.diff(ks) > 0) == (np.diff(vs) > 0)).all(), "equal keys for different values, or different keys for equal ones"


def test_argmax_key_matches_torch_argmax():
    """Rows built from the strata, with many ±0 and NaN entries and exact ties: the key's argmax equals torch.argmax's on each.
    The appendix cases show what the sign-bit-only key returned instead."""
    cases = [[-0.0, 0.0, -1.0], [-0.0, -0.0, 0.0, -0.0], [1.0, -np.nan, 2.0], [0.0, -0.0], [-1.0, -0.0, 0.0],
             [np.nan, np.inf], [np.inf, -np.nan, np.nan], [-np.inf, -np.inf], [2.0, 3.0, 3.0]]
    nan_payload = np.array([0x7FC00001, 0x7FC00000, 0xFFC00005], dtype=np.uint32).view(np.float32)
    for row in [np.array(c, dtype=np.float32) for c in cases] + [np.concatenate([[1.0], nan_payload]).astype(np.float32)]:
        assert _argmax_by_key(_key_hi, row) == int(torch.from_numpy(row).argmax()), row
    assert _argmax_by_key(_old_key_hi, np.array([-0.0, 0.0, -1.0], dtype=np.float32)) == 1  # torch: 0
    assert _argmax_by_key(_old_key_hi, np.array([1.0, -np.nan, 2.0], dtype=np.float32)) == 2  # torch: 1
    bits = _strata()
    rng = np.random.default_rng(5)
    pool = np.concatenate([bits, np.repeat(np.array([0, 0x80000000, 0x7FC00000, 0xFFC00000], dtype=np.uint32), 1000)])
    for n in (2, 3, 7, 64):
        for _ in range(500):
            row = rng.choice(pool, n).view(np.float32)
            assert _argmax_by_key(_key_hi, row) == int(torch.from_numpy(row.copy()).argmax()), row.view(np.uint32)
