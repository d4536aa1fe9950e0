"""generate()'s per-sequence sampling controls without a GPU: the refusals, which path each combination of arguments takes (today's
`pick` with its exact arguments, or mb200_select_tokens), and the host restatements the GPU tests compare against
(tests/sampling_controls_ref.py): Philox4x32-10 on known-answer vectors and the float32 penalty rule."""
import math

import numpy as np
import pytest
import torch

import mistral_inference_b200 as mi
from mistral_inference_b200 import _abi
from mistral_inference_b200.generate import TOP_P
from tests import sampling_controls_ref as SR

V = 64


class _Args:
    vocab_size, max_batch_size, n_kv_heads, head_dim, sliding_window = V, 4, 1, 8, None


class FakeModel:
    """What generate() needs of a Transformer, on the CPU: seeded logits, no kernels."""

    def __init__(self, seed=0):
        self.args, self.device, self.dtype, self.n_local_layers, self.last_argmax = _Args(), torch.device("cpu"), torch.bfloat16, 1, None
        self.kv_cache = "bf16"
        self.g = torch.Generator().manual_seed(seed)
        self.forwards = 0

    def eval(self):
        return self

    def forward_logprobs(self, ids, seqlens, cache, targets, images=None, **kw):
        self.forwards += 1
        return torch.zeros(ids.shape[0]), torch.randn(len(seqlens), V, generator=self.g)

    def next_token_logits(self, tokens, cache, **kw):
        self.forwards += 1
        return torch.randn(tokens.shape[0], V, generator=self.g)

    def last_argmax_valid_for(self, logits):
        return False


@pytest.fixture
def calls(monkeypatch):
    """Replaces the selection entry points with recorders that compute nothing on a device."""
    rec = []

    def sample_top_p(logits, u, temperature, top_p, out=None):
        rec.append(("sample_top_p", temperature, top_p, u.clone()))
        return out.zero_()

    def argmax_rows(logits, out=None):
        rec.append(("argmax_rows",))
        return out.copy_(logits.argmax(-1))

    def select_tokens(logits, temperature, top_p, presence, frequency, step, out, *, seeds=None, uniform=None, counts=None):
        rec.append(("select_tokens", temperature.tolist(), top_p.tolist(), presence.tolist(), frequency.tolist(),
                    None if seeds is None else seeds.tolist(), None if uniform is None else uniform.clone(), counts is not None))
        step += 1
        return out.zero_()

    monkeypatch.setattr(_abi, "sample_top_p", sample_top_p)
    monkeypatch.setattr(_abi, "argmax_rows", argmax_rows)
    monkeypatch.setattr(_abi, "select_tokens", select_tokens)
    monkeypatch.setattr(_abi, "logprob_gather", lambda logits, tok, out=None: out)
    return rec


PROMPTS = [[1, 2, 3], [4, 5]]


def _gen(**kw):
    kw.setdefault("max_tokens", 3)
    kw.setdefault("temperature", 0.7)
    return mi.generate(PROMPTS, FakeModel(), **kw)


# ------------------------------------------------------------------------------------------------------------ the two paths
def test_default_arguments_are_todays_pick(calls):
    torch.manual_seed(5)
    _gen()
    assert [c[:3] for c in calls] == [("sample_top_p", 0.7, TOP_P)] * 3
    assert TOP_P == 0.8 and all(type(c[2]) is float for c in calls)
    calls.clear()
    _gen(temperature=0.0)
    assert calls == [("argmax_rows",)] * 3
    calls.clear()
    _gen(top_p=0.5, random_seed=None, presence_penalty=0.0, frequency_penalty=0)
    assert [c[:3] for c in calls] == [("sample_top_p", 0.7, 0.5)] * 3  # a scalar top_p is today's path with that top_p


def test_default_path_draws_the_same_uniforms_as_before(calls):
    torch.manual_seed(11)
    _gen()
    first = [c[3] for c in calls]
    calls.clear()
    torch.manual_seed(11)
    _gen(temperature=[0.7, 0.7])  # the controls path without seeds: torch.rand(B) per step, as pick draws
    assert [c[0] for c in calls] == ["select_tokens"] * 3
    assert all(torch.equal(a, c[6]) for a, c in zip(first, calls))


@pytest.mark.parametrize("kw, counts", [
    ({"temperature": [0.0, 0.7]}, False),
    ({"top_p": [0.8, 0.9]}, False),
    ({"random_seed": 7}, False),
    ({"random_seed": [3, 2 ** 64 - 1]}, False),
    ({"presence_penalty": 0.5}, True),
    ({"frequency_penalty": [0.0, -1.0]}, True),
    ({"presence_penalty": [0.0, 0.0]}, False),
])
def test_any_other_combination_takes_the_controls_path(calls, kw, counts):
    _gen(**kw)
    assert [c[0] for c in calls] == ["select_tokens"] * 3
    c = calls[0]
    assert c[7] is counts
    if "random_seed" in kw:
        seeds = SR.sequence_seeds(kw["random_seed"], 2)
        assert [s & (2 ** 64 - 1) for s in c[5]] == seeds and c[6] is None  # uint64 bit patterns, no uniforms
    else:
        assert c[5] is None


def test_controls_are_expanded_per_sequence(calls):
    _gen(temperature=[0.0, 1.5], top_p=0.25, random_seed=2 ** 64 - 1, presence_penalty=[1.0, -2.0], frequency_penalty=0.5)
    _, t, p, pres, freq, seeds, u, counts = calls[0]
    assert t == [0.0, 1.5] and p == [0.25, 0.25] and pres == [1.0, -2.0] and freq == [0.5, 0.5] and counts
    assert [s & (2 ** 64 - 1) for s in seeds] == [2 ** 64 - 1, 0]  # (s + b) mod 2^64
    assert u is None


def test_all_greedy_controls_leave_the_generator_alone(calls):
    torch.manual_seed(3)
    _gen(temperature=[0.0, 0.0])
    after = torch.rand(1)
    torch.manual_seed(3)
    assert torch.equal(after, torch.rand(1))


# ------------------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("kw", [
    {"temperature": [0.7]},
    {"temperature": [0.7, 0.7, 0.7]},
    {"top_p": [0.8]},
    {"random_seed": [1, 2, 3]},
    {"presence_penalty": [0.0]},
    {"frequency_penalty": [0.0, 0.0, 0.0]},
    {"temperature": -0.1},
    {"temperature": [0.5, -1e-30]},
    {"temperature": math.inf},
    {"temperature": math.nan},
    {"top_p": -0.01},
    {"top_p": 1.0000001},
    {"top_p": [0.5, math.nan]},
    {"presence_penalty": 2.0001},
    {"presence_penalty": -2.5},
    {"frequency_penalty": math.inf},
    {"frequency_penalty": [0.0, math.nan]},
    {"random_seed": -1},
    {"random_seed": 2 ** 64},
    {"random_seed": 1.0},
    {"random_seed": True},
    {"random_seed": [0, 2 ** 64]},
    {"random_seed": [0, "1"]},
    {"temperature": "0.7"},
])
def test_refusals_come_before_any_work(calls, kw):
    m = FakeModel()
    with pytest.raises(ValueError):
        mi.generate(PROMPTS, m, max_tokens=3, **{"temperature": 0.7, **kw})
    assert m.forwards == 0 and not calls


def test_edges_of_the_ranges_are_accepted(calls):
    _gen(temperature=[0.0, 1e6], top_p=[0.0, 1.0], presence_penalty=[-2.0, 2.0], frequency_penalty=[2.0, -2.0],
         random_seed=[0, 2 ** 64 - 1])
    _gen(temperature=np.float32(0.5), random_seed=np.int64(3))
    assert [c[0] for c in calls] == ["select_tokens"] * 6


@pytest.mark.parametrize("kw", [{"temperature": [0.0, 0.7]}, {"top_p": 0.9}, {"random_seed": 1}, {"presence_penalty": 0.1},
                                {"frequency_penalty": [0.0, 0.1]}])
def test_draft_refuses_every_non_default_control(calls, kw):
    m, d = FakeModel(), FakeModel(1)
    with pytest.raises(ValueError, match="draft"):
        mi.generate(PROMPTS, m, max_tokens=3, **{"temperature": 0.7, **kw}, draft=d)
    assert m.forwards == 0 and d.forwards == 0


# ------------------------------------------------------------------------------------------------------------ restatements
def _hex(words):
    return [f"{int(w):08x}" for w in words]


def test_philox_known_answers():
    z = np.uint32(0)
    assert _hex(SR.philox4x32_10((z, z, z, z), (z, z))) == ["6627e8d5", "e169c58d", "bc57ac4c", "9b00dbd8"]
    f = np.uint32(0xFFFFFFFF)
    assert _hex(SR.philox4x32_10((f, f, f, f), (f, f))) == ["408f276d", "41c83b0e", "a20bc7c6", "6d5451fd"]
    ctr = tuple(np.uint32(x) for x in (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344))
    key = (np.uint32(0xA4093822), np.uint32(0x299F31D0))
    assert _hex(SR.philox4x32_10(ctr, key)) == ["d16cfe09", "94fdcceb", "5001e420", "24126ea1"]


def test_uniforms_are_exact_24_bit_values_in_the_unit_interval():
    for seed in (0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1):
        u = SR.uniforms(seed, np.arange(4096))
        assert u.dtype == np.float32 and (u >= 0).all() and (u < 1).all()
        assert np.array_equal(u * np.float32(2 ** 24), np.floor(u * np.float32(2 ** 24)))
        assert len(np.unique(u)) > 4000  # a stream, not a constant
    # the key is (seed mod 2^32, seed >> 32): seeds differing only in the high word give other streams
    assert not np.array_equal(SR.uniforms(5, np.arange(16)), SR.uniforms(5 + 2 ** 32, np.arange(16)))
    # the counter is the step: step t of one seed is word 0 of Philox at (t, 0, 0, 0)
    x0 = SR.philox4x32_10((np.uint32(9), np.uint32(0), np.uint32(0), np.uint32(0)), (np.uint32(7), np.uint32(0)))[0]
    assert SR.uniforms(7, [9])[0] == np.float32(int(x0) >> 8) * np.float32(2 ** -24)


def test_penalty_rule_in_float32():
    l = np.array([1.0, 1.0, -0.0, 0.0, 3.5, np.nan, -np.inf, 1e-8], dtype=np.float32)
    c = np.array([0, 2, 0, 1, 7, 1, 3, 1], dtype=np.int32)
    got = SR.penalised(l, c, 0.3, 0.1)
    for v in range(l.size):
        pen = np.float32(np.float32(c[v]) * np.float32(0.1))
        if c[v] > 0:
            pen = np.float32(pen + np.float32(0.3))
        want = np.float32(l[v] - pen)
        assert (np.isnan(want) and np.isnan(got[v])) or got[v].tobytes() == want.tobytes(), v
    # one add then one subtract, each rounded: not the fused or float64 value
    assert SR.penalised(np.float32([1.0]), np.int32([3]), 0.0, 0.1)[0] == np.float32(1.0) - np.float32(np.float32(3) * np.float32(0.1))
    # ties created by a penalty: 2.0 with one occurrence at presence 1.0 equals an unseen 1.0
    assert SR.penalised(np.float32([2.0, 1.0]), np.int32([1, 0]), 1.0, 0.0).tolist() == [1.0, 1.0]
    # both penalties 0: the row bit for bit, NaN payloads and -0.0 included
    bits = np.array([0x7FC12345, 0x80000000, 0x3F800000], dtype=np.uint32).view(np.float32)
    assert SR.penalised(bits, np.int32([4, 0, 9]), 0.0, -0.0).view(np.uint32).tolist() == [0x7FC12345, 0x80000000, 0x3F800000]
    # rows carry their own penalties
    two = SR.penalised(np.float32([[1.0, 1.0], [1.0, 1.0]]), np.int32([[1, 0], [1, 0]]), [0.5, 0.0], [0.0, 0.25])
    assert two.tolist() == [[0.5, 1.0], [0.75, 1.0]]
