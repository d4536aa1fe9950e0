"""Multi-adapter LoRA without a GPU: the host side of `Transformer(..., lora_slots=n)` -- keyword-only parameters and their defaults,
the slot packing of LoraAdapter, `load_lora(slot=k)`, the per-token slot vector of a ragged batch, and the refusals, which all come
before anything is allocated.  tests/test_gpu_multi_lora.py checks what the kernels compute."""
import inspect

import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200.args import LoraArgs
from mistral_inference_b200.generate import _PromptPlan
from mistral_inference_b200.transformer import MAX_LORA_SLOTS, Transformer, expand_lora_ids
from mistral_inference_b200.transformer_layers import LoraAdapter

RANK = 4


def _args(name="tiny", lora=True, **over):
    p = synth.shape(name, **over)
    a = mi.TransformerArgs.from_dict(dict(p, lora=dict(rank=RANK, scaling=2.0)) if lora else dict(p))
    a.max_batch_size = 8
    return p, a


def _meta(args, **kw):
    with torch.device("meta"):
        return Transformer(args, **kw)


def _adapters(m):
    return [mod for mod in m.modules() if isinstance(mod, LoraAdapter)]


# ----------------------------------------------------------------------------- API
@pytest.mark.parametrize("fn,name,default", [
    (Transformer.__init__, "lora_slots", 1), (Transformer.from_folder, "lora_slots", 1), (Transformer.load_lora, "slot", 0),
    (mi.generate, "lora_ids", None), (Transformer.forward, "lora_ids", None), (Transformer.forward_logprobs, "lora_ids", None),
    (Transformer.last_token_logits, "lora_ids", None), (Transformer.next_token_logits, "lora_ids", None),
    (Transformer.decode_static, "lora_ids", None),
])
def test_keyword_only_with_todays_default(fn, name, default):
    prm = inspect.signature(fn).parameters[name]
    assert prm.kind == inspect.Parameter.KEYWORD_ONLY and prm.default == default


def test_one_slot_is_todays_model():
    """lora_slots=1: the same parameters (names and shapes) and state-dict keys as a model built without the keyword."""
    _, a = _args()
    m0, m1 = _meta(a), _meta(a, lora_slots=1)
    assert [(n, tuple(t.shape)) for n, t in m0.named_parameters()] == [(n, tuple(t.shape)) for n, t in m1.named_parameters()]
    assert list(m0.state_dict()) == list(m1.state_dict())
    assert all(ad.slots == 1 and ad.a.shape[0] == ad.rank_cols for ad in _adapters(m1))


def test_slot_bank_shapes():
    _, a = _args()
    m1, m4 = _meta(a), _meta(a, lora_slots=4)
    assert list(m1.state_dict()) == list(m4.state_dict())  # the reference's keys, addressing slot 0
    for ad1, ad4 in zip(_adapters(m1), _adapters(m4)):
        assert ad4.rank_cols == ad1.rank_cols
        assert tuple(ad4.a.shape) == (4 * ad1.rank_cols, ad1.a.shape[1])
        assert tuple(ad4.b.shape) == (ad1.b.shape[0], 4 * ad1.rank_cols)


# ----------------------------------------------------------------------------- packing
@pytest.mark.parametrize("segments,interleaved", [([48, 16, 16], False), ([32, 32], True), ([40], False)])
@pytest.mark.parametrize("rank,slots", [(4, 3), (8, 2), (64, 2), (16, 16)])
def test_slot_views_and_zeros_outside(segments, interleaved, rank, slots):
    ad = LoraAdapter(24, segments, LoraArgs(rank, 2.0), interleaved=interleaved, slots=slots)
    Rc = ad.rank_cols
    assert Rc == -(-len(segments) * rank // 64) * 64
    g = torch.Generator().manual_seed(rank * 100 + slots)
    want_a = torch.zeros_like(ad.a)
    want_b = torch.zeros_like(ad.b)
    for j in range(slots):
        for s, n in enumerate(segments):
            A = torch.randn(rank, 24, generator=g) + 3
            B = torch.randn(n, rank, generator=g) + 3
            ad.put_A(s, A, slot=j)
            ad.put_B(s, B, slot=j)
            c0 = j * Rc + s * rank
            want_a[c0: c0 + rank] = A
            rows = torch.arange(n) * 2 + s if interleaved else torch.arange(n) + sum(segments[:s])
            want_b[rows, c0: c0 + rank] = B
            assert torch.equal(ad.lora_A(s, j), A) and torch.equal(ad.lora_B(s, j), B)
    assert torch.equal(ad.a, want_a) and torch.equal(ad.b, want_b)  # and nothing outside the views
    for j in range(slots):
        for s in range(len(segments)):
            ad.zero(s, j)
    assert not ad.a.any() and not ad.b.any()
    with pytest.raises(AssertionError):
        ad.lora_A(0, slots)


def _write_adapter(tmp_path, p, seed, name):
    import safetensors.torch

    sd = synth.synth_lora_state_dict(p, RANK, seed, torch.bfloat16, 1.0)
    path = tmp_path / f"{name}.safetensors"
    safetensors.torch.save_file(sd, str(path))
    return sd, path


def test_load_lora_touches_only_its_slot(tmp_path):
    p, a = _args()
    m = Transformer.empty(a, "cpu", torch.bfloat16, lora_slots=3)
    sd, path = _write_adapter(tmp_path, p, 5, "x")
    m.load_lora(path, scaling=99.0, slot=2)  # scaling is ignored, as in the reference
    for ad in _adapters(m):
        Rc = ad.rank_cols
        assert ad.a[2 * Rc:].any() and ad.b[:, 2 * Rc:].any()
        assert not ad.a[: 2 * Rc].any() and not ad.b[:, : 2 * Rc].any()
        assert ad.scaling == 2.0
    st = m.state_dict()
    for k, v in sd.items():  # the state-dict keys are slot 0's: still zero
        assert not st[k].any(), k
    m.load_lora(path, slot=0)
    for k, v in sd.items():
        assert torch.equal(st[k], v), k
    for ad in _adapters(m):  # slot 1 untouched by either load
        Rc = ad.rank_cols
        assert not ad.a[Rc: 2 * Rc].any() and not ad.b[:, Rc: 2 * Rc].any()
    bad = synth.synth_lora_state_dict(p, 2 * RANK, 1, torch.bfloat16, 1.0)  # today's rank check, per slot
    with pytest.raises(AssertionError):
        m._load_lora_state_dict(bad, slot=1)
    for s in (-1, 3, 1.0):
        with pytest.raises(ValueError, match="slot"):
            m.load_lora(path, slot=s)


# ----------------------------------------------------------------------------- per-token ids
@pytest.mark.parametrize("chunk", [None, 4, 6])
def test_token_ids_of_ragged_chunks(chunk):
    """Each chunk of generate()'s prompt plan gets one upload whose entry t is the id of token t's sequence."""
    _, a = _args()
    m = Transformer.empty(a, "cpu", torch.bfloat16, lora_slots=4)
    prompts = [list(range(n)) for n in (9, 10, 12, 11, 9)]  # ragged inside a chunk, every prompt in every chunk
    plan = _PromptPlan(prompts, chunk)
    ids = [3, -1, 0, 3, 1]
    for flat, seqlens, _, where in plan.chunks:
        rows = m._lora_rows(ids, seqlens)
        assert rows.dtype == torch.int32 and rows.tolist() == [ids[b] for b, _ in where]
        assert torch.equal(expand_lora_ids(ids, seqlens), rows)
    assert m._lora_rows(None, [2, 3]) is None
    assert m._default_rows(None, 5).tolist() == [0] * 5  # a multi-slot model without ids: slot 0, never the summed bank
    one = Transformer.empty(a, "cpu", torch.bfloat16)
    assert one._default_rows(None, 5) is None  # one slot without ids: today's unmasked call


def test_ids_checked_before_work():
    _, a = _args()
    m = _meta(a, lora_slots=2)
    for ids in ([0, 1], [0, 2, 1], [0, -2, 1], [0, 1.0, 1], [0, None, 1]):
        with pytest.raises(ValueError, match="lora_ids"):
            mi.generate([[1], [2], [3]], m, max_tokens=2, temperature=0.0, lora_ids=ids)
    m.check_lora_ids([0, 1, -1], 3)
    with pytest.raises(ValueError, match="un-merged adapters"):
        _meta(_args(lora=False)[1]).check_lora_ids([0], 1)


# ----------------------------------------------------------------------------- refusals, on meta
def test_refused_slot_counts():
    _, a = _args()
    for n in (0, MAX_LORA_SLOTS + 1, 2.0):
        with pytest.raises(ValueError, match="lora_slots"):
            _meta(a, lora_slots=n)
    _meta(a, lora_slots=MAX_LORA_SLOTS)
    with pytest.raises(ValueError, match="needs un-merged adapters"):
        _meta(_args(lora=False)[1], lora_slots=2)


def test_refused_on_mixture_of_experts():
    _, a = _args("tiny-moe")
    with pytest.raises(ValueError, match="mixture-of-experts"):
        _meta(a, lora_slots=2, expert_weights="fp8")
    m = _meta(a, expert_weights="fp8")  # one slot: today's MoE adapters, but no per-sequence ids
    with pytest.raises(ValueError, match="mixture-of-experts"):
        mi.generate([[1]], m, max_tokens=1, temperature=0.0, lora_ids=[0])


def test_refused_with_pipeline_ranks_and_expert_parallelism():
    _, a = _args()
    with pytest.raises(ValueError, match="pipeline"):
        mi.generate([[1]], _meta(a, pipeline_rank=0, num_pipeline_ranks=2), max_tokens=1, temperature=0.0, lora_ids=[0])
    _, am = _args("tiny-moe")
    ep = _meta(am, expert_parallel=(0, 2), expert_weights="fp8")
    with pytest.raises(ValueError, match="expert parallelism"):
        mi.generate([[1]], ep, max_tokens=1, temperature=0.0, lora_ids=[0])


def test_refused_with_draft():
    _, a = _args()
    with pytest.raises(ValueError, match="draft"):
        mi.generate([[1], [2]], _meta(a, lora_slots=2), max_tokens=2, temperature=0.0, draft=_meta(a), lora_ids=[0, 1])
