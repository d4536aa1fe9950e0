"""Speculative decoding on the GPU: the verify step's device metadata, the acceptance kernels, and generate(..., draft=...) at model
level against the CPU oracle (teacher-forced on the tokens it emitted)."""
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.transformer import Transformer
from oracle import restatement as R

from . import int4_dense_ref as I4
from . import kv_fp8_ref as KF
from . import spec_ref as ref
from .util import LOGPROB_TOL, RouterProbe, launched_kernels, logit_tol, oracle_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
TEMP, TOP_P = 0.7, 0.8


# ----------------------------------------------------------------------------------------------------------- mb200_spec_meta
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("k", [1, 4])
def test_spec_meta_matches_host_metadata(B, k):
    """mb200_spec_meta == BufferCache.build_metadata_host for seqlens [k + 1] * B, bit for bit: ragged positions, four distinct
    windows (the smallest one reached exactly by the last verified token), and seqpos left as it was."""
    S = k + 1
    windows = [16, 24, None, 40]  # cache sizes 16, 24, 64, 40
    cache = BufferCache(4, B, 64, 2, 128, windows)
    pos = [max(1, 16 - S - 3 * b) for b in range(B)]
    pos[-1] = 16 - S  # the last token lands on slot W - 1 of the 16-token ring: no wrap
    cache._kv_seqlens_host = list(pos)
    host, layout = cache.build_metadata_host([S] * B)
    distinct = layout["windows"]
    assert len(distinct) == 4 and max(p + S for p in pos) <= min(distinct)
    seqpos = torch.tensor(pos, dtype=torch.int32, device=DEV)
    meta = torch.full((_abi.spec_meta_words(B, S, len(distinct)),), -7, dtype=torch.int32, device=DEV)
    assert meta.numel() == host.size
    _abi.spec_meta(seqpos, meta, S, distinct)
    assert meta.cpu().tolist() == host.tolist()
    assert seqpos.cpu().tolist() == pos


# ----------------------------------------------------------------------------------------------------- greedy acceptance
@pytest.mark.parametrize("k", [1, 4])
def test_accept_greedy_exact(k):
    """Crafted rows: every sequence rejects at a different j (k = all accepted), plus argmax ties where the first index wins."""
    S, V = k + 1, 1000
    g = torch.Generator().manual_seed(k)
    cases = list(range(k + 1)) + ["tie_accept", "tie_reject"]
    B = len(cases)
    logits = torch.randn(B, S, V, generator=g)
    amax = logits.argmax(-1)
    tokens = torch.zeros(B, S, dtype=torch.long)
    tokens[:, 0] = torch.arange(B) + 3
    for b, c in enumerate(cases):
        tokens[b, 1:] = amax[b, :k]
        if isinstance(c, int) and c < k:
            tokens[b, c + 1] = (amax[b, c] + 1) % V
        elif c in ("tie_accept", "tie_reject"):
            j = k - 1
            lo, hi = sorted(torch.randperm(V, generator=g)[:2].tolist())
            logits[b, j, lo] = logits[b, j, hi] = logits[b, j].max() + 1.0
            tokens[b, j + 1] = lo if c == "tie_accept" else hi
    dev_logits = logits.reshape(B * S, V).to(DEV)
    out = torch.full((B, S), -5, dtype=torch.long, device=DEV)
    n = torch.zeros(B, dtype=torch.int32, device=DEV)
    seqpos = torch.arange(B, dtype=torch.int32, device=DEV) * 10 + 7
    _abi.spec_accept_greedy(dev_logits, tokens.to(DEV), out, n, seqpos)
    for b, c in enumerate(cases):
        want, wn = ref.accept_greedy(logits[b].double().numpy(), tokens[b].tolist())
        if isinstance(c, int):
            assert wn == c
        else:
            assert wn == (k if c == "tie_accept" else k - 1)
        assert int(n[b]) == wn, (c, int(n[b]), wn)
        assert out[b].tolist() == want + [-1] * (S - len(want)), c
        assert int(seqpos[b]) == b * 10 + 7 + wn + 1


# ----------------------------------------------------------------------------------------------------- sampled acceptance
def _rows(V: int, seed: int, scale: float = 1.0) -> torch.Tensor:
    return torch.randn(V, generator=torch.Generator().manual_seed(seed)) * scale


def _run_sample(p_rows: torch.Tensor, q_rows: torch.Tensor, trials: int, batch: int = 4096):
    """p_rows [k + 1, V], q_rows [k, V] shared by every sequence; proposals drawn from the draft's nucleus by mb200_sample_top_p.
    Returns (out [trials, k + 1], n [trials]) on the host."""
    k, V = q_rows.shape
    S = k + 1
    logits = p_rows.to(DEV).repeat(batch, 1).contiguous()
    draft = q_rows.to(DEV).repeat(batch, 1).contiguous()
    outs, ns = [], []
    gen = torch.Generator(device=DEV).manual_seed(1234)
    for _ in range(trials // batch):
        tokens = torch.zeros(batch, S, dtype=torch.long, device=DEV)
        for j in range(k):
            u = torch.rand(batch, generator=gen, device=DEV)
            tokens[:, j + 1] = _abi.sample_top_p(draft.view(batch, k, V)[:, j].contiguous(), u, TEMP, TOP_P)
        uni = torch.rand(batch, S, generator=gen, device=DEV)
        out = torch.empty(batch, S, dtype=torch.long, device=DEV)
        n = torch.empty(batch, dtype=torch.int32, device=DEV)
        seqpos = torch.zeros(batch, dtype=torch.int32, device=DEV)
        _abi.spec_accept_sample(logits, draft, tokens, uni, out, n, seqpos, TEMP, TOP_P)
        assert torch.equal(seqpos, n + 1)
        outs.append(out.cpu())
        ns.append(n.cpu())
    return torch.cat(outs), torch.cat(ns)


def _nucleus(row: torch.Tensor):
    """float64 nucleus of an fp32 row, refusing rows whose cut is within rounding of top_p (the kernel decides it in fp32)."""
    p = ref.nucleus(row.double().numpy(), TEMP, TOP_P)
    z = row.double().numpy() / TEMP
    full = torch.softmax(torch.from_numpy(z), 0).numpy()
    before = torch.tensor([full[full > x].sum() for x in full])
    assert (before - TOP_P).abs().min() > 1e-4, "fixture: a token sits on the nucleus cut"
    return p


def test_accept_sample_distribution_and_rate():
    """2^20 seeded trials, k = 2, V = 512: the first emitted token is distributed as the target's nucleus P_0 (chi-square over P_0's
    support below the 1 - 1e-6 quantile; no token outside it), and the first proposal is accepted at the rate sum(min(P_0, Q_0))
    (within 6 standard errors)."""
    from scipy.stats import chi2

    V, k, N = 512, 2, 1 << 20
    p_rows = torch.stack([_rows(V, 10 + j) for j in range(k + 1)])
    q_rows = torch.stack([0.7 * p_rows[j] + 0.7 * _rows(V, 20 + j) for j in range(k)])
    p0, q0 = _nucleus(p_rows[0]), _nucleus(q_rows[0])
    out, n = _run_sample(p_rows, q_rows, N)
    first = torch.bincount(out[:, 0], minlength=V).double().numpy()
    support = p0 > 0
    assert first[~support].sum() == 0, "a token outside the target's nucleus was emitted"
    expect = N * p0[support]
    stat = float((((first[support] - expect) ** 2) / expect).sum())
    limit = float(chi2.ppf(1 - 1e-6, int(support.sum()) - 1))
    a = ref.acceptance_rate(p0, q0)
    got = float((n >= 1).double().mean())
    se = (a * (1 - a) / N) ** 0.5
    print(f"\n[spec] sampled acceptance: chi2 {stat:.1f} (limit {limit:.1f}, {int(support.sum())} bins); accept rate {got:.5f} vs "
          f"sum(min(p, q)) {a:.5f} (se {se:.5f})")
    assert stat < limit
    assert abs(got - a) < 6 * se
    assert 0.2 < a < 0.95  # the fixture exercises both outcomes
    assert ((out == -1) == (torch.arange(k + 1)[None, :] > n[:, None].long())).all()


def test_accept_sample_exact_cases():
    """P == Q accepts every proposal; disjoint nuclei reject at row 0 and emit from P_0's nucleus."""
    V, k = 512, 4
    p_rows = torch.stack([_rows(V, 40 + j) for j in range(k + 1)])
    _, n = _run_sample(p_rows, p_rows[:k].clone(), 4096)
    assert (n == k).all()
    far = torch.full((k, V), -30.0)
    support = torch.from_numpy(_nucleus(p_rows[0]) > 0)
    for j in range(k):
        far[j, p_rows[j].argsort()[:3]] = 10.0  # the draft's nucleus: the target's three least likely tokens
    out, n = _run_sample(p_rows, far, 4096)
    assert (n == 0).all()
    assert support[out[:, 0]].all()


# ---------------------------------------------------------------------------------------------------------------- model level
def _model(p: dict, B: int, seed: int, **kw) -> Transformer:
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = B
    m = Transformer.empty(args, DEV, torch.bfloat16, **kw)
    m.load_state_dict(synth.synth_state_dict(p, seed, torch.bfloat16, DEV))
    return m.eval()


# name: (target shape, overrides, target kwargs, draft overrides, draft kwargs)
CONFIGS = {
    "tiny": ("tiny", {}, {}, {"n_layers": 1}, {}),
    "7b": ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, {}, {"n_layers": 1}, {}),
    "nemo": ("mistral-nemo-12b", {"n_layers": 2, "vocab_size": 8192}, {}, {"n_layers": 1}, {}),
    "large2-int4": ("mistral-large-2", {"n_layers": 2, "vocab_size": 4096}, {"dense_weights": "int4"}, {"n_layers": 1}, {"dense_weights": "int4"}),
    "tiny-kv-fp8": ("tiny", {}, {"kv_cache": "fp8"}, {"n_layers": 1}, {}),
    "tiny-moe": ("tiny-moe", {}, {}, {"n_layers": 1}, {}),
}
DRAFT_SHAPE = {"large2-int4": "mistral-7b"}  # the draft of Large 2 is a 7B-shaped model with its vocabulary


def _oracle(name: str, p: dict, B: int):
    sd = {k: v.cpu() for k, v in synth.synth_state_dict(p, 1, torch.bfloat16, DEV).items()}
    if CONFIGS[name][2].get("dense_weights") == "int4":
        sd = I4.int4_dense_checkpoint(sd)
    return R.OracleTransformer(oracle_args(p, B), sd)


def _teacher_forced(name, om, p, prompts, toks, lps):
    """Teacher-forces the oracle on prompt + emitted tokens: every emitted token is the oracle's argmax wherever its top-2 margin is
    decisive (2x the logit tolerance), and every log-probability is within LOGPROB_TOL.  MoE: rows at or after a router near-tie
    of their sequence are exempt (tests/test_gpu_model.py)."""
    from .test_gpu_model import Contamination

    moe = p.get("moe") is not None
    full = [pr + t for pr, t in zip(prompts, toks)]
    lens = [len(f) for f in full]
    ctx = KF.fp8_kv_cache() if CONFIGS[name][2].get("kv_cache") == "fp8" else _null()
    with ctx, RouterProbe() as probe:
        logits = om.forward(torch.tensor(sum(full, [])), lens, om.new_cache(max(lens)))
        exempt = Contamination(len(full), moe).rows(probe.end_forward(), lens)
    lsm = torch.log_softmax(logits.double(), -1)
    decisive_n = checked = 0
    o = 0
    for b, (pr, f) in enumerate(zip(prompts, full)):
        rows = logits[o:o + len(f)]
        for i in range(len(f) - 1):
            r = o + i
            if exempt is not None and exempt[r]:
                continue
            assert abs(float(lsm[r, f[i + 1]]) - lps[b][i]) <= LOGPROB_TOL, (name, b, i, float(lsm[r, f[i + 1]]), lps[b][i])
            checked += 1
            if i >= len(pr) - 1:  # an emitted token
                top2 = rows[i].topk(2).values
                if float(top2[0] - top2[1]) > 2 * logit_tol(rows[i]):
                    assert int(rows[i].argmax()) == f[i + 1], (name, b, i - len(pr) + 1)
                    decisive_n += 1
        o += len(f)
    print(f"[spec] {name}: {decisive_n} decisive emitted tokens equal the oracle's argmax, {checked} log-probabilities within {LOGPROB_TOL}")
    assert checked > 0 and (moe or decisive_n > 0)  # MoE: a router near-tie early in a prompt exempts the rest of its sequence


class _null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _pair(name: str, B: int):
    shape, over, tkw, dover, dkw = CONFIGS[name]
    p = synth.shape(shape, **over)
    dp = synth.shape(DRAFT_SHAPE.get(name, shape), **{**over, **dover})
    return p, _model(p, B, 1, **tkw), _model(dp, B, 2, **dkw)


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("lens,k,max_tokens", [([37], 4, 13), ([11, 19, 14], 3, 10)])
def test_generate_with_draft_vs_oracle(name, lens, k, max_tokens):
    """Greedy generate(draft=...): batch 1 (a megakernel draft where the draft has one) and a ragged batch of 3, max_tokens not a
    multiple of k + 1; teacher-forced against the oracle.  The accept kernel runs; the verify step is captured once and replayed."""
    p, m, d = _pair(name, len(lens))
    prompts = [synth.synth_prompt(n, p["vocab_size"], 30 + i) for i, n in enumerate(lens)]
    res = {}
    names = launched_kernels(lambda: res.setdefault("out", mi.generate(prompts, m, max_tokens=max_tokens, temperature=0.0, draft=d,
                                                                          draft_tokens=k)))
    toks, lps = res["out"]
    assert len(toks) == len(lens) and all(len(t) == max_tokens for t in toks)
    assert all(len(lp) == n - 1 + max_tokens for lp, n in zip(lps, lens))
    rounds = names.count("spec_accept_greedy_kernel")
    assert rounds >= 2 and names.count("spec_meta_kernel") == 2  # eager, then captured: every later round is one graph replay
    _teacher_forced(name, _oracle(name, p, len(lens)), p, prompts, toks, lps)


@pytest.mark.parametrize("B", [1, 3])
def test_draft_with_the_targets_weights_accepts_every_decisive_proposal(B, monkeypatch):
    """A draft holding the target's own weights: a proposal is rejected only where the target's verify row has it within the logit
    tolerance of its maximum (the draft's one-token step and the verify step round differently)."""
    p = synth.shape("mistral-7b", n_layers=2, vocab_size=4096)
    m, d = _model(p, B, 1), _model(p, B, 1)
    k = 4
    seen = []
    orig = _abi.spec_accept_greedy

    def record(logits, tokens, out, n, seqpos):
        orig(logits, tokens, out, n, seqpos)
        seen.append((logits.clone().cpu(), tokens.clone().cpu(), n.clone().cpu()))

    monkeypatch.setattr(_abi, "spec_accept_greedy", record)
    prompts = [synth.synth_prompt(20 + 3 * b, p["vocab_size"], 50 + b) for b in range(B)]
    mi.generate(prompts, m, max_tokens=21, temperature=0.0, draft=d, draft_tokens=k)
    accepted = rejected = 0
    for logits, tokens, n in seen:
        rows = logits.view(B, k + 1, -1)
        for b in range(B):
            nb = int(n[b])
            accepted += nb
            if nb < k:
                row, dtok = rows[b, nb], int(tokens[b, nb + 1])
                assert float(row.max() - row[dtok]) <= 2 * logit_tol(row), (b, nb)
                rejected += 1
    print(f"\n[spec] self-draft B={B}: {accepted} proposals accepted, {rejected} rejected at near-ties, over {len(seen)} rounds")
    assert accepted >= 3 * rejected


def test_eos_and_lengths_follow_the_reference_rule():
    """eos: a sequence is finished from its first eos on; the output stops at the first step where every sequence is finished (that
    step excluded).  max_tokens 0 returns [] and the prompt log-probabilities."""
    p = synth.shape("tiny")
    m, d = _model(p, 2, 1), _model(synth.shape("tiny", n_layers=1), 2, 2)
    prompts = [[1, 2, 3], [4, 5, 6, 7]]
    toks, _ = mi.generate(prompts, m, max_tokens=30, temperature=0.0, draft=d, draft_tokens=3)
    for eos in (toks[0][5], toks[1][2], toks[0][0]):
        steps = [min([s for s, t in enumerate(seq) if t == eos] or [10 ** 9]) for seq in toks]
        expect = max(steps) if max(steps) < 10 ** 9 else 30
        toks2, lp2 = mi.generate(prompts, m, max_tokens=30, temperature=0.0, eos_id=eos, draft=d, draft_tokens=3)
        assert toks2 == ([t[:expect] for t in toks] if expect > 0 else [])
        assert [len(x) for x in lp2] == [len(pr) - 1 + expect for pr in prompts]
    t0, l0 = mi.generate(prompts, m, max_tokens=0, temperature=0.0, draft=d)
    assert t0 == [] and [len(x) for x in l0] == [2, 3]
    t1, l1 = mi.generate(prompts, m, max_tokens=1, temperature=0.0, draft=d)
    want1, _ = mi.generate(prompts, m, max_tokens=1, temperature=0.0)
    assert t1 == want1 and [len(x) for x in l1] == [3, 4]


def test_sampled_generate_runs():
    p = synth.shape("tiny")
    m, d = _model(p, 3, 1), _model(synth.shape("tiny", n_layers=1), 3, 2)
    torch.manual_seed(0)
    res = {}
    names = launched_kernels(lambda: res.setdefault("o", mi.generate([[1, 2, 3], [4, 5, 6, 7], [9]], m, max_tokens=17, temperature=0.7,
                                                                      draft=d, draft_tokens=3)))
    toks, lps = res["o"]
    assert "spec_accept_sample_kernel" in names
    assert all(len(t) == 17 for t in toks) and all(0 <= x < p["vocab_size"] for t in toks for x in t)
    assert all(v <= 0 for x in lps for v in x) and [len(x) for x in lps] == [2 + 17, 3 + 17, 17]


def test_verify_step_replays_without_launches():
    """The third verify step of a (cache, B, S) is a graph replay: the library launches nothing from the host."""
    p = synth.shape("tiny")
    m = _model(p, 2, 1)
    cache = BufferCache(m.n_local_layers, 2, 64, p["n_kv_heads"], p["head_dim"]).to(m.device, m.dtype)
    cache.reset()
    m.forward(torch.arange(1, 12, device=DEV), [5, 6], cache)
    toks = torch.randint(0, p["vocab_size"], (2, 4), device=DEV)
    first = launched_kernels(lambda: m.verify_static(toks, cache))
    assert "spec_meta_kernel" in first and any(n.startswith("attn_prefill") for n in first)
    captured = m.verify_static(toks, cache)[0].clone()
    assert launched_kernels(lambda: m.verify_static(toks, cache)) == []
    assert torch.equal(m.verify_static(toks, cache)[0], captured)
