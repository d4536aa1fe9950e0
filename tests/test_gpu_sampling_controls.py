"""Per-sequence sampling controls on the GPU (mb200_select_tokens, csrc/sampling.cuh), bit for bit.

Every expected token is the existing selection kernels' answer on the host restatement (tests/sampling_controls_ref.py):
_abi.sample_top_p at the row's (temperature, top_p) with the restated Philox uniform, and _abi.argmax_rows on the float32-restated
penalised logits.  The model-level tests check the generate() paths: today's path untouched, seeded runs reproducible and
independent of their batch companions, greedy rows unaffected by sampled ones, and the penalty rule on the model's own logits.
"""
import sys

import numpy as np
import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.transformer import Transformer

from . import sampling_controls_ref as SR
from . import spec_ref as ref
from .test_gpu_token_selection import _argmax_rows
from .util import launched_kernels

pytestmark = pytest.mark.gpu
DEV = "cuda"
SEEDS = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 64 - 1]


def _i64(seeds):
    """uint64 seeds as the int64 bit patterns the binding takes."""
    return torch.tensor([s - (1 << 64) if s >= 1 << 63 else s for s in seeds], dtype=torch.int64, device=DEV)


def _f32(v, B=None):
    return torch.tensor(v if B is None else [v] * B, dtype=torch.float32, device=DEV)


def _select(logits, temperature, top_p, presence, frequency, step, *, seeds=None, uniform=None, counts=None):
    B = logits.shape[0]
    out = torch.full((B,), -7, dtype=torch.long, device=DEV)
    _abi.select_tokens(logits, _f32(temperature), _f32(top_p), _f32(presence), _f32(frequency), step, out,
                       seeds=None if seeds is None else _i64(seeds), uniform=uniform, counts=counts)
    return out


# ------------------------------------------------------------------------------------------------------------ the uniforms
def test_seeded_uniforms_equal_the_restatement():
    """Equal logits over V = 2^17 make the draw floor(u * 2^17) exactly (every weight, prefix and the total are exact in fp32), so the
    token shows the top 17 bits of the device uniform.  Seeds 0, 1, 2^32 - 1, 2^32, 2^64 - 1 at steps 0 .. 4095, every step's
    token exact; step advances by one per call.  The remaining bits enter every sampled-row test below."""
    V, steps = 1 << 17, 4096
    row = torch.zeros(1, V, device=DEV)
    for seed in SEEDS:
        logits = row.expand(steps, V).contiguous()
        step = torch.arange(steps, dtype=torch.int32, device=DEV)
        got = _select(logits, [1.0] * steps, [1.0] * steps, [0.0] * steps, [0.0] * steps, step, seeds=[seed] * steps).cpu().numpy()
        u = SR.uniforms(seed, np.arange(steps))
        want = np.floor(u.astype(np.float64) * V).astype(np.int64)
        assert np.array_equal(got, want), (seed, np.nonzero(got != want)[0][:5])
        assert torch.equal(step.cpu(), torch.arange(steps, dtype=torch.int32) + 1)


# ------------------------------------------------------------------------------------------------------------ sampled rows
def _mixed_rows(B: int, V: int, seed: int):
    g = torch.Generator().manual_seed(seed)
    temps = [[0.05, 0.7, 1.0, 4.0][b % 4] for b in range(B)]
    tops = [[0.0, 0.5, 0.8, 0.95, 1.0][(b * 3) % 5] for b in range(B)]
    logits = torch.randn(B, V, generator=g) * torch.tensor([4.0 * t + 0.5 for t in temps])[:, None]
    return logits, temps, tops


def _expected_sampled(logits, temps, tops, u):
    """_abi.sample_top_p row by row at the row's own (temperature, top_p) and uniform."""
    want = torch.empty(logits.shape[0], dtype=torch.long)
    for b in range(logits.shape[0]):
        want[b] = _abi.sample_top_p(logits[b:b + 1], u[b:b + 1], temps[b], tops[b]).cpu()[0]
    return want


@pytest.mark.parametrize("V", [32000, 131072, 131073])
def test_sampled_rows_equal_sample_top_p(V):
    """A batch mixing temperatures 0.05..4 and top_p 0..1: with seeds each row's token is sample_top_p at the row's controls and the
    restated uniform of its (seed, step); with caller uniforms, sample_top_p at those uniforms."""
    B = 64
    logits, temps, tops = _mixed_rows(B, V, 10 + V)
    dl = logits.to(DEV)
    seeds = [SEEDS[b % 5] + 977 * b for b in range(B)]
    seeds = [s % (1 << 64) for s in seeds]
    steps0 = [(b * 131) % 5000 for b in range(B)]
    step = torch.tensor(steps0, dtype=torch.int32, device=DEV)
    got = _select(dl, temps, tops, [0.0] * B, [0.0] * B, step, seeds=seeds).cpu()
    u = torch.tensor([float(SR.uniforms(s, [t])[0]) for s, t in zip(seeds, steps0)], dtype=torch.float32, device=DEV)
    want = _expected_sampled(dl, temps, tops, u)
    assert torch.equal(got, want), [(b, int(got[b]), int(want[b])) for b in range(B) if got[b] != want[b]][:5]
    assert torch.equal(step.cpu(), torch.tensor(steps0, dtype=torch.int32) + 1)
    uc = torch.rand(B, generator=torch.Generator().manual_seed(V)).to(DEV)
    got = _select(dl, temps, tops, [0.0] * B, [0.0] * B, step, uniform=uc).cpu()
    assert torch.equal(got, _expected_sampled(dl, temps, tops, uc))


# ------------------------------------------------------------------------------------------------------------ greedy rows
@pytest.mark.parametrize("V", [1025, 32000, 131072, 131073])
def test_greedy_rows_equal_argmax_rows_on_the_penalised_logits(V):
    """The designed argmax rows (ties, +-0, NaN payloads, -inf rows) with and without penalties and random counts: each token is
    argmax_rows of the float32-restated l'.  Rows with both penalties 0 read their logits as they are."""
    rows, _ = _argmax_rows(V, 40 + V)
    R = rows.shape[0]
    g = torch.Generator().manual_seed(V)
    counts = (torch.rand(R, V, generator=g) < 0.01).int() * torch.randint(1, 4, (R, V), generator=g, dtype=torch.int32)
    pres = [[0.0, 0.5, -1.0, 2.0][r % 4] for r in range(R)]
    freq = [[0.0, 0.0, 0.25, -2.0][(r // 4) % 4] for r in range(R)]
    lp = torch.from_numpy(SR.penalised(rows.numpy(), counts.numpy(), pres, freq))
    want = _abi.argmax_rows(lp.to(DEV)).cpu()
    step = torch.zeros(R, dtype=torch.int32, device=DEV)
    dc = counts.to(DEV)
    got = _select(rows.to(DEV), [0.0] * R, [0.8] * R, pres, freq, step, seeds=list(range(R)), counts=dc).cpu()
    assert torch.equal(got, want), [(r, int(got[r]), int(want[r])) for r in range(R) if got[r] != want[r]][:5]
    # no penalty anywhere: exactly argmax_rows of the raw rows
    raw = _select(rows.to(DEV), [0.0] * R, [0.8] * R, [0.0] * R, [0.0] * R, step, uniform=torch.zeros(R, device=DEV)).cpu()
    assert torch.equal(raw, _abi.argmax_rows(rows.to(DEV)).cpu())
    # the counts advanced by one at each row's token
    counts[torch.arange(R), got] += 1
    assert torch.equal(dc.cpu(), counts)


# ------------------------------------------------------------------------------------------------------------ penalties
def _tie_rows(V: int, R: int, seed: int):
    """Rows where a penalty makes an earlier-seen token tie the best unseen one exactly: 5.0 seen once at presence 1, or seen 4 times
    at frequency 0.25, against 4.0 unseen -- before and after it in index order."""
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn(R, V, generator=g) - 8.0
    counts = torch.zeros(R, V, dtype=torch.int32)
    pres, freq = [], []
    for r in range(R):
        i, j = sorted(torch.randperm(V, generator=g)[:2].tolist())
        seen, other = (i, j) if r % 2 == 0 else (j, i)
        rows[r, seen], rows[r, other] = 5.0, 4.0
        if r % 4 < 2:
            counts[r, seen], p, f = 1, 1.0, 0.0
        else:
            counts[r, seen], p, f = 4, 0.0, 0.25
        pres.append(p)
        freq.append(f)
    return rows, counts, pres, freq


@pytest.mark.parametrize("V", [32000, 131073])
def test_penalty_ties_and_counts_over_steps(V):
    """Ties a penalty creates go to the first index, as argmax_rows on the restated l'.  Sampled rows with penalties equal
    sample_top_p on the restated l'.  Then k = 24 steps on fixed logits: every step's tokens equal the restatement at that step's
    counts, and the counts equal the host histogram of the tokens."""
    R = 32
    rows, counts, pres, freq = _tie_rows(V, R, 70 + V)
    lp = torch.from_numpy(SR.penalised(rows.numpy(), counts.numpy(), pres, freq))
    assert all(int(lp[r].argmax()) == int((lp[r] == 4.0).nonzero()[0]) for r in range(R))  # the tie goes to the first of the two
    step = torch.zeros(R, dtype=torch.int32, device=DEV)
    got = _select(rows.to(DEV), [0.0] * R, [0.8] * R, pres, freq, step, uniform=torch.zeros(R, device=DEV), counts=counts.to(DEV)).cpu()
    assert torch.equal(got, _abi.argmax_rows(lp.to(DEV)).cpu())
    assert torch.equal(got, lp.argmax(-1))

    # k steps, half the rows sampled, seeded: the penalised row changes every step
    g = torch.Generator().manual_seed(V + 1)
    base = torch.randn(R, V, generator=g) * 1.5
    temps = [0.0 if r % 2 == 0 else [0.5, 1.0, 2.0][r % 3] for r in range(R)]
    tops = [[0.8, 0.95, 1.0][r % 3] for r in range(R)]
    pres = [[0.0, 0.7, 2.0, -0.5][r % 4] for r in range(R)]
    freq = [[0.3, 0.0, 1.0, -0.25][(r // 2) % 4] for r in range(R)]
    seeds = [1000 + r for r in range(R)]
    dl = base.to(DEV)
    dc = torch.zeros(R, V, dtype=torch.int32, device=DEV)
    step = torch.zeros(R, dtype=torch.int32, device=DEV)
    host = np.zeros((R, V), dtype=np.int32)
    for t in range(24):
        l1 = torch.from_numpy(SR.penalised(base.numpy(), host, pres, freq)).to(DEV)
        u = torch.tensor([float(SR.uniforms(s, [t])[0]) for s in seeds], device=DEV)
        want = _abi.argmax_rows(l1).cpu()
        for r in range(R):
            if temps[r] > 0:
                want[r] = _abi.sample_top_p(l1[r:r + 1], u[r:r + 1], temps[r], tops[r]).cpu()[0]
        got = _select(dl, temps, tops, pres, freq, step, seeds=seeds, counts=dc).cpu()
        assert torch.equal(got, want), (t, [(r, int(got[r]), int(want[r])) for r in range(R) if got[r] != want[r]][:5])
        host[np.arange(R), got.numpy()] += 1
    assert np.array_equal(dc.cpu().numpy(), host)
    assert (step.cpu() == 24).all()


# ------------------------------------------------------------------------------------------------------------ capture
def test_captured_selection_replays_like_eager_calls():
    """One graph with one selection, replayed n times, advances steps and counts and picks the tokens of n eager calls."""
    B, V, n = 8, 32000, 12
    g = torch.Generator().manual_seed(5)
    logits = (torch.randn(B, V, generator=g) * 2).to(DEV)
    temps = [0.0, 0.7, 1.0, 0.0, 1.3, 0.7, 0.0, 2.0]
    ctl = [_f32(temps), _f32([0.9] * B), _f32([0.4] * B), _f32([0.2] * B)]
    seeds = _i64([7 * b + 3 for b in range(B)])

    def state():
        return torch.zeros(B, dtype=torch.int32, device=DEV), torch.zeros(B, V, dtype=torch.int32, device=DEV), \
            torch.zeros(B, dtype=torch.long, device=DEV)

    step_e, counts_e, out_e = state()
    eager = []
    for _ in range(n):
        _abi.select_tokens(logits, *ctl, step_e, out_e, seeds=seeds, counts=counts_e)
        eager.append(out_e.clone())
    step_g, counts_g, out_g = state()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up outside the capture, then undo its advance
        _abi.select_tokens(logits, *ctl, step_g, out_g, seeds=seeds, counts=counts_g)
    torch.cuda.current_stream().wait_stream(s)
    step_g.zero_()
    counts_g.zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _abi.select_tokens(logits, *ctl, step_g, out_g, seeds=seeds, counts=counts_g)
    assert (step_g == 0).all()  # capturing ran nothing
    replayed = []
    for _ in range(n):
        graph.replay()
        replayed.append(out_g.clone())
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, replayed))
    assert torch.equal(step_g, step_e) and torch.equal(counts_g, counts_e) and (step_g == n).all()
    assert len({tuple(x.tolist()) for x in eager}) > 1  # the stream moves with the step


# ------------------------------------------------------------------------------------------------------------ distribution
def test_seeded_draws_follow_the_nucleus_distribution():
    """V = 24, 2^20 seeded draws from one fixed row (seeds 0 .. 2^18 - 1 at steps 0 .. 3): the token counts follow the float64
    nucleus at (0.7, 0.8) (chi-square below the 1 - 1e-6 quantile) and no token outside the nucleus appears."""
    from scipy.stats import chi2

    V, temp, top_p, batch, steps = 24, 0.7, 0.8, 1 << 18, 4
    row = torch.randn(1, V, generator=torch.Generator().manual_seed(1300))
    nuc = ref.nuclei(ref.scaled_logits(row.numpy(), temp), top_p)[0]
    assert nuc.decisive
    p = nuc.dense()
    logits = row.to(DEV).expand(batch, V).contiguous()
    seeds = _i64(list(range(batch)))
    ctl = [_f32(temp, batch), _f32(top_p, batch), _f32(0.0, batch), _f32(0.0, batch)]
    step = torch.zeros(batch, dtype=torch.int32, device=DEV)
    out = torch.empty(batch, dtype=torch.long, device=DEV)
    counts = np.zeros(V)
    for _ in range(steps):
        _abi.select_tokens(logits, *ctl, step, out, seeds=seeds)
        counts += np.bincount(out.cpu().numpy(), minlength=V)
    N = batch * steps
    assert counts[p == 0].sum() == 0, "a token outside the nucleus"
    obs, exp = counts[p > 0], p[p > 0] * N
    stat = float(((obs - exp) ** 2 / exp).sum())
    limit = float(chi2.ppf(1 - 1e-6, exp.size - 1))
    print(f"\n[controls] {int((p > 0).sum())} tokens in the nucleus, chi2 {stat:.1f} < {limit:.1f}")
    assert stat < limit


# ------------------------------------------------------------------------------------------------------------ model level
CONFIGS = {
    "7b": ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}),
    "nemo": ("mistral-nemo-12b", {"n_layers": 2, "vocab_size": 8192}),
}


def _model(name: str, B: int) -> Transformer:
    shape, over = CONFIGS[name]
    p = synth.shape(shape, **over)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = B
    m = Transformer.empty(args, DEV, torch.bfloat16)
    m.load_state_dict(synth.synth_state_dict(p, 1, torch.bfloat16, DEV))
    return m.eval()


def _prompts(name: str, lens, seed: int):
    V = CONFIGS[name][1]["vocab_size"]
    return [synth.synth_prompt(n, V, seed + i) for i, n in enumerate(lens)]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_default_path_and_equivalent_controls_agree(name):
    """Default arguments (today's path) and explicit defaults give the same output under one torch.manual_seed; a list of equal
    temperatures without seeds takes the controls path with the same torch.rand draws and the same nucleus, so it gives it too."""
    B = 3
    m = _model(name, B)
    prompts = _prompts(name, [9, 14, 6], 10)
    runs = []
    for kw in ({}, {"top_p": 0.8, "random_seed": None, "presence_penalty": 0.0, "frequency_penalty": 0.0},
               {"temperature": [0.7] * B}):
        torch.manual_seed(123)
        runs.append(mi.generate(prompts, m, max_tokens=12, **{"temperature": 0.7, **kw}))
    assert runs[0] == runs[1] == runs[2]
    g0 = mi.generate(prompts, m, max_tokens=12, temperature=0.0)
    assert g0 == mi.generate(prompts, m, max_tokens=12, temperature=[0.0] * B)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_seeded_output_is_reproducible_and_batch_independent(name):
    """A seeded call repeats exactly, whatever torch.manual_seed says.  Sequence a gives the same tokens and log-probabilities
    next to companion b or c (other prompt, seed and temperature; same batch size and max_batch_size)."""
    m = _model(name, 2)
    a, b, c = _prompts(name, [11], 1)[0], _prompts(name, [7], 2)[0], _prompts(name, [7], 3)[0]  # b, c: one length, one GEMM regime
    kw = dict(max_tokens=16, top_p=0.9, presence_penalty=0.3, frequency_penalty=0.2)
    torch.manual_seed(1)
    r1 = mi.generate([a, b], m, temperature=[0.8, 1.2], random_seed=[42, 5], **kw)
    torch.manual_seed(2)
    r2 = mi.generate([a, b], m, temperature=[0.8, 1.2], random_seed=[42, 5], **kw)
    assert r1 == r2
    r3 = mi.generate([a, c], m, temperature=[0.8, 0.0], random_seed=[42, 2 ** 64 - 1], **kw)
    assert r3[0][0] == r1[0][0] and r3[1][0] == r1[1][0]
    assert b != c and r1[0][1] != r3[0][1]  # the companions really differ
    r4 = mi.generate([a, c], m, temperature=0.8, random_seed=41, **kw)  # one int: sequence b runs on 41 + b
    assert r4 == mi.generate([a, c], m, temperature=[0.8, 0.8], random_seed=[41, 42], **kw)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_greedy_rows_of_a_mixed_batch_equal_an_all_greedy_run(name):
    m = _model(name, 4)
    prompts = _prompts(name, [8, 12, 5, 9], 20)
    greedy = mi.generate(prompts, m, max_tokens=14, temperature=0.0)
    mixed = mi.generate(prompts, m, max_tokens=14, temperature=[0.0, 0.9, 0.0, 1.5], random_seed=3)
    for b in (0, 2):
        assert mixed[0][b] == greedy[0][b] and mixed[1][b] == greedy[1][b], b


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("B", [1, 3])
def test_presence_penalty_on_the_models_logits(name, B, monkeypatch):
    """Greedy with presence_penalty = 2 on both decode paths (the batch-1 megakernel, the graph step): every step's token is the
    argmax of the restated l' of that step's logits, no token repeats where the logits' spread is under the penalty, and the
    returned log-probabilities are log_softmax of the raw logits at the chosen token.  The launch log shows the selection kernel once
    per step and the generate() `pick` is never used."""
    G = sys.modules["mistral_inference_b200.generate"]  # the module: the package re-exports its generate()

    m = _model(name, B)
    prompts = _prompts(name, [10, 6, 13][:B], 30)
    seen = []
    orig = _abi.select_tokens

    def record(logits, *a, counts=None, **kw):
        seen.append((logits.clone().cpu(), counts.clone().cpu()))
        return orig(logits, *a, counts=counts, **kw)

    monkeypatch.setattr(_abi, "select_tokens", record)
    monkeypatch.setattr(G, "pick", lambda *a, **k: pytest.fail("pick (and its fused argmax) ran on the controls path"))
    steps = 20
    res = {}
    names = launched_kernels(lambda: res.setdefault("o", mi.generate(prompts, m, max_tokens=steps, temperature=0.0, presence_penalty=2.0)))
    toks, lps = res["o"]
    assert names.count("select_tokens_kernel<uniform, counts>") == steps
    assert ("decode_megakernel" in " ".join(names)) == (B == 1) == m._megakernel_ok(B)
    assert len(seen) == steps
    for b in range(B):
        for t, (logits, counts) in enumerate(seen):
            want = torch.from_numpy(SR.penalised(logits[b:b + 1].numpy(), counts[b:b + 1].numpy(), 2.0, 0.0)).argmax(-1)
            assert toks[b][t] == int(want), (b, t)
            raw = torch.log_softmax(logits[b].double(), -1)[toks[b][t]]
            assert abs(lps[b][len(prompts[b]) - 1 + t] - float(raw)) <= 1e-5, (b, t)
        spread = max(float(l[b].max() - l[b].min()) for l, _ in seen)
        if spread < 2.0:
            assert len(set(toks[b])) == len(toks[b]), (b, toks[b])
