"""Multi-adapter LoRA on the GPU: the three `_lora` entry points with a bank of adapter slots and one slot per row, each row against
its own slot's rounding chain bit for bit (the integer method of tests/test_gpu_lora.py), and at model level batch invariance (a
sequence of a mixed batch gives exactly the bits of a batch that uses its id throughout), agreement with the oracle, and id and
adapter changes under captured decode graphs."""
import re

import pytest
import torch

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.args import LoraArgs
from mistral_inference_b200.rope import precompute_freqs_cis
from mistral_inference_b200.transformer import Transformer
from mistral_inference_b200.transformer_layers import LoraAdapter
from oracle import lora as OL
from oracle import restatement as R

from .test_gpu_lora import SHAPES, T_LIST, _normed_input, bf, chain, ints
from .test_gpu_model import new_cache
from .util import LOGPROB_TOL, launched_kernels, oracle_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
SLOTS = [2, 4, 8, 16]
RANKS = [8, 16, 64]


def cases():
    return [(("7b", "nemo")[i % 2], T, SLOTS[i % 4], RANKS[i % 3]) for i, T in enumerate(T_LIST)]


def row_ids(T, slots, seed):
    """Seeded per-row slots with -1 (no adapter) and runs of equal ids."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(-1, slots, (T,), generator=g)
    if T >= 8:
        ids[T // 4: T // 4 + max(2, T // 8)] = slots - 1  # a run
        ids[T // 2: T // 2 + 3] = -1
    if T > 1:
        ids[0], ids[-1] = -1, 0
    return ids


def bank(in_f, segments, r, slots, seed, interleaved=False):
    """An adapter bank of integer A / B per slot: (adapter, A[slot][segment], B[slot][segment])."""
    ad = LoraAdapter(in_f, segments, LoraArgs(r, 2.0), interleaved=interleaved, slots=slots).to(DEV, torch.bfloat16)
    A = [[ints(r, in_f, seed=seed + 100 * j + s) for s in range(len(segments))] for j in range(slots)]
    B = [[ints(n, r, seed=seed + 100 * j + 10 + s) for s, n in enumerate(segments)] for j in range(slots)]
    for j in range(slots):
        for s in range(len(segments)):
            ad.put_A(s, A[j][s], slot=j)
            ad.put_B(s, B[j][s], slot=j)
    return ad, A, B


def per_row(xn, W, A, B, ids, seg):
    """out of every row through its own slot's chain (segment `seg`); -1 rows: the base Linear alone."""
    out = bf(xn.double() @ W.double().T)
    for j in ids.unique().tolist():
        if j < 0:
            continue
        rows = (ids == j).nonzero().flatten().to(DEV)
        out[rows] = chain(xn[rows], W, A[j][seg], B[j][seg], 2.0)[2]
    return out


def a_want(xn, A, ids, Rc, slots, r):
    """The masked down projection: row t holds its slot's segments' a, zero everywhere else."""
    a = torch.zeros(xn.shape[0], slots * Rc, dtype=torch.bfloat16, device=DEV)
    for j in ids.unique().tolist():
        if j < 0:
            continue
        rows = (ids == j).nonzero().flatten().to(DEV)
        for s, As in enumerate(A[j]):
            a[rows, j * Rc + s * r: j * Rc + (s + 1) * r] = bf(xn[rows].double() @ As.double().T)
    return a


def check_masked_launches(call_masked, call_single, T, normed):
    """The masked call ran the masked down kernel (T <= 4: the skinny EPI_STORE GEMV with the slot mask, norm fused when the call
    norms) and issued no more launches than the same call with one adapter."""
    names = launched_kernels(call_masked)
    torch.cuda.synchronize()
    single = launched_kernels(call_single)
    torch.cuda.synchronize()
    assert not [n for n in names if n.startswith("lora_down_kernel<") or n == "lora_down_reduce_kernel"], names
    if T > 4:
        down = [n for n in names if n.startswith("lora_down_masked_kernel<")]
        assert len(down) == 1, names
        splits = int(down[0][len("lora_down_masked_kernel<"):-1])
        assert names.count("lora_down_reduce_masked_kernel") == (1 if splits > 1 else 0), names
    else:
        assert f"skinny_linear_kernel<{T}, 64, {'true' if normed else 'false'}>" in names, names
    assert len(names) <= len(single), (names, single)
    return names


@pytest.mark.parametrize("shape,T,slots,r", cases())
def test_qkv_rows_bit_exact(shape, T, slots, r):
    dim, H, KV, _ = SHAPES[shape]
    hd = 128
    x, nw, xn = _normed_input(T, dim, 1)
    Ws = [ints(H * hd, dim, seed=3), ints(KV * hd, dim, seed=4), ints(KV * hd, dim, seed=5)]
    segs = [H * hd, KV * hd, KV * hd]
    ad, A, B = bank(dim, segs, r, slots, 20)
    one, _, _ = bank(dim, segs, r, 1, 20)
    ids = row_ids(T, slots, T)
    rows = ids.to(torch.int32).to(DEV)
    table = precompute_freqs_cis(hd, 8192, 1e6)
    positions = ((torch.arange(T, dtype=torch.int32) * 7) % 8000).to(DEV)
    rope = torch.view_as_real(table).contiguous().to(DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, H, KV, hd, 14336, 0, 4), torch.device(DEV))
    q = torch.empty(T, H * hd, dtype=torch.bfloat16, device=DEV)
    k = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
    v = torch.empty_like(k)
    w = torch.cat(Ws)
    st = ad.call(T, rows)
    check_masked_launches(lambda: _abi.attn_qkv_lora(x, nw, w, rope, positions, q, k, v, None, None, None, H, KV, hd, 1e-5, ws, st),
                          lambda: _abi.attn_qkv_lora(x, nw, w, rope, positions, q.clone(), k.clone(), v.clone(), None, None, None, H, KV,
                                                     hd, 1e-5, ws, one.call(T)), T, True)
    assert torch.equal(st.keep[0], a_want(xn, A, ids, ad.rank_cols, slots, r))
    outs = [per_row(xn, W, A, B, ids, s) for s, W in enumerate(Ws)]
    q_ref, k_ref = R.apply_rope(outs[0].cpu().view(T, H, hd), outs[1].cpu().view(T, KV, hd), table[positions.long().cpu()])
    assert torch.equal(q.cpu(), q_ref.reshape(T, -1))
    assert torch.equal(k.cpu(), k_ref.reshape(T, -1))
    assert torch.equal(v, outs[2])


@pytest.mark.parametrize("shape,T,slots,r", cases())
def test_gateup_rows_bit_exact(shape, T, slots, r):
    import torch.nn.functional as F

    dim, _, _, hidden = SHAPES[shape]
    x, nw, xn = _normed_input(T, dim, 2)
    W1, W3 = ints(hidden, dim, seed=6), ints(hidden, dim, seed=7)
    ad, A, B = bank(dim, [hidden, hidden], r, slots, 40, interleaved=True)
    one, _, _ = bank(dim, [hidden, hidden], r, 1, 40, interleaved=True)
    ids = row_ids(T, slots, T + 1)
    rows = ids.to(torch.int32).to(DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 32, 8, 128, hidden, 0, 4), torch.device(DEV))
    g = torch.empty(T, hidden, dtype=torch.bfloat16, device=DEV)
    w13 = torch.stack([W1, W3], 1).reshape(2 * hidden, dim)
    st = ad.call(T, rows)
    check_masked_launches(lambda: _abi.ffn_gateup_lora(x, nw, w13, g, 1e-5, ws, st),
                          lambda: _abi.ffn_gateup_lora(x, nw, w13, g.clone(), 1e-5, ws, one.call(T)), T, True)
    assert torch.equal(st.keep[0], a_want(xn, A, ids, ad.rank_cols, slots, r))
    o1, o3 = per_row(xn, W1, A, B, ids, 0), per_row(xn, W3, A, B, ids, 1)
    assert torch.equal(g, (F.silu(o1.float()).to(torch.bfloat16).float() * o3.float()).to(torch.bfloat16))


@pytest.mark.parametrize("which", ["wo", "w2"])
@pytest.mark.parametrize("shape,T,slots,r", cases())
def test_linear_residual_rows_bit_exact(which, shape, T, slots, r):
    dim, H, _, hidden = SHAPES[shape]
    K = H * 128 if which == "wo" else hidden
    x = ints(T, K, seed=8)
    W = ints(dim, K, seed=9)
    res = ints(T, dim, lo=-4, hi=4, seed=10)
    ad, A, B = bank(K, [dim], r, slots, 60)
    one, _, _ = bank(K, [dim], r, 1, 60)
    ids = row_ids(T, slots, T + 2)
    rows = ids.to(torch.int32).to(DEV)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 32, 8, 128, hidden, 0, 4), torch.device(DEV))
    out = torch.empty(T, dim, dtype=torch.bfloat16, device=DEV)
    st = ad.call(T, rows)
    check_masked_launches(lambda: _abi.linear_residual_lora(x, W, res, out, ws, st),
                          lambda: _abi.linear_residual_lora(x, W, res, out.clone(), ws, one.call(T)), T, False)
    assert torch.equal(st.keep[0], a_want(x, A, ids, ad.rank_cols, slots, r))
    assert torch.equal(out, (per_row(x, W, A, B, ids, 0).float() + res.float()).to(torch.bfloat16))


@pytest.mark.parametrize("T", [3, 512, 4096])
def test_masked_down_projection_deterministic(T):
    """Random (non-integer) inputs, where another split or summation order would change the fp32 sums: two runs give the same bits,
    a row's result does not depend on the other rows' ids, and at T > 4 the K split really happened."""
    K, N, r, slots = 14336, 4096, 16, 4
    g = torch.Generator().manual_seed(T)
    x = torch.randn(T, K, generator=g).to(torch.bfloat16).to(DEV)
    W = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16).to(DEV)
    ad = LoraAdapter(K, [N], LoraArgs(r, 2.0), slots=slots).to(DEV, torch.bfloat16)
    for j in range(slots):
        ad.put_A(0, (torch.randn(r, K, generator=g) * K ** -0.5).to(torch.bfloat16).to(DEV), slot=j)
        ad.put_B(0, (torch.randn(N, r, generator=g) * r ** -0.5).to(torch.bfloat16).to(DEV), slot=j)
    ws = _abi.Workspace(_abi.workspace_bytes(T, N, 32, 8, 128, K, 0, 4), torch.device(DEV))
    ids = row_ids(T, slots, 7)

    def run(ids):
        out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
        st = ad.call(T, ids.to(torch.int32).to(DEV))
        names = launched_kernels(lambda: _abi.linear_residual_lora(x, W, None, out, ws, st))
        torch.cuda.synchronize()
        return st.keep[0].clone(), out, names

    a0, o0, names = run(ids)
    a1, o1, _ = run(ids)
    assert torch.equal(a0, a1) and torch.equal(o0, o1)
    if T > 4:
        down = [n for n in names if n.startswith("lora_down_masked_kernel<")]
        assert len(down) == 1 and int(down[0][len("lora_down_masked_kernel<"):-1]) > 1, names
    for j in range(-1, slots):  # every row against the call in which all rows use its id
        sel = ids == j
        if sel.any():
            aj, oj, _ = run(torch.full_like(ids, j))
            rows = sel.nonzero().flatten().to(DEV)
            assert torch.equal(a0[rows], aj[rows]) and torch.equal(o0[rows], oj[rows]), j


# ----------------------------------------------------------------------------- whole model
MODELS = {"tiny": synth.shape("tiny"), "7b": synth.shape("mistral-7b", n_layers=2, vocab_size=4096)}
RANK = 16


def _model(p, slots, B, n_adapters=3, rank=RANK):
    """A model with `slots` slots on seeded weights, adapter j (seed 7 + j, an adapter term about as large as the base Linear's)
    in slot j for j < n_adapters; returns (model, base state dict, the adapters)."""
    args = mi.TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=2.0)))
    args.max_batch_size = B
    m = Transformer.empty(args, "cuda", torch.bfloat16, lora_slots=slots)
    sd = synth.synth_state_dict(p, 1, torch.bfloat16, "cuda")
    m.load_state_dict(sd)
    ads = [synth.synth_lora_state_dict(p, rank, 7 + j, torch.bfloat16, 0.5) for j in range(n_adapters)]
    for j, ad in enumerate(ads):
        m._load_lora_state_dict(ad, slot=j)
    return m.eval(), sd, ads


PROMPT_LENS = [19, 23, 17, 21, 18]
MIXED = [0, 1, 2, -1, 1]


def _prompts(p, lens=PROMPT_LENS):
    return [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate(lens)]


@pytest.mark.parametrize("name", list(MODELS))
@pytest.mark.parametrize("chunk", [None, 8])
def test_batch_invariance(name, chunk):
    """Each sequence of a mixed batch: the tokens and log-probabilities (prompt and decoded, the decode on the captured graph)
    of the batch in which every sequence uses its id, bit for bit."""
    p = MODELS[name]
    B = len(MIXED)
    m, _, _ = _model(p, 4, B)
    prompts = _prompts(p)
    gen = lambda ids: mi.generate(prompts, m, max_tokens=6, temperature=0.0, chunk_size=chunk, lora_ids=ids)  # noqa: E731
    toks, lps = gen(MIXED)
    uniform = {j: gen([j] * B) for j in set(MIXED)}
    for b, j in enumerate(MIXED):
        assert toks[b] == uniform[j][0][b], (b, j)
        assert lps[b] == uniform[j][1][b], (b, j)
    for j in (0, 1, 2):  # the adapters do change the output
        assert uniform[j][1] != uniform[-1][1]
    if chunk is None:  # a multi-slot model without ids is slot 0 everywhere
        assert mi.generate(prompts, m, max_tokens=6, temperature=0.0) == uniform[0]


def test_no_adapter_rows_are_the_base_model():
    p = MODELS["7b"]
    B = len(MIXED)
    m, sd, _ = _model(p, 4, B)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = B
    plain = Transformer.empty(args, "cuda", torch.bfloat16)
    plain.load_state_dict(sd)
    prompts = _prompts(p)
    assert mi.generate(prompts, m, max_tokens=6, temperature=0.0, lora_ids=[-1] * B) == \
        mi.generate(prompts, plain.eval(), max_tokens=6, temperature=0.0)


def _oracle_worst(toks, lps, o_toks, o_lps):
    worst = 0.0
    for tg, to, lg, lo in zip(toks, o_toks, lps, o_lps):  # logprobs agree up to the first diverging pick
        n = next((i for i, (a, b) in enumerate(zip(tg, to)) if a != b), len(tg))
        k = len(lo) - len(to) + n
        worst = max([worst] + [abs(a - b) for a, b in zip(lg[:k], lo[:k])])
    return worst


@pytest.mark.parametrize("chunk", [None, 8])
def test_mixed_batch_vs_oracle(chunk):
    p = MODELS["7b"]
    B = len(MIXED)
    m, sd, ads = _model(p, 4, B)
    prompts = _prompts(p)
    toks, lps = mi.generate(prompts, m, max_tokens=5, temperature=0.0, chunk_size=chunk, lora_ids=MIXED)
    sd_cpu = {k: v.cpu() for k, v in sd.items()}
    for j in sorted(set(MIXED)):
        mine = [b for b, i in enumerate(MIXED) if i == j]
        oa = oracle_args(p, len(mine))
        om = R.OracleTransformer(oa, sd_cpu) if j < 0 else OL.OracleLoraTransformer(oa, OL.lora_weights(sd_cpu, ads[j]), 2.0)
        o_toks, o_lps = R.generate([prompts[b] for b in mine], om, max_tokens=5, chunk_size=chunk)
        worst = _oracle_worst([toks[b] for b in mine], [lps[b] for b in mine], o_toks, o_lps)
        print(f"[parity] slot {j} vs oracle: logprob max|d|={worst:.4f}")
        assert worst <= LOGPROB_TOL, j


def _decode_run(m, prompts, steps, plan, graph, monkeypatch):
    """Prefill with plan[0]'s ids, then `steps` decode steps; plan[s] = (ids, action) for step s (action: a callable run before
    the step).  graph False: the same calls on the eager per-step path.  Returns every step's logits."""
    monkeypatch.setenv("MB200_DECODE_GRAPH", "1" if graph else "0")
    B = len(prompts)
    c = new_cache(m, 64)
    flat = torch.tensor(sum(prompts, []), device=DEV)
    logits = m.forward(flat, [len(x) for x in prompts], c, lora_ids=plan[0][0])
    nxt = logits[torch.tensor([len(x) for x in prompts]).cumsum(0) - 1].argmax(-1)
    outs = []
    for s in range(steps):
        ids, action = plan[s]
        if action is not None:
            action()
        out = m.forward(nxt, [1] * B, c, lora_ids=ids)
        outs.append(out.clone())
        nxt = out.argmax(-1)
    return outs


def test_ids_and_adapters_change_under_captured_graphs(monkeypatch):
    """On one cache, decode steps replayed from a captured graph see new lora_ids and a slot reloaded in place: every step's logits
    equal, bit for bit, the same sequence of calls on the eager per-step path."""
    p = MODELS["7b"]
    B = len(MIXED)
    m, _, ads = _model(p, 4, B)
    other = synth.synth_lora_state_dict(p, RANK, 99, torch.bfloat16, 0.5)
    prompts = _prompts(p)
    ids2 = [2, -1, 1, 0, 3]
    plan = [(MIXED, None)] * 4 + [(ids2, None)] * 2 + [(ids2, lambda: m._load_lora_state_dict(other, slot=1))] + [(ids2, None)] * 2
    runs = []
    for graph in (False, True):
        m._load_lora_state_dict(ads[1], slot=1)
        runs.append(_decode_run(m, prompts, len(plan), plan, graph, monkeypatch))
    for s, (a, b) in enumerate(zip(*runs)):
        assert torch.equal(a, b), s
    # and both changes took effect: against the same graph path without the id change, and without the reload
    m._load_lora_state_dict(ads[1], slot=1)
    keep = _decode_run(m, prompts, len(plan), [(MIXED, None)] * len(plan), True, monkeypatch)
    assert all(torch.equal(a, b) for a, b in zip(keep[:4], runs[1][:4])) and not torch.equal(keep[4], runs[1][4])
    no_reload = _decode_run(m, prompts, len(plan), [(MIXED, None)] * 4 + [(ids2, None)] * (len(plan) - 4), True, monkeypatch)
    assert all(torch.equal(a, b) for a, b in zip(no_reload[:6], runs[1][:6])) and not torch.equal(no_reload[6], runs[1][6])


def test_one_slot_without_ids_is_todays_path():
    """lora_slots=1 and no ids: the unmasked kernels, in prefill and batched decode; with ids the masked ones run."""
    p = MODELS["7b"]
    m, _, _ = _model(p, 1, 3, n_adapters=1)
    prompts = _prompts(p, [9, 11, 10])

    def run(ids):
        c = new_cache(m, 64)
        pre = launched_kernels(lambda: m.forward(torch.tensor(sum(prompts, []), device=DEV), [len(x) for x in prompts], c, lora_ids=ids))
        dec = launched_kernels(lambda: m.forward(torch.tensor([1, 2, 3], device=DEV), [1] * 3, c, lora_ids=ids))
        torch.cuda.synchronize()
        return pre, dec

    pre, dec = run(None)
    assert any(n.startswith("lora_down_kernel<") for n in pre) and not any("masked" in n for n in pre), pre
    assert "skinny_linear_kernel<3, 0, true>" in dec and not any(re.match(r"skinny_linear_kernel<\d, 64,", n) for n in dec), dec
    pre, dec = run([0, -1, 0])
    assert any(n.startswith("lora_down_masked_kernel<") for n in pre) and not any(n.startswith("lora_down_kernel<") for n in pre), pre
    assert "skinny_linear_kernel<3, 64, true>" in dec and "skinny_linear_kernel<3, 0, true>" not in dec, dec
