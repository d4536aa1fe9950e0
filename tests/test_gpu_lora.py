"""Un-merged LoRA adapters on the GPU: the three `_lora` entry points against the rounding chain bit for bit, zero adapters against
the plain model, the whole model against the oracle (oracle/lora.py), and adapter swaps under captured decode graphs.

Bit-exact inputs: x, A, B and W hold small integers (and the normed entry points see x = +-1, so RMSNorm gives exactly x * w with
integer w), so every fp32 accumulation is exact in any order and only the bf16 roundings of the chain
    a = bf16(xn A^T);  l = bf16(a B^T);  out = bf16(bf16(xn W^T) + bf16(l * scaling))
remain.  The expected values come from float64 products of the same integers, rounded at the same points.
"""
import re

import pytest
import torch
import torch.nn.functional as F

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.args import LoraArgs
from mistral_inference_b200.rope import precompute_freqs_cis
from mistral_inference_b200.transformer import Transformer
from mistral_inference_b200.transformer_layers import LoraAdapter
from oracle import lora as OL
from oracle import restatement as R

from .test_gpu_model import check_rows, new_cache, report
from .util import LOGPROB_TOL, assert_bf16_close, launched_kernels, logit_tol, oracle_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
SHAPES = {"7b": (4096, 32, 8, 14336), "nemo": (5120, 32, 8, 14336)}  # dim, H, KV, hidden (Nemo: H * hd = 4096 != dim)
T_LIST = [1, 3, 4, 5, 32, 64, 127, 128, 129, 512, 4096]
RANKS = [8, 16, 64, 128]
SCALINGS = [2.0, 0.3]


def ints(*shape, lo=-1, hi=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, shape, generator=g).to(torch.bfloat16).to(DEV)


def bf(x64: torch.Tensor) -> torch.Tensor:
    """float64 holding an exact integer sum -> the bf16 rounding of its fp32 value."""
    return x64.float().to(torch.bfloat16)


def adapter(in_f, segments, r, scaling, seed, interleaved=False):
    ad = LoraAdapter(in_f, segments, LoraArgs(r, scaling), interleaved=interleaved).to(DEV, torch.bfloat16)
    A = [ints(r, in_f, seed=seed + s) for s in range(len(segments))]
    B = [ints(n, r, seed=seed + 10 + s) for s, n in enumerate(segments)]
    for s in range(len(segments)):
        ad.put_A(s, A[s])
        ad.put_B(s, B[s])
    return ad, A, B


def chain(xn, W, A, B, scaling):
    """(a per segment, l per segment, out) of LoRALinear.forward for one segment."""
    a = bf(xn.double() @ A.double().T)
    l = bf(a.double() @ B.double().T)
    s = (l.float() * scaling).to(torch.bfloat16)
    y = bf(xn.double() @ W.double().T)
    return a, l, (y.float() + s.float()).to(torch.bfloat16)


def cases():
    out = []
    for i, T in enumerate(T_LIST):
        for shape in SHAPES:
            out.append((shape, T, RANKS[i % 4], SCALINGS[(i + (shape == "nemo")) % 2]))
    return out


def _check_launches(names, mode, T, normed):
    """T > 4: one split-K down kernel (plus its reduce when it split), no GEMV; T <= 4: the down projection is the skinny
    EPI_STORE GEMV (norm fused when the call norms), the up projection a second EPI_STORE GEMV.  Then exactly one base GEMM with
    the LoRA flag."""
    pat = re.compile(rf"(gemm_\w+_kernel<{mode | 16}[,>]|skinny_linear_kernel<\d, {mode | 16},)")
    assert sum(bool(pat.search(n)) for n in names) == 1, names
    down = [n for n in names if n.startswith("lora_down_kernel<")]
    store_gemv = [n for n in names if re.match(r"skinny_linear_kernel<\d, 0, (true|false)>", n)]
    if T > 4:
        assert len(down) == 1 and not [n for n in names if n.startswith("skinny")], names
        splits = int(down[0][len("lora_down_kernel<"):-1])
        assert names.count("lora_down_reduce_kernel") == (1 if splits > 1 else 0), names
    else:
        assert not down and "lora_down_reduce_kernel" not in names, names
        assert store_gemv == [f"skinny_linear_kernel<{T}, 0, {'true' if normed else 'false'}>", f"skinny_linear_kernel<{T}, 0, false>"], names


def _normed_input(T, dim, seed):
    x = ints(T, dim, seed=seed)
    x = torch.where(x == 0, torch.ones_like(x), x)  # +-1: mean(x^2) = 1, so bf16(x * rsqrt(1 + eps)) = x
    nw = ints(dim, lo=1, hi=2, seed=seed + 1)
    return x, nw, x * nw


@pytest.mark.parametrize("shape,T,r,scaling", cases())
def test_qkv_lora_chain_bit_exact(shape, T, r, scaling):
    dim, H, KV, _ = SHAPES[shape]
    hd = 128
    x, nw, xn = _normed_input(T, dim, 1)
    Ws = [ints(H * hd, dim, seed=3), ints(KV * hd, dim, seed=4), ints(KV * hd, dim, seed=5)]
    ad, A, B = adapter(dim, [H * hd, KV * hd, KV * hd], r, scaling, 20)
    table = precompute_freqs_cis(hd, 8192, 1e6)
    positions = (torch.arange(T, dtype=torch.int32) * 7) % 8000
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, H, KV, hd, 14336, 0, 4), torch.device(DEV))
    q = torch.empty(T, H * hd, dtype=torch.bfloat16, device=DEV)
    k = torch.empty(T, KV * hd, dtype=torch.bfloat16, device=DEV)
    v = torch.empty_like(k)
    scatter = T % 2 == 1
    n_rows = max(T, 8)
    ck = torch.zeros(n_rows, KV * hd, dtype=torch.bfloat16, device=DEV) if scatter else None
    cv = torch.zeros_like(ck) if scatter else None
    rows = torch.arange(T, dtype=torch.int32, device=DEV).flip(0) if scatter else None
    st = ad.call(T)
    names = launched_kernels(lambda: _abi.attn_qkv_lora(x, nw, torch.cat(Ws), torch.view_as_real(table).contiguous().to(DEV), positions.to(DEV),
                                                        q, k, v, ck, cv, rows, H, KV, hd, 1e-5, ws, st))
    torch.cuda.synchronize()
    _check_launches(names, 4, T, True)
    a_buf, l_buf = st.keep
    outs = [chain(xn, W, A[s], B[s], scaling) for s, W in enumerate(Ws)]
    a_want = torch.zeros(T, ad.rank_cols, dtype=torch.bfloat16, device=DEV)
    a_want[:, :3 * r] = torch.cat([o[0] for o in outs], 1)
    assert torch.equal(a_buf, a_want)
    assert torch.equal(l_buf, torch.cat([o[1] for o in outs], 1))
    q_ref, k_ref = R.apply_rope(outs[0][2].cpu().view(T, H, hd), outs[1][2].cpu().view(T, KV, hd), table[positions.long()])
    assert torch.equal(q.cpu(), q_ref.reshape(T, -1))
    assert torch.equal(k.cpu(), k_ref.reshape(T, -1))
    assert torch.equal(v, outs[2][2])
    if scatter:
        assert torch.equal(ck[rows.long()], k) and torch.equal(cv[rows.long()], v)


@pytest.mark.parametrize("shape,T,r,scaling", cases())
def test_gateup_lora_chain_bit_exact(shape, T, r, scaling):
    dim, _, _, hidden = SHAPES[shape]
    x, nw, xn = _normed_input(T, dim, 2)
    W1, W3 = ints(hidden, dim, seed=6), ints(hidden, dim, seed=7)
    ad, A, B = adapter(dim, [hidden, hidden], r, scaling, 40, interleaved=True)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 32, 8, 128, hidden, 0, 4), torch.device(DEV))
    g = torch.empty(T, hidden, dtype=torch.bfloat16, device=DEV)
    w13 = torch.stack([W1, W3], 1).reshape(2 * hidden, dim)
    st = ad.call(T)
    names = launched_kernels(lambda: _abi.ffn_gateup_lora(x, nw, w13, g, 1e-5, ws, st))
    torch.cuda.synchronize()
    _check_launches(names, 3, T, True)
    a1, l1, o1 = chain(xn, W1, A[0], B[0], scaling)
    a3, l3, o3 = chain(xn, W3, A[1], B[1], scaling)
    a_buf, l_buf = st.keep
    assert torch.equal(a_buf[:, :2 * r], torch.cat([a1, a3], 1)) and not a_buf[:, 2 * r:].any()
    assert torch.equal(l_buf, torch.stack([l1, l3], 2).reshape(T, 2 * hidden))
    want = (F.silu(o1.float()).to(torch.bfloat16).float() * o3.float()).to(torch.bfloat16)
    assert torch.equal(g, want)


@pytest.mark.parametrize("which", ["wo", "w2"])
@pytest.mark.parametrize("shape,T,r,scaling", cases())
def test_linear_residual_lora_chain_bit_exact(which, shape, T, r, scaling):
    dim, H, _, hidden = SHAPES[shape]
    K = H * 128 if which == "wo" else hidden
    x = ints(T, K, seed=8)
    W = ints(dim, K, seed=9)
    res = ints(T, dim, lo=-4, hi=4, seed=10)
    ad, A, B = adapter(K, [dim], r, scaling, 60)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 32, 8, 128, hidden, 0, 4), torch.device(DEV))
    out = torch.empty(T, dim, dtype=torch.bfloat16, device=DEV)
    st = ad.call(T)
    names = launched_kernels(lambda: _abi.linear_residual_lora(x, W, res, out, ws, st))
    torch.cuda.synchronize()
    _check_launches(names, 1, T, False)
    a, l, o = chain(x, W, A[0], B[0], scaling)
    a_buf, l_buf = st.keep
    assert torch.equal(a_buf[:, :r], a) and torch.equal(l_buf, l)
    assert torch.equal(out, (o.float() + res.float()).to(torch.bfloat16))


@pytest.mark.parametrize("T", [512, 4096])
def test_down_projection_deterministic(T):
    """The split-K down projection on random (non-integer) inputs, where a different split or summation order would change the
    fp32 sums: two runs give the same bits, and the K split really happened."""
    K, N, r = 14336, 4096, 64
    g = torch.Generator().manual_seed(T)
    x = torch.randn(T, K, generator=g).to(torch.bfloat16).to(DEV)
    W = (torch.randn(N, K, generator=g) * K ** -0.5).to(torch.bfloat16).to(DEV)
    ad = LoraAdapter(K, [N], LoraArgs(r, 2.0)).to(DEV, torch.bfloat16)
    ad.put_A(0, (torch.randn(r, K, generator=g) * K ** -0.5).to(torch.bfloat16).to(DEV))
    ad.put_B(0, (torch.randn(N, r, generator=g) * r ** -0.5).to(torch.bfloat16).to(DEV))
    ws = _abi.Workspace(_abi.workspace_bytes(T, N, 32, 8, 128, K, 0, 4), torch.device(DEV))
    out = torch.empty(T, N, dtype=torch.bfloat16, device=DEV)
    runs = []
    for _ in range(2):
        st = ad.call(T)
        names = launched_kernels(lambda: _abi.linear_residual_lora(x, W, None, out, ws, st))
        torch.cuda.synchronize()
        runs.append((st.keep[0].clone(), out.clone()))
    down = [n for n in names if n.startswith("lora_down_kernel<")]
    assert len(down) == 1 and int(down[0][len("lora_down_kernel<"):-1]) > 1, names
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])
    a64 = x.double() @ ad.lora_A(0).double().T  # and the sums are right to fp32-reordering noise
    assert_bf16_close(runs[0][0], a64.float(), what="a")


# ----------------------------------------------------------------------------- whole model
def _models(p, rank, scaling, max_batch, adapter_seed=None, scale=1.0):
    """(LoRA model, oracle) on the same weights; adapter_seed None = zero adapters."""
    args = mi.TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=scaling)))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16)
    sd = synth.synth_state_dict(p, 1, torch.bfloat16, "cuda")
    m.load_state_dict(sd)
    ad = {}
    if adapter_seed is not None:
        ad = synth.synth_lora_state_dict(p, rank, adapter_seed, torch.bfloat16, scale, "cuda")
        m._load_lora_state_dict(ad)
    om = OL.OracleLoraTransformer(oracle_args(p, max_batch), OL.lora_weights({k: v.cpu() for k, v in sd.items()},
                                                                             {k: v.cpu() for k, v in ad.items()} or
                                                                             synth.synth_lora_state_dict(p, rank, 0, torch.bfloat16, 0.0)), scaling)
    return m.eval(), om


def _plain(p, max_batch):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16)
    m.load_state_dict(synth.synth_state_dict(p, 1, torch.bfloat16, "cuda"))
    return m.eval()


@pytest.mark.parametrize("B", [1, 8])
def test_zero_adapters_equal_plain_model(B, monkeypatch):
    monkeypatch.setenv("MB200_MEGAKERNEL", "0")  # the LoRA model never takes the megakernel: compare like with like
    p = synth.shape("mistral-7b", n_layers=2, vocab_size=4096)
    lm, _ = _models(p, 16, 2.0, B)
    pm = _plain(p, B)
    prompts = [synth.synth_prompt(37 + 3 * i, p["vocab_size"], 70 + i) for i in range(B)]
    flat = torch.tensor(sum(prompts, []), device=DEV)
    sl = [len(x) for x in prompts]
    assert torch.equal(lm.forward(flat, sl), pm.forward(flat, sl))  # cache-less
    outs = []
    for m in (lm, pm):
        c = new_cache(m, 128)
        first, rest = [x[:20] for x in prompts], [x[20:] for x in prompts]
        got = [m.forward(torch.tensor(sum(first, []), device=DEV), [20] * B, c)]  # first prefill
        got.append(m.forward(torch.tensor(sum(rest, []), device=DEV), [len(x) for x in rest], c))  # chunked prefill
        nxt = torch.tensor([x[0] for x in prompts], device=DEV)
        for _ in range(3):  # graph decode: warm-up, capture, replay
            got.append(m.forward(nxt, [1] * B, c).clone())
        outs.append(got)
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("shape,over,lens,chunk", [
    ("mistral-7b", {"n_layers": 2, "vocab_size": 4096}, [19, 23, 17, 21, 18, 22, 20, 17], 8),
    ("mistral-nemo-12b", {"n_layers": 1, "vocab_size": 4096}, [33], None),
])
def test_model_vs_oracle(shape, over, lens, chunk):
    p = synth.shape(shape, **over)
    B, max_tokens = len(lens), 5
    m, om = _models(p, 16, 2.0, B, adapter_seed=7, scale=0.5)  # an adapter term about as large as the base Linear's
    prompts = [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate(lens)]
    # the adapters move the logits well beyond the tolerance
    flat = torch.tensor(sum(prompts, []))
    with torch.inference_mode():
        plain = R.OracleTransformer(oracle_args(p, B), {k: v for k, v in om.w.items()}).forward(flat, lens)
        want0 = om.forward(flat, lens)
    assert (plain - want0).abs().max() > 4 * logit_tol(want0)
    d = report(f"{shape} cache-less", m.forward(flat.cuda(), lens), want0)
    check_rows(d, want0, what=f"{shape} cache-less")
    o_toks, o_lp, o_step = R.generate(prompts, om, max_tokens=max_tokens, chunk_size=chunk, return_logits=True)
    cache, ocache = new_cache(m, max(lens) + max_tokens), om.new_cache(max(lens) + max_tokens)
    last = None
    for s in range(0, max(lens), chunk or max(lens)):
        chunks = [pr[s:s + (chunk or max(lens))] for pr in prompts]
        sl = [len(c) for c in chunks]
        flat = torch.tensor(sum(chunks, []))
        logits = m.forward(flat.cuda(), sl, cache)
        want = om.forward(flat, sl, ocache)
        check_rows(report(f"{shape} prefill @{s}", logits, want), want, what=f"{shape} prefill @{s}")
        last = logits[torch.tensor(sl).cumsum(0) - 1]
    for step in range(max_tokens):
        check_rows(report(f"{shape} step {step}", last, o_step[step]), o_step[step], what=f"{shape} step {step}")
        top2 = o_step[step].topk(2, dim=-1).values
        decisive = (top2[:, 0] - top2[:, 1]) > 2 * logit_tol(o_step[step])
        assert torch.equal(last.argmax(-1).cpu()[decisive], torch.tensor([t[step] for t in o_toks])[decisive])
        nxt = torch.tensor([t[step] for t in o_toks])
        last = m.forward(nxt.cuda(), [1] * B, cache)
        om.forward(nxt, [1] * B, ocache)
    # the reference's property through generate(): decode logprobs == re-prefill logprobs
    toks, lp = mi.generate(prompts, m, max_tokens=max_tokens, temperature=0.0)
    full = [pr + t for pr, t in zip(prompts, toks)]
    _, lp2 = mi.generate(full, m, max_tokens=0, temperature=0.0)
    assert max(abs(a - b) for x, y in zip(lp, lp2) for a, b in zip(x, y)) <= LOGPROB_TOL


def test_adapter_swap_under_captured_graphs(tmp_path):
    import safetensors.torch

    p = synth.shape("mistral-7b", n_layers=2, vocab_size=4096)
    synth.write_model_folder(tmp_path, p, seed=1, lora=dict(rank=16, scaling=2.0))
    m = Transformer.from_folder(tmp_path, max_batch_size=8, device="cuda")
    ad_a = synth.synth_lora_state_dict(p, 16, 7, torch.bfloat16, 2.0)
    ad_b = synth.synth_lora_state_dict(p, 16, 8, torch.bfloat16, 2.0)
    safetensors.torch.save_file(ad_a, str(tmp_path / "a.safetensors"))
    safetensors.torch.save_file(ad_b, str(tmp_path / "b.safetensors"))
    prompts = [synth.synth_prompt(12 + i, p["vocab_size"], 90 + i) for i in range(8)]
    runs = []
    for name in ("a", "b", "a"):
        m.load_lora(tmp_path / f"{name}.safetensors", scaling=123.0)  # ignored
        for B in (1, 8):
            runs.append(mi.generate(prompts[:B], m, max_tokens=6, temperature=0.0))
    assert runs[0] == runs[4] and runs[1] == runs[5]
    assert runs[2] != runs[0]
    om = OL.OracleLoraTransformer(oracle_args(p, 8), OL.lora_weights(synth.synth_state_dict(p, 1), ad_b), 2.0)
    o_toks, o_lp = R.generate(prompts, om, max_tokens=6)
    worst = 0.0
    for tg, to, lg, lo in zip(runs[3][0], o_toks, runs[3][1], o_lp):  # logprobs agree up to the first diverging pick
        n = next((i for i, (a, b) in enumerate(zip(tg, to)) if a != b), len(tg))
        m_ = len(lo) - len(to) + n
        worst = max([worst] + [abs(a - b) for a, b in zip(lg[:m_], lo[:m_])])
    print(f"[parity] adapter B vs oracle: logprob max|d|={worst:.4f}")
    assert worst <= LOGPROB_TOL
