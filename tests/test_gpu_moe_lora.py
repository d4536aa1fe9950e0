"""Un-merged LoRA on FP8 experts on the GPU (csrc/lora.cuh grouped down projection, csrc/moe.cuh, mb200_moe_grouped_ffn_fp8_lora).

Kernel level, bit for bit.  Inputs make every fp32 sum of the chain exact, so only the chain's bf16 roundings remain, and the
expected values are float64 products rounded at the same points (tests/test_gpu_moe_edges.py's `bf16r`, extended to bf16's
subnormals, and `certain`):
  w13 stage  hn, A13, B13 small integers; W13 rows small integers with one +-448 entry (FP8 scale 1, so W' = W exactly)
  w2 stage   W2, A2, B2 rows with a single nonzero entry (+-448, small integers), so every sum over g is one product
The SiLU inside g is certified in float64 (`certain`); each later stage is checked on the kernel's own input read back from the
buffers, so a failure names its stage.
Model level: zero adapters equal the plain FP8 model; an adapted model follows OracleLoraTransformer on the W' checkpoint;
adapter swaps under captured decode graphs; from_folder's peak; expert parallelism; a speculative draft."""
import ctypes
import os
import socket
import sys
from pathlib import Path

import pytest
import torch
import torch.multiprocessing as mp

import mistral_inference_b200 as mi
import synth
from mistral_inference_b200 import _abi
from mistral_inference_b200.cache import BufferCache
from mistral_inference_b200.moe import MoeBuffers
from mistral_inference_b200.transformer import Transformer
from oracle import fp8 as F8
from oracle import lora as OL
from oracle import moe_lora as OM
from oracle import restatement as R

from .test_gpu_moe_edges import assert_same, bf16r, certain
from .util import launched_kernels, oracle_args

pytestmark = pytest.mark.gpu
DEV = "cuda"
REPO = Path(__file__).resolve().parents[1]


def bf16s(v: torch.Tensor) -> torch.Tensor:
    """bf16r extended to bf16's subnormal range (multiples of 2^-133), as the device's fp32 -> bf16 conversion rounds: small routing
    weights times small expert outputs land there."""
    return torch.where(v.abs() < 2.0 ** -126, torch.round(v * 2.0 ** 133) / 2.0 ** 133, bf16r(v))


def table(vals):
    t = (ctypes.c_void_p * len(vals))()
    for i, v in enumerate(vals):
        t[i] = v.data_ptr() if v is not None else None
    return t


def ints(g, shape, lim):
    return torch.randint(-lim, lim + 1, shape, generator=g, device=DEV).double()


def one_per_row(g, rows, cols, vals):
    """[rows, cols] float64 with one entry per row, drawn from `vals`, at a random column."""
    out = torch.zeros(rows, cols, dtype=torch.float64, device=DEV)
    v = torch.tensor(vals, dtype=torch.float64, device=DEV)[torch.randint(0, len(vals), (rows,), generator=g, device=DEV)]
    out[torch.arange(rows, device=DEV), torch.randint(0, cols, (rows,), generator=g, device=DEV)] = v
    return out


def fp8_exact(w):
    """e4m3 q and scales of a float64 matrix whose rows each hold +-448 (scale 1, so W' == W); asserts the round trip."""
    wb = w.to(torch.bfloat16)
    q, s = torch.empty(w.shape, dtype=torch.uint8, device=DEV), torch.empty(w.shape[0], device=DEV)
    _abi.quantize_e4m3_rows(wb, q, s)
    assert torch.equal(s, torch.ones_like(s)) and torch.equal(F8.dequantize_rows(q, s).double(), w)
    return q, s


def make_experts(E, D, H, r, seed, shard):
    R13, R2 = -(-2 * r // 64) * 64, -(-r // 64) * 64
    ex = []
    for e in range(E):
        if e % shard[1] != shard[0]:
            ex.append(None)
            continue
        g = torch.Generator(device=DEV).manual_seed(seed * 131 + e)
        w13 = ints(g, (2 * H, D), 3)
        w13[torch.arange(2 * H, device=DEV), torch.randint(0, D, (2 * H,), generator=g, device=DEV)] = 448.0 * (
            torch.randint(0, 2, (2 * H,), generator=g, device=DEV).double() * 2 - 1)
        w2 = one_per_row(g, D, H, (448.0, -448.0))
        a13 = torch.zeros(R13, D, dtype=torch.float64, device=DEV)
        a13[: 2 * r] = ints(g, (2 * r, D), 2)
        b13 = torch.zeros(2 * H, R13, dtype=torch.float64, device=DEV)  # interleaved rows: w1 rows 2i use cols [0, r), w3 rows [r, 2r)
        b13[0::2, :r] = ints(g, (H, r), 2)
        b13[1::2, r: 2 * r] = ints(g, (H, r), 2)
        a2 = torch.zeros(R2, H, dtype=torch.float64, device=DEV)
        a2[:r] = one_per_row(g, r, H, (1.0, -2.0, 0.5))
        b2 = torch.zeros(D, R2, dtype=torch.float64, device=DEV)
        b2[:, :r] = one_per_row(g, D, r, (1.0, -1.0, 2.0))
        q13, s13 = fp8_exact(w13)
        q2, s2 = fp8_exact(w2)
        bf = lambda t: t.to(torch.bfloat16).contiguous()  # noqa: E731
        ex.append(dict(w13=w13, w2=w2, a13=a13, b13=b13, a2=a2, b2=b2, q13=q13, s13=s13, q2=q2, s2=s2,
                       A13=bf(a13), B13=bf(b13), A2=bf(a2), B2=bf(b2)))
    return ex, R13, R2


def run_lora_ffn(T, E, k, D, H, r, seed, shard=(0, 1), scaling=2.0, env=None, runs=1):
    ex, R13, R2 = make_experts(E, D, H, r, seed, shard)
    g = torch.Generator(device=DEV).manual_seed(seed)
    hn = ints(g, (T, D), 2).to(torch.bfloat16)
    res = ints(g, (T, D), 4).to(torch.bfloat16)
    gate = ints(g, (E, D), 3).to(torch.bfloat16)
    ws = _abi.Workspace(_abi.workspace_bytes(T, D, 1, 1, 128, H, 0, 1), torch.device(DEV))
    b = MoeBuffers(T, D, H, E, k, torch.device(DEV), torch.bfloat16)
    _abi.moe_route(hn, gate, E, k, shard[0], shard[1], b)
    col = lambda n: table([x[n] if x is not None else None for x in ex])  # noqa: E731
    bufs = dict(a13=torch.empty(b.rows_cap, R13, dtype=torch.bfloat16, device=DEV), l13=torch.empty(b.rows_cap, 2 * H, dtype=torch.bfloat16, device=DEV),
                a2=torch.empty(b.rows_cap, R2, dtype=torch.bfloat16, device=DEV), l2=torch.empty(b.rows_cap, D, dtype=torch.bfloat16, device=DEV))
    tabs = [col(n) for n in ("q13", "s13", "q2", "s2", "A13", "B13", "A2", "B2")]
    l13 = _abi.moe_lora_struct(tabs[4], tabs[5], R13, scaling, bufs["a13"], bufs["l13"])
    l2 = _abi.moe_lora_struct(tabs[6], tabs[7], R2, scaling, bufs["a2"], bufs["l2"])
    outs, logs = [], []
    old = {key: os.environ.get(key) for key in (env or {})}
    os.environ.update(env or {})
    try:
        for _ in range(runs):
            for t in list(bufs.values()) + [b.g, b.yw]:
                t.fill_(float("nan"))
            out = torch.full((T, D), float("nan"), dtype=torch.bfloat16, device=DEV)
            logs.append(launched_kernels(lambda: _abi.moe_grouped_ffn_fp8_lora(b, *tabs[:4], res, out, T, D, H, E, k, None, ws, l13, l2)))
            torch.cuda.synchronize()
            outs.append({**{n: t.clone() for n, t in bufs.items()}, "g": b.g.clone(), "yw": b.yw.clone(), "out": out})
    finally:
        for key, v in old.items():
            if v is None:
                os.environ.pop(key, None)
            else:
                os.environ[key] = v
    return ex, b, hn, res, outs, logs, scaling


def check_chain(T, E, k, shard, ex, b, res, o, scaling):
    """Every stage of the chain, on the rows of this rank's experts."""
    sel, slot = b.sel.view(T, k).long(), b.slot.view(T, k).long()
    mine = (sel % shard[1]) == shard[0]
    H = ex[next(e for e in range(E) if ex[e] is not None)]["w2"].shape[1]
    xs = b.xs.double()
    for e in range(E):
        if ex[e] is None:
            continue
        rows = slot[sel == e]
        if rows.numel() == 0:
            continue
        P = ex[e]
        x = xs[rows]
        a13 = bf16s(x @ P["a13"].T)
        assert_same(o["a13"][rows], a13, f"expert {e}: a13")
        L13 = bf16s(o["a13"][rows].double() @ P["b13"].T)
        assert_same(o["l13"][rows], L13, f"expert {e}: L13")
        y = bf16s(bf16s(x @ P["w13"].T) + bf16s(o["l13"][rows].double() * scaling))
        y0, y1 = y[:, 0::2], y[:, 1::2]
        s = y0 / (1 + torch.exp(-y0))
        ok = certain(s)  # (bf16(s) * y1 is an exact fp32 product: its rounding needs no certificate)
        want_g = bf16s(bf16s(s) * y1)
        got_g = o["g"][rows].double()
        # far below y0 = -16 silu(y0) underflows (fp32 expf overflows to inf), where `certain` makes no claim; the w2 stage below
        # takes the kernel's own g either way
        assert ok[y0 >= -16].float().mean().item() > 0.95
        assert_same(got_g[ok], want_g[ok], f"expert {e}: g")
        gk = got_g
        a2 = bf16s(gk @ P["a2"].T)
        assert_same(o["a2"][rows], a2, f"expert {e}: a2")
        L2 = bf16s(o["a2"][rows].double() @ P["b2"].T)
        assert_same(o["l2"][rows], L2, f"expert {e}: L2")
        w = b.row_w[rows].double()[:, None]
        yw = bf16s(w * bf16s(bf16s(gk @ P["w2"].T) + bf16s(o["l2"][rows].double() * scaling)))
        assert_same(o["yw"][rows], yw, f"expert {e}: yw")
    if shard[1] == 1:
        yw = o["yw"].double()
        acc = yw[slot[:, 0]]
        for j in range(1, k):
            acc = bf16s(acc + yw[slot[:, j]])
        assert_same(o["out"], bf16s(res.double() + acc), "out")
    assert mine.any()


CASES = [  # (T, E, k, r, env)
    (1, 8, 2, 16, {}), (2, 4, 1, 8, {}), (4, 16, 4, 64, {}), (5, 2, 2, 128, {}), (31, 8, 3, 16, {}), (32, 8, 2, 64, {}),
    (33, 16, 4, 8, {}), (64, 4, 2, 16, {}), (65, 8, 2, 128, {}), (128, 2, 1, 64, {}), (129, 8, 4, 16, {}), (512, 16, 2, 64, {}),
    (4096, 8, 2, 16, {}),
    (8, 8, 2, 16, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "256"}), (8, 8, 2, 64, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "128"}),
    (8, 4, 2, 8, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "64"}), (8, 4, 2, 128, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "32"}),
    (40, 8, 2, 16, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "256"}), (40, 8, 2, 64, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "128"}),
    (40, 2, 1, 16, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "64"}), (40, 16, 4, 8, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "32"}),
    (40, 8, 2, 16, {}), (300, 4, 2, 64, {"MB200_GEMM_CLUSTER": "0"}),
]


@pytest.mark.parametrize("T,E,k,r,env", CASES, ids=[f"T{c[0]}-E{c[1]}-k{c[2]}-r{c[3]}-{'-'.join(f'{a[5:]}{b}' for a, b in c[4].items()) or 'auto'}"
                                                    for c in CASES])
def test_grouped_ffn_fp8_lora_chain(T, E, k, r, env):
    D, H = 1024, 1536  # deep enough for the down projection to split K (at least 4 k-blocks per split)
    ex, b, hn, res, outs, logs, scaling = run_lora_ffn(T, E, k, D, H, r, seed=T * 31 + E + r, env=env, runs=2)
    check_chain(T, E, k, (0, 1), ex, b, res, outs[0], scaling)
    for n in outs[0]:  # the split-K sum is in a fixed order: the same bits on every run
        assert torch.equal(outs[0][n].view(torch.int16), outs[1][n].view(torch.int16)), n
    log = logs[0]
    down = [n for n in log if n.startswith("lora_down_grouped_kernel<")]
    assert len(down) == 2, log
    splits = [int(n[len("lora_down_grouped_kernel<"):-1]) for n in down]
    assert log.count("lora_down_reduce_kernel") == sum(s > 1 for s in splits), log
    grouped = [n for n in log if "grouped" in n and "lora_down" not in n]
    base = [n for n in grouped if "_fp8_kernel" in n]
    up = [n for n in grouped if "_fp8_kernel" not in n]
    assert len(base) == 2 and len(up) == 2, log
    assert base[0].split("<")[1].startswith("19,") and base[1].split("<")[1].startswith("21,"), base  # EPI_SWIGLU|EPI_LORA, EPI_MOE_SCALE|EPI_LORA
    assert all(n.split("<")[1].startswith("0,") for n in up), up  # EPI_STORE on the bf16 B tables
    if env.get("MB200_STREAMK") == "0":
        assert not any("streamk" in n for n in grouped), grouped
        if env.get("MB200_GEMM_BN"):
            assert all(f", {env['MB200_GEMM_BN']}, " in n for n in base), base
    elif T <= 64:
        assert all("streamk" in n for n in grouped), grouped
    if T <= 4:
        assert all(s > 1 for s in splits), splits  # decode-sized calls fill the SMs through the split


@pytest.mark.parametrize("T,k", [(1, 2), (48, 2), (300, 3)])
def test_grouped_ffn_fp8_lora_shard_with_null_experts(T, k):
    E, D, H = 8, 1024, 1536
    ex, b, hn, res, outs, logs, scaling = run_lora_ffn(T, E, k, D, H, 16, seed=T + 3, shard=(1, 2))
    check_chain(T, E, k, (1, 2), ex, b, res, outs[0], scaling)


# ----------------------------------------------------------------------------- models
def lora_args(p, rank, scaling, max_batch):
    a = mi.TransformerArgs.from_dict(dict(p, lora=dict(rank=rank, scaling=scaling)))
    a.max_batch_size = max_batch
    return a


def plain_model(p, sd, max_batch):
    a = mi.TransformerArgs.from_dict(dict(p))
    a.max_batch_size = max_batch
    m = Transformer.empty(a, DEV, torch.bfloat16, expert_weights="fp8")
    m.load_state_dict(sd)
    return m.eval()


def lora_model(p, sd, max_batch, rank=4, scaling=2.0, adapter=None):
    m = Transformer.empty(lora_args(p, rank, scaling, max_batch), DEV, torch.bfloat16, expert_weights="fp8")
    m.load_state_dict(sd)
    if adapter is not None:
        m._load_lora_state_dict(adapter)
    return m.eval()


def run_model(m, p, batch1: bool, steps: int = 4):
    outs = []
    if batch1:
        cache = BufferCache(m.n_local_layers, 1, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
        toks = torch.tensor(synth.synth_prompt(21, p["vocab_size"], 9), device=DEV)
        outs.append(m.forward(toks[:13], [13], cache))
        outs.append(m.forward(toks[13:], [8], cache))  # chunked prefill
        nxt = outs[-1][-1:].argmax(-1)
        for _ in range(steps):  # eager warm-up, graph capture, replays
            lg = m.forward(nxt, [1], cache)
            outs.append(lg)
            nxt = lg.argmax(-1)
        return torch.cat(outs).cpu()
    cache = BufferCache(m.n_local_layers, 2, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
    seqlens = [37, 150]
    toks = torch.tensor(synth.synth_prompt(sum(seqlens), p["vocab_size"], 4), device=DEV)
    outs.append(m.forward(toks, seqlens, cache))
    nxt = torch.tensor([5, 7], device=DEV)
    for _ in range(steps):
        lg = m.forward(nxt, [1, 1], cache)
        outs.append(lg)
        nxt = lg.argmax(-1)
    return torch.cat(outs).cpu()


@pytest.mark.parametrize("shape", ["tiny-moe", "mixtral-8x7b-2layers"])
def test_zero_adapters_equal_the_plain_fp8_model(shape):
    if shape == "tiny-moe":
        p = synth.shape("tiny-moe", sliding_window=64)
    else:
        p = synth.shape("mixtral-8x7b", n_layers=2, vocab_size=4096)
    sd = synth.synth_state_dict(p, 2, torch.bfloat16, DEV)
    m, ml = plain_model(p, sd, 2), lora_model(p, sd, 2, rank=16)
    del sd
    for batch1 in (False, True):
        want, got = run_model(m, p, batch1), run_model(ml, p, batch1)
        assert torch.equal(got, want), f"batch1={batch1}: max |diff| {(got - want).abs().max().item()}"  # (== holds +0 == -0)
    log = launched_kernels(lambda: ml.forward(torch.tensor([1, 2, 3], device=DEV), [3]))
    assert any(n.startswith("gemm_streamk_grouped_fp8_kernel<19,") for n in log) and any(n.startswith("lora_down_grouped_kernel<") for n in log), log
    if shape == "tiny-moe":
        prompts = [synth.synth_prompt(n, p["vocab_size"], s) for n, s in ((25, 1), (30, 2))]
        assert mi.generate(prompts, ml, max_tokens=10, temperature=0.0, chunk_size=6) == \
            mi.generate(prompts, m, max_tokens=10, temperature=0.0, chunk_size=6)


def _teacher_forced(m_oracle, prompts, toks, lps, tol):
    full = [pr + t for pr, t in zip(prompts, toks)]
    _, o_lp = R.generate(full, m_oracle, max_tokens=0, chunk_size=None)
    worst = max(abs(a - b) for x, y in zip(lps, o_lp) for a, b in zip(x, y))
    assert worst <= tol, worst
    return worst


def _adapted(p, rank, scaling, max_batch, seed=7):
    sd = synth.synth_state_dict(p, 3)
    ad = OM.synth_moe_lora_state_dict(p, rank, seed, scale=0.5)
    m = lora_model(p, {k: v.to(DEV) for k, v in sd.items()}, max_batch, rank, scaling, ad)
    oracle = OL.OracleLoraTransformer(oracle_args(p, max_batch), OM.moe_lora_weights(F8.fp8_checkpoint(sd), ad), scaling)
    return m, oracle, sd, ad


@pytest.mark.parametrize("lens", [[29], [29, 25, 31]])
def test_adapted_model_vs_oracle_on_dequantised_checkpoint(lens):
    p = synth.shape("tiny-moe", sliding_window=64)
    m, oracle, sd, _ = _adapted(p, 8, 2.0, len(lens))
    prompts = [synth.synth_prompt(n, p["vocab_size"], 70 + i) for i, n in enumerate(lens)]
    toks, lps = mi.generate(prompts, m, max_tokens=10, temperature=0.0, chunk_size=8)
    _teacher_forced(oracle, prompts, toks, lps, 0.05)
    plain_toks, _ = mi.generate(prompts, plain_model(p, {k: v.to(DEV) for k, v in sd.items()}, len(lens)), max_tokens=10, temperature=0.0,
                                chunk_size=8)
    assert plain_toks != toks  # the adapters change the generation


def test_adapter_swap_under_captured_decode_graphs():
    p = synth.shape("tiny-moe", sliding_window=64)
    sd = {k: v.to(DEV) for k, v in synth.synth_state_dict(p, 3).items()}
    a, b = OM.synth_moe_lora_state_dict(p, 4, 7, scale=0.5), OM.synth_moe_lora_state_dict(p, 4, 8, scale=0.5)
    fresh = run_model(lora_model(p, sd, 2, adapter=a), p, False, steps=7)
    m = lora_model(p, sd, 2, adapter=a)
    cache = BufferCache(m.n_local_layers, 2, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
    seqlens = [37, 150]
    toks = torch.tensor(synth.synth_prompt(sum(seqlens), p["vocab_size"], 4), device=DEV)
    outs = [m.forward(toks, seqlens, cache)]
    nxt = torch.tensor([5, 7], device=DEV)
    for i in range(6):
        if i == 3:  # the decode graphs are captured by now: swap b in and a back, in place
            m._load_lora_state_dict(b)
            m._load_lora_state_dict(a)
        lg = m.forward(nxt, [1, 1], cache)
        outs.append(lg)
        nxt = lg.argmax(-1)
    assert torch.equal(torch.cat(outs).cpu(), fresh[:-2])
    m._load_lora_state_dict(b)  # a replayed step reads the adapters in place
    assert not torch.equal(m.forward(nxt, [1, 1], cache).cpu(), fresh[-2:])


def test_from_folder_peak_memory_with_adapters(tmp_path):
    p = synth.shape("tiny-moe", dim=512, hidden_dim=1536, n_layers=2)
    synth.write_model_folder(tmp_path, p, 4, lora=dict(rank=16, scaling=2.0))
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = Transformer.from_folder(tmp_path, max_batch_size=1, device=DEV, expert_weights="fp8")
    torch.cuda.synchronize()
    model_bytes = sum(t.numel() * t.element_size() for t in m.parameters())
    largest_bf16 = max(2 * n for n in (p["vocab_size"] * p["dim"], p["dim"] * p["hidden_dim"]))
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= model_bytes + 2 * largest_bf16, (peak, model_bytes, largest_bf16)
    assert m.args.lora is not None and all(not x.any() for k, x in m.state_dict().items() if "lora_" in k)
    q, s = F8.quantize_rows(synth.synth_state_dict(p, 4)["layers.1.feed_forward.experts.5.w3.weight"])
    sd = m.state_dict()
    assert torch.equal(sd["layers.1.feed_forward.experts.5.w3.linear.weight_e4m3"].view(torch.uint8).cpu(), q)
    assert torch.equal(sd["layers.1.feed_forward.experts.5.w3.linear.weight_scale"].cpu(), s)


def test_generate_with_draft_and_an_adapted_fp8_target():
    p = synth.shape("tiny-moe", sliding_window=None)
    m, oracle, _, _ = _adapted(p, 8, 2.0, 2)
    dp = synth.shape("tiny")
    dp["vocab_size"] = p["vocab_size"]
    da = mi.TransformerArgs.from_dict(dict(dp))
    da.max_batch_size = 2
    d = Transformer.empty(da, DEV, torch.bfloat16)
    d.load_state_dict({k: v.to(DEV) for k, v in synth.synth_state_dict(dp, 2).items()})
    prompts = [synth.synth_prompt(n, p["vocab_size"], 80 + i) for i, n in enumerate((19, 26))]
    res = {}
    names = launched_kernels(lambda: res.setdefault("out", mi.generate(prompts, m, max_tokens=11, temperature=0.0, draft=d, draft_tokens=3)))
    toks, lps = res["out"]
    assert names.count("spec_accept_greedy_kernel") >= 2 and any(n.startswith("lora_down_grouped_kernel<") for n in names)
    _teacher_forced(oracle, prompts, toks, lps, 0.05)


# ----------------------------------------------------------------------------- expert parallel
def _free_port() -> int:
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ep_worker(rank: int, world: int, port: int, q):
    try:
        sys.path.insert(0, str(REPO))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        torch.cuda.set_device(0)
        torch.distributed.init_process_group("gloo", rank=rank, world_size=world)
        import mistral_inference_b200 as mi
        import synth
        from mistral_inference_b200.cache import BufferCache
        from mistral_inference_b200.transformer import Transformer

        p = synth.shape("tiny-moe", sliding_window=16)
        sd = synth.synth_state_dict(p, 2, torch.bfloat16, "cuda")
        ad = OM.synth_moe_lora_state_dict(p, 8, 7, scale=0.5, device="cuda")

        def build(expert_parallel):
            args = mi.TransformerArgs.from_dict(dict(p, lora=dict(rank=8, scaling=2.0)))
            args.max_batch_size = 2
            m = Transformer.empty(args, "cuda", torch.bfloat16, expert_parallel=expert_parallel, expert_weights="fp8")
            m.load_state_dict(sd)
            m._load_lora_state_dict(ad)
            return m.eval()

        def run(m):
            cache = BufferCache(m.n_local_layers, 2, 64, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
            seqlens = [12, 9]
            toks = torch.tensor(synth.synth_prompt(sum(seqlens), p["vocab_size"], 4), device="cuda")
            outs = [m.forward(toks, seqlens, cache)]
            nxt = torch.tensor([5, 7], device="cuda")
            for _ in range(4):
                lg = m.forward(nxt, [1, 1], cache)
                outs.append(lg)
                nxt = lg.argmax(-1)
            return torch.cat(outs).cpu()

        sharded = run(build((rank, world)))
        torch.distributed.barrier()
        full = run(build(None)) if rank == 0 else None
        ok = bool(torch.equal(sharded, full)) if rank == 0 else True
        q.put((rank, ok, ""))
        torch.distributed.barrier()
        torch.distributed.destroy_process_group()
    except Exception as e:
        q.put((rank, False, repr(e)))
        raise


def test_expert_parallel_with_adapters_equals_unsharded_two_processes_one_gpu():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_ep_worker, args=(r, 2, port, q)) for r in range(2)]
    for pr in procs:
        pr.start()
    res = sorted(q.get(timeout=400) for _ in range(2))
    for pr in procs:
        pr.join(timeout=60)
    for rank, ok, err in res:
        assert ok, f"rank {rank}: {err or 'sharded adapted FP8 logits differ from the unsharded model'}"
