"""FP8 (e4m3) expert weights on the GPU: the quantiser against the CPU restatement (oracle/fp8.py), the FP8 grouped expert GEMMs
against the bf16 ones run on the dequantised weights W' in every grouped-GEMM regime, and whole models.

The FP8 model is defined as the bf16 model on W' (include/mistral_b200.h), and an FP8 call runs the same tiles, tile widths and
stream-K partition as the bf16 call over the same plan; the MMAs read the same bf16 shared-memory tiles.  So g, yw and out must be
identical bit for bit.  The one regime where the two calls differ in launch shape is the 128-row prefill with N % 256 == 0 and
enough rows for tile pairs: bf16 runs the 2-CTA cluster, FP8 the single-CTA kernel over the same tiles (each tile's k order is the
same, so the bits are too).  The bf16 path itself is checked against the float64 oracle bit for bit by tests/test_gpu_moe_edges.py.
"""
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
from mistral_inference_b200.moe import Fp8Expert, MoeBuffers
from mistral_inference_b200.transformer import Transformer
from oracle import fp8 as F8

from .util import launched_kernels

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]
DEV = "cuda"


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).cpu()


def edge_rows(K: int) -> torch.Tensor:
    """Rows with ties, +-448 after scaling, all zeros, negative zeros, subnormal e4m3 results and huge / tiny magnitudes."""
    g = torch.Generator().manual_seed(1)
    base = torch.randn(8, K, generator=g)
    base[0] = 0.0
    base[1] = -0.0
    base[1, ::3] = 0.0
    base[2, :8] = torch.tensor([448.0, 1.0625, 1.1875, -1.0625, 3 * 2.0 ** -11, 2.0 ** -10, 400.0, -432.0])
    base[2, 8:] = 0.5
    base[3] = base[3] * 2.0 ** -20
    base[3, 0] = 448 * 2.0 ** -20
    base[3, 1:5] = torch.tensor([2.0 ** -28, 2.0 ** -30, 3 * 2.0 ** -31, -(2.0 ** -29)])
    base[4] = base[4] * 1e30
    base[5] = base[5] * 1e-30
    base[6, :] = -3.0
    base[7, 5] = 1e4
    return base.to(torch.bfloat16)


@pytest.mark.parametrize("K", [64, 4096, 14336])
def test_quantize_rows_matches_oracle(K):
    g = torch.Generator().manual_seed(K)
    w = torch.cat([edge_rows(K), (torch.randn(120, K, generator=g) * torch.logspace(-3, 3, 120)[:, None]).to(torch.bfloat16)])
    q, s = F8.quantize_rows(w)
    qd = torch.full(w.shape, 0x55, dtype=torch.uint8, device=DEV)
    sd = torch.full((w.shape[0],), float("nan"), device=DEV)
    _abi.quantize_e4m3_rows(w.to(DEV), qd, sd)
    assert torch.equal(qd.cpu(), q)
    assert torch.equal(sd.cpu().view(torch.int32), s.view(torch.int32))


def test_quantize_rows_into_interleaved_w13():
    """w1 and w3 land in rows 2i and 2i + 1 of the packed gate/up matrix, their scales in the matching entries."""
    dim, hidden = 256, 128
    g = torch.Generator().manual_seed(3)
    w1 = torch.cat([edge_rows(dim), (torch.randn(hidden - 8, dim, generator=g)).to(torch.bfloat16)])
    w3 = (torch.randn(hidden, dim, generator=g) * 1e-3).to(torch.bfloat16)
    ex = Fp8Expert(dim, hidden).to(DEV)
    with torch.no_grad():
        ex.w13_q.fill_(0x55)
        ex.w13_scale_bits.fill_(-1)
    ex.quantize_("w1", w1)
    ex.quantize_("w3", w3)
    q1, s1 = F8.quantize_rows(w1)
    q3, s3 = F8.quantize_rows(w3)
    assert torch.equal(ex.w13_q.cpu(), torch.stack([q1, q3], 1).view(2 * hidden, dim))
    assert torch.equal(ex.w13_scale.cpu(), torch.stack([s1, s3], 1).view(2 * hidden))


# ----------------------------------------------------------------------------- grouped FFN: FP8 == bf16 on W'
def fp8_experts(E: int, dim: int, hidden: int, seed: int, shard=(0, 1)):
    """Per expert: (bf16 W' w13, bf16 W' w2, e4m3 w13 / scales, e4m3 w2 / scales), None for experts of other ranks."""
    out = []
    for e in range(E):
        if e % shard[1] != shard[0]:
            out.append(None)
            continue
        g = torch.Generator(device=DEV).manual_seed(seed * 100 + e)
        w13 = (torch.randn(2 * hidden, dim, generator=g, device=DEV) * dim ** -0.5 * torch.logspace(-1, 1, 2 * hidden, device=DEV)[:, None])
        w2 = torch.randn(dim, hidden, generator=g, device=DEV) * hidden ** -0.5
        w13, w2 = w13.to(torch.bfloat16), w2.to(torch.bfloat16)
        q13, s13 = torch.empty(2 * hidden, dim, dtype=torch.uint8, device=DEV), torch.empty(2 * hidden, device=DEV)
        q2, s2 = torch.empty(dim, hidden, dtype=torch.uint8, device=DEV), torch.empty(dim, device=DEV)
        _abi.quantize_e4m3_rows(w13, q13, s13)
        _abi.quantize_e4m3_rows(w2, q2, s2)
        out.append((F8.dequantize_rows(q13, s13), F8.dequantize_rows(q2, s2), q13, s13, q2, s2))
    return out


def table(vals):
    import ctypes

    t = (ctypes.c_void_p * len(vals))()
    for i, v in enumerate(vals):
        t[i] = v.data_ptr() if v is not None else None
    return t


def run_ffn(T, dim, hidden, E, k, experts, seed, shard=(0, 1), env=None):
    """Routes random tokens once, then runs the bf16 grouped FFN on W' and the FP8 one on (q, s) over the same plan.  Returns
    (bf16 outputs, fp8 outputs, bf16 launch log, fp8 launch log)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    hn = torch.randn(T, dim, generator=g, device=DEV).to(torch.bfloat16)
    res = torch.randn(T, dim, generator=g, device=DEV).to(torch.bfloat16)
    gate = (torch.randn(E, dim, generator=g, device=DEV) * dim ** -0.5).to(torch.bfloat16)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 1, 1, 128, hidden, 0, 1), torch.device(DEV))
    b = MoeBuffers(T, dim, hidden, E, k, torch.device(DEV), torch.bfloat16)
    _abi.moe_route(hn, gate, E, k, shard[0], shard[1], b)
    col = lambda i: [x[i] if x is not None else None for x in experts]  # noqa: E731
    outs, logs = [], []
    old = {key: os.environ.get(key) for key in (env or {})}
    os.environ.update(env or {})
    try:
        for fp8 in (False, True):
            b.g.fill_(float("nan"))
            b.yw.fill_(0.0)
            out = torch.full((T, dim), float("nan"), dtype=torch.bfloat16, device=DEV)
            if fp8:
                call = lambda: _abi.moe_grouped_ffn_fp8(b, table(col(2)), table(col(3)), table(col(4)), table(col(5)), res, out, T, dim,  # noqa: E731
                                                        hidden, E, k, None, ws)
            else:
                call = lambda: _abi.moe_grouped_ffn(b, table(col(0)), table(col(1)), res, out, T, dim, hidden, E, k, None, ws)  # noqa: E731
            logs.append(launched_kernels(call))
            torch.cuda.synchronize()
            outs.append((b.g.clone(), b.yw.clone(), out))
    finally:
        for key, v in old.items():
            if v is None:
                os.environ.pop(key, None)
            else:
                os.environ[key] = v
    return outs[0], outs[1], logs[0], logs[1]


def assert_same_ffn(bf, f8, what):
    for name, x, y in zip(("g", "yw", "out"), bf, f8):
        assert torch.equal(bits(x), bits(y)), f"{what}: {name} differs in {(bits(x) != bits(y)).sum().item()} elements"


def grouped_names(log):
    return [n for n in log if "grouped" in n]


# (T, E, k, dim, hidden, env): the regimes of launch_grouped (csrc/moe.cuh) -- tile rows 32 / 64 / 128, stream-K or wgmma, each BN,
# the cluster pair (bf16) against its single-CTA FP8 counterpart
REGIMES = [
    (1, 8, 2, 256, 384, {}),                                  # batch 1: stream-K, 32-row tiles, most experts empty
    (8, 4, 3, 256, 384, {}),                                  # stream-K, 32-row tiles
    (40, 16, 4, 256, 384, {}),                                # stream-K, 64-row tiles
    (8, 8, 2, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "256"}),  # wgmma 32-row tiles, BN 256
    (8, 8, 2, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "128"}),
    (40, 2, 1, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "64"}),  # wgmma 64-row tiles
    (40, 8, 2, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "32"}),
    (1200, 4, 2, 256, 384, {}),                               # 128-row tiles, BN 256, cluster pair for bf16 (rows_cap >= 512 E)
    (1200, 4, 2, 256, 384, {"MB200_GEMM_CLUSTER": "0"}),      # 128-row tiles, BN 256 single CTA both
    (200, 16, 4, 448, 320, {}),                               # 128-row tiles: w13 N = 640 -> BN 128, w2 N = 448 -> BN 64
    (2000, 8, 2, 512, 512, {}),                               # many m units: the blocked tile walk
]


@pytest.mark.parametrize("T,E,k,dim,hidden,env", REGIMES, ids=[f"T{r[0]}-E{r[1]}-k{r[2]}-{r[3]}x{r[4]}-{'-'.join(f'{a[5:]}{b}' for a, b in r[5].items()) or 'auto'}" for r in REGIMES])
def test_grouped_ffn_fp8_equals_bf16_on_dequantised_weights(T, E, k, dim, hidden, env):
    experts = fp8_experts(E, dim, hidden, seed=T + E)
    bf, f8, log_bf, log_f8 = run_ffn(T, dim, hidden, E, k, experts, seed=T * 7 + k, env=env)
    assert_same_ffn(bf, f8, f"T={T} E={E} k={k}")
    gb, gf = grouped_names(log_bf), grouped_names(log_f8)
    assert len(gb) == len(gf) == 2, (log_bf, log_f8)
    for nb, nf in zip(gb, gf):
        assert "_fp8_kernel" in nf and "_fp8_kernel" not in nb, (nb, nf)
        if "streamk" in nb:
            assert nf == nb.replace("gemm_streamk_grouped_kernel", "gemm_streamk_grouped_fp8_kernel")
        else:  # same BN and tile rows; the cluster pair becomes one CTA
            mode, cl, bn, ta = nb[nb.index("<") + 1:-1].split(", ")
            assert nf == f"gemm_wgmma_grouped_fp8_kernel<{mode}, 1, {bn}, {ta}>", (nb, nf)
    if env.get("MB200_GEMM_BN"):
        assert all(f", {env['MB200_GEMM_BN']}, " in n for n in gf), gf
    if T == 1200 and not env:
        assert any(", 2, 256, 128>" in n for n in gb), gb


@pytest.mark.parametrize("T,k", [(1, 2), (48, 2), (300, 3)])
def test_grouped_ffn_fp8_expert_shard_with_null_experts(T, k):
    E, dim, hidden = 8, 256, 384
    experts = fp8_experts(E, dim, hidden, seed=5, shard=(1, 2))
    bf, f8, _, log_f8 = run_ffn(T, dim, hidden, E, k, experts, seed=T, shard=(1, 2))
    # rows of the other rank's experts are never written (no peers here): compare g and yw, which cover every local row
    for name, x, y in zip(("g", "yw"), bf[:2], f8[:2]):
        assert torch.equal(bits(x), bits(y)), name
    assert all("_fp8_kernel" in n for n in grouped_names(log_f8))


# ----------------------------------------------------------------------------- models
def build_pair(p, sd, max_batch):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m8 = Transformer.empty(args, DEV, torch.bfloat16, expert_weights="fp8")
    m8.load_state_dict(sd)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    mb = Transformer.empty(args, DEV, torch.bfloat16)
    mb.load_state_dict(F8.fp8_checkpoint(sd))
    return m8.eval(), mb.eval()


def run_model(m, p, batch1: bool):
    cache = BufferCache(m.n_local_layers, 2, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
    outs = []
    if batch1:
        toks = torch.tensor(synth.synth_prompt(21, p["vocab_size"], 9), device=DEV)
        cache = BufferCache(m.n_local_layers, 1, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
        outs.append(m.forward(toks[:13], [13], cache))
        outs.append(m.forward(toks[13:], [8], cache))  # chunked prefill
        nxt = outs[-1][-1:].argmax(-1)
        for _ in range(4):  # eager warm-up, graph capture, replays (per-layer path: the megakernel reads bf16 experts only)
            lg = m.forward(nxt, [1], cache)
            outs.append(lg)
            nxt = lg.argmax(-1)
        return torch.cat(outs).cpu()
    seqlens = [37, 150]
    toks = torch.tensor(synth.synth_prompt(sum(seqlens), p["vocab_size"], 4), device=DEV)
    outs.append(m.forward(toks, seqlens, cache))
    nxt = torch.tensor([5, 7], device=DEV)
    for _ in range(4):
        lg = m.forward(nxt, [1, 1], cache)
        outs.append(lg)
        nxt = lg.argmax(-1)
    return torch.cat(outs).cpu()


@pytest.mark.parametrize("shape", ["tiny-moe", "mixtral-8x7b-2layers"])
def test_fp8_model_equals_bf16_model_on_dequantised_checkpoint(shape, monkeypatch):
    if shape == "tiny-moe":
        p = synth.shape("tiny-moe", sliding_window=64)
    else:
        p = synth.shape("mixtral-8x7b", n_layers=2, vocab_size=4096)
    sd = synth.synth_state_dict(p, 2, torch.bfloat16, DEV)
    m8, mb = build_pair(p, sd, 2)
    del sd
    assert not m8._megakernel_ok(1)
    for batch1 in (False, True):
        got = run_model(m8, p, batch1)
        monkeypatch.setenv("MB200_MEGAKERNEL", "0")  # the bf16 model on the same per-layer path for batch 1
        want = run_model(mb, p, batch1)
        monkeypatch.delenv("MB200_MEGAKERNEL")
        assert torch.equal(got, want), f"batch1={batch1}: max |diff| {(got - want).abs().max().item()}"
    log = launched_kernels(lambda: m8.forward(torch.tensor([1, 2, 3], device=DEV), [3]))
    assert any("gemm_streamk_grouped_fp8_kernel" in n for n in log) and not any("grouped_kernel<" in n for n in log), log


def test_fp8_generate_equals_bf16_generate():
    from mistral_inference_b200.generate import generate

    p = synth.shape("tiny-moe", sliding_window=64)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, DEV)
    m8, mb = build_pair(p, sd, 2)
    prompts = [synth.synth_prompt(n, p["vocab_size"], s) for n, s in ((25, 1), (30, 2))]  # 6-token chunks: both prompts in all 5
    got = generate(prompts, m8, max_tokens=12, temperature=0.0, chunk_size=6)
    os.environ["MB200_MEGAKERNEL"] = "0"
    try:
        want = generate(prompts, mb, max_tokens=12, temperature=0.0, chunk_size=6)
    finally:
        os.environ.pop("MB200_MEGAKERNEL")
    assert got[0] == want[0]
    for a, b in zip(got[1], want[1]):
        assert a == b


def test_from_folder_fp8_peak_memory(tmp_path):
    p = synth.shape("tiny-moe", dim=512, hidden_dim=1536, n_layers=2)
    synth.write_model_folder(tmp_path, p, 4)
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
    bf16_expert_bytes = 2 * p["moe"]["num_experts"] * 3 * p["dim"] * p["hidden_dim"] * 2
    assert model_bytes < bf16_expert_bytes  # the bf16 experts alone would not fit the bound
    sd = m.state_dict()
    ref = synth.synth_state_dict(p, 4)
    q, s = F8.quantize_rows(ref["layers.1.feed_forward.experts.5.w3.weight"])
    assert torch.equal(sd["layers.1.feed_forward.experts.5.w3.weight_e4m3"].view(torch.uint8).cpu(), q)
    assert torch.equal(sd["layers.1.feed_forward.experts.5.w3.weight_scale"].cpu(), s)


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

        def build(expert_parallel):
            args = mi.TransformerArgs.from_dict(dict(p))
            args.max_batch_size = 2
            m = Transformer.empty(args, "cuda", torch.bfloat16, expert_parallel=expert_parallel, expert_weights="fp8")
            m.load_state_dict(sd)
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


def test_fp8_expert_parallel_equals_unsharded_two_processes_one_gpu():
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
        assert ok, f"rank {rank}: {err or 'sharded FP8 logits differ from the unsharded FP8 model'}"
    assert all(pr.exitcode == 0 for pr in procs)
