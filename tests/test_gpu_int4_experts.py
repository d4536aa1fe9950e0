"""INT4 expert weights on the GPU: the quantiser into an expert's interleaved w13 rows against the restatement
(tests/int4_dense_ref.py), the INT4 grouped expert GEMMs against the bf16 ones run on the dequantised weights W' in every grouped-GEMM
regime, and whole models, also with INT4 attention Linears (dense_weights="int4").

An INT4 grouped call runs the same tiles, tile widths and stream-K partition as the bf16 call over the same plan, and its converter
warps write exactly the bf16 W' tiles the MMAs read; so g, yw and out must be identical bit for bit at every T.  The one launch-shape
difference is the 128-row prefill where bf16 runs the 2-CTA cluster: INT4 runs single CTAs at the same BN (each tile's k order is the
same, so the bits are too).

Expert K (dim and hidden) is a multiple of 128, so every expert N (2 * hidden, dim) is a multiple of 128 too.  Hence: calls of up to
64 tokens always take stream-K unless MB200_STREAMK=0, which gives the small-batch wgmma kernel at any BN of 256, 128, 64 and 32;
128-row prefill tiles take BN 256 (N % 256 == 0) or 128, never 64 or 32.
"""
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
from mistral_inference_b200.moe import Int4Expert, MoeBuffers
from mistral_inference_b200.transformer import Transformer
from tests import int4_dense_ref as I4

from .util import launched_kernels, logit_tol

pytestmark = pytest.mark.gpu
REPO = Path(__file__).resolve().parents[1]
DEV = "cuda"


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16).cpu()


def wprime(w: torch.Tensor) -> torch.Tensor:
    return I4.dequantize(*I4.quantize(w))


def int4_checkpoint(sd, attention: bool = False):
    """The reference-keyed checkpoint whose bf16 model is the INT4-expert model (and, with `attention`, the model with INT4 attention
    Linears too): those weights replaced by W', everything else the same tensor.  Replaces in place, one tensor at a time."""
    for k in list(sd):
        if (".experts." in k and k.endswith(".weight")) or (attention and I4.is_dense_key(k)):
            sd[k] = wprime(sd[k])
    return sd


def test_quantize_into_interleaved_w13_equals_restatement():
    dim, hidden = 384, 256
    g = torch.Generator().manual_seed(3)
    w1 = (torch.randn(hidden, dim, generator=g) * torch.logspace(-4, 4, hidden)[:, None]).to(torch.bfloat16)
    w1[0] = 0.0
    w1[1, :128] = 0.0
    w1[2, 5] = 1e-40  # a group whose scale rounds to 0 and is raised to 2^-133
    w1[2, :5] = 0.0
    w1[2, 6:128] = 0.0
    w3 = (torch.randn(hidden, dim, generator=g) * 1e-3).to(torch.bfloat16)
    w2 = (torch.randn(dim, hidden, generator=g)).to(torch.bfloat16)
    ex = Int4Expert(dim, hidden).to(DEV)
    with torch.no_grad():
        ex.w13.fill_(0x55)
        ex.w13_gscale_bits.fill_(-1)
    for name, w in (("w1", w1), ("w3", w3), ("w2", w2)):
        ex.quantize_int4_(name, w.to(DEV))
    c13, s13 = I4.quantize(torch.stack([w1, w3], 1).view(2 * hidden, dim))
    assert torch.equal(ex.w13.cpu(), c13)
    assert torch.equal(ex.w13_gscale_bits.cpu(), s13.view(torch.int16))
    c2, s2 = I4.quantize(w2)
    assert torch.equal(ex.w2_weight.cpu(), c2) and torch.equal(ex.w2_gscale_bits.cpu(), s2.view(torch.int16))


# ----------------------------------------------------------------------------- grouped FFN: INT4 == bf16 on W'
def int4_experts(E: int, dim: int, hidden: int, seed: int, shard=(0, 1)):
    """Per expert: (bf16 W' w13, bf16 W' w2, w13 codes, w13 scales, w2 codes, w2 scales), None for experts of other ranks."""
    out = []
    for e in range(E):
        if e % shard[1] != shard[0]:
            out.append(None)
            continue
        g = torch.Generator(device=DEV).manual_seed(seed * 100 + e)
        w13 = torch.randn(2 * hidden, dim, generator=g, device=DEV) * dim ** -0.5 * torch.logspace(-1, 1, 2 * hidden, device=DEV)[:, None]
        w2 = torch.randn(dim, hidden, generator=g, device=DEV) * hidden ** -0.5
        w13, w2 = w13.to(torch.bfloat16), w2.to(torch.bfloat16)
        c13, s13 = I4.quantize(w13)
        c2, s2 = I4.quantize(w2)
        out.append((I4.dequantize(c13, s13), I4.dequantize(c2, s2), c13, s13, c2, s2))
    return out


def table(vals):
    t = (ctypes.c_void_p * len(vals))()
    for i, v in enumerate(vals):
        t[i] = v.data_ptr() if v is not None else None
    return t


def run_ffn(T, dim, hidden, E, k, experts, seed, shard=(0, 1), env=None):
    """Routes random tokens once, then runs the bf16 grouped FFN on W' and the INT4 one on the codes over the same plan.  Returns
    (bf16 outputs, int4 outputs, bf16 launch log, int4 launch log)."""
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
        for int4 in (False, True):
            b.g.fill_(float("nan"))
            b.yw.fill_(0.0)
            out = torch.full((T, dim), float("nan"), dtype=torch.bfloat16, device=DEV)
            if int4:
                call = lambda: _abi.moe_grouped_ffn_int4(b, table(col(2)), table(col(3)), table(col(4)), table(col(5)), res, out, T, dim,  # noqa: E731
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


def grouped_names(log):
    return [n for n in log if "grouped" in n]


# (T, E, k, dim, hidden, env): the regimes of launch_grouped (csrc/moe.cuh) that INT4 expert shapes reach
REGIMES = [
    (1, 8, 2, 256, 384, {}),                                  # batch 1: stream-K, 32-row tiles, most experts empty
    (1, 8, 2, 256, 384, {"MB200_STREAMK": "0"}),              # batch 1 on the small-batch wgmma kernel
    (8, 4, 3, 256, 384, {}),                                  # stream-K, 32-row tiles
    (40, 16, 4, 256, 384, {}),                                # stream-K, 64-row tiles
    (8, 8, 2, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "256"}),  # wgmma 32-row tiles, each BN
    (8, 8, 2, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "128"}),
    (40, 2, 1, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "64"}),  # wgmma 64-row tiles
    (40, 8, 2, 256, 384, {"MB200_STREAMK": "0", "MB200_GEMM_BN": "32"}),
    (1200, 4, 2, 256, 384, {}),                               # 128-row tiles, BN 256; bf16 runs the cluster pair (rows_cap >= 512 E)
    (1200, 4, 2, 256, 384, {"MB200_GEMM_CLUSTER": "0"}),      # 128-row tiles, BN 256, single CTA both
    (200, 16, 4, 384, 256, {}),                               # 128-row tiles, no cluster: w13 N = 512 -> BN 256, w2 N = 384 -> BN 128
    (2000, 8, 2, 512, 512, {}),                               # many m units: the blocked tile walk
]


@pytest.mark.parametrize("T,E,k,dim,hidden,env", REGIMES, ids=[f"T{r[0]}-E{r[1]}-k{r[2]}-{r[3]}x{r[4]}-{'-'.join(f'{a[5:]}{b}' for a, b in r[5].items()) or 'auto'}" for r in REGIMES])
def test_grouped_ffn_int4_equals_bf16_on_dequantised_weights(T, E, k, dim, hidden, env):
    experts = int4_experts(E, dim, hidden, seed=T + E)
    bf, i4, log_bf, log_i4 = run_ffn(T, dim, hidden, E, k, experts, seed=T * 7 + k, env=env)
    for name, x, y in zip(("g", "yw", "out"), bf, i4):
        assert torch.equal(bits(x), bits(y)), f"T={T} E={E} k={k}: {name} differs in {(bits(x) != bits(y)).sum().item()} elements"
    gb, gi = grouped_names(log_bf), grouped_names(log_i4)
    assert len(gb) == len(gi) == 2, (log_bf, log_i4)
    for nb, ni in zip(gb, gi):
        assert "_int4_kernel" in ni and "_int4_kernel" not in nb, (nb, ni)
        if "streamk" in nb:
            assert ni == nb.replace("gemm_streamk_grouped_kernel", "gemm_streamk_grouped_int4_kernel")
        else:  # same BN and tile rows; the cluster pair becomes one CTA
            mode, cl, bn, ta = nb[nb.index("<") + 1:-1].split(", ")
            assert ni == f"gemm_wgmma_grouped_int4_kernel<{mode}, {bn}, {ta}>", (nb, ni)
    if env.get("MB200_GEMM_BN"):
        assert all(f", {env['MB200_GEMM_BN']}, " in n for n in gi), gi
    if T == 1200 and not env:
        assert any(", 2, 256, 128>" in n for n in gb), gb
    if T == 200:
        assert [n.split(", ")[1] for n in gi] == ["256", "128"], gi


@pytest.mark.parametrize("T,k", [(1, 2), (48, 2), (300, 3)])
def test_grouped_ffn_int4_expert_shard_with_null_experts(T, k):
    E, dim, hidden = 8, 256, 384
    experts = int4_experts(E, dim, hidden, seed=5, shard=(1, 2))
    bf, i4, _, log_i4 = run_ffn(T, dim, hidden, E, k, experts, seed=T, shard=(1, 2))
    # rows of the other rank's experts are never written (no peers here): compare g and yw, which cover every local row
    for name, x, y in zip(("g", "yw"), bf[:2], i4[:2]):
        assert torch.equal(bits(x), bits(y)), name
    assert all("_int4_kernel" in n for n in grouped_names(log_i4))


def test_grouped_ffn_int4_refuses_k_off_the_scale_groups():
    E, T, k, dim, hidden = 4, 8, 2, 256, 192  # hidden % 128 != 0: w2's K would split a scale group
    b = MoeBuffers(T, dim, hidden, E, k, torch.device(DEV), torch.bfloat16)
    ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 1, 1, 128, hidden, 0, 1), torch.device(DEV))
    codes = [torch.zeros(2 * hidden, dim // 2, dtype=torch.uint8, device=DEV) for _ in range(E)]
    sc = [torch.zeros(2 * hidden, dim // 128, dtype=torch.bfloat16, device=DEV) for _ in range(E)]
    out = torch.empty(T, dim, dtype=torch.bfloat16, device=DEV)
    with pytest.raises(_abi.Mb200Error, match="multiples of 128"):
        _abi.moe_grouped_ffn_int4(b, table(codes), table(sc), table(codes), table(sc), None, out, T, dim, hidden, E, k, None, ws)


# ----------------------------------------------------------------------------- models
def build(p, sd, max_batch, **kw):
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, DEV, torch.bfloat16, **kw)
    m.load_state_dict(sd)
    return m.eval()


def run_model(m, p, batch1: bool):
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
    cache = BufferCache(m.n_local_layers, 2, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
    seqlens = [37, 150]
    toks = torch.tensor(synth.synth_prompt(sum(seqlens), p["vocab_size"], 4), device=DEV)
    outs.append(m.forward(toks, seqlens, cache))
    nxt = torch.tensor([5, 7], device=DEV)
    for _ in range(4):
        lg = m.forward(nxt, [1, 1], cache)
        outs.append(lg)
        nxt = lg.argmax(-1)
    return torch.cat(outs).cpu()


MODEL_SHAPES = {"tiny-moe": dict(sliding_window=64), "mixtral-8x22b": dict(n_layers=2, vocab_size=4096)}


@pytest.mark.parametrize("shape", ["tiny-moe", "mixtral-8x22b"])
def test_int4_expert_model_equals_bf16_model_on_dequantised_checkpoint(shape, monkeypatch):
    p = synth.shape(shape, **MODEL_SHAPES[shape])
    sd = synth.synth_state_dict(p, 2, torch.bfloat16, DEV)
    m4 = build(p, sd, 2, expert_weights="int4")
    mb = build(p, int4_checkpoint(sd), 2)
    del sd
    assert not m4._megakernel_ok(1)
    for batch1 in (False, True):
        got = run_model(m4, p, batch1)
        monkeypatch.setenv("MB200_MEGAKERNEL", "0")  # the bf16 model on the same per-layer path for batch 1
        want = run_model(mb, p, batch1)
        monkeypatch.delenv("MB200_MEGAKERNEL")
        assert torch.equal(got, want), f"batch1={batch1}: max |diff| {(got - want).abs().max().item()}"
    log = launched_kernels(lambda: m4.forward(torch.tensor([1, 2, 3], device=DEV), [3]))
    assert any("gemm_streamk_grouped_int4_kernel" in n for n in log) and not any("grouped_kernel<" in n for n in log), log


def test_int4_generate_equals_bf16_generate():
    from mistral_inference_b200.generate import generate

    p = synth.shape("tiny-moe", sliding_window=64)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, DEV)
    m4 = build(p, sd, 2, expert_weights="int4")
    mb = build(p, int4_checkpoint(sd), 2)
    prompts = [synth.synth_prompt(n, p["vocab_size"], s) for n, s in ((25, 1), (30, 2))]
    got = generate(prompts, m4, max_tokens=12, temperature=0.0, chunk_size=6)
    os.environ["MB200_MEGAKERNEL"] = "0"
    try:
        want = generate(prompts, mb, max_tokens=12, temperature=0.0, chunk_size=6)
    finally:
        os.environ.pop("MB200_MEGAKERNEL")
    assert got[0] == want[0]
    for a, b in zip(got[1], want[1]):
        assert a == b


@pytest.mark.parametrize("shape", ["tiny-moe", "mixtral-8x22b"])
def test_int4_attention_on_moe_model(shape, monkeypatch):
    """dense_weights="int4" with INT4 experts: a first prefill of >= 128 tokens and batched decode at B >= 5 equal the bf16 model on
    the W' checkpoint bit for bit; batch 1 (the INT4 GEMV pairs nibbles in its own order) is held to 2 bf16 ulps at logit scale."""
    p = synth.shape(shape, **MODEL_SHAPES[shape])
    sd = synth.synth_state_dict(p, 5, torch.bfloat16, DEV)
    B = 6
    m4 = build(p, sd, B, expert_weights="int4", dense_weights="int4")
    assert m4.layers["0"].attention.wqkv.dtype == torch.uint8
    mb = build(p, int4_checkpoint(sd, attention=True), B)
    del sd
    monkeypatch.setenv("MB200_MEGAKERNEL", "0")
    lens = [130 + 3 * i for i in range(B)]
    toks = torch.tensor(sum((synth.synth_prompt(n, p["vocab_size"], 20 + i) for i, n in enumerate(lens)), []), device=DEV)
    res = {}
    for tag, m in (("int4", m4), ("bf16", mb)):
        cache = BufferCache(m.n_local_layers, B, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
        outs = [m.forward(toks, lens, cache)]
        nxt = torch.tensor([3 + i for i in range(B)], device=DEV)
        for _ in range(3):
            lg = m.forward(nxt, [1] * B, cache)
            outs.append(lg)
            nxt = lg.argmax(-1)
        res[tag] = torch.cat(outs).cpu()
        # batch 1: a 140-token first prefill (bit-equal), then decode steps on the GEMV
        c1 = BufferCache(m.n_local_layers, 1, 256, p["n_kv_heads"], p["head_dim"], p.get("sliding_window")).to(m.device, m.dtype)
        first = m.forward(toks[:140], [140], c1)
        steps = [m.forward(torch.tensor([11 + s], device=DEV), [1], c1) for s in range(2)]
        res[tag + "-prefill1"], res[tag + "-b1"] = first.cpu(), torch.cat(steps).cpu()
    assert torch.equal(res["int4"], res["bf16"]), f"max |diff| {(res['int4'] - res['bf16']).abs().max().item()}"
    assert torch.equal(res["int4-prefill1"], res["bf16-prefill1"])
    got, want = res["int4-b1"], res["bf16-b1"]
    tol = logit_tol(want)
    assert (got - want).abs().max().item() <= tol, ((got - want).abs().max().item(), tol)


def test_from_folder_int4_peak_memory(tmp_path):
    p = synth.shape("tiny-moe", dim=512, hidden_dim=1536, n_layers=2)
    synth.write_model_folder(tmp_path, p, 4)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = Transformer.from_folder(tmp_path, max_batch_size=1, device=DEV, expert_weights="int4", dense_weights="int4")
    torch.cuda.synchronize()
    model_bytes = sum(t.numel() * t.element_size() for t in m.parameters())
    largest_bf16 = max(2 * n for n in (p["vocab_size"] * p["dim"], p["dim"] * p["hidden_dim"]))
    peak = torch.cuda.max_memory_allocated() - base
    assert peak <= model_bytes + largest_bf16 + (1 << 20), (peak, model_bytes, largest_bf16)
    sd = m.state_dict()
    ref = synth.synth_state_dict(p, 4)
    c, s = I4.quantize(ref["layers.1.feed_forward.experts.5.w3.weight"])
    assert torch.equal(sd["layers.1.feed_forward.experts.5.w3.weight_int4"].cpu(), c)
    assert torch.equal(sd["layers.1.feed_forward.experts.5.w3.weight_gscale"].cpu().view(torch.int16), s.view(torch.int16))


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
            m = Transformer.empty(args, "cuda", torch.bfloat16, expert_parallel=expert_parallel, expert_weights="int4")
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


def test_int4_expert_parallel_equals_unsharded_two_processes_one_gpu():
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
        assert ok, f"rank {rank}: {err or 'sharded INT4 logits differ from the unsharded INT4 model'}"
    assert all(pr.exitcode == 0 for pr in procs)
