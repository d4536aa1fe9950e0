"""Mixtral on one H100 with quantised expert weights: Mixtral-8x7B with FP8 (e4m3) or INT4 experts, Mixtral-8x22B with INT4 experts.

Builds the full model (`--model mixtral-8x7b`: 32 layers, `mixtral-8x22b`: 56 layers) with `expert_weights=--experts` from seeded
synthetic weights (synth.py), each matrix generated in bf16 on the device and quantised into place, so the bf16 model never exists.
With INT4 experts the attention Linears are INT4 too (`dense_weights="int4"`, `--dense-weights` overrides): Mixtral-8x22B with bf16
attention is 80.4 GB and leaves no room for a 4k prefill.  Reports:
  * model bytes and the peak device memory of the build;
  * a 4096-token prefill, batch-1 decode ms/token at a 4k context with its share of 3.35 TB/s on the step's own bytes (one token's
    two experts, attention and router weights of every layer, the lm head, the K/V ring), and one batched decode step that fits
    (8x7B: batch 32 at a 512 context; 8x22B: batch 8 at a 2k context) with its peak memory (graph replays);
  * the grouped expert FFN (gate/up GEMM + down GEMM + combine of one MoE layer) of both shapes in bf16, FP8 and INT4, alternated in
    one run, at T = 1, 8, 32 and 4096 tokens, with each call's share of the HBM byte roofline (the bytes of the experts the routed
    tokens touch, in the call's own format, over 3.35 TB/s).  These run after the model is freed, on one layer's synthetic bf16
    weights and their FP8 and INT4 quantisations (the bf16 call's time does not depend on whether its weights are W').
Prints the card's name and power limit with the numbers, then one JSON line.
Run: python scripts/bench_moe_experts.py [--model mixtral-8x7b|mixtral-8x22b] [--experts fp8|int4]
"""
import argparse
import ctypes
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.moe import Fp8Expert, Int4Expert, MoeBuffers  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})"


def build(p, seed: int, experts: str, dense: str, max_batch: int) -> Transformer:
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    m = Transformer.empty(args, "cuda", torch.bfloat16, expert_weights=experts, dense_weights=dense)
    with torch.no_grad():
        for k, shape in synth.state_dict_shapes(p):
            assert m._assign(k, synth.synth_tensor(k, shape, seed, torch.bfloat16, "cuda")), k
    return m.eval()


def timed(fn, reps: int) -> float:
    """Mean ms of fn() over reps calls, CUDA events around the whole loop."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def step_bytes(m: Transformer, ctx: int, B: int = 1) -> int:
    """HBM bytes of one batch-1 decode step: top-k experts, attention, router and norm weights of every layer, the lm head, one
    embedding row and the K/V ring (a batch of B reads the same weights once and B rings)."""
    a = m.args
    k = a.moe.num_experts_per_tok
    nbytes = lambda mod: sum(t.numel() * t.element_size() for t in mod.parameters())  # noqa: E731
    layer = 0
    for blk in m.layers.values():
        ff = blk.feed_forward
        layer += k * nbytes(next(iter(ff.experts.values()))) + nbytes(blk.attention) + ff.gate_weight.numel() * 2 + 4 * a.dim
    return layer + m.output_weight.numel() * 2 + B * a.dim * 2 + a.dim * 2 + B * 2 * ctx * a.n_kv_heads * a.head_dim * 2 * m.n_local_layers


def model_numbers(m: Transformer, p, batch: tuple) -> dict:
    V = p["vocab_size"]
    out = {}
    toks = torch.tensor(synth.synth_prompt(4096, V, 1), device="cuda")

    def prefill():
        cache = BufferCache(m.n_local_layers, 1, 4096 + 256, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
        m.forward(toks, [4096], cache)
        return cache

    prefill()  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cache = prefill()
    torch.cuda.synchronize()
    out["prefill_4096_ms"] = (time.perf_counter() - t0) * 1e3
    nxt = torch.tensor([3], device="cuda")
    for _ in range(8):  # eager step, capture, replays
        nxt = m.next_token_logits(nxt, cache).argmax(-1)
    n = 64
    ms = [timed(lambda: m.next_token_logits(m.last_argmax, cache), n) for _ in range(3)]
    out["decode_b1_ctx4k_ms_per_token"] = min(ms)
    out["decode_b1_ctx4k_all_ms"] = [round(x, 3) for x in ms]
    out["decode_b1_tok_s"] = 1e3 / min(ms)
    b = step_bytes(m, 4096)
    out["decode_b1_step_gb"] = b / 1e9
    out["decode_b1_hbm_share"] = b / (min(ms) * 1e-3) / HBM_BPS
    out["decode_b1_finite"] = bool(torch.isfinite(m.next_token_logits(m.last_argmax, cache)).all())
    del cache
    torch.cuda.empty_cache()
    B, L = batch
    torch.cuda.reset_peak_memory_stats()
    cache = BufferCache(m.n_local_layers, B, L + 128, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
    toks = torch.tensor(synth.synth_prompt(B * L, V, 2), device="cuda").view(B, L)
    for c0 in range(0, L, 512):  # chunked prefill: B x 512 tokens per forward keeps its logits and row buffers small
        m.forward(toks[:, c0:c0 + 512].reshape(-1), [min(512, L - c0)] * B, cache)
    nxt = torch.arange(B, device="cuda")
    for _ in range(4):
        nxt = m.next_token_logits(nxt, cache).argmax(-1)
    out[f"decode_b{B}_ctx{L}_step_ms"] = timed(lambda: m.next_token_logits(m.last_argmax, cache), 16)
    out[f"decode_b{B}_ctx{L}_peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    out[f"decode_b{B}_finite"] = bool(torch.isfinite(m.next_token_logits(m.last_argmax, cache)).all())
    return out


def ffn_numbers(p, seed: int) -> list:
    """One layer's grouped expert FFN in bf16, FP8 and INT4 over the same routing, alternated."""
    dim, hidden = p["dim"], p["hidden_dim"]
    E, k = p["moe"]["num_experts"], p["moe"]["num_experts_per_tok"]
    key = lambda e, n: f"layers.0.feed_forward.experts.{e}.{n}.weight"  # noqa: E731
    w = lambda e, n, shape: synth.synth_tensor(key(e, n), shape, seed, torch.bfloat16, "cuda")  # noqa: E731
    gate = synth.synth_tensor("layers.0.feed_forward.gate.weight", (E, dim), seed, torch.bfloat16, "cuda")
    w13, w2, f8, i4 = [], [], [], []
    for e in range(E):
        w1, w3 = w(e, "w1", (hidden, dim)), w(e, "w3", (hidden, dim))
        w13.append(torch.stack((w1, w3), 1).view(2 * hidden, dim))
        w2.append(w(e, "w2", (dim, hidden)))
        x8, x4 = Fp8Expert(dim, hidden).cuda(), Int4Expert(dim, hidden).cuda()
        for n, t in (("w1", w1), ("w3", w3), ("w2", w2[-1])):
            x8.quantize_(n, t)
            x4.quantize_int4_(n, t)
        f8.append(x8)
        i4.append(x4)
        del w1, w3
    tab = lambda ts: (ctypes.c_void_p * E)(*[t.data_ptr() for t in ts])  # noqa: E731
    t_bf = (tab(w13), tab(w2))
    t_f8 = (tab([x.w13_q for x in f8]), tab([x.w13_scale_bits for x in f8]), tab([x.w2_q for x in f8]), tab([x.w2_scale_bits for x in f8]))
    t_i4 = (tab([x.w13 for x in i4]), tab([x.w13_gscale_bits for x in i4]), tab([x.w2_weight for x in i4]), tab([x.w2_gscale_bits for x in i4]))
    ebytes = {"bf16": 2 * 3 * dim * hidden, "fp8": 3 * dim * hidden + 4 * (2 * hidden + dim),
              "int4": 3 * dim * hidden // 2 + 2 * 3 * dim * hidden // 128}  # one expert's bytes in each format
    rows = []
    for T in (1, 8, 32, 4096):
        g = torch.Generator(device="cuda").manual_seed(T)
        hn = (torch.randn(T, dim, generator=g, device="cuda")).to(torch.bfloat16)
        res = torch.zeros_like(hn)
        ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 1, 1, 128, hidden, 0, 1), torch.device("cuda"))
        b = MoeBuffers(T, dim, hidden, E, k, torch.device("cuda"), torch.bfloat16)
        _abi.moe_route(hn, gate, E, k, 0, 1, b)
        touched = int(torch.unique(b.sel).numel())
        out = torch.empty_like(hn)
        runs = {"bf16": lambda: _abi.moe_grouped_ffn(b, *t_bf, res, out, T, dim, hidden, E, k, None, ws),
                "fp8": lambda: _abi.moe_grouped_ffn_fp8(b, *t_f8, res, out, T, dim, hidden, E, k, None, ws),
                "int4": lambda: _abi.moe_grouped_ffn_int4(b, *t_i4, res, out, T, dim, hidden, E, k, None, ws)}
        reps = 10 if T == 4096 else 100
        for f in runs.values():
            f()
        torch.cuda.synchronize()
        ms = {n: [] for n in runs}
        for _ in range(5):  # alternated
            for n, f in runs.items():
                ms[n].append(timed(f, reps))
        med = {n: sorted(v)[2] for n, v in ms.items()}
        flops = 2 * T * k * 3 * dim * hidden
        row = dict(shape=f"{dim}x{hidden}", T=T, experts_touched=touched)
        for n, t in med.items():
            row[f"{n}_ms"] = round(t, 4)
            row[f"{n}_hbm_roofline"] = round(touched * ebytes[n] / HBM_BPS * 1e3 / t, 3)
            row[f"{n}_tflops"] = round(flops / t / 1e9, 1)
        rows.append(row)
        print("  " + json.dumps(row), flush=True)
        del ws, b
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=("mixtral-8x7b", "mixtral-8x22b"), default="mixtral-8x7b")
    ap.add_argument("--experts", choices=("fp8", "int4"), default="fp8")
    ap.add_argument("--dense-weights", choices=("bf16", "int4"), default=None, help="attention Linears (default: int4 with INT4 experts)")
    ap.add_argument("--layers", type=int, default=None, help="default: the model's own depth")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dense = a.dense_weights or ("int4" if a.experts == "int4" else "bf16")
    p = synth.shape(a.model, **({"n_layers": a.layers} if a.layers else {}))
    batch = (32, 512) if a.model == "mixtral-8x7b" else (8, 2048)
    print(f"card: {card()}", flush=True)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m = build(p, a.seed, a.experts, dense, batch[0])
    torch.cuda.synchronize()
    res = {"card": card(), "model": a.model, "experts": a.experts, "dense_weights": dense, "layers": p["n_layers"],
           "build_s": round(time.perf_counter() - t0, 1),
           "model_gb": round(sum(t.numel() * t.element_size() for t in m.parameters()) / 1e9, 2),
           "build_peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}
    print(f"model {res['model_gb']} GB, build peak {res['build_peak_gb']} GB, built in {res['build_s']} s", flush=True)
    torch.cuda.reset_peak_memory_stats()
    res.update({k: (round(v, 3) if isinstance(v, float) else v) for k, v in model_numbers(m, p, batch).items()})
    res["decode_b1_bound_ms"] = round(res["decode_b1_step_gb"] * 1e9 / HBM_BPS * 1e3, 2)
    print({k: v for k, v in res.items()}, flush=True)
    del m
    torch.cuda.empty_cache()
    res["grouped_ffn"] = [r for name in ("mixtral-8x7b", "mixtral-8x22b") for r in ffn_numbers(synth.shape(name), a.seed)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
