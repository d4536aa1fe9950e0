"""Mixtral-8x7B on one H100 with FP8 (e4m3) expert weights.

Builds a full 32-layer Mixtral-8x7B-shaped model with `expert_weights="fp8"` from seeded synthetic weights (synth.py), each
expert matrix generated in bf16 on the device and quantised into place, so the bf16 model never exists.  Reports:
  * peak device memory of the build;
  * a 4096-token prefill, batch-1 decode ms/token at a 4k context, and one batch-32 decode step (graph replays);
  * the grouped expert FFN (gate/up GEMM + down GEMM + combine of one MoE layer) in FP8 and in bf16, alternated in one run, at
    T = 1, 8, 32 and 4096 tokens, with each call's share of the HBM byte roofline (expert bytes the routed tokens touch, FP8
    bytes for the FP8 call, over 3.35 TB/s).  The bf16 side uses one layer's dequantised experts W' (2.8 GB): a bf16 model of
    more than a few layers does not fit next to the FP8 one.
Prints the card's name and power limit with the numbers, then one JSON line.  Run: python scripts/bench_moe_fp8.py
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
from mistral_inference_b200.moe import MoeBuffers  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})"


def build(p, seed: int) -> Transformer:
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 32
    m = Transformer.empty(args, "cuda", torch.bfloat16, expert_weights="fp8")
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


def model_numbers(m: Transformer, p) -> dict:
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
    out["decode_b1_ctx4k_ms_per_token"] = timed(lambda: m.next_token_logits(m.last_argmax, cache), n)
    del cache
    B, L = 32, 512
    cache = BufferCache(m.n_local_layers, B, L + 128, p["n_kv_heads"], p["head_dim"], None).to(m.device, m.dtype)
    toks = torch.tensor(synth.synth_prompt(B * L, V, 2), device="cuda")
    m.forward(toks, [L] * B, cache)
    nxt = torch.arange(B, device="cuda")
    for _ in range(4):
        nxt = m.next_token_logits(nxt, cache).argmax(-1)
    out["decode_b32_ctx512_step_ms"] = timed(lambda: m.next_token_logits(m.last_argmax, cache), 32)
    return out


def ffn_numbers(m: Transformer, p) -> list:
    dim, hidden = p["dim"], p["hidden_dim"]
    E, k = p["moe"]["num_experts"], p["moe"]["num_experts_per_tok"]
    layer = m.layers["0"].feed_forward
    ex = [layer.experts[str(e)] for e in range(E)]
    # bf16 W' of layer 0: W'[n, k] = bf16(float(q) * s), built on the device
    deq = lambda q, s: (q.view(torch.float8_e4m3fn).float() * s[:, None]).to(torch.bfloat16)  # noqa: E731
    w13 = [deq(x.w13_q, x.w13_scale) for x in ex]
    w2 = [deq(x.w2_q, x.w2_scale) for x in ex]
    tab = lambda ts: (ctypes.c_void_p * E)(*[t.data_ptr() for t in ts])  # noqa: E731
    t_bf = (tab(w13), tab(w2))
    t_f8 = (tab([x.w13_q for x in ex]), tab([x.w13_scale_bits for x in ex]), tab([x.w2_q for x in ex]), tab([x.w2_scale_bits for x in ex]))
    rows = []
    for T in (1, 8, 32, 4096):
        g = torch.Generator(device="cuda").manual_seed(T)
        hn = (torch.randn(T, dim, generator=g, device="cuda")).to(torch.bfloat16)
        res = torch.zeros_like(hn)
        ws = _abi.Workspace(_abi.workspace_bytes(T, dim, 1, 1, 128, hidden, 0, 1), torch.device("cuda"))
        b = MoeBuffers(T, dim, hidden, E, k, torch.device("cuda"), torch.bfloat16)
        _abi.moe_route(hn, layer.gate_weight, E, k, 0, 1, b)
        touched = int(torch.unique(b.sel).numel())
        out = torch.empty_like(hn)
        run_bf = lambda: _abi.moe_grouped_ffn(b, *t_bf, res, out, T, dim, hidden, E, k, None, ws)  # noqa: E731
        run_f8 = lambda: _abi.moe_grouped_ffn_fp8(b, *t_f8, res, out, T, dim, hidden, E, k, None, ws)  # noqa: E731
        reps = 20 if T == 4096 else 100
        run_bf(), run_f8()
        torch.cuda.synchronize()
        ms_bf, ms_f8 = [], []
        for _ in range(5):  # alternated
            ms_bf.append(timed(run_bf, reps))
            ms_f8.append(timed(run_f8, reps))
        bf, f8 = sorted(ms_bf)[2], sorted(ms_f8)[2]
        w_elems = touched * 3 * dim * hidden
        bytes_f8 = w_elems + touched * (2 * hidden + dim) * 4  # e4m3 weights + fp32 row scales
        bytes_bf = 2 * w_elems
        flops = 2 * T * k * 3 * dim * hidden
        rows.append(dict(T=T, experts_touched=touched, bf16_ms=round(bf, 4), fp8_ms=round(f8, 4), speedup=round(bf / f8, 3),
                         bf16_hbm_roofline=round(bytes_bf / HBM_BPS * 1e3 / bf, 3), fp8_hbm_roofline=round(bytes_f8 / HBM_BPS * 1e3 / f8, 3),
                         bf16_tflops=round(flops / bf / 1e9, 1), fp8_tflops=round(flops / f8 / 1e9, 1)))
        print(f"  T={T:5d} touched={touched}  bf16 {bf:8.3f} ms  fp8 {f8:8.3f} ms  x{bf / f8:5.2f}  "
              f"HBM roofline bf16 {rows[-1]['bf16_hbm_roofline']:.0%} fp8 {rows[-1]['fp8_hbm_roofline']:.0%}  "
              f"TFLOP/s bf16 {rows[-1]['bf16_tflops']} fp8 {rows[-1]['fp8_tflops']}", flush=True)
        del ws, b
    return rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    p = synth.shape("mixtral-8x7b", n_layers=a.layers)
    print(f"card: {card()}", flush=True)
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m = build(p, a.seed)
    torch.cuda.synchronize()
    res = {"card": card(), "layers": a.layers, "build_s": round(time.perf_counter() - t0, 1),
           "model_gb": round(sum(t.numel() * t.element_size() for t in m.parameters()) / 1e9, 2),
           "build_peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 2)}
    print(f"model {res['model_gb']} GB, build peak {res['build_peak_gb']} GB, built in {res['build_s']} s", flush=True)
    torch.cuda.reset_peak_memory_stats()
    res.update({k: round(v, 3) for k, v in model_numbers(m, p).items()})
    res["run_peak_gb"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
    # algorithmic bound of a batch-1 token at 4k context: experts of 2 of 8 per layer in FP8, attention + router weights, lm head, KV
    dim, hd, hid, L = p["dim"], p["head_dim"], p["hidden_dim"], p["n_layers"]
    attn = (p["n_heads"] + 2 * p["n_kv_heads"]) * hd * dim + dim * p["n_heads"] * hd
    tok_bytes = L * (2 * 3 * dim * hid + 2 * attn + 2 * 8 * dim) + 2 * p["vocab_size"] * dim + L * 2 * 4096 * p["n_kv_heads"] * hd * 2
    res["decode_b1_bound_ms"] = round(tok_bytes / HBM_BPS * 1e3, 2)
    res["decode_b1_hbm_roofline"] = round(res["decode_b1_bound_ms"] / res["decode_b1_ctx4k_ms_per_token"], 3)
    print({k: v for k, v in res.items()}, flush=True)
    res["grouped_ffn"] = ffn_numbers(m, p)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
