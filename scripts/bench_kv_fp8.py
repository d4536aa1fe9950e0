"""FP8 (e4m3) KV cache on one H100: what it costs and what it saves.

Reports, with the card's name, power limit and maximum SM clock read in the same run:
  * decode attention alone (attn_decode_tma_kernel vs attn_decode_tma_fp8_kernel, alternated in one process) at the Nemo-12B head
    shape (32 query / 8 kv heads) for B = 32 at kv_len 1k, 4k, 8k, 16k and B = 1 at 32k: time, and the share of 3.35 TB/s from
    each format's own algorithmic bytes (bf16: 2 * kv_len * KV * 128 * 2 B per sequence; e4m3: 2 * kv_len * KV * (128 + 1) B);
  * the decode step of a 40-layer Nemo-12B-shaped model at B = 32 (graph replays) at a 1k and an 8k context in both formats (the
    caches are allocated one after the other), and at 16k in FP8 only: the bf16 cache of that case is 85.9 GB by arithmetic;
  * one 512-token chunk of chunked-prefill attention against a 16k ring in both formats;
  * the drift between the FP8-cache and the bf16-cache model on seeded synthetic weights (a 4-layer Mistral-7B shape): the largest
    logit difference and the top-1 agreement over a greedy generate run, teacher-forced on the bf16 model's tokens.
Weights and caches of the timing runs are random, not a checkpoint.  Run: python scripts/bench_kv_fp8.py [--quick]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402
from mistral_inference_b200.transformer_layers import decode_splits  # noqa: E402

HBM_BPS = 3.35e12  # H100 SXM data sheet
HD = 128


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e!r})"


def timed(fn, reps: int) -> float:
    """Mean ms of fn() over reps calls, CUDA events around the whole loop."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def rings(B: int, W: int, KV: int, fmt: str):
    """K, V rings (and exponents) of random rows: bf16 N(0, 1), or e4m3 codes of N(0, 1) rows with exponent -6."""
    if fmt == "bf16":
        return [torch.randn(B, W, KV, HD, device="cuda").to(torch.bfloat16) for _ in range(2)], None
    codes = [(torch.randn(B, W, KV, HD, device="cuda") * 64).clamp(-448, 448).to(torch.float8_e4m3fn) for _ in range(2)]
    return codes, [torch.full((B, W, KV), -6, dtype=torch.int8, device="cuda") for _ in range(2)]


def attn_decode_alone(reps: int, out: dict) -> None:
    H, KV = 32, 8
    for B, L in [(32, 1024), (32, 4096), (32, 8192), (32, 16384), (1, 32768)]:
        ws = _abi.Workspace(_abi.workspace_bytes(B, H * HD, H, KV, HD, H * HD, 0, B), torch.device("cuda"))
        q = torch.randn(B, H * HD, device="cuda").to(torch.bfloat16)
        o = torch.empty_like(q)
        lens = torch.full((B,), L, dtype=torch.int32, device="cuda")
        S = decode_splits(B, KV, L)
        (kb, vb), _ = rings(B, L, KV, "bf16")
        (k8, v8), (ek, ev) = rings(B, L, KV, "fp8")
        f_b = lambda: _abi.attn_decode(q, kb, vb, lens, o, H, KV, HD, S, ws)  # noqa: E731
        f_8 = lambda: _abi.attn_decode_fp8(q, k8, v8, ek, ev, lens, o, H, KV, HD, S, ws)  # noqa: E731
        f_b(), f_8()
        t_b, t_8 = [], []
        for _ in range(5):  # alternated
            t_b.append(timed(f_b, reps))
            t_8.append(timed(f_8, reps))
        tb, t8 = min(t_b), min(t_8)
        bytes_b, bytes_8 = 2 * B * L * KV * HD * 2, 2 * B * L * KV * (HD + 1)
        row = {"B": B, "kv_len": L, "splits": S, "bf16_us": round(tb * 1e3, 1), "fp8_us": round(t8 * 1e3, 1),
               "bf16_hbm_share": round(bytes_b / (tb * 1e-3) / HBM_BPS, 3), "fp8_hbm_share": round(bytes_8 / (t8 * 1e-3) / HBM_BPS, 3),
               "speedup": round(tb / t8, 3)}
        print("attn_decode", json.dumps(row), flush=True)
        out.setdefault("attn_decode", []).append(row)
        del kb, vb, k8, v8, ek, ev


def prefill_chunk(reps: int, out: dict) -> None:
    H, KV, T, L = 32, 8, 512, 16384
    q = torch.randn(T, H * HD, device="cuda").to(torch.bfloat16)
    kn, vn = (torch.randn(T, KV * HD, device="cuda").to(torch.bfloat16) for _ in range(2))
    o = torch.empty_like(q)
    qs = torch.tensor([0, T], dtype=torch.int32, device="cuda")
    sp = torch.tensor([L], dtype=torch.int32, device="cuda")
    W = L + T
    (kb, vb), _ = rings(1, W, KV, "bf16")
    (k8, v8), (ek, ev) = rings(1, W, KV, "fp8")
    f_b = lambda: _abi.attn_prefill(q, kn, vn, kb, vb, qs, sp, o, 1, T, W, H, KV, HD, causal=True)  # noqa: E731
    f_8 = lambda: _abi.attn_prefill_fp8(q, kn, vn, k8, v8, ek, ev, qs, sp, o, 1, T, W, H, KV, HD)  # noqa: E731
    f_b(), f_8()
    tb = min(timed(f_b, reps) for _ in range(3))
    t8 = min(timed(f_8, reps) for _ in range(3))
    row = {"chunk": T, "ring_tokens": L, "bf16_ms": round(tb, 3), "fp8_ms": round(t8, 3), "ratio_fp8_over_bf16": round(t8 / tb, 3)}
    print("prefill_chunk", json.dumps(row), flush=True)
    out["prefill_chunk"] = row


def nemo_decode_step(steps: int, out: dict, quick: bool) -> None:
    p = synth.shape("mistral-nemo-12b", n_layers=40 if not quick else 4)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = 32
    B = 32
    m = Transformer.empty(args, "cuda", torch.bfloat16).eval()
    with torch.no_grad():
        for prm in m.parameters():
            prm.normal_(0.0, 0.02)
    weights_gb = sum(t.numel() * t.element_size() for t in m.parameters()) / 1e9
    cases = [("bf16", 1024), ("fp8", 1024), ("bf16", 8192), ("fp8", 8192), ("fp8", 16384)]
    for fmt, ctx in cases:
        m.kv_cache = fmt  # one set of weights; the cache format is the model's, switched between runs
        cache = BufferCache(m.n_local_layers, B, ctx + steps + 4, args.n_kv_heads, HD, None, kv_cache=fmt).to("cuda", torch.bfloat16)
        with torch.no_grad():
            for i in cache.cache_k:
                if fmt == "bf16":
                    cache.cache_k[i].normal_()
                    cache.cache_v[i].normal_()
                else:
                    cache.cache_k[i].view(torch.uint8).random_(0, 0x7E)
                    cache.cache_v[i].view(torch.uint8).random_(0, 0x7E)
                    cache.cache_k_exp[i].fill_(-6)
                    cache.cache_v_exp[i].fill_(-6)
        cache.init_kvseqlens(B)
        cache._kv_seqlens_host = [ctx] * B  # as if a ctx-token prompt had been prefilled
        tok = torch.zeros(B, dtype=torch.long, device="cuda")
        for _ in range(3):  # eager warm-up, capture, replay
            m.next_token_logits(tok, cache)
        torch.cuda.synchronize()
        ms = timed(lambda: m.next_token_logits(tok, cache), steps)
        row = {"format": fmt, "B": B, "context": ctx, "layers": m.n_local_layers, "step_ms": round(ms, 2),
               "cache_gb": round(cache.nbytes / 1e9, 1), "weights_gb": round(weights_gb, 1),
               "peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 1)}
        print("nemo_decode", json.dumps(row), flush=True)
        out.setdefault("nemo_decode", []).append(row)
        del cache
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
    m.kv_cache = "bf16"
    bf16_16k = 2 * 2 * B * 16384 * args.n_kv_heads * HD * m.n_local_layers / 1e9
    out["nemo_16k_bf16_cache_gb"] = round(bf16_16k, 1)
    print(f"nemo_decode: a bf16 cache at B={B}, 16k context would take {bf16_16k:.1f} GB next to {weights_gb:.1f} GB of weights: not run")
    del m
    torch.cuda.empty_cache()


def drift(out: dict, quick: bool) -> None:
    p = synth.shape("mistral-7b", n_layers=4, vocab_size=32768)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, "cuda")
    ms = {}
    for fmt in ("bf16", "fp8"):
        args = mi.TransformerArgs.from_dict(dict(p))
        args.max_batch_size = 4
        m = Transformer.empty(args, "cuda", torch.bfloat16, kv_cache=fmt)
        m.load_state_dict(sd)
        ms[fmt] = m.eval()
    prompts = [synth.synth_prompt(n, p["vocab_size"], 7 + i) for i, n in enumerate((512, 300, 700, 64))]
    n_new = 16 if quick else 64
    toks, _ = mi.generate(prompts, ms["bf16"], max_tokens=n_new, temperature=0.0)
    full = [pr + t for pr, t in zip(prompts, toks)]
    worst, agree, total = 0.0, 0, 0
    # teacher-forced: prefill the prompt, then decode the bf16 model's tokens one step at a time in both models
    caches = {f: BufferCache(4, 4, max(len(x) for x in full) + 1, p["n_kv_heads"], HD, p.get("sliding_window"), kv_cache=f)
              .to("cuda", torch.bfloat16) for f in ms}
    logits = {}
    for f, m in ms.items():
        ids = torch.tensor(sum(prompts, []), device="cuda")
        logits[f] = [m.forward(ids, [len(x) for x in prompts], caches[f])[torch.tensor([len(x) for x in prompts]).cumsum(0) - 1]]
        for s in range(n_new - 1):
            nxt = torch.tensor([t[s] for t in toks], device="cuda")
            logits[f].append(m.forward(nxt, [1] * 4, caches[f]))
    for lb, l8 in zip(logits["bf16"], logits["fp8"]):
        worst = max(worst, (lb - l8).abs().max().item())
        agree += int((lb.argmax(-1) == l8.argmax(-1)).sum())
        total += lb.shape[0]
    row = {"shape": "mistral-7b x4 layers, synthetic", "prompts": [len(x) for x in prompts], "new_tokens": n_new,
           "max_abs_logit_diff": round(worst, 4), "top1_agreement": round(agree / total, 4), "picks": total,
           "logit_absmax": round(max(x.abs().max().item() for x in logits["bf16"]), 2)}
    print("drift", json.dumps(row), flush=True)
    out["drift"] = row


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="4 Nemo layers and fewer steps (a check that the script runs)")
    ap.add_argument("--skip-model", action="store_true")
    a = ap.parse_args()
    torch.manual_seed(0)
    out = {"card": card(), "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}
    print("card:", out["card"], flush=True)
    attn_decode_alone(20 if a.quick else 100, out)
    prefill_chunk(5 if a.quick else 20, out)
    if not a.skip_model:
        nemo_decode_step(5 if a.quick else 20, out, a.quick)
        drift(out, a.quick)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
