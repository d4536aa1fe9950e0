"""FP8 (e4m3) dense weights on one H100: what they buy and what they cost.

Reports, with the card's name, power limit and maximum SM clock read in the same run (bf16 and FP8 alternated in one process):
  1. Mistral-7B shape, 32 layers, and Nemo-12B shape, 40 layers, batch 1 at a 4k context: decode-megakernel tok/s in both formats,
     and each format's share of 3.35 TB/s from its own bytes per step (layer weights, scales, the bf16 lm head, the embedding row,
     the K/V ring);
  2. Nemo-12B shape, 40 layers, batch 32 at a 1k context: the decode step as a CUDA-graph replay;
  3. a 4096-token Mistral-7B prefill (one forward over the prompt);
  4. the Linear kernels alone at T = 1, 4, 32, 128, 4096 for the 7B wqkv, w13 and w2 shapes: time, and the share of 3.35 TB/s
     from each format's weight bytes (e4m3: N * K + 4 N);
  5. drift on seeded synthetic weights (a 4-layer 7B shape): the largest logit difference and the top-1 agreement between the FP8
     and the bf16 model, teacher-forced on the bf16 model's greedy tokens;
  6. the peak device memory of Transformer.from_folder(dense_weights="fp8") on a synthetic 8-layer 7B-shaped checkpoint, next to the
     FP8 model's bytes and the largest bf16 tensor.
Weights of the timing runs are random (the FP8 model holds the e4m3 rows of the bf16 model's weights), not a checkpoint.
Run: python scripts/bench_fp8_dense.py [--quick]
"""
import argparse
import json
import subprocess
import sys
import tempfile
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import mistral_inference_b200 as mi  # noqa: E402
import synth  # noqa: E402
from mistral_inference_b200 import _abi  # noqa: E402
from mistral_inference_b200.cache import BufferCache  # noqa: E402
from mistral_inference_b200.transformer import Transformer  # noqa: E402

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


def model_pair(name: str, n_layers: int, max_batch: int):
    """A bf16 model with random weights and the FP8 model holding the e4m3 rows of the same weights."""
    p = synth.shape(name, n_layers=n_layers)
    args = mi.TransformerArgs.from_dict(dict(p))
    args.max_batch_size = max_batch
    bf = Transformer.empty(args, "cuda", torch.bfloat16).eval()
    with torch.no_grad():
        for prm in bf.parameters():
            prm.normal_(0.0, 0.02)
        for prm in (bf.layers[k].attention_norm.weight for k in bf.layers):
            prm.fill_(1.0)
    f8 = Transformer.empty(args, "cuda", torch.bfloat16, dense_weights="fp8").eval()
    with torch.no_grad():
        f8.tok_embeddings.weight.copy_(bf.tok_embeddings.weight)
        f8.norm.weight.copy_(bf.norm.weight)
        f8.output_weight.copy_(bf.output_weight)
        for k in bf.layers:
            b8, bb = f8.layers[k], bf.layers[k]
            b8.attention_norm.weight.copy_(bb.attention_norm.weight)
            b8.ffn_norm.weight.copy_(bb.ffn_norm.weight)
            for n in ("wq", "wk", "wv", "wo"):
                b8.attention.quantize_(n, getattr(bb.attention, n).weight)
            for n in ("w1", "w2", "w3"):
                b8.feed_forward.quantize_(n, getattr(bb.feed_forward, n).weight)
    return p, args, {"bf16": bf, "fp8": f8}


def nbytes(m: Transformer) -> int:
    return sum(t.numel() * t.element_size() for t in m.parameters())


def filled_cache(m: Transformer, B: int, ctx: int, extra: int) -> BufferCache:
    a = m.args
    cache = BufferCache(m.n_local_layers, B, ctx + extra, a.n_kv_heads, HD, None).to("cuda", torch.bfloat16)
    with torch.no_grad():
        for i in cache.cache_k:
            cache.cache_k[i].normal_()
            cache.cache_v[i].normal_()
    cache.init_kvseqlens(B)
    cache._kv_seqlens_host = [ctx] * B  # as if a ctx-token prompt had been prefilled
    return cache


def step_bytes(m: Transformer, fmt: str, ctx: int) -> int:
    """Bytes one batch-1 decode step must read: every layer matrix (and its scales), the lm head, one embedding row, the norms, the
    K/V ring up to ctx."""
    a = m.args
    layer = sum(t.numel() * t.element_size() for n, t in m.named_parameters() if n.startswith("layers."))
    return layer + m.output_weight.numel() * 2 + a.dim * 2 + a.dim * 2 + 2 * ctx * a.n_kv_heads * HD * 2 * m.n_local_layers


def decode_b1(ms: dict, key: str, out: dict, quick: bool) -> None:
    """Batch-1 decode on the megakernel at a 4k context, the two formats alternated."""
    ctx, steps = 4096, 30 if quick else 200
    caches = {f: filled_cache(m, 1, ctx, 4 * steps + 16) for f, m in ms.items()}
    tok = torch.zeros(1, dtype=torch.long, device="cuda")
    for f, m in ms.items():
        assert m._megakernel_ok(1), f"{f}: the megakernel refuses this shape"
        for _ in range(3):
            m.decode_static(tok, caches[f])
    res = {f: [] for f in ms}
    for _ in range(3 if quick else 5):  # alternated
        for f, m in ms.items():
            res[f].append(timed(lambda: m.decode_static(tok, caches[f]), steps))
    for f, m in ms.items():
        ms_step = min(res[f])
        b = step_bytes(m, f, ctx)
        row = {"format": f, "layers": m.n_local_layers, "context": ctx, "step_ms": round(ms_step, 3), "tok_s": round(1e3 / ms_step, 1),
               "all_tok_s": [round(1e3 / t, 1) for t in res[f]], "step_bytes_gb": round(b / 1e9, 3),
               "hbm_share": round(b / (ms_step * 1e-3) / HBM_BPS, 3)}
        print(key, json.dumps(row), flush=True)
        out.setdefault(key, []).append(row)
    out[key + "_speedup"] = round(min(res["bf16"]) / min(res["fp8"]), 3)
    print(key, "speedup fp8 over bf16:", out[key + "_speedup"], flush=True)
    del caches


def decode_7b(out: dict, quick: bool) -> None:
    _, args, ms = model_pair("mistral-7b", 4 if quick else 32, 1)
    decode_b1(ms, "decode_7b_b1", out, quick)
    # 3. prefill of 4096 tokens (the same models)
    T = 4096
    ids = torch.randint(0, args.vocab_size, (T,), device="cuda")
    pf = {f: BufferCache(m.n_local_layers, 1, T, args.n_kv_heads, HD, None).to("cuda", torch.bfloat16) for f, m in ms.items()}

    def prefill(f):
        pf[f].reset()
        ms[f].forward(ids, [T], pf[f])

    for f in ms:
        prefill(f)
    res = {f: [] for f in ms}
    for _ in range(3):
        for f in ms:
            res[f].append(timed(lambda: prefill(f), 2 if quick else 5))
    row = {"tokens": T, "layers": ms["bf16"].n_local_layers, "bf16_ms": round(min(res["bf16"]), 2), "fp8_ms": round(min(res["fp8"]), 2),
           "ratio_fp8_over_bf16": round(min(res["fp8"]) / min(res["bf16"]), 3)}
    print("prefill_7b", json.dumps(row), flush=True)
    out["prefill_7b"] = row
    del ms, pf
    torch.cuda.empty_cache()
    _, _, ms = model_pair("mistral-nemo-12b", 4 if quick else 40, 1)
    decode_b1(ms, "decode_nemo_b1", out, quick)
    del ms
    torch.cuda.empty_cache()


def decode_nemo(out: dict, quick: bool) -> None:
    B, ctx = 32, 1024
    _, args, ms = model_pair("mistral-nemo-12b", 4 if quick else 40, B)
    steps = 5 if quick else 20
    caches = {f: filled_cache(m, B, ctx, 4 * steps + 16) for f, m in ms.items()}
    tok = torch.zeros(B, dtype=torch.long, device="cuda")
    for f, m in ms.items():
        for _ in range(3):  # eager warm-up, capture, replay
            m.next_token_logits(tok, caches[f])
    res = {f: [] for f in ms}
    for _ in range(3):
        for f, m in ms.items():
            res[f].append(timed(lambda: m.next_token_logits(tok, caches[f]), steps))
    for f, m in ms.items():
        row = {"format": f, "B": B, "context": ctx, "layers": m.n_local_layers, "step_ms": round(min(res[f]), 3),
               "weights_gb": round(nbytes(m) / 1e9, 2)}
        print("decode_nemo_b32", json.dumps(row), flush=True)
        out.setdefault("decode_nemo_b32", []).append(row)
    del ms, caches
    torch.cuda.empty_cache()


def linears(out: dict, quick: bool) -> None:
    dim, hidden, q_dim, kv_dim = 4096, 14336, 4096, 1024
    shapes = {"wqkv": (q_dim + 2 * kv_dim, dim), "w13": (2 * hidden, dim), "w2": (dim, hidden)}
    for name, (N, K) in shapes.items():
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        q = torch.empty(N, K, dtype=torch.uint8, device="cuda")
        s = torch.empty(N, dtype=torch.float32, device="cuda")
        _abi.quantize_e4m3_rows(w, q, s)
        for T in (1, 4, 32, 128, 4096):
            ws = _abi.Workspace(_abi.workspace_bytes(T, max(K, dim), 32, 8, 128, max(K, hidden), 0, 1), torch.device("cuda"))
            x = torch.randn(T, K, device="cuda").to(torch.bfloat16)
            o = torch.empty(T, N, dtype=torch.bfloat16, device="cuda")
            calls = {"bf16": lambda: _abi.linear_residual(x, w, None, o, ws), "fp8": lambda: _abi.linear_residual_fp8(x, q, s, None, o, ws)}
            names = {f: ",".join(sorted({n.split("<")[0] for n in launched(c)})) for f, c in calls.items()}
            reps = 5 if T == 4096 else (20 if quick else 200)
            res = {f: [] for f in calls}
            for _ in range(3):
                for f, c in calls.items():
                    res[f].append(timed(c, reps))
            tb, t8 = min(res["bf16"]), min(res["fp8"])
            row = {"linear": name, "N": N, "K": K, "T": T, "bf16_us": round(tb * 1e3, 1), "fp8_us": round(t8 * 1e3, 1),
                   "bf16_hbm_share": round(N * K * 2 / (tb * 1e-3) / HBM_BPS, 3), "fp8_hbm_share": round((N * K + 4 * N) / (t8 * 1e-3) / HBM_BPS, 3),
                   "fp8_tflops": round(2 * T * N * K / (t8 * 1e-3) / 1e12, 1), "bf16_tflops": round(2 * T * N * K / (tb * 1e-3) / 1e12, 1),
                   "speedup": round(tb / t8, 3), "kernels": names}
            print("linear", json.dumps(row), flush=True)
            out.setdefault("linears", []).append(row)
        del w, q, s
        torch.cuda.empty_cache()


def launched(fn):
    from tests.util import launched_kernels

    return launched_kernels(fn)


def drift(out: dict, quick: bool) -> None:
    p = synth.shape("mistral-7b", n_layers=4, vocab_size=32768)
    sd = synth.synth_state_dict(p, 3, torch.bfloat16, "cuda")
    ms = {}
    for fmt in ("bf16", "fp8"):
        args = mi.TransformerArgs.from_dict(dict(p))
        args.max_batch_size = 4
        m = Transformer.empty(args, "cuda", torch.bfloat16, dense_weights=fmt)
        m.load_state_dict(sd)
        ms[fmt] = m.eval()
    del sd
    prompts = [synth.synth_prompt(n, p["vocab_size"], 7 + i) for i, n in enumerate((512, 300, 700, 64))]
    n_new = 16 if quick else 64
    toks, _ = mi.generate(prompts, ms["bf16"], max_tokens=n_new, temperature=0.0)
    full = [pr + t for pr, t in zip(prompts, toks)]
    caches = {f: BufferCache(4, 4, max(len(x) for x in full) + 1, p["n_kv_heads"], HD, p.get("sliding_window")).to("cuda", torch.bfloat16)
              for f in ms}
    logits = {}
    for f, m in ms.items():
        ids = torch.tensor(sum(prompts, []), device="cuda")
        logits[f] = [m.forward(ids, [len(x) for x in prompts], caches[f])[torch.tensor([len(x) for x in prompts]).cumsum(0) - 1]]
        for s in range(n_new - 1):
            nxt = torch.tensor([t[s] for t in toks], device="cuda")
            logits[f].append(m.forward(nxt, [1] * 4, caches[f]).clone())
    worst, agree, total = 0.0, 0, 0
    for lb, l8 in zip(logits["bf16"], logits["fp8"]):
        worst = max(worst, (lb - l8).abs().max().item())
        agree += int((lb.argmax(-1) == l8.argmax(-1)).sum())
        total += lb.shape[0]
    row = {"shape": "mistral-7b x4 layers, synthetic", "prompts": [len(x) for x in prompts], "new_tokens": n_new,
           "max_abs_logit_diff": round(worst, 4), "top1_agreement": round(agree / total, 4), "picks": total,
           "logit_absmax": round(max(x.abs().max().item() for x in logits["bf16"]), 2)}
    print("drift", json.dumps(row), flush=True)
    out["drift"] = row
    del ms
    torch.cuda.empty_cache()


def load_peak(out: dict, quick: bool) -> None:
    p = synth.shape("mistral-7b", n_layers=2 if quick else 8)
    with tempfile.TemporaryDirectory() as d:
        synth.write_model_folder(d, p, seed=1)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        m = Transformer.from_folder(d, dense_weights="fp8")
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    largest = max(2 * a * b for _, (a, b) in ((k, s) for k, s in synth.state_dict_shapes(p) if len(s) == 2))
    row = {"shape": f"mistral-7b x{p['n_layers']} layers", "model_gb": round(nbytes(m) / 1e9, 3), "peak_gb": round(peak / 1e9, 3),
           "largest_bf16_tensor_gb": round(largest / 1e9, 3)}
    print("from_folder", json.dumps(row), flush=True)
    out["from_folder"] = row
    del m
    torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="few layers and steps (a check that the script runs)")
    ap.add_argument("--only", default="", help="comma-separated sections: decode7b,nemo,linears,drift,load")
    a = ap.parse_args()
    torch.manual_seed(0)
    out = {"card": card(), "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}
    print("card:", out["card"], flush=True)
    only = set(filter(None, a.only.split(",")))
    for key, fn in (("decode7b", decode_7b), ("nemo", decode_nemo), ("linears", linears), ("drift", drift), ("load", load_peak)):
        if not only or key in only:
            fn(out, a.quick)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
